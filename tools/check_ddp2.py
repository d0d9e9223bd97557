"""2-GPU check of the data-parallel step (torchrun --nproc-per-node 2 tools/check_ddp2.py):
  modes (argv[1], comma separated): single = eager step, one all-reduce after backward; graph = captured graphs A / B
  with the all-reduce between them; sync_bn = eager step with `sync_bn: True` (SyncBatchNorm over NCCL).
  * every mode except sync_bn gives the same weights as the first one listed (to bf16-training run-to-run noise),
  * replicas stay bit-identical (student weights) across ranks,
  * BatchNorm running statistics at the start of a forward equal rank 0's (DDP broadcast_buffers semantics); with sync_bn
    they are equal across ranks after the steps even without that broadcast, and a captured step refuses sync_bn.
Prints PASS / FAIL lines; exit code != 0 on failure.  The sync_bn mode has not been run on a multi-GPU machine yet."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def run(mode, rank, world, dev, steps=3):
    import synth
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep
    torch.manual_seed(0)
    img, bl, bu = 256, 2, 2
    cfg = yolov5_ssod_cfg('l_shallow', batch_size=(bl + bu) * world, img_size=img)
    cfg.SSOD.fixed_accumulate = True
    cfg.sync_bn = mode == "sync_bn"
    st = SSODTrainerStep(cfg, dev, rank=rank, world_size=world, epochs=300)
    st.ema.updates = 100000
    with torch.no_grad():
        for mm in (st.model, st.ema.ema, st.semi_ema.ema):
            for h in mm.head.m:
                h.bias.view(3, -1)[:, 4] += 6.5
                h.bias.view(3, -1)[:, 5:] += 5.0
    r = np.random.RandomState(10 + rank)
    imgs = torch.from_numpy(r.rand(bl, 3, img, img).astype(np.float32)).to(dev)
    uw = torch.from_numpy(r.rand(bu, 3, img, img).astype(np.float32)).to(dev)
    us = uw.flip(3).contiguous()
    tg = torch.from_numpy(synth.make_targets(7 + rank, 8 * bl, bl)).to(dev)
    Ms = torch.from_numpy(synth.make_Ms(9 + rank, bu, img)).to(dev)
    bn_equal = True
    for i in range(steps):
        f = st.train_instance_graphed if mode == "graph" else st.train_instance
        f(imgs, tg, us, uw, None, Ms, i)
        torch.cuda.synchronize()
        if rank == 0:
            print("   %s step %d done" % (mode, i), flush=True)
        # after the step every rank has updated its own copy of the running statistics from rank 0's: they differ now,
        # and the NEXT forward must start from rank 0's again -- checked through the flat buffer after an explicit broadcast
    torch.cuda.synchronize()
    if mode == "sync_bn":
        try:
            st.train_instance_graphed(imgs, tg, us, uw, None, Ms, steps)
            bn_equal = False
        except NotImplementedError:
            pass
    else:
        st._bn_sync.broadcast(world)
    flat = st._bn_sync.flat.clone()
    g = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(g, flat)
    bn_equal = bn_equal and all(torch.equal(g[0], t) for t in g)
    w = torch.cat([p.detach().flatten() for p in st.model.parameters()])
    gw = [torch.zeros_like(w) for _ in range(world)]
    dist.all_gather(gw, w)
    return w, all(torch.equal(gw[0], t) for t in gw), bn_equal


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    import __graft_entry__ as g
    if rank == 0:
        g.build()
    dist.barrier()
    ok = True
    res = {}
    modes = sys.argv[1].split(",") if len(sys.argv) > 1 else ["single", "graph"]
    for mode in modes:
        w, same, bn_same = run(mode, rank, world, dev)
        res[mode] = w
        if rank == 0:
            print("%s: replicas identical %s, BN buffers follow rank 0 %s" % (mode, same, bn_same), flush=True)
        ok = ok and same and bn_same
    for mode in [m for m in modes[1:] if m != "sync_bn" and modes[0] != "sync_bn"]:
        d = float((res[mode] - res[modes[0]]).abs().max())
        rel = float((res[mode] - res[modes[0]]).norm() / res[modes[0]].norm())
        if rank == 0:
            print("%s vs %s: max |dw| %.3g rel %.3g" % (mode, modes[0], d, rel), flush=True)
        ok = ok and rel < 5e-3          # eager vs graph replay of 3 bf16 training steps: run-to-run noise of the step itself (measured 1.1e-3)
    if rank == 0:
        print("PASS" if ok else "FAIL", flush=True)
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
    os._exit(0 if ok else 1)


if __name__ == "__main__":
    main()
