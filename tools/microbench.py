"""Per-kernel timings on one H100 (CUDA events, warm-up, L2 flushed between iterations).  Writes JSON lines.
  python tools/microbench.py [--out bench_out/microbench.json]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth  # noqa: E402


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "fallback": "H100 SXM data sheet"}


_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    _flush.zero_()


def timeit(fn, iters=10, warmup=3, flush=True):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        if flush:
            flush_l2()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "microbench.json"))
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from efficientteacher_b200 import nms as N
    from efficientteacher_b200.ema import ModelEMA, CosineEMA, update_ema_pair
    from efficientteacher_b200.loss import ComputeLoss
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from efficientteacher_b200.pseudo_label import FairPseudoLabel
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    pk = peaks()
    dev = "cuda:0"
    res = []

    def rec(name, med, mn, **kw):
        d = dict(name=name, ms_median=med, ms_min=mn, **kw)
        print(json.dumps(d), flush=True)
        res.append(d)

    # EMA at YOLOv5l-SSOD state size: 518 tensors / 48,003,599 elements -> emulate with a mixed-size parameter list
    class Blob(torch.nn.Module):
        def __init__(self):
            super().__init__()
            r = np.random.RandomState(0)
            sizes, tot = [], 0
            while tot < 48_003_599 - 2_400_000:
                s = int(r.choice([64, 128, 256, 512, 1024, 36864, 147456, 589824, 2359296]))
                sizes.append(s); tot += s
            sizes.append(48_003_599 - tot)
            self.ps = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(s)) for s in sizes])
    m = Blob().to(dev)
    ema = ModelEMA(m)
    n_el = sum(p.numel() for p in m.parameters())
    med, mn = timeit(lambda: ema.update(m))
    rec("ema_single", med, mn, elements=n_el, tensors=len(m.ps), bytes=12 * n_el, gbs=12 * n_el / med / 1e6, frac_hbm=12 * n_el / med / 1e6 / pk["hbm_gbs"])
    semi = CosineEMA(ema.ema, 0.999, 0.9999, 10)
    med, mn = timeit(lambda: update_ema_pair(ema, semi, m))
    rec("ema_fused_pair", med, mn, elements=n_el, bytes=20 * n_el, gbs=20 * n_el / med / 1e6, frac_hbm=20 * n_el / med / 1e6 / pk["hbm_gbs"])
    del m, ema, semi
    torch.cuda.empty_cache()

    cfg = ssod_cfg()
    fpl = FairPseudoLabel(cfg)
    for (B, P, img) in ((16, 25200, 640), (8, 100800, 1280)):
        pred = torch.from_numpy(synth.make_teacher_pred(0, B, P, img=img)).to(dev)
        Ms = torch.from_numpy(synth.make_Ms(1, B, img=img))
        Ms_dev = Ms.to(dev)
        med, mn = timeit(lambda: fpl.create_pseudo_label_device(pred, Ms_dev, img, img))
        rec("nms_pseudo_label_device", med, mn, B=B, P=P, read_bytes=B * P * 85 * 4)
        imgs = torch.empty(B, 3, 8, 8, device=dev)
        med, mn = timeit(lambda: fpl.create_pseudo_label_online_with_gt(pred, torch.empty(B, 3, img, img, device="meta"), Ms, None))
        rec("nms_pseudo_label_api_host_rows", med, mn, B=B, P=P)
        del pred

    model = HeadOnlyModel().to(dev)
    sup, ssod = ComputeLoss(model, cfg), ComputeStudentMatchLoss(model, cfg)
    B = 16
    p = [torch.from_numpy(x).to(dev).requires_grad_(True) for x in synth.make_head_logits(3, B)]
    tg = torch.from_numpy(synth.make_targets(4, 128, B)).to(dev)
    rows = torch.from_numpy(synth.make_pseudo_rows(5, 2000, B)).to(dev)
    dense = sum(x.numel() for x in p) * 4

    def fb(crit, t):
        for x in p:
            x.grad = None
        loss, _ = crit(p, t)
        loss.backward()
    med, mn = timeit(lambda: sup(p, tg))
    rec("compute_loss_fwd", med, mn, B=B, targets=128)
    med, mn = timeit(lambda: fb(sup, tg))
    rec("compute_loss_fwd_bwd", med, mn, B=B, targets=128, grad_bytes=dense, gbs_write=dense / med / 1e6)
    med, mn = timeit(lambda: ssod(p, rows))
    rec("ssod_loss_fwd", med, mn, B=B, rows=2000)
    med, mn = timeit(lambda: fb(ssod, rows))
    rec("ssod_loss_fwd_bwd", med, mn, B=B, rows=2000)

    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(dict(peaks=pk, results=res, gpu=torch.cuda.get_device_name(0)), open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
