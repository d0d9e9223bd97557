"""Diagnostic: parameter-gradient agreement of (a) native wgmma convs under bf16 autocast and (b) torch/cuDNN under bf16
autocast, each against an fp32 (no autocast, TF32 off) torch reference of the same step."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def run(m, crit, x, tg, native, amp):
    from efficientteacher_b200 import model as M
    M.Conv.NATIVE = native
    m.zero_grad(set_to_none=True)
    if amp:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            pred, feat = m(x.contiguous(memory_format=torch.channels_last))
    else:
        pred, feat = m(x)
    loss, _ = crit([p.float() for p in pred], tg)
    (loss + sum(f.float().mean() for f in feat) * 0.1).backward()
    M.Conv.NATIVE = True
    return loss.item(), {k: p.grad.detach().float().clone() for k, p in m.named_parameters()}


def main():
    import __graft_entry__ as g
    g.build()
    import synth
    from efficientteacher_b200 import model as M
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.loss import ComputeLoss
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda:0"
    torch.manual_seed(0)
    cfg = yolov5_ssod_cfg('l_shallow', batch_size=4, img_size=256)
    m = M.Model(cfg).to(dev).train()
    crit = ComputeLoss(m, cfg)
    x = torch.rand(4, 3, 256, 256, generator=torch.Generator().manual_seed(1)).to(dev)
    tg = torch.from_numpy(synth.make_targets(2, 32, 4)).to(dev)
    l32, g32 = run(m, crit, x, tg, False, False)
    ln, gn = run(m, crit, x, tg, True, True)
    lc, gc = run(m, crit, x, tg, False, True)
    print("loss fp32 %.5f native-bf16 %.5f cudnn-bf16 %.5f" % (l32, ln, lc))
    cos = torch.nn.functional.cosine_similarity
    rows = []
    for k in g32:
        a = cos(gn[k].flatten(), g32[k].flatten(), dim=0).item()
        b = cos(gc[k].flatten(), g32[k].flatten(), dim=0).item()
        rows.append((k, a, b))
    import numpy as np
    A = np.array([r[1] for r in rows]); B = np.array([r[2] for r in rows])
    print("cos vs fp32: native mean %.4f min %.4f | cudnn-bf16 mean %.4f min %.4f" % (A.mean(), A.min(), B.mean(), B.min()))
    for k, a, b in rows[:12] + rows[-8:]:
        print("%-40s native %.4f cudnn %.4f" % (k, a, b))
    worse = [(k, a, b) for k, a, b in rows if a < b - 0.05]
    print("native worse than cudnn by >0.05:", len(worse), worse[:10])


if __name__ == "__main__":
    main()
