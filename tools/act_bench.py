#!/usr/bin/env python
"""Cost of the trunk activation on one GPU:
  1. the training BatchNorm apply and backward kernels per activation (SiLU, ReLU, Hardswish) on YOLOv5l activation shapes
     at batch 32 / 640 (CUDA events, L2 flushed, median of tools/conv_bench.timeit);
  2. the `sup32`-shaped supervised step (YOLOv5l, 640, 32 images, captured graph) per trunk mode: SiLU, ReLU, the
     reference's default (Hardswish backbone, ReLU neck) and Hardswish; the modes take turns over --repeats windows.

  python tools/act_bench.py [--steps K] [--warmup W] [--repeats R] [--no-step]

Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

ACTS = ("silu", "relu", "hard_swish")
MODES = {"silu": ("SiLU", "SiLU"), "relu": ("ReLU", "ReLU"), "default": ("LeakyReLU", "ReLU"), "hswish": ("Hardswish", "Hardswish")}
SHAPES = ((32, 320, 64), (32, 160, 128), (32, 80, 256), (32, 40, 512), (32, 20, 1024))   # N, H = W, C


def bn_kernels(dev):
    from efficientteacher_b200 import _lib, convops as co
    from tools.conv_bench import timeit
    lib = _lib.lib()
    rows = []
    for N, H, C_ in SHAPES:
        M = N * H * H
        g = torch.Generator(device=dev).manual_seed(0)
        y = (torch.randn(N, H, H, C_, device=dev, generator=g) * 2.0).to(torch.bfloat16)
        da = torch.randn(N, H, H, C_, device=dev, generator=g).to(torch.bfloat16)
        gamma, beta = torch.ones(C_, device=dev), torch.zeros(C_, device=dev)
        out = torch.empty_like(y)
        _, stats = co.bn_forward(y, C_, gamma, beta, None, None, 1e-3, 0.03, "silu", out=out)
        sums = torch.zeros(2 * C_, dtype=torch.float32, device=dev)
        rows1 = int(lib.etb_bn_partial_rows(M, C_, 1))
        part = torch.empty(rows1, 2, C_, device=dev)
        p = [_lib.ptr(t) for t in (y, da, stats[0], stats[1], stats[2], stats[3], out, part, sums)]
        for act in ACTS:
            a, s = co.ACT[act], _lib.stream_ptr()
            t = {"apply": timeit(lambda: lib.etb_bn_act_apply_res(p[0], p[2], p[3], None, p[6], M, C_, C_, 0, C_, a, s)),
                 "bwd_reduce": timeit(lambda: lib.etb_bn_act_bwd_reduce(p[1], p[0], p[2], p[3], p[4], p[5], M, C_, C_, C_, a, p[7], rows1, s)),
                 "bwd_apply": timeit(lambda: lib.etb_bn_act_bwd_apply(p[1], p[0], p[2], p[3], p[4], p[5], p[8], M, C_, C_, C_, C_, a, p[6], s))}
            rows.append(dict(N=N, H=H, C=C_, act=act, **{k + "_us": round(v * 1e3, 2) for k, v in t.items()}))
            print(json.dumps(rows[-1]), flush=True)
    return rows


def sup_steps(dev, steps, warmup, repeats):
    from bench import synth_batch
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.trainer import SupTrainerStep
    host = synth_batch(0, bl=32, bu=0, img=640)
    imgs, tg = (host["imgs"].to(dev).float() / 255.0), host["targets"].to(dev)
    res = {m: [] for m in MODES}
    for _ in range(repeats):               # one model at a time (four YOLOv5l steps at batch 32 do not fit together)
        for mode, (bb, nk) in MODES.items():
            torch.manual_seed(0)
            st = SupTrainerStep(yolov5_sup_cfg('l', batch_size=32, img_size=640, backbone_act=bb, neck_act=nk), dev, epochs=300)
            for i in range(warmup):
                st.train_step_graphed(imgs, tg, i)
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for i in range(warmup, warmup + steps):
                loss = st.train_step_graphed(imgs, tg, i)
            e.record()
            torch.cuda.synchronize()
            assert torch.isfinite(loss).all(), mode
            res[mode].append(round(32 * steps / (s.elapsed_time(e) / 1e3), 1))
            print(json.dumps({"mode": mode, "images_per_s": res[mode][-1]}), flush=True)
            del st, loss
            torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("act_bench.py measures on a CUDA device; none found")
    import __graft_entry__ as g
    g.build()
    from tools.burnin_bench import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    t0 = time.time()
    out = {"card": card(), "bn_kernels": bn_kernels(dev)}
    if not args.no_step:
        out["sup32_images_per_s"] = sup_steps(dev, args.steps, args.warmup, args.repeats)
    out["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
