"""Per-layer-shape timing of the wgmma conv kernels on the YOLOv5l@640 shapes, CUDA events, L2 flushed between iterations.
Modes: fwd (folded BN + SiLU), fwd_res (folded BN + SiLU + shortcut: the Bottleneck's second conv, on the 3x3 s1 C->C
shapes only), raw (raw output: the student's training forward), dgrad, dgrad_acc (dgrad added into the existing input
gradient: gradient fan-in), wgrad.
  python tools/conv_bench.py [--batch 16] [--modes fwd,dgrad,wgrad] [--out bench_out/conv_bench.json]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, Cin, Cout, k, s, H_in, count in the trunk)   -- SURVEY.md Appendix B
SHAPES = [
    ("stem_gemm K128", 128, 64, 1, 1, 320, 1),
    ("s2 64->128 @320", 64, 128, 3, 2, 320, 1),
    ("1x1 128->64 @160", 128, 64, 1, 1, 160, 2),
    ("1x1 64->64 @160", 64, 64, 1, 1, 160, 3),
    ("3x3 64->64 @160", 64, 64, 3, 1, 160, 3),
    ("1x1 128->128 @160", 128, 128, 1, 1, 160, 1),
    ("s2 128->256 @160", 128, 256, 3, 2, 160, 1),
    ("1x1 256->128 @80", 256, 128, 1, 1, 80, 4),
    ("1x1 128->128 @80", 128, 128, 1, 1, 80, 9),
    ("3x3 128->128 @80", 128, 128, 3, 1, 80, 9),
    ("1x1 256->256 @80", 256, 256, 1, 1, 80, 2),
    ("s2 256->512 @80", 256, 512, 3, 2, 80, 1),
    ("1x1 512->256 @40", 512, 256, 1, 1, 40, 5),
    ("1x1 256->256 @40", 256, 256, 1, 1, 40, 15),
    ("3x3 256->256 @40", 256, 256, 3, 1, 40, 15),
    ("1x1 512->512 @40", 512, 512, 1, 1, 40, 3),
    ("s2 512->1024 @40", 512, 1024, 3, 2, 40, 1),
    ("1x1 1024->512 @20", 1024, 512, 1, 1, 20, 6),
    ("1x1 512->512 @20", 512, 512, 1, 1, 20, 6),
    ("3x3 512->512 @20", 512, 512, 3, 1, 20, 6),
    ("1x1 1024->1024 @20", 1024, 1024, 1, 1, 20, 2),
    ("1x1 2048->1024 @20", 2048, 1024, 1, 1, 20, 1),
    ("1x1 1024->256 @40", 1024, 256, 1, 1, 40, 2),
    ("1x1 512->128 @80", 512, 128, 1, 1, 80, 2),
    ("s2 256->256 @80", 256, 256, 3, 2, 80, 1),
    ("s2 512->512 @40", 512, 512, 3, 2, 40, 1),
    ("head 256->255 @80", 256, 255, 1, 1, 80, 1),
]

_flush = None


ITERS = 5


def timeit(fn, iters=None):
    iters = iters or ITERS
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        _flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "conv_bench.json"))
    ap.add_argument("--modes", default="fwd,dgrad,wgrad")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--only", default="", help="substring filter on the shape name")
    args = ap.parse_args()
    global ITERS
    ITERS = args.iters
    import __graft_entry__ as g
    g.build()
    from efficientteacher_b200 import convops as co
    dev = "cuda:0"
    N = args.batch
    res = []
    tot = {m: [0.0, 0.0] for m in args.modes.split(",")}
    for name, Cin, Cout, k, s, H, cnt in SHAPES:
        if args.only and args.only not in name:
            continue
        p = k // 2
        Ho = (H + 2 * p - k) // s + 1
        x = torch.randn(N, H, H, Cin, device=dev).to(torch.bfloat16)
        w = torch.randn(Cout, Cin, k, k, device=dev) * (Cin * k * k) ** -0.5
        cpad = (Cout + 7) // 8 * 8
        dy = torch.randn(N, Ho, Ho, cpad, device=dev).to(torch.bfloat16)
        flops = 2.0 * N * Ho * Ho * Cout * Cin * k * k
        row = dict(name=name, count=cnt, gflop=flops / 1e9)
        if "fwd" in tot:
            wp = co.pack_weight(w)
            sc = torch.ones(Cout, device=dev); bi = torch.zeros(Cout, device=dev)
            y = torch.empty(N, Ho, Ho, cpad, dtype=torch.bfloat16, device=dev)
            ms = timeit(lambda: co.conv_fwd(x, wp, Cin, Cout, k, s, p, sc, bi, "silu", out=y))
            row["fwd_us"], row["fwd_tflops"] = ms * 1e3, flops / ms / 1e9
            tot["fwd"][0] += ms * cnt; tot["fwd"][1] += flops * cnt
        if "fwd_res" in tot and name.startswith("3x3"):   # Bottleneck cv2: the shortcut is added in the epilogue
            wp = co.pack_weight(w)
            sc = torch.ones(Cout, device=dev); bi = torch.zeros(Cout, device=dev)
            y = torch.empty(N, Ho, Ho, cpad, dtype=torch.bfloat16, device=dev)
            r = torch.randn(N, Ho, Ho, cpad, device=dev).to(torch.bfloat16)
            ms = timeit(lambda: co.conv_fwd(x, wp, Cin, Cout, k, s, p, sc, bi, "silu", out=y, residual=r))
            row["fwd_res_us"], row["fwd_res_tflops"] = ms * 1e3, flops / ms / 1e9
            tot["fwd_res"][0] += ms * cnt; tot["fwd_res"][1] += flops * cnt
        if "raw" in tot:        # the student's training forward: raw bf16 conv output (BN statistics come next)
            wp = co.pack_weight(w)
            y = torch.empty(N, Ho, Ho, cpad, dtype=torch.bfloat16, device=dev)
            ms = timeit(lambda: co.conv_fwd(x, wp, Cin, Cout, k, s, p, None, None, None, out=y))
            row["raw_us"], row["raw_tflops"] = ms * 1e3, flops / ms / 1e9
            tot["raw"][0] += ms * cnt; tot["raw"][1] += flops * cnt
        if "dgrad" in tot and Cout % 64 == 0:
            wd = co.pack_weight_dgrad(w, s, p)
            dx = torch.empty(N, H, H, Cin, dtype=torch.bfloat16, device=dev)
            ms = timeit(lambda: co.conv_dgrad(dy, wd, N, H, H, Cin, Cout, k, s, p, out=dx))
            row["dgrad_us"], row["dgrad_tflops"] = ms * 1e3, flops / ms / 1e9
            tot["dgrad"][0] += ms * cnt; tot["dgrad"][1] += flops * cnt
        if "dgrad_acc" in tot and Cout % 64 == 0:   # gradient fan-in: the dgrad is added into the existing input gradient
            wd = co.pack_weight_dgrad(w, s, p)
            dx = torch.zeros(N, H, H, Cin, dtype=torch.bfloat16, device=dev)
            ms = timeit(lambda: co.conv_dgrad(dy, wd, N, H, H, Cin, Cout, k, s, p, out=dx, accumulate=True))
            row["dgrad_acc_us"], row["dgrad_acc_tflops"] = ms * 1e3, flops / ms / 1e9
            tot["dgrad_acc"][0] += ms * cnt; tot["dgrad_acc"][1] += flops * cnt
        if "wgrad" in tot:
            ms = timeit(lambda: co.conv_wgrad(x, dy, Cin, Cout, k, s, p))
            row["wgrad_us"], row["wgrad_tflops"] = ms * 1e3, flops / ms / 1e9
            tot["wgrad"][0] += ms * cnt; tot["wgrad"][1] += flops * cnt
        # floors: HBM (read x + write y, bf16) at 3.35 TB/s vs tensor pipe at 989 TF/s dense bf16 (H100 SXM data sheet)
        row["floor_us"] = max((N * H * H * Cin + N * Ho * Ho * Cout) * 2 / 3.35e6, flops / 989e6)
        print("%-22s x%-2d %6.1fGF floor %6.1fus | " % (name, cnt, flops / 1e9, row["floor_us"]) +
              " ".join("%s %6.1fus" % (m, row[m + "_us"]) for m in tot if m + "_us" in row), flush=True)
        res.append(row)
        del x, dy
    summ = {m: dict(ms=v[0], tflops=v[1] / v[0] / 1e9 if v[0] else None) for m, v in tot.items()}
    print(json.dumps(dict(batch=N, trunk_totals=summ)))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(dict(batch=N, layers=res, trunk_totals=summ), open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
