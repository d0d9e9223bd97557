"""GB/s of the fused training BatchNorm+SiLU kernels on YOLOv5l activation shapes (batch 32), CUDA events, L2 flushed."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import __graft_entry__ as g
    g.build()
    from efficientteacher_b200 import _lib, convops as co
    from tools.conv_bench import timeit
    dev = "cuda:0"
    lib = _lib.lib()
    pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0   # H100 SXM data sheet
    for (N, H, C_) in ((32, 320, 64), (32, 160, 64), (32, 160, 128), (32, 80, 128), (32, 80, 256), (32, 40, 256), (32, 40, 512), (32, 20, 512), (32, 20, 1024)):
        M = N * H * H
        y = torch.randn(N, H, H, C_, device=dev).to(torch.bfloat16)
        da = torch.randn(N, H, H, C_, device=dev).to(torch.bfloat16)
        gamma = torch.ones(C_, device=dev); beta = torch.zeros(C_, device=dev)
        rm = torch.zeros(C_, device=dev); rv = torch.ones(C_, device=dev)
        out = torch.empty_like(y)
        a, stats = co.bn_forward(y, C_, gamma, beta, rm, rv, 1e-3, 0.03, "silu", out=out)
        sums = torch.zeros(2 * C_, dtype=torch.float32, device=dev)
        rows0, rows1 = int(lib.etb_bn_partial_rows(M, C_, 0)), int(lib.etb_bn_partial_rows(M, C_, 1))
        part = torch.empty(max(rows0, rows1), 2, C_, device=dev)
        nb = M * C_ * 2
        r = {}
        r["stats(1R)"] = (timeit(lambda: lib.etb_bn_stats(_lib.ptr(y), M, C_, C_, _lib.ptr(part), rows0, _lib.stream_ptr())), 1)
        r["apply(1R1W)"] = (timeit(lambda: lib.etb_bn_act_apply_res(_lib.ptr(y), _lib.ptr(stats[0]), _lib.ptr(stats[1]), None, _lib.ptr(out), M, C_, C_, 0, C_, 1, _lib.stream_ptr())), 2)
        r["bwd_reduce(2R)"] = (timeit(lambda: lib.etb_bn_act_bwd_reduce(_lib.ptr(da), _lib.ptr(y), _lib.ptr(stats[0]), _lib.ptr(stats[1]), _lib.ptr(stats[2]), _lib.ptr(stats[3]), M, C_, C_, C_, 1, _lib.ptr(part), rows1, _lib.stream_ptr())), 2)
        r["bwd_apply(2R1W)"] = (timeit(lambda: lib.etb_bn_act_bwd_apply(_lib.ptr(da), _lib.ptr(y), _lib.ptr(stats[0]), _lib.ptr(stats[1]), _lib.ptr(stats[2]), _lib.ptr(stats[3]), _lib.ptr(sums), M, C_, C_, C_, C_, 1, _lib.ptr(out), _lib.stream_ptr())), 3)
        print("M=%8d C=%4d (%6.1f MB/pass): " % (M, C_, nb / 1e6) + "  ".join("%s %6.1fus %4.0fGB/s(%.2f)" % (k, ms * 1e3, p * nb / ms / 1e6, p * nb / ms / 1e6 / pk) for k, (ms, p) in r.items()), flush=True)


if __name__ == "__main__":
    main()
