"""Cost of the SyncBatchNorm split on one GPU (no communication), CUDA events:
  1. per YOLOv5l / YOLOv5m activation shape (batch 32): etb_bn_stats_sums + etb_bn_finalize_global against
     etb_bn_stats + etb_bn_finalize (L2 flushed, median of 20);
  2. the eager ssod640 step (YOLOv5l, 16 + 16 images at 640) with every fused BatchNorm on the synced kernels through the
     identity reducer (parallel.BnSync(loopback=True)) against the default per-rank path, alternating the two.
Prints one JSON line per measurement and writes them all to --out.  The collectives themselves (two small all-reduces per
BatchNorm layer and step at world > 1) are not measured here; the layer count and the bytes they move are printed."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = ((32, 320, 64), (32, 160, 128), (32, 80, 256), (32, 40, 512), (32, 20, 1024), (32, 80, 192), (32, 40, 384), (32, 20, 768))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def kernels(emit):
    from efficientteacher_b200 import _lib
    from tools.conv_bench import timeit
    lib, P = _lib.lib(), _lib.ptr
    dev = "cuda:0"
    for N, H, C_ in SHAPES:
        M = N * H * H
        y = torch.randn(N, H, H, C_, device=dev).to(torch.bfloat16)
        gamma, beta = torch.ones(C_, device=dev), torch.zeros(C_, device=dev)
        rm, rv = torch.zeros(C_, device=dev), torch.ones(C_, device=dev)
        stats = torch.empty(4, C_, device=dev)
        rows = int(lib.etb_bn_partial_rows(M, C_, 0))
        part = torch.empty(rows, 2, C_, device=dev)
        sums = torch.empty(2 * C_ + 1, dtype=torch.float64, device=dev)
        sp = _lib.stream_ptr()
        st = [P(stats[i]) for i in range(4)]

        def per_rank():
            lib.etb_bn_stats(P(y), M, C_, C_, P(part), rows, sp)
            lib.etb_bn_finalize(P(part), rows, M, C_, P(gamma), P(beta), 1e-3, 0.03, P(rm), P(rv), *st, sp)

        def synced():
            lib.etb_bn_stats_sums(P(y), M, C_, C_, P(part), rows, P(sums), sp)
            lib.etb_bn_finalize_global(P(sums), C_, P(gamma), P(beta), 1e-3, 0.03, P(rm), P(rv), *st, sp)
        t0, t1 = timeit(per_rank, 20), timeit(synced, 20)
        emit(dict(what="bn_forward_statistics", N=N, H=H, C=C_, M=M, per_rank_us=round(t0 * 1e3, 2), synced_us=round(t1 * 1e3, 2),
                  delta_us=round((t1 - t0) * 1e3, 2)))


def step(emit, steps, rounds):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Conv
    from efficientteacher_b200.parallel import BnSync
    from efficientteacher_b200.trainer import SSODTrainerStep
    import synth
    dev = torch.device("cuda:0")
    bl = bu = 16
    img = 640
    torch.manual_seed(0)
    cfg = yolov5_ssod_cfg('l', batch_size=bl + bu, img_size=img)
    cfg.SSOD.fixed_accumulate = True
    st = SSODTrainerStep(cfg, dev, epochs=300)
    st.ema.updates = 100000
    tg = synth.make_targets(100, 8 * bl, bl)
    imgs = torch.from_numpy(synth.make_images(1, bl, img, tg)).to(dev).float() / 255
    uw = torch.from_numpy(synth.make_images(1001, bu, img)).to(dev).float() / 255
    us = uw.flip(3).contiguous()
    tg, Ms = torch.from_numpy(tg).to(dev), torch.from_numpy(synth.make_Ms(200, bu, img)).to(dev)
    convs = [m for m in st.model.modules() if isinstance(m, Conv)]
    n_bn = len(convs)
    floats = sum(2 * m.conv.out_channels for m in convs)
    emit(dict(what="collectives_per_step_not_measured", model="YOLOv5l", bn_layers=n_bn, all_reduces=2 * n_bn,
              forward_bytes=8 * (floats + n_bn), backward_bytes=4 * floats))
    ni = [0]

    def run(mode, n):
        st.model.set_bn_sync(BnSync(loopback=True) if mode == "loopback" else None)
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(n):
            st.train_instance(imgs, tg, us, uw, None, Ms, ni[0])
            ni[0] += 1
        torch.cuda.synchronize()
        return (time.perf_counter() - t) / n * 1e3
    for mode in ("default", "loopback"):
        run(mode, 8)                        # warm-up of both paths
    res = {"default": [], "loopback": []}
    for _ in range(rounds):
        for mode in ("default", "loopback"):
            res[mode].append(run(mode, steps))
    st.model.set_bn_sync(None)
    d, l = float(np.median(res["default"])), float(np.median(res["loopback"]))
    emit(dict(what="eager_ssod640_step", steps_per_round=steps, rounds=rounds, default_ms=[round(v, 2) for v in res["default"]],
              loopback_ms=[round(v, 2) for v in res["loopback"]], default_median_ms=round(d, 2), loopback_median_ms=round(l, 2),
              delta_pct=round(100 * (l - d) / d, 2), images_per_s_default=round((bl + bu) / d * 1e3, 1),
              images_per_s_loopback=round((bl + bu) / l * 1e3, 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--no-step", action="store_true")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)
    lines = []
    gpu = gpu_info()

    def emit(d):
        d = dict(gpu=gpu, **d)
        lines.append(d)
        print(json.dumps(d), flush=True)
    kernels(emit)
    if not a.no_step:
        step(emit, a.steps, a.rounds)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
