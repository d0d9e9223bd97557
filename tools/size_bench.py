#!/usr/bin/env python
"""Throughput of every YOLOv5 size the reference ships (n, s, m, l, x) on one GPU:
  1. the captured supervised step, 32 images at 640;
  2. the captured SSOD step, 16 labeled + 16 unlabeled images at 640 (the per-GPU batch is halved until it fits);
  3. the same SSOD step with stock PyTorch eager (oracle/eager_ref.EagerSSODStep through bench.gpu_eager_baseline: same
     weights, same batch);
  4. the training BatchNorm kernels at a YOLOv5m / YOLOv5l width pair (96 / 128) and a YOLOv5x / YOLOv5l pair (160 / 256) on
     the batch-32 maps of 640-pixel images, as a share of the H100 SXM's 3.35 TB/s HBM bandwidth.
Each step is set up like bench.py's: BatchNorm running statistics from one pass over the synthetic batch, teacher = student,
and bench.py's teacher calibration (objectness logits widened to std 3, then the bias placed so about 2 % of the 25 200
predictions per image are NMS candidates; the teacher is re-calibrated before each timed window of --window steps and
before the eager step).  Every SSOD line reports the measured candidates per image, at the start and end of each window, and
whether each window meets bench.py's load rule.

  python tools/size_bench.py [--steps K] [--warmup W] [--window S] [--sizes n,s,m,l,x] [--no-bn]

Prints one JSON line per result, each with the card's name and power limit read in the same run."""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BPS = 3.35e12            # H100 SXM data sheet
CARD = {}


def emit(**kw):
    print(json.dumps(dict(card=CARD, **kw)), flush=True)


def _steady_state(st, imgs):
    """bench.py's synthetic steady state: running statistics = batch statistics of the data, teacher(s) = student"""
    with torch.no_grad():
        bns = [m for m in st.model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
        for m in bns:
            m.momentum = 1.0
        with torch.autocast("cuda", dtype=torch.bfloat16):
            st.model(imgs.contiguous(memory_format=torch.channels_last))
        for m in bns:
            m.momentum = 0.03
        for e in (st.ema, getattr(st, "semi_ema", None)):
            if e is not None:
                e.ema.load_state_dict(st.model.state_dict())


def _calibrate_teacher(st, uw, conf_thres, first):
    """bench.py's teacher calibration: (2a) scale the three objectness rows of every head conv so the teacher's objectness
    logits have std 3 (a random-init head gives ~0.15, which would put nearly every prediction above the NMS threshold),
    (2b) set the objectness bias so the 98th percentile is obj = 0.3, and on the first call (2c) raise the class biases
    by 8 and give the student and semi-teacher heads the same values.  bench.py scales only on its first call; here every
    call scales the teacher (a no-op once the std is 3), because the EMA moves a random-init YOLOv5x teacher's logit
    spread within 20 steps and the bias alone then no longer holds the load.  Returns the NMS candidates per image
    (objectness above conf_thres) of the calibrated teacher on uw."""
    with torch.no_grad():
        (_, raw), _ = st.ema.ema(uw)
        for l, m in enumerate(st.ema.ema.head.m):
            b = m.bias.view(3, -1)
            w = m.weight.view(3, -1, m.weight.shape[1])
            lin = (raw[l][..., 4].float() - b[:, 4].float().view(1, 3, 1, 1)).flatten()
            sc = 3.0 / max(float(lin.std()), 1e-6)
            q98 = torch.quantile(sc * lin[:2_000_000], 0.98).item()
            w[:, 4] *= sc
            b[:, 4] = float(np.log(0.3 / 0.7)) - q98
            if first:
                b[:, 5:] += 8.0
                for other in (st.model, st.semi_ema.ema):
                    other.head.m[l].bias.data.copy_(m.bias.data)
                    other.head.m[l].weight.data.copy_(m.weight.data)
        return _candidates(st, uw, conf_thres)


def _candidates(st, uw, conf_thres):
    with torch.no_grad():
        (pred, _), _ = st.ema.ema(uw)
        return round(float((pred[..., 4] > conf_thres).sum(1).float().mean().item()), 1)


def _time(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(warmup, warmup + steps):
        loss = fn(i)
    e.record()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    return s.elapsed_time(e) / steps


def sup_step(size, dev, steps, warmup):
    from bench import NB, synth_batch
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.trainer import SupTrainerStep
    torch.manual_seed(0)
    host = synth_batch(0, bl=32, bu=0, img=640)
    imgs, tg = host["imgs"].to(dev).float() / 255.0, host["targets"].to(dev)
    st = SupTrainerStep(yolov5_sup_cfg(size, batch_size=32, img_size=640), dev, epochs=300, nb=NB)
    _steady_state(st, imgs)
    ms = _time(lambda i: st.train_step_graphed(imgs, tg, i), steps, warmup)
    emit(size=size, step="sup", batch="32", img=640, images_per_s=round(32 / (ms / 1e3), 1), ms_per_step=round(ms, 2),
         steps=steps, warmup=warmup, peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 1))


def ssod_steps(size, dev, steps, warmup, window, bl):
    from bench import NB, gpu_eager_baseline, synth_batch
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep
    torch.manual_seed(0)
    host = synth_batch(0, bl=bl, bu=bl, img=640)
    f01 = lambda t: t.to(dev).float() / 255.0  # noqa: E731
    imgs, uw, us = f01(host["imgs"]), f01(host["u_weak"]), f01(host["u_strong"])
    tg, Ms = host["targets"].to(dev), host["Ms"].to(dev)
    cfg = yolov5_ssod_cfg(size, batch_size=2 * bl, img_size=640)
    cfg.SSOD.fixed_accumulate = True
    st = SSODTrainerStep(cfg, dev, epochs=300, nb=NB)
    st.ema.updates = 100000
    _steady_state(st, torch.cat([imgs, us], 0))
    thr = cfg.SSOD.nms_conf_thres
    first = _calibrate_teacher(st, uw, thr, True)
    f = lambda i: st.train_instance_graphed(imgs, tg, us, uw, None, Ms, i)  # noqa: E731
    for i in range(warmup):
        f(i)
    # timed windows of at most `window` steps, the teacher re-calibrated before each (bench.py does so before its timed
    # window): a random-init teacher's candidate load drifts as the EMA moves it, by ~3x over 20 YOLOv5x steps
    ms_total, loads, ni = 0.0, [], warmup
    while ni < warmup + steps:
        n = min(window, warmup + steps - ni)
        start = _calibrate_teacher(st, uw, thr, False)
        ms_total += _time(lambda i: f(ni + i), n, 0) * n
        loads.append((start, _candidates(st, uw, thr)))
        ni += n
    ms = ms_total / steps
    native = 2 * bl / (ms / 1e3)
    load = dict(predictions_per_img=int(sum(3 * (640 // s) ** 2 for s in (8, 16, 32))), nms_candidates_per_img_after_first_calibration=first,
                nms_candidates_per_img_start_end_of_timed_windows=loads,
                load_valid=all(c0 > 0 and 0.5 * c0 <= c1 <= 2.0 * c0 for c0, c1 in loads),
                load_rule="bench.py's: NMS candidates/img at the end of each timed window within [0.5, 2] x its start")
    emit(size=size, step="ssod", impl="native graphed", batch="%d+%d" % (bl, bl), img=640, images_per_s=round(native, 1),
         ms_per_step=round(ms, 2), steps=steps, window=window, warmup=warmup,
         pseudo_label_rows_last_step=int(st.pseudo_label_creator.last_count_dev.item()),
         peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), **load)
    st.model.zero_grad(set_to_none=True)
    cand_eager = _calibrate_teacher(st, uw, thr, False)       # the eager step starts from the same teacher load
    eg = gpu_eager_baseline(st, host, dict(bl=bl, bu=bl), dev)
    emit(size=size, step="ssod", impl="eager PyTorch", batch="%d+%d" % (bl, bl), img=640, images_per_s=round(eg["value"], 1),
         ms_per_step=round(eg["ms_per_step"], 2), steps=eg["steps"], warmup=eg["warmup"], what=eg["what"],
         nms_candidates_per_img_at_start=cand_eager, pseudo_label_rows_last_step=eg["pseudo_label_rows_last_step"],
         native_over_eager=round(native / eg["value"], 2))


def bn_kernels(dev):
    from efficientteacher_b200 import _lib, convops as co
    from tools.conv_bench import timeit
    lib = _lib.lib()
    for C_ in (96, 128, 160, 256):
        for H in (160, 80):
            N, M = 32, 32 * H * H
            g = torch.Generator(device=dev).manual_seed(0)
            y = (torch.randn(N, H, H, C_, device=dev, generator=g) * 2.0).to(torch.bfloat16)
            da = torch.randn(N, H, H, C_, device=dev, generator=g).to(torch.bfloat16)
            gamma, beta = torch.ones(C_, device=dev), torch.zeros(C_, device=dev)
            out = torch.empty_like(y)
            _, stats = co.bn_forward(y, C_, gamma, beta, None, None, 1e-3, 0.03, "silu", out=out)
            rows0, rows1 = int(lib.etb_bn_partial_rows(M, C_, 0)), int(lib.etb_bn_partial_rows(M, C_, 1))
            part0, part1 = torch.empty(rows0, 2, C_, device=dev), torch.empty(rows1, 2, C_, device=dev)
            sums = torch.zeros(2 * C_, dtype=torch.float32, device=dev)
            p = [_lib.ptr(t) for t in (y, da, stats[0], stats[1], stats[2], stats[3], out, part1, sums, part0)]
            a, s = co.ACT["silu"], _lib.stream_ptr()
            kern = {"stats": (lambda: lib.etb_bn_stats(p[0], M, C_, C_, p[9], rows0, s), 2),
                    "apply": (lambda: lib.etb_bn_act_apply_res(p[0], p[2], p[3], None, p[6], M, C_, C_, 0, C_, a, s), 4),
                    "bwd_reduce": (lambda: lib.etb_bn_act_bwd_reduce(p[1], p[0], p[2], p[3], p[4], p[5], M, C_, C_, C_, a, p[7], rows1, s), 4),
                    "bwd_apply": (lambda: lib.etb_bn_act_bwd_apply(p[1], p[0], p[2], p[3], p[4], p[5], p[8], M, C_, C_, C_, C_, a, p[6], s), 6)}
            for name, (fn, bytes_per_elem) in kern.items():
                ms = timeit(fn)
                emit(bn_kernel=name, C=C_, N=N, H=H, W=H, act="silu", us=round(ms * 1e3, 2),
                     hbm_fraction=round(bytes_per_elem * M * C_ / (ms / 1e3) / HBM_BPS, 3),
                     pow2=(C_ // 8) & (C_ // 8 - 1) == 0)
            del y, da, out, part0, part1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--window", type=int, default=5, help="SSOD steps per timed window (teacher load re-placed before each)")
    ap.add_argument("--sizes", default="n,s,m,l,x")
    ap.add_argument("--no-bn", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("size_bench.py measures on a CUDA device; none found")
    import __graft_entry__ as g
    g.build()
    from tools.burnin_bench import card
    CARD.update(card())
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    if not args.no_bn:
        bn_kernels(dev)
    for size in args.sizes.split(","):
        for kind in ("sup", "ssod"):
            bl = 16
            while True:
                gc.collect()
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                try:
                    if kind == "sup":
                        sup_step(size, dev, args.steps, args.warmup)
                    else:
                        ssod_steps(size, dev, args.steps, args.warmup, args.window, bl)
                    break
                except torch.cuda.OutOfMemoryError:
                    if kind == "sup" or bl == 1:
                        emit(size=size, step=kind, images_per_s="not measured", reason="out of memory")
                        break
                    emit(size=size, step=kind, batch="%d+%d" % (bl, bl), images_per_s="not measured", reason="out of memory")
                    bl //= 2


if __name__ == "__main__":
    main()
