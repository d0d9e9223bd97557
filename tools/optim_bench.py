#!/usr/bin/env python
"""The optimizer of `adam: True`: FusedAdamW (csrc/adamw.cu) against torch.optim.AdamW, and what it costs the whole step.

Part 1, the optimizer step alone, over the parameters of the YOLOv5l SSOD student and of the supervised student, in the
reference's three groups (TrainerStep.build_optimizer):
  native          FusedAdamW.step()  (one launch; also zeroes the gradients)
  torch_foreach   torch.optim.AdamW (the default implementation) step() + zero_grad(set_to_none=False), so both legs end
                  with zeroed gradients; the step alone is reported too
  torch_fused     torch.optim.AdamW(fused=True), the same two numbers
Times are CUDA events over --iters back-to-back steps after --warmup; the HBM fraction is 32 B per parameter (read p, g,
m, v; write p, m, v, g) over the time, against the H100 SXM data-sheet 3.35 TB/s.

Part 2, the captured training steps ssod640 and sup32 (bench.py's set-up, imported as is: synthetic batch, steady state,
teacher calibration), `adam` off and on, alternated --windows times, images/s over --steps replays after --warmup.

  python tools/optim_bench.py [--iters N] [--warmup W] [--steps K] [--windows R] [--no-steps] [--out FILE]

Prints one JSON line per measurement with the card's name and power limit read in the same run; --out appends them."""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (HERE, os.path.join(HERE, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet
BYTES_PER_PARAM = 32


def _groups(kind, dev):
    """the reference's [bias, conv weight, BN weight] groups of the YOLOv5l student, as TrainerStep.build_optimizer builds them"""
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.model import Model, SupModel
    from efficientteacher_b200.trainer import TrainerStep
    cfg = yolov5_ssod_cfg('l', batch_size=32) if kind == "ssod" else yolov5_sup_cfg('l', batch_size=32)
    cfg.adam = True
    st = TrainerStep.__new__(TrainerStep)
    st.model, st.epochs, st.epoch, st.batch_size = (Model(cfg) if kind == "ssod" else SupModel(cfg)).to(dev), 300, 0, 32
    st.build_optimizer(cfg)
    return [dict(params=g["params"], weight_decay=g["weight_decay"]) for g in st.optimizer.param_groups], cfg


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters      # us per call


def optimizer_legs(kind, dev, args, emit):
    from efficientteacher_b200.optim import FusedAdamW
    groups, cfg = _groups(kind, dev)
    params = [p for g in groups for p in g["params"]]
    n = sum(p.numel() for p in params)
    gen = torch.Generator(device=dev).manual_seed(0)
    for p in params:
        p.grad = torch.randn(p.shape, device=dev, generator=gen) * 1e-3

    def make(which):
        gs = [dict(g) for g in groups]
        kw = dict(lr=cfg.hyp.lr0, betas=(cfg.hyp.momentum, 0.999))
        if which == "native":
            return FusedAdamW(gs, **kw)
        return torch.optim.AdamW(gs, fused=(which == "torch_fused"), **kw)

    for which in ("native", "torch_foreach", "torch_fused"):
        opt = make(which)
        if which == "native":
            us = {"step_and_zero_grad": _time(opt.step, args.iters, args.warmup)}
        else:
            def both(o=opt):
                o.step()
                o.zero_grad(set_to_none=False)
            us = {"step_and_zero_grad": _time(both, args.iters, args.warmup), "step": _time(opt.step, args.iters, args.warmup)}
        t = us["step_and_zero_grad"]
        emit(part="optimizer", model="YOLOv5l %s student" % kind, impl=which, params=n, tensors=len(params),
             us={k: round(v, 1) for k, v in us.items()},
             hbm_fraction_at_32B_per_param=round(n * BYTES_PER_PARAM / (t * 1e-6) / HBM_BYTES_PER_S, 3),
             iters=args.iters, warmup=args.warmup)
        del opt
        gc.collect()
        torch.cuda.empty_cache()


def step_legs(name, dev, args, emit):
    from bench import CONFIGS, NB, synth_batch
    from tools.size_bench import _calibrate_teacher, _steady_state
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    cb = CONFIGS[name]
    bl, bu, img, ssod = cb["bl"], cb["bu"], cb["img"], cb["kind"] == "ssod"
    host = synth_batch(0, pinned=True, bl=bl, bu=bu, img=img)
    b = {k: v.to(dev) for k, v in host.items()}
    f01 = lambda t: t.float() / 255.0  # noqa: E731
    rates = {False: [], True: []}
    for _ in range(args.windows):
        for adam in (False, True):
            gc.collect()
            torch.cuda.empty_cache()
            torch.manual_seed(0)
            if ssod:
                cfg = yolov5_ssod_cfg('l', batch_size=bl + bu, img_size=img)
                cfg.adam = adam
                st = SSODTrainerStep(cfg, dev, epochs=300, nb=NB)
                st.ema.updates = 100000
                _steady_state(st, torch.cat([f01(b["imgs"]), f01(b["u_strong"])], 0))
                _calibrate_teacher(st, f01(b["u_weak"]), cfg.SSOD.nms_conf_thres, True)
                f = lambda ni: st.train_instance_graphed(b["imgs"], b["targets"], b["u_strong"], b["u_weak"], None, b["Ms"], ni)  # noqa: E731
            else:
                cfg = yolov5_sup_cfg('l', batch_size=bl, img_size=img)
                cfg.adam = adam
                st = SupTrainerStep(cfg, dev, epochs=300, nb=NB)
                _steady_state(st, f01(b["imgs"]))
                f = lambda ni: st.train_step_graphed(b["imgs"], b["targets"], ni)  # noqa: E731
            for ni in range(args.warmup):
                f(ni)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for ni in range(args.warmup, args.warmup + args.steps):
                loss = f(ni)
            e1.record()
            torch.cuda.synchronize()
            assert torch.isfinite(loss).all(), (name, adam)
            rates[adam].append(round((bl + bu) * args.steps / (e0.elapsed_time(e1) / 1e3), 1))
            del st, f
    for adam in (False, True):
        emit(part="step", config=name, adam=adam, images_per_s_per_window=rates[adam],
             images_per_s_median=float(np.median(rates[adam])), steps_per_window=args.steps, warmup=args.warmup,
             schedule="reference warm-up from ni=0 (optimizer every step)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=2)
    ap.add_argument("--no-steps", action="store_true", help="part 1 only")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim_bench needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from tools.burnin_bench import card
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    info = dict(card(), torch=torch.__version__)

    def emit(**kw):
        line = json.dumps(dict(**kw, card=info))
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(line + "\n")

    for kind in ("ssod", "sup"):
        optimizer_legs(kind, dev, args, emit)
    if not args.no_steps:
        for name in ("ssod640", "sup32"):
            step_legs(name, dev, args, emit)


if __name__ == "__main__":
    main()
