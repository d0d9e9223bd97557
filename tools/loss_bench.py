#!/usr/bin/env python
"""Cost of the loss options (cfg.Loss.fl_gamma / cls_pw / obj_pw / autobalance) on the H100.

Part 1, the loss kernels: etb_loss_forward + etb_loss_backward at the head shapes of bench.py's `sup32` (ComputeLoss,
B = 32) and `ssod640` (ComputeLoss on 16 labeled + ComputeStudentMatchLoss on 16 unlabeled) at 640, Poisson(8) labels (and
pseudo-label rows) per image, for the variants default / focal (fl_gamma 1.5) / pos_weight (cls_pw 2, obj_pw 1.3) /
autobalance / all three.  The target sets are built once; --iters forward+backward pairs are captured in one CUDA graph
and timed with CUDA events over --reps replays, the variants alternated round by round (--rounds); the median per call.

Part 2, the captured training step: bench.py's `sup32` step (YOLOv5l, batch 32, 640) captured with the default loss and
with fl_gamma=1.5 + autobalance, two step objects timed in alternated --steps windows after --warmup steps.

  python tools/loss_bench.py [--iters 10] [--reps 20] [--rounds 5] [--steps 20] [--warmup 5] [--windows 4] [--out FILE]

Prints one JSON line per measurement with the card's name and power limit read in the same run; --out appends them."""
import argparse
import ctypes as C
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

VARIANTS = {
    "default": dict(),
    "focal": dict(fl_gamma=1.5),
    "pos_weight": dict(cls_pw=2.0, obj_pw=1.3),
    "autobalance": dict(autobalance=True),
    "all": dict(fl_gamma=1.5, cls_pw=2.0, obj_pw=1.3, autobalance=True),
}


def card():
    q = "name,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=10).stdout.strip()
        return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
    except Exception as exc:
        return {"unavailable": repr(exc)[:200]}


def poisson_targets(seed, b, mean=8.0):
    import synth
    counts = np.random.RandomState(seed).poisson(mean, b)
    t = synth.make_targets(seed, int(counts.sum()), b)
    t[:, 0] = np.repeat(np.arange(b), counts)
    return t


def poisson_rows(seed, b, mean=8.0):
    import synth
    counts = np.random.RandomState(seed).poisson(mean, b)
    rows = synth.make_pseudo_rows(seed, int(counts.sum()), b)
    rows[:, 0] = np.repeat(np.arange(b), counts)
    return rows


class LossCall:
    """one loss's etb_loss_forward + etb_loss_backward on fixed target sets, as the mirror calls them"""

    def __init__(self, crit, p, targets, ssod):
        from efficientteacher_b200 import _lib
        from efficientteacher_b200._lib import EtbAssignOut
        from efficientteacher_b200.loss import make_loss_params
        self.lib, self._lib = _lib.lib(), _lib
        if ssod:
            sel, cnt = crit._select_device(targets)
            cap = sel.shape[1]
            self.sets = [crit.assigner.assign(p, sel[0, :, :6], nt_dev=cnt[0:1], cap_rows=cap)] + \
                [crit.assigner.assign(p, sel[s], nt_dev=cnt[s:s + 1], cap_rows=cap, with_pseudo_score=True) for s in (1, 2, 3)]
            self.lp = make_loss_params(p, crit.na, crit.balance, crit.box_w, crit.obj_w, crit.cls_w, crit.cp, crit.cn, nsets=4,
                                       ignore_obj=crit.ignore_obj, with_bbox=crit.pseudo_label_with_bbox,
                                       with_cls=crit.pseudo_label_with_cls, cls_pw=crit.cls_pw, obj_pw=crit.obj_pw)
        else:
            self.sets = [crit.assigner.assign(p, targets)]
            bal = crit.balance if crit.balance_state is None else [0.0] * crit.nl
            self.lp = make_loss_params(p, crit.na, bal, crit.box_w, crit.obj_w, crit.cls_w, crit.cp, crit.cn, cls_pw=crit.cls_pw,
                                       obj_pw=crit.obj_pw, fl_gamma=crit.fl_gamma, balance_state=crit.balance_state, ssi=crit.ssi)
        nbytes = self.lib.etb_loss_workspace_bytes(C.byref(self.lp), self.sets[0].cap)
        dev = p[0].device
        self.ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
        self.out4 = torch.empty(4, dtype=torch.float32, device=dev)
        self.gs = torch.ones(1, dtype=torch.float32, device=dev)
        self.grads = [torch.empty_like(t) for t in p]
        self.parr = (C.c_void_p * len(p))(*[t.data_ptr() for t in p])
        self.garr = (C.c_void_p * len(p))(*[t.data_ptr() for t in self.grads])
        self.sarr = (EtbAssignOut * len(self.sets))(*[s.struct for s in self.sets])

    def __call__(self):
        L, lp, st = self._lib, C.byref(self.lp), self._lib.stream_ptr()
        L.check(self.lib.etb_loss_forward(self.parr, lp, self.sarr, L.ptr(self.out4), L.ptr(self.ws), self.ws.numel(), st),
                "etb_loss_forward")
        L.check(self.lib.etb_loss_backward(self.parr, self.garr, lp, self.sarr, L.ptr(self.gs), L.ptr(self.ws), self.ws.numel(),
                                           st), "etb_loss_backward")


def kernel_legs(args, dev, emit, info):
    import synth
    from efficientteacher_b200.loss import ComputeLoss
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import HeadOnlyModel, ssod_cfg
    shapes = dict(sup32=(32, 0), ssod640=(16, 16))
    for name, (bl, bu) in shapes.items():
        pl = [torch.from_numpy(x).to(dev) for x in synth.make_head_logits(11, bl)]
        tl = torch.from_numpy(poisson_targets(1000, bl)).to(dev)
        pu = [torch.from_numpy(x).to(dev) for x in synth.make_head_logits(12, bu)] if bu else None
        tu = torch.from_numpy(poisson_rows(2000, bu)).to(dev) if bu else None
        graphs, nlabels = {}, int(tl.shape[0])
        for var, opt in VARIANTS.items():
            cfg = ssod_cfg()
            for k, v in opt.items():
                setattr(cfg.Loss, k, v)
            calls = [LossCall(ComputeLoss(HeadOnlyModel().to(dev), cfg), pl, tl, False)]
            if bu:
                calls.append(LossCall(ComputeStudentMatchLoss(HeadOnlyModel().to(dev), cfg), pu, tu, True))
            for c in calls:
                c()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(args.iters):
                    for c in calls:
                        c()
            graphs[var] = (g, calls)
        times = {v: [] for v in VARIANTS}
        order = list(VARIANTS)
        for rnd in range(args.rounds):
            for var in (order if rnd % 2 == 0 else order[::-1]):
                g = graphs[var][0]
                g.replay()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    g.replay()
                e1.record()
                torch.cuda.synchronize()
                times[var].append(e0.elapsed_time(e1) * 1e3 / (args.reps * args.iters))
        base = float(np.median(times["default"]))
        for var in VARIANTS:
            med = float(np.median(times[var]))
            emit(part="loss_kernels", shape=name, variant=var, options=VARIANTS[var], labeled=bl, unlabeled=bu, img=640,
                 labels=nlabels, us_per_fwd_bwd_median=round(med, 2), us_per_round=[round(t, 2) for t in times[var]],
                 vs_default=round(med / base, 4), iters_per_graph=args.iters, replays=args.reps, **info)
        del graphs
        gc.collect()
        torch.cuda.empty_cache()


def step_legs(args, dev, emit, info):
    from bench import NB, synth_batch
    from tools.size_bench import _steady_state
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.trainer import SupTrainerStep
    bl, img = 32, 640
    host = synth_batch(0, bl=bl, bu=0, img=img)
    imgs = host["imgs"].to(dev).float() / 255.0
    tg = host["targets"].to(dev)
    steps = {}
    for var in ("default", "focal_autobalance"):
        torch.manual_seed(0)
        cfg = yolov5_sup_cfg('l', batch_size=bl, img_size=img)
        if var != "default":
            cfg.Loss.fl_gamma, cfg.Loss.autobalance = 1.5, True
        st = SupTrainerStep(cfg, dev, epochs=300, nb=NB)
        _steady_state(st, imgs)
        steps[var] = dict(st=st, ni=0, rates=[])
    def window(s, k):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(k):
            loss = s["st"].train_step_graphed(imgs, tg, s["ni"])
            s["ni"] += 1
        e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(loss).all()
        return bl * k / (e0.elapsed_time(e1) / 1e3)
    for s in steps.values():
        window(s, args.warmup)
    for w in range(args.windows):
        for var in (list(steps) if w % 2 == 0 else list(steps)[::-1]):
            steps[var]["rates"].append(round(window(steps[var], args.steps), 1))
    base = float(np.median(steps["default"]["rates"]))
    for var, s in steps.items():
        med = float(np.median(s["rates"]))
        emit(part="captured_step", config="sup32", variant=var, images_per_s_per_window=s["rates"], images_per_s_median=med,
             vs_default=round(med / base, 4), steps_per_window=args.steps, warmup=args.warmup, captures=s["st"].captures,
             balance_after=(s["st"].compute_loss.balance if s["st"].compute_loss.autobalance else None), **info)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10, help="forward+backward pairs per captured graph")
    ap.add_argument("--reps", type=int, default=20, help="graph replays per timed round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, default=4)
    ap.add_argument("--no-step", action="store_true", help="only the loss-kernel part")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    info = dict(card=card(), torch=torch.__version__)

    def emit(**kw):
        line = json.dumps(kw)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
    kernel_legs(args, dev, emit, info)
    if not args.no_step:
        step_legs(args, dev, emit, info)


if __name__ == "__main__":
    main()
