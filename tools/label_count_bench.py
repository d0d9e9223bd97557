#!/usr/bin/env python
"""Images/s of the YOLOv5l 640 steps when every labeled batch has its own label count, as a real loader delivers them.

Workloads (bench.py's): `ssod640` (SSOD step, 16 labeled + 16 unlabeled) and `sup32` (supervised step, batch 32).  The label
count of every image is drawn from a seeded Poisson with mean 8 (bench.py feeds a fixed 8 per image), over a cycle of
--label-sets batches.  Legs, alternated window by window on one step object:
  eager         train_instance / train_step;
  graph_fixed   the captured step (train_instance_graphed / train_step_graphed) with bench.py's fixed 8 labels per image;
  graph         the captured step with the varying label counts;
  graph_labelmatch  (ssod640 only) the captured step of a second SSOD step with pseudo_label_type = 'LabelMatch'.
Every leg takes its batches (pinned uint8 images, labels, affine matrices) through trainer.DevicePrefetcher, as a training
loop would.  With --pad-labels (for a tree whose prefetcher cannot take a changing label count) the labels go through
padded to the largest count and are sliced after get(); the line says which ("labels_through").  Set-up, teacher
calibration (re-done before each SSOD window) and the batches are bench.py's / tools/size_bench.py's.

Only the public step methods are called, so the script also measures another tree of this project: --root DIR imports the
package, bench.py and tools/ from DIR (built by DIR's own build()).  Captures are counted from the identity of the step's
captured-graph record, which both trees keep in `_graph`.

  python tools/label_count_bench.py [--root DIR] [--tag NAME] [--configs ssod640,sup32] [--steps K] [--warmup W]
                                    [--windows R] [--no-labelmatch] [--pad-labels] [--out FILE]

Prints one JSON line per (config, leg), each with the card's name and power limit read in the same run; --out appends
them to FILE."""
import argparse
import gc
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def poisson_targets(seed, bl, mean=8.0):
    """[n,6] labels whose per-image counts are Poisson(mean) draws (boxes / classes from synth.make_targets)"""
    import synth
    counts = np.random.RandomState(seed).poisson(mean, bl)
    t = synth.make_targets(seed, int(counts.sum()), bl)
    t[:, 0] = np.repeat(np.arange(bl), counts)
    return t


class Feeder:
    """batches through DevicePrefetcher: put() one step ahead, get() / release() around the step"""

    def __init__(self, dev, host, keys, label_sets, pad_labels):
        from efficientteacher_b200.trainer import DevicePrefetcher
        self.pf, self.host, self.keys, self.sets = DevicePrefetcher(dev), host, keys, label_sets
        self.pad = max(int(t.shape[0]) for t in label_sets)
        self.grows = not pad_labels
        self.i, self.counts = 0, []           # batches put so far / label counts of the batches put and not yet handed out
        if not self.grows:
            padded = []
            for t in label_sets:
                p = torch.zeros((self.pad, 6), dtype=t.dtype).pin_memory()
                p[:t.shape[0]] = t
                padded.append(p)
            self.padded = padded

    def _batch(self, i):
        k = i % len(self.sets)
        b = {key: self.host[key] for key in self.keys}
        b["targets"] = self.sets[k] if self.grows else self.padded[k]
        return b, int(self.sets[k].shape[0])

    def get(self):
        if self.pf.pending == 0:
            self._put()
        b = dict(self.pf.get())      # a tree whose get() returns the slot's own dict must not see the slice below
        n = self.counts.pop(0)
        if not self.grows:
            b["targets"] = b["targets"][:n]
        return b

    def _put(self):
        b, n = self._batch(self.i)
        self.counts.append(n)
        self.pf.put(b)
        self.i += 1

    def done(self):
        self.pf.release()
        self._put()


def run_config(name, dev, args, emit):
    from bench import CONFIGS, NB, synth_batch
    from tools.size_bench import _calibrate_teacher, _steady_state
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    cb = CONFIGS[name]
    bl, bu, img, ssod = cb["bl"], cb["bu"], cb["img"], cb["kind"] == "ssod"
    host = synth_batch(0, pinned=True, bl=bl, bu=bu, img=img)
    keys = ("imgs", "u_strong", "u_weak", "Ms") if ssod else ("imgs",)
    varying = [torch.from_numpy(poisson_targets(1000 + i, bl)).pin_memory() for i in range(args.label_sets)]
    counts = [int(t.shape[0]) for t in varying]
    f01 = lambda t: t.to(dev).float() / 255.0  # noqa: E731
    uw = f01(host["u_weak"]) if ssod else None

    def make(labelmatch):
        torch.manual_seed(0)
        if ssod:
            cfg = yolov5_ssod_cfg('l', batch_size=bl + bu, img_size=img)
            cfg.SSOD.fixed_accumulate = True
            if labelmatch:
                cfg.SSOD.pseudo_label_type = "LabelMatch"
                cfg.SSOD.resample_high_percent, cfg.SSOD.resample_low_percent = 0.0, 0.0
            st = SSODTrainerStep(cfg, dev, epochs=300, nb=NB)
            st.ema.updates = 100000
            _steady_state(st, torch.cat([f01(host["imgs"]), f01(host["u_strong"])], 0))
            _calibrate_teacher(st, uw, cfg.SSOD.nms_conf_thres, True)
        else:
            cfg = yolov5_sup_cfg('l', batch_size=bl, img_size=img)
            st = SupTrainerStep(cfg, dev, epochs=300, nb=NB)
            _steady_state(st, f01(host["imgs"]))
        return st, cfg

    def leg_fn(st, graphed):
        if ssod:
            f = st.train_instance_graphed if graphed else st.train_instance
            return lambda b, ni: f(b["imgs"], b["targets"], b["u_strong"], b["u_weak"], None, b["Ms"], ni)
        f = st.train_step_graphed if graphed else st.train_step
        return lambda b, ni: f(b["imgs"], b["targets"], ni)

    legs = [("eager", False, varying), ("graph_fixed", False, [host["targets"]]), ("graph", False, varying)]
    if ssod and not args.no_labelmatch:
        legs.append(("graph_labelmatch", True, varying))
    steps = {}
    for labelmatch in sorted({lm for _, lm, _ in legs}):
        gc.collect()
        torch.cuda.empty_cache()
        st, cfg = make(labelmatch)
        mine = [(n, sets) for n, lm, sets in legs if lm == labelmatch]
        state = {n: dict(feeder=Feeder(dev, host, keys, sets, args.pad_labels), fn=leg_fn(st, n != "eager"), rates=[], captures=[], peak=0.0)
                 for n, sets in mine}
        ni = 0

        def window(leg, k):
            nonlocal ni
            s = state[leg]
            if ssod:
                _calibrate_teacher(st, uw, cfg.SSOD.nms_conf_thres, False)     # outside the timed region, as bench.py
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            caps, last = 0, st._graph
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(k):
                b = s["feeder"].get()
                loss = s["fn"](b, ni)
                s["feeder"].done()
                ni += 1
                if st._graph is not last:
                    caps, last = caps + 1, st._graph
            ev1.record()
            torch.cuda.synchronize()
            assert torch.isfinite(loss).all(), (name, leg)
            s["peak"] = max(s["peak"], torch.cuda.max_memory_allocated() / 2 ** 30)
            s["cap"] = st._graph.get("cap") if leg != "eager" and st._graph is not None else None   # None: a tree without one
            return (bl + bu) * k / (ev0.elapsed_time(ev1) / 1e3), caps

        for leg, _ in mine:
            state[leg]["warmup_captures"] = window(leg, args.warmup)[1]
        for _ in range(args.windows):
            for leg, _ in mine:
                rate, caps = window(leg, args.steps)
                state[leg]["rates"].append(round(rate, 1))
                state[leg]["captures"].append(caps)
        for leg, _ in mine:
            s = state[leg]
            steps[leg] = dict(config=name, leg=leg, images_per_s_per_window=s["rates"],
                              images_per_s_median=float(np.median(s["rates"])), captures_per_window=s["captures"],
                              captures_in_warmup=s["warmup_captures"], steps_per_window=args.steps, warmup=args.warmup,
                              peak_mem_gb=round(s["peak"], 2), labels_through="DevicePrefetcher" if s["feeder"].grows else
                              "DevicePrefetcher, padded to %d rows and sliced after get()" % s["feeder"].pad,
                              label_counts=("fixed %d per image" % (int(host["targets"].shape[0]) // bl)) if leg == "graph_fixed" else
                              dict(per_image="Poisson(8), seeded", batches=len(counts), min=min(counts), max=max(counts),
                                   mean_per_image=round(float(np.mean(counts)) / bl, 2)),
                              label_capacity_after_last_window=s["cap"])
            emit(**steps[leg])
        del st, state
    return steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=HERE, help="tree of this project to measure (default: the one this script is in)")
    ap.add_argument("--tag", default="", help="name of the tree in the output lines")
    ap.add_argument("--configs", default="ssod640,sup32")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--label-sets", type=int, default=40, help="distinct labeled batches, cycled")
    ap.add_argument("--no-labelmatch", action="store_true", help="skip the LabelMatch leg")
    ap.add_argument("--pad-labels", action="store_true",
                    help="put the labels through the prefetcher padded to the largest count and slice them after get() "
                         "(for a tree whose DevicePrefetcher needs fixed shapes)")
    ap.add_argument("--out", default="", help="append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("label_count_bench.py measures on a CUDA device; none found")
    root = os.path.abspath(args.root)
    sys.path.insert(0, os.path.join(root, "tests"))
    sys.path.insert(0, root)
    import __graft_entry__ as g
    g.build()
    import efficientteacher_b200
    assert os.path.dirname(os.path.abspath(efficientteacher_b200.__file__)).startswith(root), efficientteacher_b200.__file__
    from tools.burnin_bench import card
    info = dict(card(), torch=torch.__version__)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)

    def emit(**kw):
        line = json.dumps(dict(tree=args.tag or root, **kw, card=info))
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")

    for name in args.configs.split(","):
        run_config(name, dev, args, emit)


if __name__ == "__main__":
    main()
