#!/usr/bin/env python
"""Images/s of the SSOD burn-in step (SSODTrainerStep.train_without_unlabeled, trainer/ssod_trainer.py:421-456) on one GPU:
YOLOv5l, 640, 32 labeled images per step, optimizer + EMA every step; eager launches vs the captured graphs.

  python tools/burnin_bench.py [--steps K] [--warmup W] [--batches N] [--repeats R] [--da]

The graphed step is first fed N batches whose label counts vary (0 .. 16 per image) and the number of captures this takes
is reported; a graph keyed on the label count would capture once per distinct count.  The timed windows alternate eager
and graphed (R windows each, K steps per window, device events around the window) and cycle through the same label sets.
`native_launches_per_step` counts the project's kernel launches issued from the host per step (a replayed graph issues none).
Prints one JSON line with the card's name, power limit and the SM clock sampled during the timed windows."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=10).stdout.strip()
        return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
    except Exception as exc:
        return {"unavailable": repr(exc)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batches", type=int, default=50, help="batches with varying label counts fed to the graphed step")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--img", type=int, default=640)
    ap.add_argument("--da", action="store_true", help="train_without_unlabeled_da with as many weak unlabeled images")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("burnin_bench.py measures on a CUDA device; none found")
    import __graft_entry__ as g
    g.build()
    import synth
    from bench import ClockSampler
    from efficientteacher_b200 import _lib
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    lib = _lib.lib()
    B, img = args.batch, args.img
    bu = B if args.da else 0
    torch.manual_seed(0)
    cfg = yolov5_ssod_cfg('l', batch_size=B + bu, img_size=img)
    cfg.hyp.burn_epochs = 220                   # configs/ssod/coco-standard/yolov5l_coco_ssod_{1,2,5}_percent.yaml
    cfg.SSOD.with_da_loss = args.da
    cfg.SSOD.fixed_accumulate = True            # optimizer + EMA every iteration, as bench.py
    st = SSODTrainerStep(cfg, dev, epochs=300, nb=369)
    r = np.random.RandomState(0)
    counts = [0] + [int(c) for c in r.randint(0, 16 * B + 1, args.batches - 1)]
    tgs = [torch.from_numpy(synth.make_targets(500 + i, n, B)).pin_memory() for i, n in enumerate(counts)]
    imgs = torch.from_numpy(synth.make_images(1, B, img, tgs[1].numpy())).to(dev)       # uint8, read in place by the stem
    uw = torch.from_numpy(synth.make_images(2, bu, img)).to(dev) if args.da else None
    ni = 0

    def step(graphed, i):
        tg = tgs[i % len(tgs)]
        if args.da:
            f = st.train_without_unlabeled_da_graphed if graphed else st.train_without_unlabeled_da
            return f(imgs, tg, uw, i)
        f = st.train_without_unlabeled_graphed if graphed else st.train_without_unlabeled
        return f(imgs, tg, i)

    for _ in range(args.warmup):
        step(False, ni); ni += 1
    torch.cuda.synchronize()
    l0 = lib.etb_launch_count()
    for _ in range(3):
        step(False, ni); ni += 1
    torch.cuda.synchronize()
    launches_eager = (lib.etb_launch_count() - l0) / 3
    for i in range(args.batches):               # every label set once through the graphed step
        loss = step(True, ni); ni += 1
        assert torch.isfinite(loss).all(), i
    torch.cuda.synchronize()
    captures = st.burn_in_captures
    l0 = lib.etb_launch_count()
    for _ in range(3):
        step(True, ni); ni += 1
    torch.cuda.synchronize()
    launches_graph = (lib.etb_launch_count() - l0) / 3

    def window(graphed):
        nonlocal ni
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.steps):
            step(graphed, ni); ni += 1
        e.record()
        torch.cuda.synchronize()
        return (B + bu) * args.steps / (s.elapsed_time(e) / 1e3)

    sampler = ClockSampler(0)
    sampler.start()
    rates = {"eager": [], "graph": []}
    for _ in range(args.repeats):
        for graphed in (False, True):
            rates["graph" if graphed else "eager"].append(window(graphed))
    clocks = sampler.summary()
    loss = float(step(True, ni).item())
    assert np.isfinite(loss) and st.burn_in_captures == captures
    eager, graph = float(np.median(rates["eager"])), float(np.median(rates["graph"]))
    print(json.dumps({
        "metric": "images/s YOLOv5l SSOD burn-in step (train_without_unlabeled%s) @%d, %d labeled%s" % (
            "_da" if args.da else "", img, B, " + %d unlabeled" % bu if bu else ""),
        "eager_images_per_s": eager, "graph_images_per_s": graph, "graph_over_eager": graph / eager,
        "windows_images_per_s": rates, "steps_per_window": args.steps,
        "native_launches_per_step": {"eager": launches_eager, "graph_replay": launches_graph},
        "captures": {"batches": args.batches, "count": captures, "label_counts_min_max": [min(counts), max(counts)],
                     "label_capacity": st._burn_graph["cap"]},
        "last_loss": loss, "card": card(), "clocks": clocks,
    }), flush=True)


if __name__ == "__main__":
    main()
