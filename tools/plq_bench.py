"""Pseudo-label quality statistics: time of the native mirror against the CPU restatement, and the cost the statistics and
the meter add to the SSOD step's graph A.

    python tools/plq_bench.py [--images 16] [--rows 300] [--gt 10] [--iters 200] [--out results/h100_plq.json]

mirror: efficientteacher_b200.pl_quality.check_pseudo_label_with_gt on CPU inputs (upload, etb_pl_quality, one read-back),
host clock over calls that end in that read-back; cpu_port: tests/plq_port.py (torch-CPU / numpy, the reference's
algorithm without its per-row .cpu() loop); in_graph: the three launches the step adds (etb_pl_quality's two kernels and
one etb_meter_update of the twelve logged values), captured in a CUDA graph and replayed, device events per replay."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def make_case(seed, B, rows_per_img, gt_per_img, nc=80):
    r = np.random.default_rng(seed)
    gt, rows = [], []
    for b in range(B):
        g = np.concatenate([np.full((gt_per_img, 1), b), r.integers(0, nc, (gt_per_img, 1)), r.uniform(0.05, 0.95, (gt_per_img, 2)),
                            r.uniform(0.03, 0.4, (gt_per_img, 2))], 1)
        src = g[r.integers(0, gt_per_img, rows_per_img)]
        x = np.zeros((rows_per_img, 9))
        x[:, 0] = b
        x[:, 1] = np.where(r.random(rows_per_img) < 0.7, src[:, 1], r.integers(0, nc, rows_per_img))
        x[:, 2:4] = src[:, 2:4] + r.normal(0, 0.05, (rows_per_img, 2)) * src[:, 4:6]
        x[:, 4:6] = src[:, 4:6] * np.exp(r.normal(0, 0.25, (rows_per_img, 2)))
        x[:, 6:] = r.uniform(0.1, 1, (rows_per_img, 3))
        gt.append(g)
        rows.append(x)
    return np.concatenate(rows), np.concatenate(gt).astype(np.float32), list(r.uniform(0.1, 0.3, nc)), list(r.uniform(0.4, 0.8, nc))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--rows", type=int, default=300)
    ap.add_argument("--gt", type=int, default=10)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import plq_port
    import __graft_entry__ as g
    g.build()
    from efficientteacher_b200 import pl_quality
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rows, gt, lo, hi = make_case(0, a.images, a.rows, a.gt)
    rows_t, gt_t = torch.from_numpy(rows), torch.from_numpy(gt)
    bs = a.images
    want = plq_port.check_pseudo_label_with_gt(rows, gt, (0.5,), lo, hi, bs)
    got = pl_quality.check_pseudo_label_with_gt(rows_t, gt_t, torch.tensor([0.5]), lo, hi, bs)
    agree = all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(got, want))

    def host_time(fn, n):
        fn()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        return (time.perf_counter() - t0) / n * 1e3

    mirror_ms = host_time(lambda: pl_quality.check_pseudo_label_with_gt(rows_t, gt_t, torch.tensor([0.5]), lo, hi, bs), a.iters)
    port_ms = host_time(lambda: plq_port.check_pseudo_label_with_gt(rows, gt, (0.5,), lo, hi, bs), max(a.iters // 20, 5))

    # the step's launches: statistics over the device rows, then one meter update of the twelve logged values
    plq = pl_quality.PLQuality(dev)
    meter = pl_quality.DeviceMetricMeter(dev)
    rows_d, gt_d = rows_t.to(dev), gt_t.to(dev)
    n_dev = torch.tensor([rows.shape[0]], dtype=torch.int32, device=dev)
    m_dev = torch.tensor([gt.shape[0]], dtype=torch.int32, device=dev)
    hi_d, lo_d = (torch.tensor(t, dtype=torch.float64, device=dev) for t in (hi, lo))
    items = torch.rand(8, device=dev)

    def step():
        v = plq.run(rows_d, n_dev, hi_d, lo_d, gt_d, m_dev, bs, True)
        d = {k: items[i:i + 1] for i, k in enumerate(("box", "obj", "cls", "loss", "ss_box", "ss_obj", "ss_cls"))}
        d.update({k: v[i, 0] for i, k in enumerate(pl_quality.HIT_KEYS)})
        meter.update(d)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for _ in range(20):
        graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    graph_us = e0.elapsed_time(e1) / a.iters * 1e3
    meter.reset()
    props = torch.cuda.get_device_properties(dev)
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        power = "unknown"
    res = dict(gpu=props.name, power_limit=power, images=a.images, rows=int(rows.shape[0]), gt=int(gt.shape[0]),
               mirror_ms=round(mirror_ms, 4), cpu_port_ms=round(port_ms, 3), mirror_agrees_with_port=bool(agree),
               in_graph_us_per_step=round(graph_us, 2), launches_in_graph=3)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
