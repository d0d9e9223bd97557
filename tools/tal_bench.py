"""Device timing of the anchor-free operators (csrc/tal.cu) with CUDA events: etb_tal_assign at BASELINE configs[3]'s per-GPU shape
(32 images x 8400 anchors x 80 classes, 8 and 32 gts per image) and etb_v8_decode (eval decode + assigner inputs).
Prints one JSON object.  Usage: python tools/tal_bench.py [--iters 50]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def timed(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import synth
    from efficientteacher_b200 import _lib, tal
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    pk_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    peaks = json.load(open(pk_path)) if os.path.exists(pk_path) else {"hbm_gbs": 3350.0}   # H100 SXM data sheet
    out = {"hbm_peak_gbs": peaks["hbm_gbs"], "iters": args.iters, "cases": {}}
    B, img, nc = 32, 640, 80
    A = sum(h * w for h, w in synth.level_shapes(img))
    for M in (8, 32):
        d = synth.make_tal_inputs(90 + M, B, [M] * B, img=img)
        t = {k: torch.from_numpy(v).to(dev) for k, v in d.items()}
        asg = tal.TaskAlignedAssigner(13, nc)
        l0 = _lib.lib().etb_launch_count()
        res = asg(t["pd_scores"], t["pd_bboxes"], t["anc_points"], t["gt_labels"], t["gt_bboxes"], t["mask_gt"])
        launches = _lib.lib().etb_launch_count() - l0
        ms = timed(lambda: asg(t["pd_scores"], t["pd_bboxes"], t["anc_points"], t["gt_labels"], t["gt_bboxes"], t["mask_gt"]), args.iters)
        # algorithmic bytes: read scores once for the gathers' sectors is data dependent; the fixed part is the output pass
        out_bytes = B * A * (nc * 4 + 8 + 16 + 1)
        in_bytes = B * A * 16 + B * A * nc * 4            # boxes + (upper bound) the score tensor once
        out["cases"]["tal_assign_B%d_A%d_M%d" % (B, A, M)] = {
            "ms": ms, "kernel_launches": launches, "fg_anchors": int(res[3].sum()), "output_bytes": out_bytes,
            "output_GBps": out_bytes / (ms * 1e-3) / 1e9, "io_upper_bound_bytes": in_bytes + out_bytes,
            "frac_of_hbm_peak_on_output_bytes": out_bytes / (ms * 1e-3) / 1e9 / peaks["hbm_gbs"]}
    cls, reg = synth.make_v8_head_logits(95, B, img=img)
    cls, reg = torch.from_numpy(cls).to(dev), torch.from_numpy(reg).to(dev)
    shapes = synth.level_shapes(img)
    ms = timed(lambda: tal.decode_eval(cls, reg, shapes, synth.STRIDES, 16), args.iters)
    by = B * A * ((nc + 68) * 4 + (5 + nc) * 4)
    out["cases"]["v8_decode_eval_B%d_A%d" % (B, A)] = {"ms": ms, "bytes": by, "GBps": by / (ms * 1e-3) / 1e9, "frac_of_hbm_peak": by / (ms * 1e-3) / 1e9 / peaks["hbm_gbs"]}
    ms = timed(lambda: tal.assigner_inputs(cls, reg, shapes, synth.STRIDES, 16), args.iters)
    by = B * A * ((nc + 68) * 4 + (4 + 4 + nc) * 4)
    out["cases"]["v8_assigner_inputs_B%d_A%d" % (B, A)] = {"ms": ms, "bytes": by, "GBps": by / (ms * 1e-3) / 1e9, "frac_of_hbm_peak": by / (ms * 1e-3) / 1e9 / peaks["hbm_gbs"]}
    out["note"] = ("ms include the mirror's host work (torch.empty of the outputs / workspace, ctypes call): these are small launches, so the "
                   "figures are upper bounds on the kernel time")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
