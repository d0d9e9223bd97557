"""Frames per second of batched inference on raw frames, two ways on the same GPU:

  native:   detect.Predictor -- pinned uploads, etb_letterbox_u8, the bf16 engine, the device NMS, etb_detect_rescale, one
            read-back of the detection counts per call;
  detect.py way: per frame, letterbox on the CPU with cv2 (resize INTER_LINEAR + copyMakeBorder), BGR -> RGB, HWC -> CHW, one
            upload, / 255, the eager fp32 torch / cuDNN forward of oracle/eager_ref.py (TrunkRef + decode_t; detect.py's
            default half=False), the per-image torchvision NMS (nms_ssod_t) and scale_coords(...).round() with torch ops.

Synthetic uint8 BGR frames in host memory (as cv2.imread returns them) at 1080p, 720p and 480x640; batches of 1, 8 and 32
frames per Predictor call (detect.py takes one frame at a time, so its rate does not depend on the batch); YOLOv5s and
YOLOv5l with seeded weights whose heads keep a few classes above conf 0.25.  Times are CUDA events around whole calls that end
in a device synchronise.  Writes one JSON file (--out).

    python tools/detect_bench.py --out results/h100_detect.json
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RES = {"1080p": (1080, 1920), "720p": (720, 1280), "480x640": (480, 640)}


def _model(size, dev):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(0)
    m = Model(yolov5_ssod_cfg(size, batch_size=1, img_size=640)).to(dev)
    with torch.no_grad():
        for h in m.head.m:
            b = h.bias.view(3, -1)
            b[:, 4] += 6.0
            b[:, 5:] = -12.0
            b[:, 5:9] = 1.0
    return m.eval()


def _frames(n, hw, seed):
    r = np.random.RandomState(seed)
    return [np.frombuffer(bytearray(r.bytes(hw[0] * hw[1] * 3)), np.uint8).reshape(hw[0], hw[1], 3) for _ in range(n)]


def _timed(fn, iters, warmup):
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


def native(model, frames, iters, warmup):
    from efficientteacher_b200.detect import Predictor
    p = Predictor(model, img_size=640)
    ms = _timed(lambda: p(frames), iters, warmup)
    return ms, sum(int(d.shape[0]) for d in p(frames))


def detect_py_way(model, frames, iters, warmup):
    import cv2
    from efficientteacher_b200 import val
    from efficientteacher_b200.detect import letterbox_geometry
    from oracle.eager_ref import STRIDES, decode_t, nms_ssod_t
    from oracle.trunk_ref import TrunkRef
    import synth
    dev = next(model.parameters()).device
    torch.backends.cudnn.benchmark = True
    depth = tuple(len(getattr(model.backbone, n).m) for n in ("stage2_2", "stage3_2", "stage4_2", "stage5_2"))
    trunk = TrunkRef({k: v.detach().clone() for k, v in model.state_dict().items()}, depth, len(model.neck.C1.m))
    count = [0]

    def one(im0):
        new_h, new_w, top, left, H, W = letterbox_geometry(im0.shape[0], im0.shape[1], 640)[:6]
        im = cv2.resize(im0, (new_w, new_h), interpolation=cv2.INTER_LINEAR) if im0.shape[:2] != (new_h, new_w) else im0
        im = cv2.copyMakeBorder(im, top, H - new_h - top, left, W - new_w - left, cv2.BORDER_CONSTANT, value=(114, 114, 114))
        im = np.ascontiguousarray(im[:, :, ::-1].transpose(2, 0, 1))
        x = (torch.from_numpy(im).to(dev).float() / 255.0)[None]
        with torch.no_grad():
            raw, _ = trunk.forward(x, train=False)
            det = nms_ssod_t(decode_t(raw, synth.ANCHORS_GRID, STRIDES), 0.25, 0.45, max_det=1000)[0][:, :6]
            det[:, :4] = val.scale_coords_((H, W), det[:, :4], im0.shape).round()
        count[0] += int(det.shape[0])

    def run():
        for f in frames:
            one(f)
    ms = _timed(run, iters, warmup)
    count[0] = 0
    run()
    return ms, count[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="s,l")
    ap.add_argument("--res", default="1080p,720p,480x640")
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--frames", type=int, default=64, help="frames per timed window (at least one call)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    gpu = {"name": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        gpu["power_limit_and_max_sm_clock"] = q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        gpu["power_limit_and_max_sm_clock"] = "not read"
    rows = []
    for size in a.sizes.split(","):
        model = _model(size, dev)
        for res in a.res.split(","):
            hw = RES[res]
            base = _frames(8, hw, 1)
            ms, n = detect_py_way(model, base, 2, 1)
            rows.append(dict(model="yolov5" + size, res=res, way="detect.py", batch=1, fps=len(base) / (ms / 1e3),
                             ms_per_frame=ms / len(base), detections=n))
            print(json.dumps(rows[-1]), flush=True)
            for B in [int(b) for b in a.batches.split(",")]:
                frames = _frames(B, hw, 2)
                iters = max(1, a.frames // B)
                ms, n = native(model, frames, iters, a.warmup)
                rows.append(dict(model="yolov5" + size, res=res, way="native", batch=B, fps=B / (ms / 1e3), ms_per_call=ms,
                                 calls=iters, detections=n))
                print(json.dumps(rows[-1]), flush=True)
        del model
        torch.cuda.empty_cache()
    out = {"gpu": gpu, "torch": torch.__version__, "img_size": 640, "conf_thres": 0.25, "iou_thres": 0.45, "max_det": 1000,
           "frames": "synthetic uint8 BGR in host memory", "rows": rows}
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
