"""Times one validation epoch of a YOLOv5l teacher: N synthetic letterboxed images in rect batches, conf 0.001 / IoU 0.6.

  native : val.run -- engine forward, etb_nms_val, etb_val_epoch_append per batch, etb_ap_per_class + the numpy tail once
  host   : val.val_batch per batch (per-image host lists) + the numpy ap_per_class of tests/ap_port.py on the host
  ap     : ap_per_class alone on a synthetic 1.5 M-row, 80-class epoch, native vs numpy

The Detect head is calibrated so that most images reach max_det = 300 detections at conf 0.001 (objectness bias +4, class
biases +2).  Prints one JSON line; --out writes it to a file too.

    python tools/val_bench.py --images 5000 --out results/h100_val.json
"""
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

SHAPES = ((640, 640), (480, 640), (640, 480), (384, 640))     # rect batch shapes (H, W), multiples of 32


def _loader(n_images, batch, seed=0):
    """uint8 batches on the device (a few distinct ones, reused), targets [nt, 6] with ~7 labels per image, loader shapes"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = np.random.RandomState(seed)
    distinct = {}
    out = []
    for bi in range((n_images + batch - 1) // batch):
        B = min(batch, n_images - bi * batch)
        H, W = SHAPES[bi % len(SHAPES)]
        key = (B, H, W, bi % 8)
        if key not in distinct:
            distinct[key] = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, device="cuda", generator=g)
        nt = r.poisson(7, B)
        rows = [(b, r.randint(0, 80), r.rand(), r.rand(), r.uniform(0.02, 0.4), r.uniform(0.02, 0.4)) for b in range(B) for _ in range(nt[b])]
        tg = torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)
        shapes = []
        for _ in range(B):
            h0, w0 = int(r.randint(300, 900)), int(r.randint(300, 900))
            gain = min(H / h0, W / w0)
            shapes.append(((h0, w0), ((gain, gain), ((W - w0 * gain) / 2, (H - h0 * gain) / 2))))
        out.append((distinct[key], tg, ["%d.jpg" % i for i in range(B)], shapes))
    return out


def _teacher():
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.model import SupModel
    torch.manual_seed(0)
    m = SupModel(yolov5_sup_cfg('l', batch_size=32, img_size=640)).cuda()
    with torch.no_grad():
        for h in m.head.m:
            h.bias.view(3, -1)[:, 4] += 4.0
            h.bias.view(3, -1)[:, 5:] += 2.0
    return m.eval()


def _host_leg(model, loader):
    """today's path: val_batch per batch, the reference's per-image .cpu() lists, numpy ap_per_class"""
    import ap_port
    from efficientteacher_b200 import val
    stats, dets = [], 0
    for img, tg, _, shapes in loader:
        for correct, conf, pcls, tcls in val.val_batch(model, img, tg.cuda(), shapes):
            stats.append((correct.cpu(), conf.cpu(), pcls.cpu(), tcls))
            dets += correct.shape[0]
    stats = [np.concatenate(x, 0) for x in zip(*stats)]
    res = ap_port.ap_per_class(*stats)
    return res, dets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--ap-rows", type=int, default=1500000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import ap_port
    from efficientteacher_b200 import metrics, val
    torch.cuda.set_device(0)
    model = _teacher()
    loader = _loader(a.images, a.batch)
    res = {"gpu": torch.cuda.get_device_name(0), "images": a.images, "batch": a.batch, "shapes": SHAPES}
    try:
        import subprocess
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        res["power_limit_w"] = None
    # warm-up: one short epoch (engine packing, workspaces)
    val.run({'nc': 80}, model=model, dataloader=loader[:2], plots=False, half=False)
    torch.cuda.synchronize()
    native = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        r_native = val.run({'nc': 80}, model=model, dataloader=loader, plots=False, half=False)
        torch.cuda.synchronize()
        native.append(time.perf_counter() - t0)
    res["native_s"] = native
    res["native_ms_per_image"] = [1e3 * x / a.images for x in native]
    res["native_t_ms_per_image"] = list(r_native[2])
    res["native_results"] = [float(x) for x in r_native[0]]
    t0 = time.perf_counter()
    (p, r, apc, f1, ap_class, thr), dets = _host_leg(model, loader)
    torch.cuda.synchronize()
    res["host_s"] = time.perf_counter() - t0
    res["detections"] = dets
    res["detections_per_image"] = dets / a.images
    res["host_map50"] = float(apc[:, 0].mean())
    res["native_map50_equal_host"] = bool(float(r_native[0][2]) == float(apc[:, 0].mean()))
    # ap_per_class alone
    tp, conf, pcls, tcls = ap_port.make_case(7, a.ap_rows, 80, labels_per_class=(50, 900), tp_rate=0.3)
    d = [torch.from_numpy(x).cuda() for x in (tp, conf, pcls)]
    metrics.ap_per_class(*d, tcls)
    torch.cuda.synchronize()
    ts = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        got = metrics.ap_per_class(*d, tcls)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    res["ap_rows"] = a.ap_rows
    res["ap_native_s"] = ts
    t0 = time.perf_counter()
    want = ap_port.ap_per_class(tp, conf, pcls, tcls)
    res["ap_numpy_s"] = time.perf_counter() - t0
    res["ap_native_equal_numpy"] = all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(got, want))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
