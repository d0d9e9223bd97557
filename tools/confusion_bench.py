"""Times the detection confusion matrix on tools/val_bench.py's workload: a YOLOv5l teacher, N synthetic letterboxed images
in rect batches, conf 0.001 / IoU 0.6 NMS (about 300 detections per image).

  per_image : ConfusionMatrix.process_batch once per image, as val.py:373 calls it.  host = the reference's per-image
              algorithm restated in numpy (tests/confusion_port.py; the reference itself is not importable here), fed with
              the same native-space rows as host arrays; native = efficientteacher_b200.metrics.ConfusionMatrix on the device
              tensors (one launch per image, one read-back at the end).  Both matrices must be equal.
  epoch     : val.run over the N images, without and with confusion_matrix= (alternating), and whether their results agree.

Prints one JSON line; --out writes it to a file too.

    python tools/confusion_bench.py --images 5000 --out results/h100_confusion.json
"""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _native_rows(model, loader):
    """(predn [n, 6], labelsn [m, 5]) on the device for every image that val.py passes to process_batch"""
    from efficientteacher_b200 import val
    out = []
    with torch.no_grad():
        for img, tg, _, shapes in loader:
            H, W = img.shape[2:]
            det, cnt = val._nms(val._unwrap(model(img)), 0.001, 0.6, False)
            t = tg.cuda().clone()
            t[:, 2:6] *= torch.tensor([W, H, W, H], device="cuda", dtype=torch.float32)
            cnt = cnt.tolist()
            for si in range(img.shape[0]):
                lab = t[t[:, 0] == si, 1:]
                if cnt[si] == 0 or lab.shape[0] == 0:
                    continue
                predn = det[si, :cnt[si], :6].clone()
                val.scale_coords_((H, W), predn[:, :4], shapes[si][0], shapes[si][1])
                box = torch.cat((lab[:, 1:3] - lab[:, 3:5] / 2, lab[:, 1:3] + lab[:, 3:5] / 2), 1)
                val.scale_coords_((H, W), box, shapes[si][0], shapes[si][1])
                out.append((predn.contiguous(), torch.cat((lab[:, 0:1], box), 1).contiguous()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import confusion_port
    import val_bench
    from efficientteacher_b200 import val
    from efficientteacher_b200.metrics import ConfusionMatrix
    torch.cuda.set_device(0)
    model = val_bench._teacher()
    loader = val_bench._loader(a.images, a.batch)
    res = {"gpu": torch.cuda.get_device_name(0), "images": a.images, "batch": a.batch, "shapes": val_bench.SHAPES, "nc": 80}
    try:
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        res["power_limit_w"] = None

    # ---- per image -----------------------------------------------------------------------------------------------------
    rows = _native_rows(model, loader)
    host_rows = [(d.cpu().numpy(), l.cpu().numpy()) for d, l in rows]
    res["per_image_calls"] = len(rows)
    res["detections_per_call"] = float(np.mean([d.shape[0] for d, _ in host_rows]))
    res["labels_per_call"] = float(np.mean([l.shape[0] for _, l in host_rows]))
    cm = ConfusionMatrix(80)
    for d, l in rows[:64]:                   # warm-up
        cm.process_batch(d, l)
    native = []
    for _ in range(a.repeats):
        cm.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for d, l in rows:
            cm.process_batch(d, l)
        m_native = cm.matrix                 # the read-back waits for the device
        native.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    m_host = np.zeros((81, 81))
    for d, l in host_rows:
        confusion_port.process_batch(m_host, d, l)
    res["per_image_host_s"] = time.perf_counter() - t0
    res["per_image_native_s"] = native
    res["per_image_host_us_per_call"] = 1e6 * res["per_image_host_s"] / len(rows)
    res["per_image_native_us_per_call"] = [1e6 * x / len(rows) for x in native]
    res["per_image_equal"] = bool(np.array_equal(m_native, m_host))
    res["matrix_total"] = float(m_host.sum())

    # ---- the val.run epoch ---------------------------------------------------------------------------------------------
    val.run({'nc': 80}, model=model, dataloader=loader[:2], plots=False, half=False)
    val.run({'nc': 80}, model=model, dataloader=loader[:2], plots=False, half=False, confusion_matrix=ConfusionMatrix(80))
    torch.cuda.synchronize()
    plain, with_cm = [], []
    for _ in range(a.repeats):
        for leg, ts in (("plain", plain), ("cm", with_cm)):
            cm = ConfusionMatrix(80) if leg == "cm" else None
            t0 = time.perf_counter()
            r = val.run({'nc': 80}, model=model, dataloader=loader, plots=False, half=False, confusion_matrix=cm)
            if cm is not None:
                m_epoch = cm.matrix
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
            if leg == "plain":
                r_plain = r
            else:
                r_cm = r
    res["epoch_plain_s"] = plain
    res["epoch_confusion_s"] = with_cm
    res["epoch_results_equal"] = bool(r_plain[0] == r_cm[0] and np.array_equal(r_plain[1], r_cm[1]))
    res["epoch_matrix_equal_per_image"] = bool(np.array_equal(m_epoch, m_host))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
