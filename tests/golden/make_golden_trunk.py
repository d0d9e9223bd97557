"""Generates the golden vectors that pin oracle/trunk_ref.TrunkRef and this package's model layouts to the LIVE, UNMODIFIED
reference (imported through oracle/ref_harness.py), and three more TaskAlignedAssigner cases on fresh seeds:
  trunk_ref.npz      the reference SSOD YOLOv5l (models/detector/yolo_ssod.py) run on THIS package's seeded initial weights:
                     a fixed seeded sample of every eval / train output and of the BN running statistics after the train pass
  model_keys.npz     state_dict keys and shapes of the reference's YOLOv5l SSOD and YOLOv5s supervised models
  tal_fresh*.npz     tests/golden/make_golden_v8.py's TAL format, seeds 101-103
Run where the reference is importable:  python tests/golden/make_golden_trunk.py"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_harness  # noqa: E402

SSOD_YAML = "configs/ssod/coco-standard/yolov5l_coco_ssod_10_percent.yaml"
SUP_YAML = "configs/sup/public/yolov5s_coco.yaml"
SAMPLE = 2048            # values kept per output tensor


def initial_state_dict():
    """The weights both sides run: this package's YOLOv5l SSOD model, seeded (no reference needed to rebuild them)."""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(0)
    return {k: v.detach().clone() for k, v in Model(yolov5_ssod_cfg('l')).state_dict().items()}


def trunk_inputs():
    return (torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(3)),
            torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(4)))


def sample_index(numel, salt):
    g = np.random.RandomState(1000 + salt)
    return np.sort(g.choice(numel, size=min(SAMPLE, numel), replace=False))


def sampled(tensors, prefix, out):
    for i, t in enumerate(tensors):
        flat = t.detach().reshape(-1).numpy()
        idx = sample_index(flat.size, len(out))
        out["%s%d_shape" % (prefix, i)] = np.array(t.shape, dtype=np.int64)
        out["%s%d_idx" % (prefix, i)] = idx
        out["%s%d" % (prefix, i)] = flat[idx]


def gen_trunk(ns):
    sd = initial_state_dict()
    ref = ns.SSODModel(ref_harness.make_cfg(SSOD_YAML))
    ref.load_state_dict(sd)
    x, x2 = trunk_inputs()
    out = {}
    ref.eval()
    with torch.no_grad():
        (pred, raw), feat = ref(x)
    sampled(raw, "eval_raw", out)
    sampled(feat, "eval_feat", out)
    ref.train()
    raw_t, feat_t = ref(x2)
    sampled(raw_t, "train_raw", out)
    sampled(feat_t, "train_feat", out)
    after = ref.state_dict()
    keys = [k for k in after if "running_" in k]
    sampled([torch.cat([after[k].reshape(-1) for k in keys])], "running", out)
    np.savez_compressed(os.path.join(HERE, "trunk_ref.npz"), **out)


def gen_keys(ns):
    out = {}
    for name, model in (("ssod_l", ns.SSODModel(ref_harness.make_cfg(SSOD_YAML))), ("sup_s", ns.SupModel(ref_harness.make_cfg(SUP_YAML)))):
        sd = model.state_dict()
        out[name + "_keys"] = np.array(list(sd.keys()))
        out[name + "_ndim"] = np.array([v.dim() for v in sd.values()], dtype=np.int64)
        out[name + "_dims"] = np.array([d for v in sd.values() for d in v.shape], dtype=np.int64)
        out[name + "_dtypes"] = np.array([str(v.dtype) for v in sd.values()])
    np.savez_compressed(os.path.join(HERE, "model_keys.npz"), **out)


def gen_tal_fresh(ns):
    import make_golden_v8 as mg
    mg.TAL_CASES = {"fresh101": (101, 2, [6, 9], 320, 4, 0), "fresh102": (102, 2, [25, 1], 320, 1, 0), "fresh103": (103, 1, [16], 640, 3, 0)}
    mg.gen_tal(ns)


if __name__ == "__main__":
    ns = ref_harness.load_reference()
    gen_trunk(ns)
    gen_keys(ns)
    gen_tal_fresh(ns)
