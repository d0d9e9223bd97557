"""Generates the golden vectors that pin this package's YOLOv5n/m/x models and oracle/trunk_ref.TrunkRef at YOLOv5m width
to the LIVE, UNMODIFIED reference (imported through oracle/ref_harness.py):
  model_keys_sizes.npz  for n, m and x: the (depth_multiple, width_multiple) of the reference's supervised config
                        (configs/sup/public/yolov5{n,m,x}_coco.yaml), and the state_dict keys, shapes and dtypes of the
                        reference's supervised model from that config and of its SSOD model (the 10 % COCO SSOD config
                        with the size's multipliers)
  trunk_m.npz           the reference SSOD model at YOLOv5m width and depth 0.33 run on THIS package's seeded initial
                        weights: the fixed seeded sample make_golden_trunk.py stores in trunk_ref.npz (eval and train
                        outputs, BN running statistics after the train pass)
Run where the reference is importable:  python tests/golden/make_golden_sizes.py"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import ref_harness  # noqa: E402
from make_golden_trunk import SSOD_YAML, sampled, trunk_inputs  # noqa: E402

SIZES = ("n", "m", "x")
SUP_YAML = "configs/sup/public/yolov5%s_coco.yaml"
TRUNK_SIZE = "m_shallow"         # width 0.75, depth 0.33: every C3 has one to three Bottlenecks
DEPTH, NECK_DEPTH = (1, 2, 3, 1), 1


def initial_state_dict(size=TRUNK_SIZE):
    """The weights both sides run: this package's SSOD model of the size, seeded (no reference needed to rebuild them)."""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(0)
    return {k: v.detach().clone() for k, v in Model(yolov5_ssod_cfg(size)).state_dict().items()}


def _keys(name, model, out):
    sd = model.state_dict()
    out[name + "_keys"] = np.array(list(sd.keys()))
    out[name + "_ndim"] = np.array([v.dim() for v in sd.values()], dtype=np.int64)
    out[name + "_dims"] = np.array([d for v in sd.values() for d in v.shape], dtype=np.int64)
    out[name + "_dtypes"] = np.array([str(v.dtype) for v in sd.values()])


def gen_keys(ns):
    out = {}
    for s in SIZES:
        sup = ref_harness.make_cfg(SUP_YAML % s)
        dm, wm = float(sup.Model.depth_multiple), float(sup.Model.width_multiple)
        out["mult_" + s] = np.array([dm, wm])
        _keys("sup_" + s, ns.SupModel(sup), out)
        _keys("ssod_" + s, ns.SSODModel(ref_harness.make_cfg(SSOD_YAML, ["Model.depth_multiple", dm, "Model.width_multiple", wm])), out)
    np.savez_compressed(os.path.join(HERE, "model_keys_sizes.npz"), **out)


def gen_trunk(ns):
    cfg = ref_harness.make_cfg(SSOD_YAML, ["Model.depth_multiple", 0.33, "Model.width_multiple", 0.75])
    ref = ns.SSODModel(cfg)
    ref.load_state_dict(initial_state_dict())
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
    np.savez_compressed(os.path.join(HERE, "trunk_m.npz"), **out)


if __name__ == "__main__":
    ns = ref_harness.load_reference()
    gen_keys(ns)
    gen_trunk(ns)
