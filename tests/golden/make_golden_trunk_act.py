"""Generates the golden vectors that pin the ReLU and Hardswish YOLOv5 trunks (this package's Model and the activation-aware
trunk reference tests/trunk_act_ref.py) to the LIVE, UNMODIFIED reference (imported through oracle/ref_harness.py).
For each mode, trunk_act_<mode>.npz holds, for the reference SSOD model at YOLOv5s widths and depth 0.33
(models/detector/yolo_ssod.py with cfg.Model.{Backbone,Neck}.activation set) run on THIS package's seeded initial weights:
  conv_paths / conv_acts   module path and activation class name of every reference `Conv`
  backbone_act / neck_act  the two config strings
  eval_* / train_* / running  the fixed seeded sample make_golden_trunk.py stores in trunk_ref.npz (eval and train
                           outputs, BN running statistics after the train pass)
Modes: 'relu' (ReLU, ReLU), 'default' (the reference's defaults, configs/defaults.py: LeakyReLU backbone -> Hardswish,
ReLU neck), 'hswish' (Hardswish, Hardswish).
Run where the reference is importable:  python tests/golden/make_golden_trunk_act.py"""
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

MODES = {"relu": ("ReLU", "ReLU"), "default": ("LeakyReLU", "ReLU"), "hswish": ("Hardswish", "Hardswish")}
SIZE = "s"                       # width 0.50, depth 0.33: every C3 has one or two Bottlenecks
DEPTH, NECK_DEPTH = (1, 2, 3, 1), 1


def initial_state_dict(mode):
    """The weights both sides run: this package's SSOD model for the mode, seeded (no reference needed to rebuild them)."""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    bb, nk = MODES[mode]
    torch.manual_seed(0)
    return {k: v.detach().clone() for k, v in Model(yolov5_ssod_cfg(SIZE, backbone_act=bb, neck_act=nk)).state_dict().items()}


def gen(ns, mode):
    bb, nk = MODES[mode]
    cfg = ref_harness.make_cfg(SSOD_YAML, ["Model.depth_multiple", 0.33, "Model.width_multiple", 0.50,
                                           "Model.Backbone.activation", bb, "Model.Neck.activation", nk])
    ref = ns.SSODModel(cfg)
    ref.load_state_dict(initial_state_dict(mode))
    conv_cls = sys.modules["models.backbone.common"].Conv
    convs = [(n, type(m.act).__name__) for n, m in ref.named_modules() if isinstance(m, conv_cls)]
    out = {"conv_paths": np.array([n for n, _ in convs]), "conv_acts": np.array([a for _, a in convs]),
           "backbone_act": np.array(bb), "neck_act": np.array(nk)}
    x, x2 = trunk_inputs()
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
    np.savez_compressed(os.path.join(HERE, "trunk_act_%s.npz" % mode), **out)


if __name__ == "__main__":
    ns = ref_harness.load_reference()
    for m in MODES:
        gen(ns, m)
