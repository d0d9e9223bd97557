"""Generates tests/golden/loss_opts_*.npz from the LIVE, UNMODIFIED reference (imported through oracle/ref_harness.py):
ComputeLoss and ComputeStudentMatchLoss under the cfg.Loss options (fl_gamma, cls_pw / obj_pw, label_smoothing,
autobalance) and the single-target assigner switches (Loss.single_targets, SSOD.uncertain_aug=False).
Run in the build container only:  python tests/golden/make_golden_loss_opts.py
Inputs are re-created from seeds by tests/synth.py (tests/loss_opts_cases.py, shared with the tests), so only outputs are stored.

Each loss case stores opts = OPT_KEYS values, and per call k: c{k}_items = [box, obj, cls, loss] and gradient samples
(c{k}_g{l}_l1 / _sv at synth.grad_sample_idx / top-128 _ti,_tv / every 7th objectness gradient _obj); autobalance
cases also store c{k}_balance, the reference's self.balance after the call."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import synth  # noqa: E402
from loss_opts_cases import inputs  # noqa: E402
from oracle import ref_harness  # noqa: E402

SSOD_YAML = 'configs/ssod/coco-standard/yolov5l_coco_ssod_10_percent.yaml'
SMALL = ['Model.depth_multiple', 0.33, 'Model.width_multiple', 0.50]   # YOLOv5s-sized model: same head/anchors
# name: (ssod loss?, nc, calls, cfg.Loss / cfg.SSOD overrides)
CASES = {
    "fl1": (False, 80, 1, dict(fl_gamma=1.0)),
    "fl15": (False, 80, 1, dict(fl_gamma=1.5)),
    "fl2": (False, 80, 1, dict(fl_gamma=2.0)),
    "pw": (False, 80, 1, dict(cls_pw=2.0, obj_pw=0.5)),
    "mix": (False, 80, 1, dict(fl_gamma=1.5, cls_pw=2.0, obj_pw=0.5, label_smoothing=0.1)),
    "nc1": (False, 1, 1, dict(fl_gamma=1.5, cls_pw=2.0, obj_pw=1.3)),
    "ssod_ign": (True, 80, 1, dict(cls_pw=2.0, obj_pw=0.5, ignore_obj=True)),
    "ssod_cls": (True, 80, 1, dict(cls_pw=2.0, obj_pw=0.5, pseudo_label_with_cls=True)),
    "autobal": (False, 80, 6, dict(autobalance=True)),
}
LOSS_KEYS = ("fl_gamma", "cls_pw", "obj_pw", "label_smoothing", "autobalance")


def grad_samples(out, prefix, p):
    for l, pi in enumerate(p):
        g = pi.grad.numpy().reshape(-1)
        si = synth.grad_sample_idx(len(g), l)
        top = np.argsort(-np.abs(g), kind="stable")[:128].astype(np.int32)
        out[f"{prefix}g{l}_l1"] = np.abs(g).sum(dtype=np.float64)
        out[f"{prefix}g{l}_sv"] = g[si]
        out[f"{prefix}g{l}_ti"], out[f"{prefix}g{l}_tv"] = top, g[top]
        out[f"{prefix}g{l}_obj"] = pi.grad.numpy()[..., 4].reshape(-1)[::7].copy()


def gen_loss(ns, name, ssod, nc, ncalls, over):
    ov = list(SMALL) + ['Dataset.nc', nc, 'Dataset.names', [str(i) for i in range(nc)]]
    for k, v in over.items():
        ov += [('Loss.' if k in LOSS_KEYS else 'SSOD.') + k, v]
    cfg = ref_harness.make_cfg(SSOD_YAML, ov)
    cfg.single_cls = nc == 1
    torch.manual_seed(0)
    model = ns.SSODModel(cfg)
    assert np.allclose(model.head.anchors.numpy(), synth.ANCHORS_GRID)
    crit = ns.ComputeStudentMatchLoss(model, cfg) if ssod else ns.ComputeLoss(model, cfg)
    L, S = cfg.Loss, cfg.SSOD
    out = dict(opts=np.array([nc, L.fl_gamma, L.cls_pw, L.obj_pw, L.label_smoothing, float(L.autobalance), float(S.ignore_obj),
                              float(S.pseudo_label_with_bbox), float(S.pseudo_label_with_cls), float(ssod), ncalls], np.float64))
    for k in range(ncalls):
        logits, tg = inputs(nc, ssod, k)
        p = [torch.from_numpy(x).requires_grad_(True) for x in logits]
        loss, items = crit(p, torch.from_numpy(tg))
        loss.backward()
        keys = ("ss_box", "ss_obj", "ss_cls") if ssod else ("box", "obj", "cls")
        out[f"c{k}_items"] = np.array([float(items[x]) for x in keys] + [float(loss.detach())], np.float32)
        grad_samples(out, f"c{k}_", p)
        if L.autobalance and not ssod:
            out[f"c{k}_balance"] = np.array(crit.balance, np.float64)
    np.savez_compressed(os.path.join(HERE, f"loss_opts_{name}.npz"), **out)
    print(name, {k: out[k] for k in out if k.endswith("_items")})


def gen_single_targets(ns):
    """Loss.single_targets=True and SSOD.uncertain_aug=False (which only sets single_targets): the reference's
    assigner stores the flag and never reads it, so both must assign like the default"""
    cfg = ref_harness.make_cfg(SSOD_YAML, SMALL + ['Loss.single_targets', True, 'SSOD.uncertain_aug', False])
    torch.manual_seed(0)
    model = ns.SSODModel(cfg)
    det = model.head
    sup = ns.ComputeLoss(model, cfg)
    uc = ns.ComputeStudentMatchLoss(model, cfg)
    assert sup.assigner.single_targets and uc.assigner.single_targets
    n = 128
    t = synth.make_targets(11, n, 16)
    sc = np.random.RandomState(5).uniform(0.1, 1, (n, 1)).astype(np.float32)
    p = [torch.zeros(16, 3, ny, nx, 85) for ny, nx in synth.level_shapes()]
    out = dict(seed=11, score_seed=5, n=n, B=16)
    for pref, asg in (("sup", sup.assigner), ("ssod", uc.assigner)):
        res = asg(p, torch.from_numpy(t))
        res7 = asg(p, torch.from_numpy(np.concatenate([t, sc], 1)), with_pseudo_score=True)
        for l in range(det.nl):
            out[f"{pref}_bt_idx{l}"] = torch.stack(res[2][l], 1).numpy().astype(np.int64)
            out[f"{pref}_bt_tbox{l}"] = res[1][l].numpy()
            out[f"{pref}_uc_idx{l}"] = torch.stack(res7[2][l], 1).numpy().astype(np.int64)
            out[f"{pref}_uc_tscore{l}"] = res7[4][l].numpy()
    np.savez_compressed(os.path.join(HERE, "loss_opts_single_targets.npz"), **out)
    print("single_targets", [len(out[f"sup_bt_idx{l}"]) for l in range(det.nl)])


def main():
    ns = ref_harness.load_reference()
    torch.set_num_threads(8)
    for name, (ssod, nc, ncalls, over) in CASES.items():
        gen_loss(ns, name, ssod, nc, ncalls, over)
    gen_single_targets(ns)


if __name__ == "__main__":
    main()
