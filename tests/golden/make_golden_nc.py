"""Generates tests/golden/class_counts_nc{20,8,2,1}.npz from the LIVE, UNMODIFIED reference (imported through
oracle/ref_harness.py) at the class counts of the reference's other datasets: VOC (20), Cityscapes (8), the custom configs (2)
and single_cls (1).  Run in the build container only:  python tests/golden/make_golden_nc.py
Inputs are re-created from seeds by tests/synth.py (the same recipes tests/test_oracle_golden_nc.py and
tests/test_gpu_class_counts.py use), so only outputs are stored; test_oracle_golden_nc.check_loss reads the loss cases."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import synth  # noqa: E402
from oracle import ref_harness  # noqa: E402

SSOD_YAML = 'configs/ssod/coco-standard/yolov5l_coco_ssod_10_percent.yaml'
SMALL = ['Model.depth_multiple', 0.33, 'Model.width_multiple', 0.50]   # YOLOv5s-sized model: same head/anchors
NCS = (20, 8, 2, 1)
IMG = 320
SWITCHES = [(a, b, c) for a in (False, True) for b in (False, True) for c in (False, True)]


def grad_samples(out, prefix, p):
    for l, pi in enumerate(p):
        g = pi.grad.numpy().reshape(-1)
        si = synth.grad_sample_idx(len(g), l)
        top = np.argsort(-np.abs(g), kind="stable")[:128].astype(np.int32)
        out[f"{prefix}g{l}_l1"] = np.abs(g).sum(dtype=np.float64)
        out[f"{prefix}g{l}_sv"] = g[si]
        out[f"{prefix}g{l}_ti"], out[f"{prefix}g{l}_tv"] = top, g[top]


def gen(ns, nc):
    out = {}
    names = [str(i) for i in range(nc)]
    cfg = ref_harness.make_cfg(SSOD_YAML, SMALL + ['Dataset.nc', nc, 'Dataset.names', names])
    torch.manual_seed(0)
    model = ns.SSODModel(cfg)
    det = model.head
    assert det.nc == nc and np.allclose(det.anchors.numpy(), synth.ANCHORS_GRID)
    shapes = synth.level_shapes(IMG)

    # ---- build_targets / build_uc_targets_aug at anchor_t 4.0 and 5.0 ----
    B, n = 4, 160
    t = synth.make_targets(50 + nc, n, B, nc=nc)
    t[: n // 8, 4:6] *= 3.0
    sc = np.random.RandomState(51 + nc).uniform(0.1, 1, (n, 1)).astype(np.float32)
    p0 = [torch.zeros(B, 3, ny, nx, nc + 5) for ny, nx in shapes]
    for at in (4.0, 5.0):
        asg = ns.YOLOAnchorAssigner(det.na, det.nl, det.anchors, at, det.stride, det.nc, 0)
        for pref, tt, ws in (("bt", t, False), ("uc", np.concatenate([t, sc], 1), True)):
            res = asg(p0, torch.from_numpy(tt), with_pseudo_score=ws)
            for l in range(3):
                out[f"a{at:g}_{pref}_idx{l}"] = torch.stack(res[2][l], 1).numpy().astype(np.int64)
                out[f"a{at:g}_{pref}_tbox{l}"] = res[1][l].numpy()
                out[f"a{at:g}_{pref}_anch{l}"] = res[3][l].numpy()
                out[f"a{at:g}_{pref}_tcls{l}"] = res[0][l].numpy().astype(np.int64)
                if ws:
                    out[f"a{at:g}_{pref}_tscore{l}"] = res[4][l].numpy()

    # ---- NMS, pseudo-label rows, multi-label val NMS (plain and tied scores) ----
    cfg.SSOD.nms_conf_thres, cfg.SSOD.nms_iou_thres = 0.1, 0.65
    fpl = ns.FairPseudoLabel(cfg)
    Bn = 2
    Ms = synth.make_Ms(30 + nc, Bn, IMG)
    for ties in (0, 1):
        pred = synth.make_teacher_pred_ties(20 + nc, Bn, nc, ties, IMG)
        tp = torch.from_numpy(pred)
        dets = ns.non_max_suppression_ssod(tp.clone(), conf_thres=0.1, iou_thres=0.65)
        imgs = torch.zeros(Bn, 3, IMG, IMG)
        rows, _ = fpl.create_pseudo_label_online_with_gt(tp.clone(), imgs, torch.from_numpy(Ms), imgs.clone())
        out[f"t{ties}_rows"] = rows.numpy() if isinstance(rows, torch.Tensor) else np.zeros((0, 9))
        val = ns.non_max_suppression(tp.clone(), conf_thres=0.05, iou_thres=0.6, multi_label=True)
        for b in range(Bn):
            out[f"t{ties}_det{b}"] = dets[b].numpy().reshape(-1, 8)
            out[f"t{ties}_val{b}"] = val[b].numpy().reshape(-1, 6)

    # ---- select_targets with per-class thresholds ----
    crit = ns.ComputeStudentMatchLoss(model, cfg)
    hi, lo = synth.make_class_thresholds(nc)
    crit.ignore_thres_high, crit.ignore_thres_low = list(hi), list(lo)
    rows = synth.make_pseudo_rows(60 + nc, 400, 4, nc=nc)
    for i, s in enumerate(crit.select_targets(torch.from_numpy(rows))):
        out[f"sel{i}"] = s.numpy().reshape(-1, 7)

    # ---- ComputeLoss at label_smoothing 0 / 0.1, ComputeStudentMatchLoss over the switch matrix ----
    Bl = 2
    logits = synth.make_head_logits(90 + nc, Bl, img=IMG, no=nc + 5)
    tg = synth.make_targets(80 + nc, 12 * Bl, Bl, nc=nc)
    srows = synth.make_pseudo_rows_dup(100 + nc, 96, Bl, nc=nc)
    for smooth in (0.0, 0.1):
        cfg.Loss.label_smoothing = smooth
        cfg.single_cls = nc == 1
        sup = ns.ComputeLoss(model, cfg)
        p = [torch.from_numpy(x).requires_grad_(True) for x in logits]
        loss, items = sup(p, torch.from_numpy(tg))
        loss.backward()
        pref = f"sup_s{smooth:g}_"
        out[pref + "items"] = np.array([float(items[k]) for k in ("box", "obj", "cls")] + [float(loss.detach())], np.float32)
        grad_samples(out, pref, p)
        for ig, wb, wc in SWITCHES:
            cfg.SSOD.ignore_obj, cfg.SSOD.pseudo_label_with_bbox, cfg.SSOD.pseudo_label_with_cls = ig, wb, wc
            crit = ns.ComputeStudentMatchLoss(model, cfg)
            crit.ignore_thres_high, crit.ignore_thres_low = list(hi), list(lo)
            p = [torch.from_numpy(x).requires_grad_(True) for x in logits]
            loss, items = crit(p, torch.from_numpy(srows))
            loss.backward()
            pref = f"ssod_s{smooth:g}_{int(ig)}{int(wb)}{int(wc)}_"
            out[pref + "items"] = np.array([float(items[k]) for k in ("ss_box", "ss_obj", "ss_cls")] + [float(loss.detach())], np.float32)
            grad_samples(out, pref, p)
    cfg.single_cls = False
    np.savez_compressed(os.path.join(HERE, f"class_counts_nc{nc}.npz"), **out)
    print("nc", nc, "keys", len(out))


def main():
    ns = ref_harness.load_reference()
    torch.set_num_threads(8)
    for nc in NCS:
        gen(ns, nc)


if __name__ == "__main__":
    main()
