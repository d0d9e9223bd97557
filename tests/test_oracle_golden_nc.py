"""CPU: the oracle restatement (oracle/port.py) against the golden vectors the live reference produced at nc 20, 8, 2 and 1
(tests/golden/make_golden_nc.py): anchor assignment at anchor_t 4.0 and 5.0, NMS and pseudo-label rows with and without
tied scores, multi-label val NMS, select_targets with per-class thresholds, ComputeLoss at label_smoothing 0 / 0.1 and
ComputeStudentMatchLoss at every ignore_obj x pseudo_label_with_bbox x pseudo_label_with_cls setting.  The GPU tests of
tests/test_gpu_class_counts.py compare the kernels with this oracle at the same class counts."""
import numpy as np
import pytest
import torch

import synth
from oracle import port

NCS = [20, 8, 2, 1]
IMG = 320         # the input size of the fixtures' maps
SWITCHES = [(a, b, c) for a in (False, True) for b in (False, True) for c in (False, True)]   # ignore_obj, with_bbox, with_cls


def check_loss(g, pref, items, grads):
    """one loss case of a class_counts fixture: items [lbox, lobj, lcls, loss], grads the dense per-level gradients of the
    implementation under test, against the stored items, gradient samples, largest gradients and L1 norms"""
    np.testing.assert_allclose(np.asarray(items, np.float64), g[pref + "items"], rtol=1e-5, atol=1e-9)
    for l, gr in enumerate(grads):
        gr = np.asarray(gr, np.float64).reshape(-1)
        tol = 1e-5 * np.abs(g[f"{pref}g{l}_tv"]).max()
        np.testing.assert_allclose(gr[synth.grad_sample_idx(len(gr), l)], g[f"{pref}g{l}_sv"], rtol=1e-4, atol=tol)
        np.testing.assert_allclose(gr[g[f"{pref}g{l}_ti"]], g[f"{pref}g{l}_tv"], rtol=1e-4, atol=tol)
        np.testing.assert_allclose(np.abs(gr).sum(), float(g[f"{pref}g{l}_l1"]), rtol=1e-4)


def loss_prefix(smooth, switches):
    return f"sup_s{smooth:g}_" if switches is None else f"ssod_s{smooth:g}_{''.join(str(int(s)) for s in switches)}_"


def loss_sets(nc, smooth, switches=None):
    """(det_loss args, sets) of the fixture's sup (switches None) or SSOD loss case"""
    shapes = synth.level_shapes(IMG)
    cp, cn = 1.0 - 0.5 * smooth, 0.5 * smooth
    cls_w = 0.3 * nc / 80. * 3. / 3
    if switches is None:
        tg = synth.make_targets(80 + nc, 12 * 2, 2, nc=nc)
        return [port.build_targets(tg, synth.ANCHORS_GRID, shapes)], dict(cls_w=cls_w, cp=cp, cn=cn)
    hi, lo = synth.make_class_thresholds(nc)
    sel = port.select_targets(synth.make_pseudo_rows_dup(100 + nc, 96, 2, nc=nc), hi, lo, True)
    sets = [port.build_targets(sel[0][:, :6], synth.ANCHORS_GRID, shapes)]
    sets += [port.build_targets(s, synth.ANCHORS_GRID, shapes, with_score=True) for s in sel[1:]]
    ig, wb, wc = switches
    return sets, dict(cls_w=cls_w, cp=cp, cn=cn, ignore_obj=ig, with_bbox=wb, with_cls=wc)


@pytest.mark.parametrize("nc", NCS)
def test_build_targets_anchor_t(golden, nc):
    g = golden(f"class_counts_nc{nc}")
    n = 160
    t = synth.make_targets(50 + nc, n, 4, nc=nc)
    t[: n // 8, 4:6] *= 3.0
    sc = np.random.RandomState(51 + nc).uniform(0.1, 1, (n, 1)).astype(np.float32)
    for at in (4.0, 5.0):
        for pref, tt, ws in (("bt", t, False), ("uc", np.concatenate([t, sc], 1), True)):
            res = port.build_targets(tt, synth.ANCHORS_GRID, synth.level_shapes(IMG), at, with_score=ws)
            for l in range(3):
                k = f"a{at:g}_{pref}_"
                assert np.array_equal(res[l]["idx"], g[f"{k}idx{l}"]), (at, pref, l)
                assert np.array_equal(res[l]["tcls"], g[f"{k}tcls{l}"])
                assert np.array_equal(res[l]["tbox"], g[f"{k}tbox{l}"])
                assert np.array_equal(res[l]["anch"], g[f"{k}anch{l}"])
                if ws:
                    assert np.array_equal(res[l]["tscore"], g[f"{k}tscore{l}"])
    assert len(g["a5_bt_idx0"]) > len(g["a4_bt_idx0"])


@pytest.mark.parametrize("ties", [0, 1])
@pytest.mark.parametrize("nc", NCS)
def test_nms_pseudo_rows_and_val_nms(golden, nc, ties):
    g = golden(f"class_counts_nc{nc}")
    pred = synth.make_teacher_pred_ties(20 + nc, 2, nc, ties, IMG)
    dets = port.nms_ssod(pred, 0.1, 0.65)
    val = port.nms_val(pred, 0.05, 0.6, multi_label=True)
    for b in range(2):
        assert np.array_equal(dets[b], g[f"t{ties}_det{b}"]), b
        assert np.array_equal(val[b], g[f"t{ties}_val{b}"]), b
    rows = port.pseudo_label_rows(dets, synth.make_Ms(30 + nc, 2, IMG), IMG, IMG)
    want = g[f"t{ties}_rows"]
    assert rows.shape == want.shape and len(rows)
    assert np.array_equal(rows[:, :2], want[:, :2])
    np.testing.assert_allclose(rows, want, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("nc", NCS)
def test_select_targets_per_class_thresholds(golden, nc):
    g = golden(f"class_counts_nc{nc}")
    hi, lo = synth.make_class_thresholds(nc)
    sel = port.select_targets(synth.make_pseudo_rows(60 + nc, 400, 4, nc=nc), hi, lo, True)
    for i in range(4):
        assert np.array_equal(sel[i], g[f"sel{i}"]), i


@pytest.mark.parametrize("switches", [None] + SWITCHES)
@pytest.mark.parametrize("smooth", [0.0, 0.1])
@pytest.mark.parametrize("nc", NCS)
def test_losses(golden, nc, smooth, switches):
    g = golden(f"class_counts_nc{nc}")
    sets, kw = loss_sets(nc, smooth, switches)
    p = [torch.from_numpy(x).requires_grad_(True) for x in synth.make_head_logits(90 + nc, 2, img=IMG, no=nc + 5)]
    loss, (lbox, lobj, lcls) = port.det_loss(p, sets, [4.0, 1.0, 0.4], 0.05, 0.7, kw.pop("cls_w"), **kw)
    loss.backward()
    pref = loss_prefix(smooth, switches)
    check_loss(g, pref, [float(lbox.detach()), float(lobj.detach()), float(lcls.detach()), float(loss.detach())], [pi.grad.numpy() for pi in p])
    if nc == 1:
        assert g[pref + "items"][2] == 0.0
