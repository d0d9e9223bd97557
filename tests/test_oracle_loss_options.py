"""CPU: the restatement of the loss options (tests/loss_opts_port.det_loss: oracle/port.det_loss with cls_pw / obj_pw /
fl_gamma / autobalance) against the live reference's ComputeLoss and ComputeStudentMatchLoss (tests/golden/loss_opts_*.npz), and the
single-target assigner switches against the default assignment.  Losses within 1e-5, gradients within 1e-4."""
import numpy as np
import pytest
import torch

import loss_opts_port
import synth
from loss_opts_cases import IMG, LOSS_CASES, check_grads, inputs, opts
from oracle import port


def oracle_sets(o, tg):
    """the per-level target sets det_loss takes, for one case's targets (supervised) or pseudo-label rows (SSOD)"""
    shapes = synth.level_shapes(IMG)
    if not o["ssod"]:
        return [port.build_targets(tg, synth.ANCHORS_GRID, shapes)]
    sel = port.select_targets(tg, [0.6] * o["nc"], [0.1] * o["nc"], with_obj=True)
    return [port.build_targets(sel[0][:, :6], synth.ANCHORS_GRID, shapes)] + \
           [port.build_targets(s, synth.ANCHORS_GRID, shapes, with_score=True) for s in sel[1:]]


@pytest.mark.parametrize("name", LOSS_CASES)
def test_det_loss_options_vs_reference(golden, name):
    g = golden("loss_opts_" + name)
    o = opts(g)
    nc = o["nc"]
    cp, cn = 1.0 - 0.5 * o["label_smoothing"], 0.5 * o["label_smoothing"]
    w = (0.05, 0.7, 0.3 * nc / 80.0)     # the yaml's Loss.box/obj/cls and SSOD.*_loss_weight agree; nl = 3
    balance = [4.0, 1.0, 0.4]
    for k in range(o["ncalls"]):
        logits, tg = inputs(nc, o["ssod"], k)
        p = [torch.from_numpy(x).requires_grad_(True) for x in logits]
        loss, (lbox, lobj, lcls) = loss_opts_port.det_loss(
            p, oracle_sets(o, tg), balance, *w, cp=cp, cn=cn, ignore_obj=o["ignore_obj"], with_bbox=o["with_bbox"],
            with_cls=o["with_cls"], cls_pw=o["cls_pw"], obj_pw=o["obj_pw"], fl_gamma=0.0 if o["ssod"] else o["fl_gamma"],
            autobalance=o["autobalance"] and not o["ssod"], ssi=1)
        got = np.array([float(v.detach()) for v in (lbox, lobj, lcls, loss)], np.float32)
        np.testing.assert_allclose(got, g[f"c{k}_items"], rtol=1e-5, atol=1e-8)
        if o["autobalance"]:
            np.testing.assert_allclose(balance, g[f"c{k}_balance"], rtol=1e-9)
        loss.backward()
        check_grads(g, f"c{k}_", [pi.grad.numpy() for pi in p], 1e-4)


def test_default_options_leave_det_loss_unchanged(golden):
    """the options at their defaults: bit for bit what oracle/port.det_loss computes, and the loss_sup fixture holds"""
    g = golden("loss_sup")
    B = int(g["B"])
    tg = synth.make_targets(int(g["target_seed"]), int(g["n"]), B)
    sets = [port.build_targets(tg, synth.ANCHORS_GRID, synth.level_shapes())]
    logits = synth.make_head_logits(int(g["logit_seed"]), B)
    a = port.det_loss([torch.from_numpy(x) for x in logits], sets, [4.0, 1.0, 0.4], 0.05, 0.7, 0.3)[0]
    b = loss_opts_port.det_loss([torch.from_numpy(x) for x in logits], sets, [4.0, 1.0, 0.4], 0.05, 0.7, 0.3, cls_pw=1.0,
                                obj_pw=1.0, fl_gamma=0.0, autobalance=False)[0]
    assert torch.equal(a, b)
    np.testing.assert_allclose(a.numpy(), g["loss"], rtol=1e-5)


@pytest.mark.parametrize("owner", ["sup", "ssod"])
def test_single_targets_assign_like_the_default(golden, owner):
    g = golden("loss_opts_single_targets")
    n, B = int(g["n"]), int(g["B"])
    t = synth.make_targets(int(g["seed"]), n, B)
    sc = np.random.RandomState(int(g["score_seed"])).uniform(0.1, 1, (n, 1)).astype(np.float32)
    bt = port.build_targets(t, synth.ANCHORS_GRID, synth.level_shapes())
    uc = port.build_targets(np.concatenate([t, sc], 1), synth.ANCHORS_GRID, synth.level_shapes(), with_score=True)
    for l in range(3):
        assert np.array_equal(bt[l]["idx"], g[f"{owner}_bt_idx{l}"])
        assert np.array_equal(bt[l]["tbox"], g[f"{owner}_bt_tbox{l}"])
        assert np.array_equal(uc[l]["idx"], g[f"{owner}_uc_idx{l}"])
        assert np.array_equal(uc[l]["tscore"], g[f"{owner}_uc_tscore{l}"])
