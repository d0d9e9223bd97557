"""GPU (H100): the anchor-free (YOLOv8 / TAL) operators of csrc/tal.cu through their reference-shaped mirrors
(efficientteacher_b200/tal.py) against the golden vectors of the live reference and the oracle (oracle/port_v8.py).
Labels / boxes / foreground masks bit-exact; target_scores within 1e-5 relative (the alignment metric goes through pow);
decoded boxes within 1e-5 relative.

This file sorts last on purpose: a failure here must never hide the results of the older suite before it (pytest -x)."""
import os

import numpy as np
import pytest
import torch

import synth
from oracle import port_v8
from test_v8_oracle import check_tal_against_golden, tal_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)


def _assign(d, **kw):
    from efficientteacher_b200.tal import TaskAlignedAssigner
    asg = TaskAlignedAssigner(top_k=13, num_classes=d["pd_scores"].shape[-1], alpha=1.0, beta=6.0, **kw)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in d.items()}
    out = asg(t["pd_scores"], t["pd_bboxes"], t["anc_points"], t["gt_labels"], t["gt_bboxes"], t["mask_gt"])
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", ["a", "b", "c", "d"])
def test_tal_assign_matches_live_reference_golden(name):
    g, d = tal_case(name)
    labels, bboxes, scores, fg = _assign(d)
    assert labels.dtype == torch.int64 and fg.dtype == torch.bool and scores.dtype == torch.float32
    check_tal_against_golden(g, labels.cpu().numpy(), bboxes.cpu().numpy(), scores.cpu().numpy(), fg.cpu().numpy(), score_tol=1e-5)


def test_tal_assign_without_gts_returns_the_reference_quirk():
    g = np.load(os.path.join(GOLD, "tal_empty.npz"))
    labels, bboxes, scores, fg = _assign(synth.make_tal_inputs(65, 2, [0, 0], img=320))
    assert labels.dtype == torch.float32 and np.array_equal(labels.cpu().numpy(), g["labels"])
    assert fg.dtype == torch.float32 and np.array_equal(fg.cpu().numpy(), g["fg"])
    assert float(bboxes.abs().max()) == 0.0 and float(scores.abs().max()) == 0.0


def test_tal_assign_batch32_vs_oracle():
    """BASELINE configs[3] per-GPU shape: 32 images x 8400 anchors x 80 classes, 8 gts per image (SURVEY.md section 8d)."""
    d = synth.make_tal_inputs(66, 32, [8] * 32, img=640)
    labels, bboxes, scores, fg = _assign(d)
    rl, rb, rs, rf = port_v8.tal_assign(d["pd_scores"], d["pd_bboxes"], d["anc_points"], d["gt_labels"], d["gt_bboxes"], d["mask_gt"])
    assert np.array_equal(fg.cpu().numpy(), rf) and np.array_equal(labels.cpu().numpy(), rl) and np.array_equal(bboxes.cpu().numpy(), rb)
    np.testing.assert_allclose(scores.cpu().numpy(), rs, rtol=1e-5, atol=1e-12)
    # properties that hold at any size: a foreground anchor carries at most one non-zero class score, a background anchor none
    s = scores.cpu().numpy()
    f = fg.cpu().numpy()
    assert ((s != 0).sum(-1)[~f] == 0).all() and ((s != 0).sum(-1)[f] <= 1).all()
    assert (s >= 0).all() and s.max() <= 1.0 + 1e-6        # normalised metric <= the gt's best IoU <= 1


def test_tal_assign_is_deterministic_and_stream_ordered():
    d = synth.make_tal_inputs(67, 4, [20, 3, 11, 7], img=640, score_pow=2)
    a = _assign(d)
    b = _assign(d)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("name", ["a", "b"])
def test_v8_decode_eval_matches_live_head(name):
    from efficientteacher_b200 import tal
    g = np.load(os.path.join(GOLD, "v8_head.npz"))
    seed, B, img, reg_max, step = [int(v) for v in g["meta_" + name]]
    cls, reg = synth.make_v8_head_logits(seed, B, img=img, reg_max=reg_max)
    y = tal.decode_eval(torch.from_numpy(cls).to(DEV), torch.from_numpy(reg).to(DEV), synth.level_shapes(img), synth.STRIDES, reg_max)
    torch.cuda.synchronize()
    assert tuple(y.shape) == (B, cls.shape[1], 85)
    np.testing.assert_allclose(y.cpu().numpy()[:, ::step], g["pred_" + name], rtol=1e-5, atol=1e-4)


def test_v8_assigner_inputs_vs_oracle_and_into_the_assigner():
    """tal_loss.py:88-101 as one pass: grid-unit boxes, sigmoid scores, pixel boxes; then the assigner on them == the oracle chain."""
    from efficientteacher_b200 import tal
    img, B, reg_max = 320, 3, 16
    cls, reg = synth.make_v8_head_logits(81, B, img=img, reg_max=reg_max)
    shapes = synth.level_shapes(img)
    bg, sc, bp = tal.assigner_inputs(torch.from_numpy(cls).to(DEV), torch.from_numpy(reg).to(DEV), shapes, synth.STRIDES, reg_max)
    torch.cuda.synchronize()
    pts, st = port_v8.generate_anchors(shapes, synth.STRIDES, 0.5, is_eval=False)
    want = port_v8.bbox_decode(pts / st, reg, reg_max)
    np.testing.assert_allclose(bg.cpu().numpy(), want, rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(bp.cpu().numpy(), want * st[None], rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(sc.cpu().numpy(), torch.sigmoid(torch.from_numpy(cls)).numpy(), rtol=1e-5, atol=1e-7)
    only = tal.bbox_decode(torch.from_numpy(reg).to(DEV), shapes, synth.STRIDES, reg_max)
    assert torch.equal(only, bg)
    # feed the device tensors straight into the assigner; the oracle gets the SAME (device-computed) inputs
    d = synth.make_tal_inputs(82, B, [6, 2, 9], img=img)
    from efficientteacher_b200.tal import TaskAlignedAssigner
    asg = TaskAlignedAssigner(13, 80)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in d.items()}
    labels, bboxes, scores, fg = asg(sc, bp, t["anc_points"], t["gt_labels"], t["gt_bboxes"], t["mask_gt"])
    rl, rb, rs, rf = port_v8.tal_assign(sc.cpu().numpy(), bp.cpu().numpy(), d["anc_points"], d["gt_labels"], d["gt_bboxes"], d["mask_gt"])
    assert np.array_equal(fg.cpu().numpy(), rf) and np.array_equal(labels.cpu().numpy(), rl) and np.array_equal(bboxes.cpu().numpy(), rb)
    np.testing.assert_allclose(scores.cpu().numpy(), rs, rtol=1e-5, atol=1e-12)


def test_generate_anchors_on_device():
    from efficientteacher_b200 import tal
    g = np.load(os.path.join(GOLD, "v8_anchors.npz"))
    feats = [torch.zeros(1, 1, h, w, device=DEV) for h, w in synth.level_shapes(640)]
    pts, st = tal.generate_anchors(feats, [8, 16, 32], 5.0, 0.5, device=DEV, is_eval=True)
    assert np.array_equal(pts.cpu().numpy(), g["eval_pts_640"]) and np.array_equal(st.cpu().numpy(), g["eval_stride_640"])
    _, pts_t, counts, st_t = tal.generate_anchors(feats, [8, 16, 32], 5.0, 0.5, device=DEV, is_eval=False)
    assert np.array_equal(pts_t.cpu().numpy(), g["train_pts_640"]) and np.array_equal(st_t.cpu().numpy(), g["train_stride_640"])
    assert counts == [6400, 1600, 400]
