"""CPU: oracle/port_v8.py (restatement of the reference's importable YOLOv8 / TAL pieces) against the golden vectors that
tests/golden/make_golden_v8.py (and, for three fresh seeds, tests/golden/make_golden_trunk.py) generated from the live,
unmodified reference."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import synth  # noqa: E402
from oracle import port_v8  # noqa: E402

GOLD = os.path.join(HERE, "golden")


def tal_case(name):
    g = np.load(os.path.join(GOLD, "tal_%s.npz" % name))
    seed, B, img, sp, tiny = [int(v) for v in g["meta"][:5]]
    n_gt = [int(v) for v in g["meta"][5:]]
    return g, synth.make_tal_inputs(seed, B, n_gt, img=img, score_pow=sp, tiny=tiny)


def check_tal_against_golden(g, labels, bboxes, scores, fg, score_tol=1e-6):
    """Shared with the GPU parity test: labels / boxes / foreground mask bit-exact, scores to score_tol (relative)."""
    assert np.array_equal(fg, g["fg"])
    assert labels.dtype == np.int64 and np.array_equal(labels, g["labels"])
    assert np.array_equal(bboxes[fg], g["bboxes_fg"])
    assert np.array_equal(np.unique(bboxes[~fg], axis=0), g["bboxes_bg_unique"])
    assert tuple(scores.shape) == tuple(g["score_shape"])
    idx = g["score_idx"]
    nz = np.argwhere(scores != 0)
    assert np.array_equal(nz, idx), "non-zero pattern of target_scores differs"
    got = scores[idx[:, 0], idx[:, 1], idx[:, 2]]
    np.testing.assert_allclose(got, g["score_val"], rtol=score_tol, atol=1e-12)


@pytest.mark.parametrize("name", ["a", "b", "c", "d"])
def test_tal_assign_matches_live_reference_golden(name):
    g, d = tal_case(name)
    labels, bboxes, scores, fg = port_v8.tal_assign(d["pd_scores"], d["pd_bboxes"], d["anc_points"], d["gt_labels"], d["gt_bboxes"], d["mask_gt"])
    check_tal_against_golden(g, labels, bboxes, scores, fg)


def test_tal_assign_without_gts():
    g = np.load(os.path.join(GOLD, "tal_empty.npz"))
    d = synth.make_tal_inputs(65, 2, [0, 0], img=320)
    labels, bboxes, scores, fg = port_v8.tal_assign(d["pd_scores"], d["pd_bboxes"], d["anc_points"], d["gt_labels"], d["gt_bboxes"], d["mask_gt"])
    assert labels.dtype == g["labels"].dtype and np.array_equal(labels, g["labels"])
    assert fg.dtype == g["fg"].dtype and np.array_equal(fg, g["fg"])
    assert float(np.abs(bboxes).max()) == 0.0 == float(g["bboxes_absmax"]) and float(np.abs(scores).max()) == 0.0


def test_generate_anchors_bit_exact():
    g = np.load(os.path.join(GOLD, "v8_anchors.npz"))
    for img in (320, 640):
        for mode, ev in (("eval", True), ("train", False)):
            pts, st = port_v8.generate_anchors(synth.level_shapes(img), synth.STRIDES, 0.5, is_eval=ev)
            assert np.array_equal(pts, g["%s_pts_%d" % (mode, img)]) and np.array_equal(st, g["%s_stride_%d" % (mode, img)])
    d = synth.make_tal_inputs(1, 1, [1], img=640)        # the synthetic assigner inputs use exactly these points
    assert np.array_equal(d["anc_points"], g["train_pts_640"]) and np.array_equal(d["stride"], g["train_stride_640"])


@pytest.mark.parametrize("name", ["a", "b"])
def test_v8_detect_eval_decode(name):
    g = np.load(os.path.join(GOLD, "v8_head.npz"))
    seed, B, img, reg_max, step = [int(v) for v in g["meta_" + name]]
    cls, reg = synth.make_v8_head_logits(seed, B, img=img, reg_max=reg_max)
    y = port_v8.v8_detect_eval(cls, reg, synth.level_shapes(img), synth.STRIDES, reg_max)
    np.testing.assert_allclose(y[:, ::step], g["pred_" + name], rtol=1e-5, atol=1e-4)


def test_preprocess_and_bbox_decode_text_restatement():
    """models/loss/tal_loss.py cannot be imported (missing modules), so these two follow the text; pinned indirectly: bbox_decode
    shares dfl_expectation with the eval decode above; preprocess is checked on a hand-computed case."""
    t = np.array([[0, 3, .5, .5, .2, .4], [2, 7, .25, .75, .1, .1], [0, 1, .1, .2, .05, .05]], np.float64)
    out, num = port_v8.preprocess(t, 3, 640)
    assert out.shape == (3, 2, 5) and num == 6          # the reference counts its dummy first rows too
    np.testing.assert_allclose(out[0, 0], [3, 256, 192, 384, 448])
    np.testing.assert_allclose(out[1], [[-1, 0, 0, 0, 0], [-1, 0, 0, 0, 0]])
    np.testing.assert_allclose(out[2, 0], [7, 128, 448, 192, 512])
    pts, st = port_v8.generate_anchors(synth.level_shapes(320), synth.STRIDES, 0.5, is_eval=False)
    _, reg = synth.make_v8_head_logits(5, 1, img=320)
    box = port_v8.bbox_decode(pts / st, reg, 16)
    assert box.shape == (1, 2100, 4) and (box[..., 2:] >= box[..., :2]).all()


def test_tal_assign_vs_live_reference_fresh_seeds():
    """Three more seeds, outside the cases the oracle was written against (tests/golden/make_golden_trunk.py stored the live
    reference's assignments)."""
    for name in ("fresh101", "fresh102", "fresh103"):
        g, d = tal_case(name)
        labels, bboxes, scores, fg = port_v8.tal_assign(d["pd_scores"], d["pd_bboxes"], d["anc_points"], d["gt_labels"], d["gt_bboxes"], d["mask_gt"])
        check_tal_against_golden(g, labels, bboxes, scores, fg)


def test_mirror_generate_anchors_and_no_cpu_fallback():
    """Host side of efficientteacher_b200/tal.py: the anchor tables equal the live reference's (they are constants, built with
    torch on any device); the operators themselves raise without CUDA -- there is no CPU path."""
    from efficientteacher_b200 import tal
    g = np.load(os.path.join(GOLD, "v8_anchors.npz"))
    for img in (320, 640):
        feats = [torch.zeros(1, 1, h, w) for h, w in synth.level_shapes(img)]
        pts, st = tal.generate_anchors(feats, [8, 16, 32], 5.0, 0.5, device='cpu', is_eval=True)
        assert np.array_equal(pts.numpy(), g["eval_pts_%d" % img]) and np.array_equal(st.numpy(), g["eval_stride_%d" % img])
        anchors, pts_t, counts, st_t = tal.generate_anchors(feats, [8, 16, 32], 5.0, 0.5, device='cpu', is_eval=False)
        assert np.array_equal(pts_t.numpy(), g["train_pts_%d" % img]) and np.array_equal(st_t.numpy(), g["train_stride_%d" % img])
        assert counts == [h * w for h, w in synth.level_shapes(img)] and anchors.shape == (sum(counts), 4)
    if not torch.cuda.is_available():
        d = synth.make_tal_inputs(1, 1, [2], img=320)
        t = {k: torch.from_numpy(v) for k, v in d.items()}
        with pytest.raises(RuntimeError):
            tal.TaskAlignedAssigner()(t["pd_scores"], t["pd_bboxes"], t["anc_points"], t["gt_labels"], t["gt_bboxes"], t["mask_gt"])
        cls, reg = synth.make_v8_head_logits(1, 1, img=320)
        with pytest.raises(RuntimeError):
            tal.decode_eval(torch.from_numpy(cls), torch.from_numpy(reg), synth.level_shapes(320), synth.STRIDES)
