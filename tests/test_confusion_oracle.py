"""CPU: tests/confusion_port.py (the numpy restatement of ConfusionMatrix.process_batch that etb_confusion_matrix follows)
against the golden matrices of the live reference's utils.metrics.ConfusionMatrix (tests/golden/confusion_*.npz,
tests/golden/make_golden_confusion.py), and its stated tie rule on hand-made ties."""
import numpy as np
import pytest

import confusion_port as cp

CASES = ("nc1", "nc2", "nc8", "nc20", "nc80", "shapes")


@pytest.mark.parametrize("name", CASES)
def test_port_matches_reference_golden(golden, name):
    nc, images = cp.golden_cases()[name]
    want = golden("confusion_" + name)["matrix"]
    assert want.dtype == np.float64 and want.shape == (nc + 1, nc + 1)
    assert all(cp.deciding_ties(d, l) == 0 for d, l in images)
    assert np.array_equal(cp.matrix_of(nc, images), want)


def test_golden_cases_cover_the_edges():
    cases = cp.golden_cases()
    edge = np.float32(cp.CONF)
    confs = np.concatenate([d[:, 4] for nc, imgs in cases.values() for d, _ in imgs])
    assert {np.nextafter(edge, np.float32(0)), edge, np.nextafter(edge, np.float32(1))} <= set(confs.tolist())
    nc, imgs = cases["nc8"]
    d, l = imgs[-1]
    iou = cp.box_iou(l[:, 1:], d[:, :4])[0]
    thr = np.float32(cp.IOU)
    assert (iou == thr).any() and (iou < thr).any() and (iou > thr).any()
    # the same box emitted with two classes, in every multi-class image with labels
    assert all(np.array_equal(d[-1, :4], d[-2, :4]) and d[-1, 5] != d[-2, 5] for d, _ in imgs[:-1])
    # shapes: no pair above the threshold -> no background column count; no detection above conf -> labels all missed
    nc, (many, one_big, far, low, none) = cases["shapes"]
    m = cp.matrix_of(nc, [far])
    assert m[:, nc].sum() == 0 and m[nc].sum() == len(far[1])
    for img in (low, none):
        m = cp.matrix_of(nc, [img])
        assert m.sum() == m[nc].sum() == len(img[1])


def test_ties_follow_the_stated_rule():
    """equal IoU: the later label wins a detection, then the later detection wins a label"""
    nc = 4
    lab = np.array([[0, 0, 0, 10, 10], [1, 0, 0, 10, 10]], np.float32)      # the same box twice, classes 0 and 1
    det = np.array([[0, 0, 10, 10, 0.9, 2], [0, 0, 10, 10, 0.8, 3]], np.float32)
    m = cp.matrix_of(nc, [(det, lab)])
    want = np.zeros((nc + 1, nc + 1))
    want[3, 1] = 1          # label 1 (the later) is both detections' best label; detection 1 (the later) is its match
    want[nc, 0] = 1         # label 0: no match
    want[2, nc] = 1         # detection 0: no label's match, and the image has pairs
    assert np.array_equal(m, want)
    # numpy's argsort()[::-1] on a short array (a stable insertion sort) gives this order too
    matches = np.array([[0, 0, 1.0], [0, 1, 1.0], [1, 0, 1.0], [1, 1, 1.0]], np.float32)
    s = matches[matches[:, 2].argsort(kind="stable")[::-1]]
    s = s[np.unique(s[:, 1], return_index=True)[1]]
    s = s[s[:, 2].argsort(kind="stable")[::-1]]
    s = s[np.unique(s[:, 0], return_index=True)[1]]
    assert s[:, :2].tolist() == [[1, 1]]


def test_out_of_range_class_raises():
    det = np.array([[0, 0, 10, 10, 0.9, 5]], np.float32)
    lab = np.array([[0, 0, 0, 10, 10]], np.float32)
    with pytest.raises(IndexError):
        cp.matrix_of(4, [(det, lab)])
    with pytest.raises(IndexError):
        cp.matrix_of(4, [(det[:, [0, 1, 2, 3, 4, 4]] * 0 + [0, 0, 10, 10, 0.9, 1], lab + [7, 0, 0, 0, 0])])
