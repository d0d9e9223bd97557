"""The reference's ConfusionMatrix.process_batch (utils/metrics.py:129-186) restated in numpy, and the seeded images of
tests/golden/confusion_*.npz.

The restatement, for one image (detections [N, 6] x1,y1,x2,y2,conf,cls; labels [M, 5] cls,x1,y1,x2,y2; fp32):
  1. keep the detections with conf > fp32(conf) (original order);
  2. iou = box_iou(labels, detections) in fp32, inter / (area1 + area2 - inter) with area1 the label's; the candidate pairs
     are those with iou > fp32(iou_thres), whatever the classes;
  3. l*(d) = the label of d's highest-IoU candidate pair; m(l) = the highest-IoU detection among those with l*(d) = l.
     TIE RULE: on equal IoU the later label, then the later detection wins.  The reference sorts the pairs with numpy's
     argsort()[::-1], which puts equal IoUs in reverse of their original (label-major) order wherever that sort is stable;
  4. every label l adds one to matrix[cls(m(l)), cls(l)], or to matrix[nc, cls(l)] without m(l);
  5. only if the image has a candidate pair: every kept detection that is no label's m(l) adds one to matrix[cls(d), nc].
Classes truncate toward zero (Tensor.int()); a class outside [0, nc) raises IndexError when it is counted."""
import numpy as np

CONF, IOU = 0.25, 0.45


def box_iou(lab, det):
    """[M, 4] x [N, 4] xyxy fp32 -> [M, N] fp32, every step rounded in fp32 as torch does it"""
    lab, det = lab.astype(np.float32), det.astype(np.float32)
    area1 = (lab[:, 2] - lab[:, 0]) * (lab[:, 3] - lab[:, 1])
    area2 = (det[:, 2] - det[:, 0]) * (det[:, 3] - det[:, 1])
    w = (np.minimum(lab[:, None, 2], det[None, :, 2]) - np.maximum(lab[:, None, 0], det[None, :, 0])).clip(0)
    h = (np.minimum(lab[:, None, 3], det[None, :, 3]) - np.maximum(lab[:, None, 1], det[None, :, 1])).clip(0)
    inter = w * h
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / (area1[:, None] + area2[None, :] - inter)


def _match(det, lab, conf, iou_thres):
    """-> (kept detections, iou [M, n], candidate mask, l* [n], m [M]) of steps 1-3"""
    det = det[det[:, 4] > np.float32(conf)]
    iou = box_iou(lab[:, 1:5], det[:, :4])
    cand = iou > np.float32(iou_thres)
    lstar = np.full(det.shape[0], -1)
    for d in range(det.shape[0]):
        ls = np.flatnonzero(cand[:, d])
        if ls.size:
            lstar[d] = ls[iou[ls, d] == iou[ls, d].max()].max()          # ties: the later label
    m = np.full(lab.shape[0], -1)
    for l in range(lab.shape[0]):
        ds = np.flatnonzero(lstar == l)
        if ds.size:
            m[l] = ds[iou[l, ds] == iou[l, ds].max()].max()              # ties: the later detection
    return det, iou, cand, lstar, m


def _cls(c, nc):
    k = int(np.float32(c))          # truncation toward zero, like Tensor.int()
    if not 0 <= k < nc:
        raise IndexError("class %r outside [0, %d)" % (c, nc))
    return k


def process_batch(matrix, detections, labels, conf=CONF, iou_thres=IOU):
    """adds one image into matrix [nc+1, nc+1] (float64, in place)"""
    nc = matrix.shape[0] - 1
    det, _, cand, _, m = _match(np.asarray(detections, np.float32), np.asarray(labels, np.float32), conf, iou_thres)
    for l in range(labels.shape[0]):
        matrix[_cls(det[m[l], 5], nc) if m[l] >= 0 else nc, _cls(labels[l, 0], nc)] += 1
    if cand.any():
        for d in range(det.shape[0]):
            if d not in m:
                matrix[_cls(det[d, 5], nc), nc] += 1
    return matrix


def deciding_ties(detections, labels, conf=CONF, iou_thres=IOU):
    """The number of exact IoU ties that decide l* or m: a detection whose highest candidate IoU is shared by two labels, or
    a label whose highest IoU among the detections that have it as best label is shared by two of them.  Where it is zero,
    numpy's sort order cannot change the reference's result."""
    det, iou, cand, lstar, _ = _match(np.asarray(detections, np.float32), np.asarray(labels, np.float32), conf, iou_thres)
    n = 0
    for d in range(det.shape[0]):
        v = iou[cand[:, d], d]
        n += v.size and int((v == v.max()).sum() > 1)
    for l in range(labels.shape[0]):
        v = iou[l, lstar == l]
        n += v.size and int((v == v.max()).sum() > 1)
    return n


# ---- the golden images ---------------------------------------------------------------------------------------------------

def _boxes(r, k, size=640.0):
    xy = r.uniform(0, size * 0.8, (k, 2))
    wh = r.uniform(8, size * 0.3, (k, 2))
    return np.concatenate([xy, np.minimum(xy + wh, size)], 1)


def _jitter(r, box, s):
    w, h = box[2] - box[0], box[3] - box[1]
    return box + r.uniform(-s, s, 4) * np.array([w, h, w, h])


def _image(r, nc, n_lab, conf_edge=False):
    """labels with Poisson-ish counts; detections: jittered copies of labels (some labels get many, with the true or a
    random class), random boxes, a box over several labels, and the same box emitted with two classes"""
    lab = np.concatenate([r.randint(0, nc, (n_lab, 1)), _boxes(r, n_lab)], 1)
    rows = []
    for l in range(n_lab):
        for _ in range(r.choice([0, 1, 1, 2, 5])):
            c = lab[l, 0] if r.rand() < 0.7 else r.randint(0, nc)
            rows.append(np.r_[_jitter(r, lab[l, 1:], r.choice([0.05, 0.15, 0.35])), r.rand(), c])
    for b in _boxes(r, r.randint(0, 6)):
        rows.append(np.r_[b, r.rand(), r.randint(0, nc)])
    if n_lab >= 2:      # one detection over many labels: the union of a few label boxes
        ls = lab[r.choice(n_lab, min(n_lab, 3), replace=False), 1:]
        rows.append(np.r_[ls[:, :2].min(0), ls[:, 2:].max(0), r.rand(), r.randint(0, nc)])
    det = np.asarray(rows, np.float64).reshape(-1, 6)
    if conf_edge and len(det):
        edge = np.float32(CONF)
        det[:, 4] = r.choice([np.nextafter(edge, np.float32(0)), edge, np.nextafter(edge, np.float32(1)), 0.1, 0.6], len(det))
    if n_lab and nc > 1:    # multi-label NMS: one box with two classes; a tighter detection holds its label (no IoU tie)
        box = _jitter(r, lab[0, 1:], 0.2)
        c1, c2 = r.choice(nc, 2, replace=False)
        det = np.concatenate([det, [np.r_[_jitter(r, lab[0, 1:], 0.01), 0.9, lab[0, 0]], np.r_[box, 0.7, c1], np.r_[box, 0.6, c2]]])
    return det.astype(np.float32), lab.astype(np.float32)


def _iou_edge_image(r, nc):
    """IoUs on both sides of fp32(0.45): label [0, 0, 100, 100], detections [0, 0, w, 100] with IoU = w / 100"""
    lab = np.array([[r.randint(0, nc), 0, 0, 100, 100]], np.float32)
    e = np.float32(45)
    ws = [np.nextafter(np.nextafter(e, np.float32(0)), np.float32(0)), np.nextafter(e, np.float32(0)), e, np.nextafter(e, np.float32(99)),
          np.float32(45.01), np.float32(44.99)]
    det = np.array([[0, 0, w, 100, 0.5 + 0.01 * i, r.randint(0, nc)] for i, w in enumerate(ws)], np.float32)
    return det, lab


def golden_cases():
    """name -> (nc, [(detections [N, 6], labels [M, 5]), ...]) fp32"""
    cases = {}
    for nc in (1, 2, 8, 20, 80):
        r = np.random.RandomState(100 + nc)
        imgs = [_image(r, nc, r.poisson(5) + 1, conf_edge=(i % 3 == 0)) for i in range(24)]
        imgs.append(_iou_edge_image(r, nc))
        cases["nc%d" % nc] = (nc, imgs)
    r = np.random.RandomState(7)
    nc = 8
    lab = np.concatenate([r.randint(0, nc, (1, 1)), [[100, 100, 300, 260]]], 1).astype(np.float32)
    many = np.array([np.r_[_jitter(r, lab[0, 1:], 0.02 + 0.01 * k), 0.3 + 0.02 * k, r.randint(0, nc)] for k in range(30)], np.float32)
    labs = np.concatenate([r.randint(0, nc, (6, 1)), [[60 * k, 40, 60 * k + 70, 120] for k in range(6)]], 1).astype(np.float32)
    big = np.array([[0, 30, 400, 130, 0.8, 3], [5, 41, 72, 119, 0.7, 1]], np.float32)
    far = np.array([[500, 500, 600, 600, 0.9, 2], [520, 10, 630, 90, 0.3, 5]], np.float32)
    low = many.copy()
    low[:, 4] = r.uniform(0.0, 0.25, len(low)).astype(np.float32)
    cases["shapes"] = (nc, [(many, lab),            # many detections on one label
                            (big, labs),            # one detection over many labels
                            (far, labs),            # no pair above the threshold: step 5 is skipped
                            (low, lab),             # no detection above conf
                            (low[:0], labs)])       # no detection at all
    return cases


def matrix_of(nc, images, conf=CONF, iou_thres=IOU):
    m = np.zeros((nc + 1, nc + 1))
    for det, lab in images:
        process_batch(m, det, lab, conf, iou_thres)
    return m
