"""Seeded synthetic inputs shared by the golden-vector generator, the CPU tests and the GPU parity tests.
numpy RandomState only (bit-reproducible across machines); recipes follow SURVEY.md section 8d."""
import numpy as np

F32 = np.float32
ANCHORS_GRID = np.array([[[1.25, 1.625], [2.0, 3.75], [4.125, 2.875]],
                         [[1.875, 3.8125], [3.875, 2.8125], [3.6875, 7.4375]],
                         [[3.625, 2.8125], [4.875, 6.1875], [11.65625, 10.1875]]], dtype=F32)  # YOLOv5 anchors / stride
STRIDES = (8, 16, 32)


def level_shapes(img=640):
    return [(img // s, img // s) for s in STRIDES]


def make_targets(seed, n, B, with_conf=False, nc=80):
    """[n,6] (img,cls,x,y,w,h) normalised, classes in [0, nc); includes exact cell-boundary (.5) cases and same-cell
    duplicates."""
    r = np.random.RandomState(seed)
    t = np.zeros((n, 6), F32)
    t[:, 0] = r.randint(0, B, n)
    t[:, 1] = r.randint(0, nc, n)
    t[:, 2:4] = r.uniform(0.1, 0.9, (n, 2))
    t[:, 4:6] = r.uniform(0.02, 0.32, (n, 2))
    k = n // 16
    if k == 0:
        return t[np.argsort(t[:, 0], kind="stable")]
    t[:k, 2] = (r.randint(8, 72, k) + 0.5) / 80.0      # gx % 1 == 0.5 exactly on P3
    t[k:2 * k, 3] = r.randint(8, 72, k) / 80.0          # gy % 1 == 0
    t[2 * k:3 * k] = t[3 * k:4 * k]                     # duplicate rows -> duplicate cells
    t = t[np.argsort(t[:, 0], kind="stable")]
    return t


def make_teacher_pred(seed, B, P, nc=80, cand_frac=0.02, img=640):
    """Decoded teacher predictions [B,P,5+nc] (SURVEY.md 8d probe4 recipe): ~cand_frac of rows have obj>0.1."""
    r = np.random.RandomState(seed)
    x = np.empty((B, P, 5 + nc), F32)
    x[..., 0:2] = r.uniform(0, img, (B, P, 2))
    x[..., 2:4] = r.uniform(4, 196, (B, P, 2))
    hot = r.uniform(0, 1, (B, P)) < cand_frac
    x[..., 4] = np.where(hot, r.uniform(0.1, 1.0, (B, P)), r.uniform(0, 0.05, (B, P)))
    x[..., 5:] = r.uniform(0, 1, (B, P, nc)) ** 4
    return x.astype(F32)


def make_Ms(seed, B, img=640):
    """[B,13] float64 = [i, M (3x3 row-major: scale about centre + translate), s, ud, lr] (datasets_ssod.py:989)."""
    r = np.random.RandomState(seed)
    Ms = np.zeros((B, 13))
    for i in range(B):
        s = r.uniform(0.5, 1.5)
        tx, ty = r.uniform(-0.1, 0.1, 2) * img
        C = np.array([[1, 0, -img / 2], [0, 1, -img / 2], [0, 0, 1.0]])
        R = np.array([[s, 0, 0], [0, s, 0], [0, 0, 1.0]])
        T = np.array([[1, 0, img / 2 + tx], [0, 1, img / 2 + ty], [0, 0, 1.0]])
        M = T @ R @ C
        Ms[i, 0] = i
        Ms[i, 1:10] = M.reshape(-1)
        Ms[i, 10] = s
        Ms[i, 11] = 1.0 if (i % 5 == 3) else 0.0
        Ms[i, 12] = float(r.uniform() < 0.5)
    return Ms


def make_pseudo_rows(seed, n, B, nc=80):
    """[n,9] float64 pseudo-label rows (classes in [0, nc)) with confidences straddling the 0.1 / 0.6 / 0.99 thresholds."""
    r = np.random.RandomState(seed)
    t = make_targets(seed + 1, n, B, nc=nc).astype(np.float64)
    conf = r.uniform(0.02, 1.0, n)
    obj = np.where(r.uniform(size=n) < 0.3, r.uniform(0.99, 1.0, n), r.uniform(0.1, 1.0, n))
    cc = np.where(r.uniform(size=n) < 0.3, r.uniform(0.99, 1.0, n), r.uniform(0.1, 1.0, n))
    conf[:4] = [0.6, 0.1, np.float64(np.float32(0.6)), np.float64(np.float32(0.1))]   # exact-threshold cases
    return np.concatenate([t, conf[:, None], obj[:, None], cc[:, None]], 1)


def make_teacher_pred_ties(seed, B, nc, ties, img=640):
    """make_teacher_pred over every prediction of an img x img input at cand_frac 0.05; ties: class scores quantized to
    quarters and candidate objectness to sixteenths, so the maximal class of a row is often shared (the first one wins) and
    rows tie on confidence"""
    P = sum(3 * ny * nx for ny, nx in level_shapes(img))
    pred = make_teacher_pred(seed, B, P, nc=nc, cand_frac=0.05, img=img)
    if ties:
        pred[..., 5:] = np.round(pred[..., 5:] * 4) / 4
        pred[..., 4] = np.where(pred[..., 4] > 0.1, np.round(pred[..., 4] * 16) / 16, pred[..., 4])
    return pred


def make_class_thresholds(nc):
    """per-class (ignore_thres_high, ignore_thres_low) of ComputeStudentMatchLoss, not uniform across classes"""
    r = np.random.RandomState(200 + nc)
    return r.uniform(0.4, 0.8, nc), r.uniform(0.05, 0.3, nc)


def make_pseudo_rows_dup(seed, n, B, nc=80):
    """make_pseudo_rows whose first n/8 boxes come again with other confidences (duplicate cells across the routed sets),
    sorted by image"""
    rows = make_pseudo_rows(seed, n, B, nc=nc)
    k = n // 8
    rows[k:2 * k, :6] = rows[:k, :6]
    return rows[np.argsort(rows[:, 0], kind="stable")]


def grad_sample_idx(numel, level):
    """the gradient elements the class-count loss fixtures store for one level"""
    return np.random.RandomState(300 + level).randint(0, numel, 1024)


def make_head_logits(seed, B, img=640, no=85, scale=1.5):
    """Raw Detect train-mode outputs: list of [B,3,ny,nx,no] fp32."""
    r = np.random.RandomState(seed)
    out = []
    for (ny, nx) in level_shapes(img):
        x = (r.standard_normal((B, 3, ny, nx, no)) * scale).astype(F32)
        x[..., 4] -= 3.0
        out.append(x)
    return out


def make_images(seed, n, img=640, targets=None):
    """Seeded synthetic images with spatial structure, uint8 [n,3,img,img] like the loaders produce: a smooth low-frequency
    colour field, ~10 textured rectangles per image (at the ground-truth boxes when `targets` [nt,6] is given, random
    otherwise) and mild pixel noise.  I.i.d. uniform noise images drive a random-init YOLOv5 into a regime where every image
    looks the same to every layer and the teacher's logits are ~7x more sensitive to parameter perturbations (DESIGN.md)."""
    r = np.random.RandomState(seed)
    g = img // 32 + 1
    out = np.empty((n, 3, img, img), np.uint8)
    yy = np.linspace(0, g - 1, img)
    y0 = np.floor(yy).astype(int).clip(0, g - 2)
    fy = (yy - y0).astype(F32)
    for i in range(n):
        lo = r.rand(3, g, g).astype(F32)
        rows = lo[:, y0, :] * (1 - fy)[None, :, None] + lo[:, y0 + 1, :] * fy[None, :, None]          # bilinear, rows
        im = rows[:, :, y0] * (1 - fy)[None, None, :] + rows[:, :, y0 + 1] * fy[None, None, :]         # bilinear, cols
        if targets is not None:
            t = np.asarray(targets)[np.asarray(targets)[:, 0] == i]
            boxes = [(int((b[2] - b[4] / 2) * img), int((b[3] - b[5] / 2) * img), max(int(b[4] * img), 2), max(int(b[5] * img), 2)) for b in t]
        else:
            boxes = []
            for _ in range(10):
                w, h = r.randint(img // 20, img // 3, 2)
                boxes.append((int(r.randint(0, img - w)), int(r.randint(0, img - h)), int(w), int(h)))
        for (x0, y0b, w, h) in boxes:
            x0, y0b = max(x0, 0), max(y0b, 0)
            x1, y1 = min(x0 + w, img), min(y0b + h, img)
            if x1 <= x0 or y1 <= y0b:
                continue
            col = r.rand(3, 1, 1).astype(F32)
            tex = (r.rand(3, y1 - y0b, x1 - x0).astype(F32) - 0.5) * 0.3
            im[:, y0b:y1, x0:x1] = col + tex
        im = im + (r.rand(3, img, img).astype(F32) - 0.5) * 0.08
        out[i] = (np.clip(im, 0, 1) * 255.0 + 0.5).astype(np.uint8)
    return out


def make_tal_inputs(seed, B, n_gt, img=640, nc=80, reg_max=16, score_pow=4, tiny=0):
    """Inputs of TaskAlignedAssigner.forward as models/loss/tal_loss.py:76-101 would build them (SURVEY.md section 8d, config #4):
    pd_scores ~ U(0,1)^score_pow [B,A,nc]; pd_bboxes = DFL-style boxes around each anchor point (ltrb distances ~ U(0, reg_max)
    grid cells, times the stride) in pixels; n_gt[b] ground-truth boxes per image (xyxy pixels, centre U(.1,.9), size U(.02,.5)),
    padded with label -1 / zero boxes to max(n_gt); `tiny` of the first image's boxes are smaller than one P3 cell (fewer than
    13 anchor points inside -> the top-k runs over zeros).  Returns fp32 arrays (labels as float, like the reference's targets)."""
    r = np.random.RandomState(seed)
    shapes = level_shapes(img)
    pts, st = [], []
    for (h, w), s in zip(shapes, STRIDES):
        yy, xx = np.meshgrid((np.arange(h, dtype=F32) + F32(0.5)) * F32(s), (np.arange(w, dtype=F32) + F32(0.5)) * F32(s), indexing="ij")
        pts.append(np.stack([xx, yy], -1).reshape(-1, 2))
        st.append(np.full((h * w, 1), s, F32))
    anc, stride = np.concatenate(pts).astype(F32), np.concatenate(st)
    A = anc.shape[0]
    pd_scores = (r.uniform(0, 1, (B, A, nc)) ** score_pow).astype(F32)
    dist = (r.uniform(0, reg_max, (B, A, 4)).astype(F32)) * stride[None]
    pd_bboxes = np.concatenate([anc[None] - dist[..., :2], anc[None] + dist[..., 2:]], -1).astype(F32)
    M = max(n_gt) if len(n_gt) else 0
    gt_labels = np.full((B, M, 1), -1, F32)
    gt_bboxes = np.zeros((B, M, 4), F32)
    for b in range(B):
        n = n_gt[b]
        c = r.uniform(0.1, 0.9, (n, 2)) * img
        wh = r.uniform(0.02, 0.5, (n, 2)) * img
        if b == 0 and tiny:
            wh[:tiny] = r.uniform(2.0, 7.0, (tiny, 2))
        gt_bboxes[b, :n] = np.concatenate([c - wh / 2, c + wh / 2], -1).astype(F32)
        gt_labels[b, :n, 0] = r.randint(0, nc, n)
    mask_gt = (gt_bboxes.sum(-1, keepdims=True) > 0).astype(F32)
    return dict(pd_scores=pd_scores, pd_bboxes=pd_bboxes, anc_points=anc, gt_labels=gt_labels, gt_bboxes=gt_bboxes, mask_gt=mask_gt,
                stride=stride)


def make_v8_head_logits(seed, B, img=640, nc=80, reg_max=16, scale=2.0):
    """Train-layout outputs of YoloV8Detect (yolov8_head.py:117-135): cls [B,A,nc], reg [B,A,4*(reg_max+1)] fp32 logits."""
    r = np.random.RandomState(seed)
    A = sum(h * w for h, w in level_shapes(img))
    return (r.randn(B, A, nc).astype(F32) * F32(scale) - F32(2.0)), (r.randn(B, A, 4 * (reg_max + 1)).astype(F32) * F32(scale))
