"""Float64 numpy restatement of ap_per_class (reference utils/metrics.py:22-126) that the native path follows: the rows of
each class in descending confidence with a STABLE sort (equal confidences keep their row order; numpy's default argsort is
not stable, so the reference agrees with this only when confidences are distinct), cumulative TP / FP counts, recall
tpc / n_l, precision tpc / (tpc + fpc), and the 101-point COCO integral of the precision envelope.  Also the case generator
shared by the golden fixture (tests/golden/make_golden_val.py) and the tests."""
import numpy as np

_trapz = getattr(np, "trapezoid", None) or np.trapz
PX = np.linspace(0, 1, 1000)
XS = np.linspace(0, 1, 101)


def class_ap(recall, precision):
    """101-point interpolated AP of one precision / recall column: the envelope is the running max from the right of
    [1, precision, 0] against [0, recall, 1]"""
    mrec = np.concatenate(([0.0], recall, [1.0]))
    env = np.maximum.accumulate(np.concatenate(([1.0], precision, [0.0]))[::-1])[::-1]
    return _trapz(np.interp(XS, mrec, env), XS)


def ap_per_class(tp, conf, pred_cls, target_cls):
    """-> (p, r, ap, f1, ap_class, cls_thr) like the reference (plots aside)"""
    tp = np.asarray(tp, dtype=bool)
    order = np.argsort(-np.asarray(conf), kind="stable")
    tp, conf, pred_cls = tp[order], np.asarray(conf)[order], np.asarray(pred_cls)[order]
    classes = np.unique(target_cls)
    T = tp.shape[1]
    ap = np.zeros((len(classes), T))
    p = np.zeros((len(classes), PX.size))
    r = np.zeros((len(classes), PX.size))
    for ci, c in enumerate(classes):
        sel = pred_cls == c
        n_l = (np.asarray(target_cls) == c).sum()
        if sel.sum() == 0 or n_l == 0:
            continue
        tpc = tp[sel].cumsum(0)
        fpc = (1 - tp[sel]).cumsum(0)
        recall = tpc / (n_l + 1e-16)
        precision = tpc / (tpc + fpc)
        r[ci] = np.interp(-PX, -conf[sel], recall[:, 0], left=0)
        p[ci] = np.interp(-PX, -conf[sel], precision[:, 0], left=1)
        for j in range(T):
            ap[ci, j] = class_ap(recall[:, j], precision[:, j])
    f1 = 2 * p * r / (p + r + 1e-16)
    best = f1.mean(0).argmax()
    cls_thr = [PX[f1[k].argmax()] for k in range(f1.shape[0])]
    return p[:, best], r[:, best], ap, f1[:, best], classes.astype('int32'), cls_thr


def make_case(seed, n, nc, label_classes=None, pred_classes=None, labels_per_class=(1, 60), tp_rate=0.4, T=10, distinct=True):
    """A synthetic epoch: (tp [n,T] bool, conf [n] fp32, pred_cls [n] fp32, target_cls [m] float64).  At most n_l true
    positives per class and column, and a TP at a stricter IoU threshold is a TP at every looser one (what process_batch
    produces).  distinct: every confidence differs from every other."""
    rng = np.random.RandomState(seed)
    label_classes = np.arange(nc) if label_classes is None else np.asarray(label_classes)
    pred_classes = np.arange(nc) if pred_classes is None else np.asarray(pred_classes)
    n_l = {int(c): int(rng.randint(labels_per_class[0], labels_per_class[1] + 1)) for c in label_classes}
    target_cls = np.concatenate([np.full(k, c, dtype=np.float64) for c, k in n_l.items()]) if n_l else np.zeros(0)
    rng.shuffle(target_cls)
    pred_cls = pred_classes[rng.randint(0, len(pred_classes), n)].astype(np.float32) if n else np.zeros(0, np.float32)
    if distinct:
        pool = np.unique(rng.uniform(0.001, 1.0, 3 * n + 16).astype(np.float32))
        conf = rng.permutation(pool)[:n]
    else:
        conf = np.round(rng.uniform(0.001, 1.0, n), 2).astype(np.float32)
    tp = np.zeros((n, T), dtype=bool)
    for c, k in n_l.items():
        rows = np.flatnonzero(pred_cls == c)
        hit = rows[rng.rand(rows.size) < tp_rate][:k]
        tp[hit, 0] = True
    for j in range(1, T):
        tp[:, j] = tp[:, j - 1] & (rng.rand(n) < 0.85)
    return tp, conf, pred_cls, target_cls


def golden_cases():
    """name -> case inputs of tests/golden/ap_per_class.npz"""
    cases = {}
    # 80 classes; 3, 11 and 42 have labels but no predictions, 75..79 have predictions but no labels
    cases["mixed"] = make_case(1, 20000, 80, label_classes=[c for c in range(75)],
                               pred_classes=[c for c in range(80) if c not in (3, 11, 42)], labels_per_class=(1, 400))
    # class 0: every prediction a TP at every threshold; class 1: none; class 2: mixed
    tp, conf, pcls, tcls = make_case(2, 600, 3, labels_per_class=(300, 300))
    tp[pcls == 0] = True
    tp[pcls == 1] = False
    tcls = np.concatenate([tcls, np.zeros(int((pcls == 0).sum()), np.float64)])
    cases["alltp_allfp"] = (tp, conf, pcls, tcls)
    # a class with a single prediction (a TP) next to regular classes
    tp, conf, pcls, tcls = make_case(3, 400, 4, pred_classes=[1, 2, 3], labels_per_class=(2, 50))
    pcls[0], tp[0] = 0.0, True
    cases["np1"] = (tp, conf, pcls, tcls)
    cases["nc1"] = make_case(4, 5000, 1, labels_per_class=(800, 800))
    cases["big"] = make_case(5, 300000, 80, labels_per_class=(50, 2000), tp_rate=0.3)
    return cases
