"""Generates tests/golden/plq_*.npz from the LIVE, UNMODIFIED reference's check_pseudo_label_with_gt and check_pseudo_label
(utils/self_supervised_utils.py:481-606, imported through oracle/ref_harness.py).  Needs the reference checkout:
    python tests/golden/make_golden_plq.py
Each file holds one seeded case -- the inputs (rows [N,9] float64 as FairPseudoLabel makes them, gt [M,6] fp32, the per-class
thresholds or none, iouv, batch_size) and both functions' outputs.  The ties case keeps every match list at 16 entries or
fewer, and no two of its rows compete for the same pair of tied labels: numpy's argsort is not stable on every CPU (its
AVX-512 sort reorders equal keys even in short arrays), so which of two tied labels the reference keeps depends on the
machine; the counts of this case do not."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import plq_port  # noqa: E402
from oracle import ref_harness  # noqa: E402


def _gt(rng, B, per_img, nc, corner=False):
    out = []
    for b in range(B):
        k = int(rng.integers(max(per_img - 3, 0), per_img + 4)) if per_img else 0
        xy = rng.uniform(0.85, 0.98, (k, 2)) if corner and b % 2 == 0 else rng.uniform(0.05, 0.95, (k, 2))
        if corner and b % 2 == 1:
            xy = rng.uniform(0.0, 0.12, (k, 2))
        wh = rng.uniform(0.03, 0.4, (k, 2))
        out.append(np.concatenate([np.full((k, 1), b), rng.integers(0, nc, (k, 1)), xy, wh], 1))
    return np.concatenate(out, 0).astype(np.float32) if out else np.zeros((0, 6), np.float32)


def _rows(rng, gt, B, per_img, nc, corner=False):
    out = []
    for b in range(B):
        g = gt[gt[:, 0] == b]
        n = int(rng.integers(per_img * 3 // 4, per_img + 1))
        r = np.zeros((n, 9))
        r[:, 0] = b
        near = rng.random(n) < (0.6 if len(g) else 0.0)
        src = g[rng.integers(0, max(len(g), 1), n) % max(len(g), 1)] if len(g) else np.zeros((n, 6))
        r[:, 2:4] = np.where(near[:, None], src[:, 2:4] + rng.normal(0, 0.04, (n, 2)) * src[:, 4:6],
                             rng.uniform(0.85, 1.0, (n, 2)) if corner else rng.uniform(0.05, 0.95, (n, 2)))
        r[:, 4:6] = np.where(near[:, None], src[:, 4:6] * np.exp(rng.normal(0, 0.2, (n, 2))), rng.uniform(0.02, 0.4, (n, 2)))
        r[:, 1] = np.where(near & (rng.random(n) < 0.7), src[:, 1], rng.integers(0, nc, n))
        r[:, 6:9] = rng.uniform(0.1, 1.0, (n, 3))
        out.append(r)
    return np.concatenate(out, 0) if out else np.zeros((0, 9))


def _thr(rng, nc):
    return rng.uniform(0.1, 0.35, nc), rng.uniform(0.4, 0.8, nc)


def cases():
    c = {}
    rng = np.random.default_rng(1001)
    gt = _gt(rng, 4, 10, 80)
    c["random_nc80"] = dict(rows=_rows(rng, gt, 4, 300, 80), gt=gt, thr=_thr(rng, 80), iouv=[0.5], bs=4)
    for nc, seed in ((1, 1002), (20, 1003)):
        rng = np.random.default_rng(seed)
        gt = _gt(rng, 3, 8, nc)
        rows = _rows(rng, gt, 3, 120, nc)
        if nc == 20:
            rows = rows[rng.permutation(len(rows))]       # rows of the images interleaved
        c["nc%d" % nc] = dict(rows=rows, gt=gt, thr=_thr(rng, nc), iouv=[0.5], bs=3)
    # ties: GT 0 and 1 are the same box and class, so a row near them has two labels at equal IoU -- in the tp set (row 0),
    # the fp_cls set (row 1) and the fp_loc set (row 2); one row per set and tied pair, so the counts do not depend on
    # which of the two the reference's sort puts first
    gt = np.array([[0, 0, .5, .5, .2, .2], [0, 0, .5, .5, .2, .2], [0, 1, .8, .2, .2, .25], [1, 2, .3, .3, .1, .1]], np.float32)
    rows = np.array([[0, 0, .51, .5, .2, .21, .3, .9, .9], [0, 1, .49, .52, .19, .2, .25, .8, .8], [0, 0, .62, .62, .1, .1, .3, .6, .6],
                     [0, 1, .81, .2, .2, .24, .2, .7, .7], [1, 2, .31, .3, .1, .11, .3, .5, .5], [1, 2, .3, .3, .1, .1, .9, .5, .5]])
    c["ties"] = dict(rows=rows, gt=gt, thr=(np.full(3, 0.1), np.full(3, 0.6)), iouv=[0.5], bs=2)
    rng = np.random.default_rng(1004)
    gt = _gt(rng, 4, 6, 5, corner=True)
    c["boundary"] = dict(rows=_rows(rng, gt, 4, 60, 5, corner=True), gt=gt, thr=_thr(rng, 5), iouv=[0.5], bs=4)
    rng = np.random.default_rng(1005)
    gt = _gt(rng, 2, 6, 10)
    rows = _rows(rng, gt, 2, 50, 10)
    c["zero_uncertain"] = dict(rows=rows, gt=gt, thr=(np.full(10, 0.5), np.full(10, 0.5)), iouv=[0.5], bs=2)
    c["zero_gt"] = dict(rows=rows, gt=np.zeros((0, 6), np.float32), thr=_thr(rng, 10), iouv=[0.5], bs=2)
    c["zero_rows"] = dict(rows=np.zeros((0, 9)), gt=gt, thr=_thr(rng, 10), iouv=[0.5], bs=2)
    c["thr_none"] = dict(rows=rows, gt=gt, thr=None, iouv=[0.5], bs=2)
    rng = np.random.default_rng(1006)
    gt = _gt(rng, 4, 10, 80)
    c["iouv10"] = dict(rows=_rows(rng, gt, 4, 200, 80), gt=gt, thr=_thr(rng, 80),
                       iouv=torch.linspace(0.5, 0.95, 10).numpy(), bs=4)
    return c


GT_KEYS = ("tp", "fp_cls", "fp_loc", "pse_num", "gt_num")
NOGT_KEYS = ("precision", "recall", "pse_num", "reliable_num")


def _pack(prefix, keys, vals):
    out = {}
    for k, v in zip(keys, vals):
        out[prefix + k] = np.asarray(v, dtype=np.float64)
        out[prefix + k + "_is_int"] = np.asarray(isinstance(v, int))
    return out


def main():
    ref_harness.load_reference()
    from utils.self_supervised_utils import check_pseudo_label, check_pseudo_label_with_gt
    for name, cs in cases().items():
        lo, hi = (None, None) if cs["thr"] is None else (list(cs["thr"][0]), list(cs["thr"][1]))
        iouv = torch.tensor(np.asarray(cs["iouv"], np.float32))
        rows = torch.from_numpy(cs["rows"]).double()
        got = check_pseudo_label_with_gt(rows.clone(), torch.from_numpy(cs["gt"]).clone(), iouv=iouv, ignore_thres_low=lo,
                                         ignore_thres_high=hi, batch_size=cs["bs"])
        out = dict(rows=cs["rows"], gt=cs["gt"], iouv=np.asarray(cs["iouv"], np.float32), bs=np.asarray(cs["bs"]),
                   has_thr=np.asarray(cs["thr"] is not None))
        if cs["thr"] is not None:
            out.update(thr_low=np.asarray(lo), thr_high=np.asarray(hi))
            out.update(_pack("nogt_", NOGT_KEYS, check_pseudo_label(rows.clone(), lo, hi, batch_size=cs["bs"])))
        out.update(_pack("gt_", GT_KEYS, got))
        port = plq_port.check_pseudo_label_with_gt(cs["rows"], cs["gt"], iouv, lo, hi, cs["bs"])
        same = all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, port))
        print(name, "N=%d M=%d" % (len(cs["rows"]), len(cs["gt"])), [np.round(np.asarray(v), 4).tolist() for v in got],
              "port agrees" if same else "PORT DIFFERS %s" % (port,))
        np.savez_compressed(os.path.join(HERE, "plq_%s.npz" % name), **out)


if __name__ == "__main__":
    main()
