"""GPU (H100): etb_pl_quality and the device training meter.  The kernel and the mirrors of check_pseudo_label_with_gt /
check_pseudo_label against the live reference's golden vectors and, on 50 seeded batches, against tests/plq_port.py;
DeviceMetricMeter against MetricMeter's float64 sums; and the SSOD, burn-in and supervised steps, eager and captured,
updating the meter every iteration with the values the reference logs."""
import glob
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import plq_port
import synth
from test_gpu_trainer_graph import _images, _make
from test_plq_port import GT_KEYS, NOGT_KEYS, assert_same, load

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plq_*.npz")))
SSOD_KEYS = ["box", "obj", "cls", "loss", "ss_box", "ss_obj", "ss_cls", "tp", "fp_cls", "fp_loc", "pse_num", "gt_num"]


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _kernel(rows, gt, iouv, lo, hi, bs, with_gt):
    from efficientteacher_b200.pl_quality import PLQuality
    plq = PLQuality(DEV, iouv)
    rows_d = torch.from_numpy(np.ascontiguousarray(rows, np.float64).reshape(-1, 9)).to(DEV)
    gt_d = torch.from_numpy(np.ascontiguousarray(gt, np.float32).reshape(-1, 6)).to(DEV)
    th = [None if t is None else torch.tensor(np.asarray(t, np.float64), device=DEV) for t in (hi, lo)]
    plq.run(rows_d, None, th[0], th[1], gt_d, None, bs, with_gt, iou64=lo is None)
    return plq.read()


@pytest.mark.parametrize("path", GOLDEN, ids=lambda p: os.path.basename(p)[:-4])
def test_kernel_and_mirrors_match_reference(path):
    from efficientteacher_b200 import pl_quality
    z, (lo, hi), bs = load(path)
    n = len(z["rows"])
    vals, c = _kernel(z["rows"], z["gt"], z["iouv"], lo, hi, bs, True)
    assert c["overflow"] == 0 and c["n"] == n and c["m"] == len(z["gt"])
    for s, k in enumerate(GT_KEYS[:3]):
        want = np.zeros(len(z["iouv"])) if bool(z["gt_" + k + "_is_int"]) else z["gt_" + k]
        assert np.array_equal(vals[s], want), (k, vals[s], want)
    # the kernel logs the invalid step's zeros when there are no rows (ssod_trainer.py:658-660)
    assert np.all(vals[3:] == (0.0 if n == 0 else np.array([[float(z["gt_pse_num"])], [float(z["gt_gt_num"])]])))
    labels = torch.from_numpy(z["gt"].copy())
    for dev in ("cpu", DEV):
        got = pl_quality.check_pseudo_label_with_gt(torch.from_numpy(z["rows"]).to(dev), labels.to(dev),
                                                    iouv=torch.from_numpy(z["iouv"]), ignore_thres_low=lo, ignore_thres_high=hi,
                                                    batch_size=bs)
        assert_same(got, z, "gt_", GT_KEYS)
    assert torch.equal(labels, torch.from_numpy(z["gt"]))
    if lo is not None:
        vals, c = _kernel(z["rows"], z["gt"], z["iouv"], lo, hi, bs, False)
        want = [z["nogt_precision"], 0.0, z["nogt_recall"], z["nogt_pse_num"], z["nogt_reliable_num"]] if n else [0.0] * 5
        assert np.array_equal(vals[:, 0], np.asarray(want, np.float64)), (vals[:, 0], want)
        assert_same(pl_quality.check_pseudo_label(torch.from_numpy(z["rows"]), lo, hi, batch_size=bs), z, "nogt_", NOGT_KEYS)


def _fuzz_case(seed):
    r = np.random.default_rng(seed)
    B, nc = int(r.integers(1, 9)), int(r.choice([1, 3, 20, 80]))
    gt, rows = [], []
    for b in range(B):
        k = int(r.integers(0, 21))
        g = np.concatenate([np.full((k, 1), b), r.integers(0, nc, (k, 1)), r.uniform(0, 1, (k, 2)), r.uniform(0.01, 0.5, (k, 2))], 1)
        gt.append(g)
        n = int(r.integers(0, 301))
        src = g[r.integers(0, k, n)] if k else np.zeros((n, 6))
        near = (r.random(n) < 0.6) & (k > 0)
        x = np.zeros((n, 9))
        x[:, 0] = b
        x[:, 1] = np.where(near & (r.random(n) < 0.7), src[:, 1], r.integers(0, nc, n))
        x[:, 2:4] = np.where(near[:, None], src[:, 2:4] + r.normal(0, 0.05, (n, 2)) * src[:, 4:6], r.uniform(0, 1, (n, 2)))
        x[:, 4:6] = np.where(near[:, None], src[:, 4:6] * np.exp(r.normal(0, 0.25, (n, 2))), r.uniform(0.01, 0.5, (n, 2)))
        x[:, 6:] = r.uniform(0.1, 1, (n, 3))
        rows.append(x)
    rows, gt = np.concatenate(rows), np.concatenate(gt).astype(np.float32)
    if seed % 3 == 0:
        rows = rows[r.permutation(len(rows))]
    thr = (None, None) if seed % 7 == 0 else (list(r.uniform(0.1, 0.4, nc)), list(r.uniform(0.3, 0.9, nc)))
    iouv = np.linspace(0.5, 0.95, 10, dtype=np.float32) if seed % 4 == 0 else np.array([0.5], np.float32)
    return rows, gt, thr, iouv, int(r.integers(1, 17))


@pytest.mark.parametrize("chunk", range(5))
def test_fuzz_against_port(chunk):
    from efficientteacher_b200 import pl_quality
    for seed in range(chunk * 10, chunk * 10 + 10):
        rows, gt, (lo, hi), iouv, bs = _fuzz_case(seed)
        n_uc, tp, fpc, fpl = plq_port.pl_quality_counts(rows, gt, torch.from_numpy(iouv), lo, hi)
        vals, c = _kernel(rows, gt, iouv, lo, hi, bs, True)
        assert (c["n_uc"], c["overflow"]) == (n_uc, 0), seed
        assert np.array_equal(c["tp"], tp) and np.array_equal(c["fp_cls"], fpc) and np.array_equal(c["fp_loc"], fpl), (seed, c, tp, fpc, fpl)
        want = plq_port.check_pseudo_label_with_gt(rows, gt, torch.from_numpy(iouv), lo, hi, bs)
        got = pl_quality.check_pseudo_label_with_gt(torch.from_numpy(rows), torch.from_numpy(gt), torch.from_numpy(iouv), lo, hi, bs)
        for a, b in zip(got, want):
            assert type(a) is type(b) and np.array_equal(np.asarray(a), np.asarray(b)), (seed, got, want)
        if lo is not None:
            assert pl_quality.check_pseudo_label(torch.from_numpy(rows), lo, hi, bs) == plq_port.check_pseudo_label(rows, lo, hi, bs)
            assert np.array_equal(_kernel(rows, gt, iouv, lo, hi, bs, False)[0][:, 0],
                                  plq_port.hit_values(rows, gt, lo, hi, bs, False))


def test_device_meter_matches_metric_meter():
    """MetricMeter's float64 sums, first-insertion key order, str and a reset that keeps the state's storage"""
    from efficientteacher_b200.pl_quality import DeviceMetricMeter
    m = DeviceMetricMeter(DEV)
    state_ptr = m.state.data_ptr()
    r = np.random.default_rng(5)
    sums, counts, last = {}, {}, {}
    for it in range(20):
        a = torch.tensor([r.normal()], dtype=torch.float32, device=DEV)
        b = torch.tensor(r.normal() * 1e-3, dtype=torch.float64, device=DEV)
        d = dict(a=a, b=b, c=float(r.normal()), e=np.float64(r.normal()))
        if it % 3 == 0:
            d["f"] = int(it)
        m.update(d)
        for k, v in d.items():
            x = torch.as_tensor(v).item() if torch.is_tensor(v) else float(v)
            sums[k] = sums.get(k, 0) + x * 1
            counts[k] = counts.get(k, 0) + 1
            last[k] = x
    got = m.meters
    assert list(got) == ["a", "b", "c", "e", "f"]
    for k, v in got.items():
        assert (v.sum, v.count, v.val, v.avg) == (sums[k], counts[k], last[k], sums[k] / counts[k]), k
    assert m.get_avg() == [sums[k] / counts[k] for k in got]
    assert str(m) == "\t".join('{} {:.4f} ({:.4f})'.format(k, last[k], sums[k] / counts[k]) for k in got)
    m.reset()
    assert m.state.data_ptr() == state_ptr and m.get_avg() == [] and str(m) == ""
    m.update(dict(b=torch.tensor([2.5], device=DEV)))
    assert m.get_avg() == [2.5] and list(m.meters) == ["b"]


def _ssod_thresholds(st):
    """even classes: every row reliable; classes 1 mod 4: every row uncertain; 3 mod 4: neither"""
    nc = st.cfg.Dataset.nc
    st.compute_un_sup_loss.ignore_thres_low = [0.0 if c % 4 != 3 else 1.5 for c in range(nc)]
    st.compute_un_sup_loss.ignore_thres_high = [0.0 if c % 2 == 0 else 2.0 for c in range(nc)]
    return st.compute_un_sup_loss.ignore_thres_low, st.compute_un_sup_loss.ignore_thres_high


@pytest.mark.parametrize("with_gt", [True, False])
@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_ssod_step_meter(mode, with_gt):
    """8 iterations with 0-30 labels, 0-90 GT boxes (the GT capacity doubles once) and one batch whose pseudo labels all
    leave the strong-augmented image (zero rows): each iteration's hit values equal the oracle on that step's device rows,
    and the meter holds the float64 running sums of all twelve values; the warm-up before a capture leaves no trace, and
    reset_meter() works between replays"""
    img, bl, bu = 256, 2, 2
    st = _make("ssod", img, bl, bu)
    st.cfg.SSOD.ssod_hyp = NS(with_gt=with_gt)
    st.pseudo_label_creator.nms_conf_thres = 1e-6       # a random-init teacher: low-confidence pseudo labels, up to 300 per image
    lo, hi = _ssod_thresholds(st)
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    us = uw.flip(3).contiguous()
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    gone = Ms.clone()
    gone[:, 3] += 1e5                                   # translate every box out of the image: no pseudo label survives
    gone[:, 6] += 1e5
    n_lab = [8, 0, 16, 3, 30, 5, 12, 9]
    n_gt = [5, 0, 30, 90, 10, None, 20, 40]
    f = st.train_instance_graphed if mode == "graph" else st.train_instance
    sums, seen_rows = [0.0] * 12, 0
    for ni in range(8):
        tg = torch.from_numpy(synth.make_targets(30 + ni, n_lab[ni], bl)).to(DEV)
        gt = None if n_gt[ni] is None else torch.from_numpy(synth.make_targets(50 + ni, n_gt[ni], bu))
        f(imgs, tg, us, uw, gt, gone if ni == 4 else Ms, ni)
        c = st.pseudo_label_creator
        n = int(c.last_count_dev.item())
        rows = c.last_rows_dev[:n].cpu().numpy()
        seen_rows += n
        assert (n == 0) == (ni == 4), (ni, n)
        want = plq_port.hit_values(rows, np.zeros((0, 6), np.float32) if gt is None else gt.numpy(), lo, hi, st.batch_size, with_gt)
        meters = st.meter.meters
        assert list(meters) == SSOD_KEYS and all(m.count == ni + 1 for m in meters.values()), (ni, meters)
        vals = [meters[k].val for k in SSOD_KEYS]
        assert vals[7:] == want, (ni, vals[7:], want)
        last = st.last
        assert vals[:7] == [float(last["sup"][k]) for k in SSOD_KEYS[:4]] + [float(last["unsup"][k]) for k in SSOD_KEYS[4:7]]
        assert [float(last["hits"][k]) for k in SSOD_KEYS[7:]] == want
        sums = [s + v for s, v in zip(sums, vals)]
    assert seen_rows > 0
    assert st.meter.get_avg() == [s / 8 for s in sums]
    if mode == "graph":
        assert st.captures == (2 if with_gt else 1)
    st.reset_meter()
    f(imgs, torch.from_numpy(synth.make_targets(70, 6, bl)).to(DEV), us, uw, None, Ms, 8)
    meters = st.meter.meters
    assert all(m.count == 1 and m.avg == m.val for m in meters.values()) and list(meters) == SSOD_KEYS
    if mode == "graph":
        assert st.captures == (2 if with_gt else 1)


@pytest.mark.parametrize("kind", ["sup", "burn_in"])
@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_burn_in_and_supervised_meter(kind, mode):
    img, bl = 256, 2
    st = _make(kind, img, bl, 2)
    imgs = _images(3, bl, img)
    if kind == "sup":
        f = st.train_step_graphed if mode == "graph" else st.train_step
    else:
        f = st.train_without_unlabeled_graphed if mode == "graph" else st.train_without_unlabeled
    keys = ["box", "obj", "cls", "loss"]
    sums = [0.0] * 4
    for ni, n in enumerate((9, 0, 24, 5)):
        f(imgs, torch.from_numpy(synth.make_targets(30 + ni, n, bl)).to(DEV), ni)
        meters = st.meter.meters
        assert list(meters) == keys and all(m.count == ni + 1 for m in meters.values()), (ni, meters)
        vals = [meters[k].val for k in keys]
        assert vals == [float(st.last["sup"][k]) for k in keys]
        assert vals[3] == float(st.last["loss"])
        sums = [s + v for s, v in zip(sums, vals)]
    assert st.meter.get_avg() == [s / 4 for s in sums]
    st.reset_meter()
    f(imgs, torch.from_numpy(synth.make_targets(40, 7, bl)).to(DEV), 4)
    assert [m.count for m in st.meter.meters.values()] == [1] * 4
    if mode == "graph":
        assert (st.captures if kind == "sup" else st.burn_in_captures) == 1
