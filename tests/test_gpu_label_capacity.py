"""GPU (H100): captured SSOD and supervised steps with any label count -- etb_label_class_hist (LabelMatch's class
histogram of a padded label buffer), the label-capacity scheme of train_step_graphed / train_instance_graphed (one capture
for any count up to the capacity, one more when a batch exceeds it), LabelMatch inside the captured SSOD step, and
DevicePrefetcher with a label count that changes between batches."""
import math

import numpy as np
import pytest
import torch

import synth
from test_gpu_trainer_graph import _flat, _float_state, _images, _make, _within_spread

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NC = 80


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _hist_call(t, n_dev, n_host, hist):
    from efficientteacher_b200 import _lib
    _lib.check(_lib.lib().etb_label_class_hist(_lib.ptr(t), _lib.ptr(n_dev), n_host, int(t.shape[0]), int(t.shape[1]), NC,
                                               _lib.ptr(hist), _lib.stream_ptr()), "etb_label_class_hist")


def _want(cls_col, n):
    """the reference's int(l[1:2]) per row, valid classes through numpy.bincount, the rest in the last slot"""
    c = [math.trunc(v) if np.isfinite(v) else None for v in cls_col[:n].tolist()]
    ok = [x for x in c if x is not None and 0 <= x < NC]
    return np.concatenate([np.bincount(np.array(ok, dtype=np.int64), minlength=NC), [n - len(ok)]]).astype(np.int32)


def _labels(seed, cap, tstride, n, bad_inside):
    r = np.random.RandomState(seed)
    t = r.uniform(0, 1, (cap, tstride)).astype(np.float32)
    t[:, 1] = r.randint(0, NC, cap) + r.uniform(0, 0.999, cap)           # fractional classes truncate toward zero
    t[:n:7, 1] = -0.75                                                     # int(-0.75) == 0
    stale = np.array([NC, 1000.0, -1.0, -7.5, np.nan, 3.0e9], np.float32)
    t[n:, 1] = stale[np.arange(cap - n) % len(stale)]                      # past the count: never read
    if bad_inside and n >= 6:
        t[1:6, 1] = stale[:5]                                              # inside the count: hist[nc]
    return t


@pytest.mark.parametrize("tstride", [6, 9])
@pytest.mark.parametrize("n", [0, 117, 300])
@pytest.mark.parametrize("bad_inside", [False, True])
def test_label_class_hist_matches_bincount(tstride, n, bad_inside):
    cap = 300
    t = _labels(11 + n + tstride, cap, tstride, n, bad_inside)
    td = torch.from_numpy(t).to(DEV)
    for use_dev in (False, True):
        hist = torch.zeros(NC + 1, dtype=torch.int32, device=DEV)
        if use_dev:
            _hist_call(td, torch.tensor([n], dtype=torch.int32, device=DEV), 0, hist)
        else:
            _hist_call(td[:n].contiguous() if n else td[:0], None, n, hist)
        got = hist.cpu().numpy()
        assert np.array_equal(got, _want(t[:, 1], n)), (use_dev, got)
        if bad_inside and n >= 6:
            assert got[NC] == 5


def test_label_class_hist_accumulates_and_replays_captured():
    """adds into the histogram over calls, and a captured call replayed with different device counts reads each replay's
    count"""
    cap = 256
    t = _labels(5, cap, 6, cap, False)
    td = torch.from_numpy(t).to(DEV)
    hist = torch.zeros(NC + 1, dtype=torch.int32, device=DEV)
    n_dev = torch.tensor([cap], dtype=torch.int32, device=DEV)
    want = np.zeros(NC + 1, np.int32)
    for n in (10, 200, 0):
        n_dev.fill_(n)
        _hist_call(td, n_dev, 0, hist)
        want += _want(t[:, 1], n)
    assert np.array_equal(hist.cpu().numpy(), want)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _hist_call(td, n_dev, 0, hist)        # warm-up outside the capture (n = 0: adds nothing)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _hist_call(td, n_dev, 0, hist)
    torch.cuda.synchronize()
    assert np.array_equal(hist.cpu().numpy(), want)          # capturing does not run the kernel
    for n in (256, 3, 0, 99):
        n_dev.fill_(n)
        graph.replay()
        want += _want(t[:, 1], n)
    assert np.array_equal(hist.cpu().numpy(), want)


def test_labelmatch_update_device_matches_update():
    """LabelMatch.update_device + flush == the reference-shaped LabelMatch.update on the host rows; a padded buffer with a
    device count ignores its stale rows; a class outside [0, nc) raises at flush, as the reference's indexing does"""
    from efficientteacher_b200.labelmatch import LabelMatch
    cfg = _make_cfg_labelmatch()
    dev_lm, host_lm = LabelMatch(cfg, 1000, 7.0, np.full(NC, 1.0 / NC)), LabelMatch(cfg, 1000, 7.0, np.full(NC, 1.0 / NC))
    pad = torch.from_numpy(_labels(3, 64, 6, 64, False)).to(DEV)
    for i, n in enumerate((16, 0, 37)):
        tg = synth.make_targets(60 + i, n, 2)
        dev_lm.update_device(torch.from_numpy(tg).to(DEV))
        pad[:n] = torch.from_numpy(tg).to(DEV)
        dev_lm.update_device(pad, torch.tensor([n], dtype=torch.int32, device=DEV))
        host_lm.update(np.concatenate([tg, tg]), n=0, pse_n=0)
    dev_lm.flush()
    assert np.array_equal(dev_lm.cls_tmp, host_lm.cls_tmp) and dev_lm.cls_tmp.sum() == 2 * (16 + 37)
    assert not dev_lm.class_hist(DEV).any()                   # flush zeroes the accumulator
    bad = torch.from_numpy(synth.make_targets(70, 5, 2)).to(DEV)
    bad[2, 1] = NC
    dev_lm.update_device(bad)
    with pytest.raises(IndexError):
        dev_lm.flush()
    with pytest.raises(IndexError):
        host_lm.update(bad.cpu().numpy())


def _make_cfg_labelmatch():
    from efficientteacher_b200.config import yolov5_ssod_cfg
    cfg = yolov5_ssod_cfg('l_shallow', batch_size=4, img_size=256)
    cfg.SSOD.pseudo_label_type = "LabelMatch"
    cfg.SSOD.resample_high_percent, cfg.SSOD.resample_low_percent = 0.0, 0.0   # the reference's defaults.py:277-278
    return cfg


COUNTS = (16, 0, 9, 24, 9, 31)


@pytest.mark.parametrize("kind", ["sup", "ssod"])
def test_graphed_step_any_label_count_matches_eager(kind):
    """(eager, eager, graph) over 6 batches with 16 / 0 / 9 / 24 / 9 / 31 labels: one capture serves them all (a 9 right
    after a 24 leaves stale rows in the buffer); then a batch over the capacity re-captures once with the capacity doubled,
    and a smaller batch after it (CPU labels) replays that graph."""
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    us = uw.flip(3).contiguous()
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    tgs = [torch.from_numpy(synth.make_targets(30 + i, n, bl)).to(DEV) for i, n in enumerate(COUNTS)]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        st = _make(kind, img, bl, bu)
        g = mode == "graph"
        if kind == "ssod":
            f = lambda tg, ni: (st.train_instance_graphed if g else st.train_instance)(imgs, tg, us, uw, None, Ms, ni)  # noqa: E731
        else:
            f = lambda tg, ni: (st.train_step_graphed if g else st.train_step)(imgs, tg, ni)  # noqa: E731
        losses = [float(f(tg, ni).item()) for ni, tg in enumerate(tgs)]
        if g:
            assert st.captures == 1 and st._graph["cap"] == st.LABEL_CAPACITY
            cap = st._graph["cap"]
        else:
            cap = st.LABEL_CAPACITY
        for i, n in enumerate((cap + 1, 3)):
            tg = torch.from_numpy(synth.make_targets(40 + i, n, bl))
            losses.append(float(f(tg if (g and i == 1) else tg.to(DEV), len(COUNTS) + i).item()))
        if g:
            assert st.captures == 2 and st._graph["cap"] == 2 * cap
        emas = [e for e in (st.ema, st.semi_ema) if e is not None]
        assert st.ema.updates == 4 and st.last_opt_step == 7, mode
        out[mode] = dict(losses=losses, ema=_flat(t for e in emas for t in _float_state(e.ema)),
                         weights=_flat(_float_state(st.model)), updates=[e.updates for e in emas])
    assert out["eager"]["updates"] == out["eager2"]["updates"] == out["graph"]["updates"]
    for i, (a, b, c) in enumerate(zip(out["eager"]["losses"], out["graph"]["losses"], out["eager2"]["losses"])):
        assert abs(a - b) <= 3.0 * abs(a - c) + (0.01 + 0.02 * i) * abs(a), (i, out)
    _within_spread(out, "ema")
    _within_spread(out, "weights")


def _labelmatch_step(img, bl, bu):
    from efficientteacher_b200.labelmatch import LabelMatch
    from efficientteacher_b200.trainer import SSODTrainerStep
    torch.manual_seed(0)
    cfg = _make_cfg_labelmatch()
    cfg.hyp.warmup_epochs = 0
    cfg.hyp.burn_epochs = 0
    st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    assert isinstance(st.pseudo_label_creator, LabelMatch)
    with torch.no_grad():
        for mm in (st.model, st.ema.ema, st.semi_ema.ema):
            for h in mm.head.m:
                h.bias.view(3, -1)[:, 4] += 6.5
                h.bias.view(3, -1)[:, 5:] += 5.0
    return st


def _labelmatch_inputs(img, bl, bu):
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    return imgs, uw.flip(3).contiguous(), uw, torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)


def _teacher_state(st):
    return [t.clone() for t in st.ema.ema.state_dict().values()]


def test_labelmatch_graphed_matches_eager():
    """LabelMatch in the captured SSOD step against the eager step: cls_tmp, count and pse_count equal exactly after flush();
    the per-class score lists are identical over the steps before the first EMA update (ni = 0 is not due, ni = 1 updates
    the teachers only after its teacher forward), with the teacher bit-identical in both runs."""
    img, bl, bu = 256, 2, 2
    imgs, us, uw, Ms = _labelmatch_inputs(img, bl, bu)
    tgs = [torch.from_numpy(synth.make_targets(50 + i, n, bl)).to(DEV) for i, n in enumerate(COUNTS)]
    out = {}
    for mode in ("eager", "graph"):
        st = _labelmatch_step(img, bl, bu)
        c = st.pseudo_label_creator
        f = st.train_instance_graphed if mode == "graph" else st.train_instance
        teachers = [_teacher_state(st)]
        f(imgs, tgs[0], us, uw, None, Ms, 0)
        teachers.append(_teacher_state(st))          # the teacher ni = 1 runs its forward with
        f(imgs, tgs[1], us, uw, None, Ms, 1)
        c.flush()
        early = [list(s) for s in c.score_list_epoch]
        for ni in range(2, len(tgs)):
            f(imgs, tgs[ni], us, uw, None, Ms, ni)
        c.flush()
        if mode == "graph":
            assert st.captures == 1
        assert st.ema.updates == 3
        out[mode] = dict(teachers=teachers, early=early, cls_tmp=c.cls_tmp.copy(), count=c.count, pse_count=c.pse_count,
                         n_scores=sum(len(s) for s in c.score_list_epoch))
    e, g = out["eager"], out["graph"]
    for t in (0, 1):
        assert all(torch.equal(a, b) for a, b in zip(e["teachers"][t], g["teachers"][t]))
        assert all(torch.equal(a, b) for a, b in zip(g["teachers"][0], g["teachers"][t]))
    assert sum(len(s) for s in e["early"]) > 0
    assert e["early"] == g["early"]
    assert np.array_equal(e["cls_tmp"], g["cls_tmp"]) and e["cls_tmp"].sum() == sum(COUNTS)
    want = np.zeros(NC)
    for tg in tgs:
        for row in tg.cpu().numpy():
            want[int(row[1])] += 1
    assert np.array_equal(g["cls_tmp"], want)
    assert e["count"] == g["count"] == bl * len(COUNTS) and e["pse_count"] == g["pse_count"] == bu * len(COUNTS)
    assert g["n_scores"] > 0


def test_labelmatch_capture_leaves_no_trace():
    """The first graphed call -- two warm-up steps that really run the LabelMatch bookkeeping, then the restore -- leaves
    every LabelMatch field as one eager call does: the device histogram, the staged detections, the counters and, after
    flush(), cls_tmp and the score lists."""
    img, bl, bu = 256, 2, 2
    imgs, us, uw, Ms = _labelmatch_inputs(img, bl, bu)
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    out = {}
    for mode in ("eager", "graph"):
        st = _labelmatch_step(img, bl, bu)
        c = st.pseudo_label_creator
        (st.train_instance_graphed if mode == "graph" else st.train_instance)(imgs, tg, us, uw, None, Ms, 0)
        torch.cuda.synchronize()
        staged = [(h_det.clone(), h_cnt.clone()) for h_det, h_cnt, _ in c._pending]
        o = dict(hist=c.class_hist(DEV).cpu().numpy(), count=c.count, pse_count=c.pse_count, staged=staged)
        c.flush()
        o.update(cls_tmp=c.cls_tmp.copy(), scores=[list(s) for s in c.score_list_epoch], pending=len(c._pending),
                 hist_after=c.class_hist(DEV).cpu().numpy())
        out[mode] = o
    e, g = out["eager"], out["graph"]
    assert np.array_equal(e["hist"], g["hist"]) and e["hist"].sum() == 8 * bl
    assert e["count"] == g["count"] == bl and e["pse_count"] == g["pse_count"] == bu
    assert len(e["staged"]) == len(g["staged"]) == 1
    (de, ce), (dg, cg) = e["staged"][0], g["staged"][0]
    assert torch.equal(ce, cg) and int(ce.sum()) > 0
    for b, n in enumerate(ce.tolist()):
        assert torch.equal(de[b, :n], dg[b, :n])
    assert np.array_equal(e["cls_tmp"], g["cls_tmp"]) and e["scores"] == g["scores"]
    assert e["pending"] == g["pending"] == 0 and not e["hist_after"].any() and not g["hist_after"].any()


def test_device_prefetcher_label_count_rises_and_falls():
    """Batches whose label count rises and falls come back exactly; the label slot grows by doubling, the fixed-shape
    image slot keeps its buffer."""
    from efficientteacher_b200.trainer import DevicePrefetcher
    pf = DevicePrefetcher(DEV)
    g = torch.Generator().manual_seed(2)
    counts = (5, 40, 3, 100, 0, 64, 7, 300, 1)
    batches = [{"imgs": torch.randint(0, 255, (2, 3, 32, 32), dtype=torch.uint8, generator=g).pin_memory(),
                "targets": torch.rand(n, 6, generator=g).pin_memory()} for n in counts]
    img_bufs = []
    pf.put(batches[0])
    for i, n in enumerate(counts):
        got = pf.get()
        assert got["targets"].shape == (n, 6) and got["imgs"].shape == (2, 3, 32, 32)
        assert torch.equal(got["targets"].cpu(), batches[i]["targets"]) and torch.equal(got["imgs"].cpu(), batches[i]["imgs"])
        if i < len(pf.slots):
            img_bufs.append(got["imgs"].data_ptr())
        pf.release()
        if i + 1 < len(counts):
            pf.put(batches[i + 1])
    # slot 0 holds 5, 3, 0, 7, 1 labels: 5 -> 10; slot 1 holds 40, 100, 64, 300: 40 -> 160 -> 320
    assert [sl["buf"]["targets"].shape[0] for sl in pf.slots] == [10, 320]
    assert [sl["buf"]["imgs"].data_ptr() for sl in pf.slots] == img_bufs
