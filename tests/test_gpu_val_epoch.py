"""GPU (H100): the native validation epoch -- etb_val_epoch_append + etb_ap_per_class (csrc/metrics.cu), metrics.ap_per_class,
val.run and the trainers' validate().

  * the kernels plus the numpy tail equal the live reference's ap_per_class bit for bit (tests/golden/ap_per_class.npz);
  * tied confidences follow the stable rule of tests/ap_port.py; empty and degenerate epochs match it too;
  * the per-batch rescale gives the fp32 bits of the torch-op path val_batch uses;
  * run() equals engine predictions -> port.nms_val -> torch rescale -> port.process_batch -> ap_port.ap_per_class;
  * the batch loop makes no host sync;
  * validate() rounds the EMA to fp16 in place, and each captured step replayed after it matches the eager step."""
import numpy as np
import pytest
import torch

import ap_port
import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = ("p", "r", "ap", "f1", "ap_class", "cls_thr")


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _same(got, want, what=""):
    for k, a, b in zip(KEYS, got, want):
        a, b = np.asarray(a), np.asarray(b)
        assert a.shape == b.shape and a.dtype == b.dtype, (what, k, a.shape, b.shape, a.dtype, b.dtype)
        assert np.array_equal(a, b), (what, k, np.abs(a.astype(np.float64) - b).max() if a.size else None)


@pytest.mark.parametrize("name", ["mixed", "alltp_allfp", "np1", "nc1", "big"])
def test_ap_per_class_matches_reference_golden(golden, name):
    from efficientteacher_b200 import metrics
    g = golden("ap_per_class")
    tp, conf, pcls, tcls = ap_port.golden_cases()[name]
    want = [g[name + "_" + k] for k in KEYS]
    _same(metrics.ap_per_class(tp, conf, pcls, tcls), want, name)
    # CUDA tensors in, the same result
    _same(metrics.ap_per_class(torch.from_numpy(tp).to(DEV), torch.from_numpy(conf).to(DEV), torch.from_numpy(pcls).to(DEV),
                               torch.from_numpy(tcls).to(DEV)), want, name + " (cuda)")


@pytest.mark.parametrize("seed", [11, 12])
def test_tied_confidences_follow_the_stable_rule(seed):
    from efficientteacher_b200 import metrics
    tp, conf, pcls, tcls = ap_port.make_case(seed, 6000, 20, labels_per_class=(1, 120), distinct=False)
    assert np.unique(conf).size < conf.size / 10
    _same(metrics.ap_per_class(tp, conf, pcls, tcls), ap_port.ap_per_class(tp, conf, pcls, tcls), "ties")


def test_empty_and_degenerate_epochs_match_the_port():
    from efficientteacher_b200 import metrics
    tp, conf, pcls, tcls = ap_port.make_case(21, 3000, 10)
    z = lambda n, T=10: np.zeros((n, T), bool)  # noqa: E731
    cases = {
        "no detections": (z(0), np.zeros(0, np.float32), np.zeros(0, np.float32), tcls),
        "no labels": (tp, conf, pcls, np.zeros(0)),
        "no TP": (z(len(conf)), conf, pcls, tcls),
        "one row": (tp[:1] | True, conf[:1], pcls[:1], pcls[:1].astype(np.float64)),
        "T=1": (tp[:, :1], conf, pcls, tcls),
    }
    import warnings
    for name, c in cases.items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")      # numpy's "mean of empty slice" when no class has labels, in both
            _same(metrics.ap_per_class(*c), ap_port.ap_per_class(*c), name)


def _shapes(B, H, W, seed):
    r = np.random.RandomState(seed)
    out = []
    for _ in range(B):
        h0, w0 = int(r.randint(H // 2, 3 * H)), int(r.randint(W // 2, 3 * W))
        g = min(H / h0, W / w0)
        out.append(((h0, w0), ((g, g), ((W - w0 * g) / 2, (H - h0 * g) / 2))))
    return out


def test_rescale_matches_the_torch_op_path():
    """etb_val_epoch_append's native-space rows and labels (its workspace) against val.scale_coords_ on fp32 CUDA tensors"""
    from efficientteacher_b200 import _ws, val
    B, max_det, H, W = 3, 50, 256, 320
    r = np.random.RandomState(5)
    det = torch.zeros((B, max_det, 8), dtype=torch.float32)
    xy = r.uniform(-20, 340, (B, max_det, 2)).astype(np.float32)
    wh = r.uniform(1, 120, (B, max_det, 2)).astype(np.float32)
    det[..., :2], det[..., 2:4] = torch.from_numpy(xy), torch.from_numpy(xy + wh)
    det[..., 4] = torch.from_numpy(r.rand(B, max_det).astype(np.float32))
    det[..., 5] = torch.from_numpy(r.randint(0, 80, (B, max_det)).astype(np.float32))
    det = det.to(DEV)
    cnt = torch.tensor([50, 0, 17], dtype=torch.int32, device=DEV)
    tg = torch.from_numpy(synth.make_targets(3, 40, B)).to(DEV)
    shapes = _shapes(B, H, W, 1)
    for single_cls in (False, True):
        ep = val.ValEpoch(DEV, 80, single_cls=single_cls)
        ep.add(det, cnt, tg, shapes, (H, W))
        ws = _ws._cache[("val_epoch", str(ep.device))]
        got = ws[:B * max_det * 24].view(torch.float32).view(B, max_det, 6)
        off = (B * max_det * 24 + 255) // 256 * 256
        got_lab = ws[off:off + tg.shape[0] * 24].view(torch.float32).view(-1, 6)
        for b in range(B):
            n = int(cnt[b])
            want = det[b, :n, :6].clone()
            if single_cls:
                want[:, 5] = 0
            val.scale_coords_((H, W), want[:, :4], shapes[b][0], shapes[b][1])
            assert torch.equal(got[b, :n], want), b
            t = tg[tg[:, 0] == b].clone()
            t[:, 2:6] *= torch.tensor([W, H, W, H], device=DEV, dtype=torch.float32)
            box = torch.cat((t[:, 2:4] - t[:, 4:6] / 2, t[:, 2:4] + t[:, 4:6] / 2), 1)
            val.scale_coords_((H, W), box, shapes[b][0], shapes[b][1])
            assert torch.equal(got_lab[tg[:, 0] == b][:, 2:], box), b
        _, nt, _ = ep.finish()
        assert np.array_equal(nt, np.bincount(tg[:, 1].long().cpu().numpy(), minlength=80))


# ---- run() against the composition of the oracles -----------------------------------------------------------------------

def _detector(seed=0, nc=80):
    """A YOLOv5s SSOD model (outputs ((pred, raw), features)) with nc classes whose head keeps classes 0..3 (objectness ~0.9)
    and pushes every other class below conf_thres, so a val batch has a few hundred detections per image at conf 0.001"""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(seed)
    cfg = yolov5_ssod_cfg('s', batch_size=4, img_size=160)
    cfg.Dataset.nc, cfg.Dataset.names = nc, [str(i) for i in range(nc)]
    m = Model(cfg).to(DEV)
    with torch.no_grad():
        for h in m.head.m:
            b = h.bias.view(3, -1)
            b[:, 4] += 6.0
            b[:, 5:] = -12.0
            b[:, 5:9] = 1.0
    return m.eval()


def _loader(model, seed=3, single_cls=False):
    """three rect batches (H x W 128x160, 160x128, 128x128) of uint8 images; labels are jittered copies of a third of the
    model's own detections (so every IoU threshold sees true positives) plus a few unmatched boxes; single_cls: every label
    is class 0, as a single_cls dataset gives them"""
    nc = model.nc
    from oracle import port
    from efficientteacher_b200 import val
    r = np.random.RandomState(seed)
    batches = []
    for bi, (B, H, W) in enumerate(((3, 128, 160), (2, 160, 128), (3, 128, 128))):
        img = torch.from_numpy(r.randint(0, 256, (B, 3, H, W)).astype(np.uint8))
        with torch.no_grad():
            pred = val._unwrap(model(img.to(DEV))[0])
        dets = port.nms_val(pred.cpu().numpy(), 0.001, 0.6)
        rows = []
        for b, d in enumerate(dets):
            pick = d[r.rand(len(d)) < 0.3][:40]
            for x1, y1, x2, y2, _, c in pick:
                j = r.uniform(0.85, 1.15, 4)
                cx, cy, w, h = (x1 + x2) / 2 * j[0] ** 0.1, (y1 + y2) / 2 * j[1] ** 0.1, (x2 - x1) * j[2], (y2 - y1) * j[3]
                rows.append((b, c, cx / W, cy / H, w / W, h / H))
            for _ in range(3):
                rows.append((b, r.randint(0, min(4, nc)), r.rand(), r.rand(), r.uniform(0.05, 0.3), r.uniform(0.05, 0.3)))
        tg = torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)
        if single_cls:
            tg[:, 1] = 0
        batches.append((img, tg, ["im%d_%d.jpg" % (bi, b) for b in range(B)], _shapes(B, H, W, 10 + bi)))
    return batches


def _composition(model, loader, nc=80, single_cls=False):
    """engine -> port.nms_val -> torch rescale -> port.process_batch -> ap_port.ap_per_class, then val.py:398-465;
    single_cls: class-agnostic NMS and every detection in class 0 (val.py:335-344), nc 1"""
    from oracle import port
    from efficientteacher_b200 import val
    iouv = torch.linspace(0.5, 0.95, 10).numpy()
    stats = []
    for img, tg, _, shapes in loader:
        B, _, H, W = img.shape
        with torch.no_grad():
            pred = val._unwrap(model(img.to(DEV))[0])
        dets = port.nms_val(pred.cpu().numpy(), 0.001, 0.6, agnostic=single_cls)
        if single_cls:
            for d in dets:
                d[:, 5] = 0
        t = tg.to(DEV).clone()
        t[:, 2:6] *= torch.tensor([W, H, W, H], device=DEV, dtype=torch.float32)
        for si, d in enumerate(dets):
            lab = t[t[:, 0] == si, 1:]
            predn = torch.from_numpy(d).to(DEV)
            val.scale_coords_((H, W), predn[:, :4], shapes[si][0], shapes[si][1])
            box = torch.cat((lab[:, 1:3] - lab[:, 3:5] / 2, lab[:, 1:3] + lab[:, 3:5] / 2), 1)
            val.scale_coords_((H, W), box, shapes[si][0], shapes[si][1])
            labn = torch.cat((lab[:, 0:1], box), 1).cpu().numpy()
            correct = port.process_batch(predn.cpu().numpy(), labn, iouv)
            stats.append((correct, d[:, 4], d[:, 5], lab[:, 0].cpu().numpy().astype(np.float64)))
    stats = [np.concatenate(x, 0) for x in zip(*stats)]
    assert stats[0].any()
    p, r, ap, f1, ap_class, cls_thr = ap_port.ap_per_class(*stats)
    ap50, ap = ap[:, 0], ap.mean(1)
    maps = np.zeros(nc) + ap.mean()
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    return (p.mean(), r.mean(), ap50.mean(), ap.mean(), 0.0, 0.0, 0.0), maps, cls_thr


def test_run_matches_the_composition_of_the_oracles():
    from efficientteacher_b200 import val
    model = _detector()
    loader = _loader(model)
    ptrs = [p.data_ptr() for p in model.parameters()]
    results, maps, t, cls_thr = val.run({'nc': 80}, model=model, dataloader=loader, plots=False, val_ssod=True)
    assert not model.training and [p.data_ptr() for p in model.parameters()] == ptrs
    assert len(t) == 3 and all(x > 0 for x in t)
    want_results, want_maps, want_thr = _composition(model, loader)   # the model is fp16-rounded now, as run() forwarded it
    assert results == want_results and np.array_equal(maps, want_maps) and np.array_equal(cls_thr, want_thr), (results, want_results)
    assert results[2] > 0.05
    # the rounding is idempotent: a second run gives the same numbers
    r2, m2, _, thr2 = val.run({'nc': 80}, model=model, dataloader=loader, plots=False, val_ssod=True)
    assert r2 == results and np.array_equal(m2, maps) and np.array_equal(thr2, cls_thr)
    # as in the reference, an SSOD model without val_ssod unwraps to (pred, raw): not a prediction tensor
    with pytest.raises(TypeError):
        val.run({'nc': 80}, model=model, dataloader=loader, plots=False)


@pytest.mark.parametrize("nc,single_cls", [(20, False), (2, False), (1, True)])
def test_run_matches_the_composition_of_the_oracles_at_class_counts(nc, single_cls):
    """run() at the class counts of VOC (20), the custom configs (2) and single_cls (a one-class model): ValEpoch's histogram
    and etb_val_epoch_append / etb_ap_per_class sized by nc, the nc 1 NMS route, class-agnostic NMS with classes zeroed"""
    from efficientteacher_b200 import val
    model = _detector(nc=nc)
    loader = _loader(model, single_cls=single_cls)
    results, maps, _, cls_thr = val.run({'nc': nc}, model=model, dataloader=loader, plots=False, val_ssod=True, single_cls=single_cls)
    want_results, want_maps, want_thr = _composition(model, loader, 1 if single_cls else nc, single_cls)
    assert results == want_results and np.array_equal(maps, want_maps) and np.array_equal(cls_thr, want_thr), (results, want_results)
    assert results[2] > 0.05 and len(maps) == (1 if single_cls else nc)


def test_run_without_true_positives_returns_zeros():
    from efficientteacher_b200 import val
    model = _detector()
    loader = [(img, tg[:0], p, s) for img, tg, p, s in _loader(model)]
    results, maps, t, cls_thr = val.run({'nc': 80}, model=model, dataloader=loader, plots=False, val_ssod=True)
    assert results == (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0) and cls_thr == [] and not maps.any()


def test_batch_loop_makes_no_host_sync():
    from efficientteacher_b200 import val
    model = _detector()
    loader = [(img.to(DEV), tg.to(DEV), p, s) for img, tg, p, s in _loader(model)]
    ep = val.ValEpoch(DEV, 80)
    val.val_step(model, *loader[0][:2], loader[0][3], ep, val_ssod=True)       # first call: allocations of the engine / workspaces
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for img, tg, _, shapes in loader:
            val.val_step(model, img, tg, shapes, ep, val_ssod=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert ep.seen == 3 + sum(x[0].shape[0] for x in loader) and ep.finish()[0]


# ---- the trainers' validate() --------------------------------------------------------------------------------------------

def _images(seed, n, img):
    return torch.from_numpy(np.random.RandomState(seed).rand(n, 3, img, img).astype(np.float32)).to(DEV)


def _flat(tensors):
    return torch.cat([t.detach().flatten().float() for t in tensors])


def _make(kind, img, bl, bu):
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    torch.manual_seed(0)
    if kind == "sup":
        cfg = yolov5_sup_cfg('l_shallow', batch_size=bl, img_size=img)
        cfg.hyp.warmup_epochs = 0
        return SupTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    cfg = yolov5_ssod_cfg('l_shallow', batch_size=bl + bu, img_size=img)
    cfg.hyp.warmup_epochs = 0
    cfg.hyp.burn_epochs = 2 if kind == "burn_in" else 0
    st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    if kind == "ssod":
        with torch.no_grad():
            for mm in (st.model, st.ema.ema, st.semi_ema.ema):
                for h in mm.head.m:
                    h.bias.view(3, -1)[:, 4] += 6.5
                    h.bias.view(3, -1)[:, 5:] += 5.0
    return st


def _val_loader(img=128):
    r = np.random.RandomState(8)
    out = []
    for bi in range(2):
        im = torch.from_numpy(r.randint(0, 256, (2, 3, img, img)).astype(np.uint8))
        out.append((im, torch.from_numpy(synth.make_targets(40 + bi, 10, 2)), ["a.jpg", "b.jpg"], _shapes(2, img, img, 30 + bi)))
    return out


def test_validate_rounds_the_ema_in_place():
    st = _make("sup", 128, 2, 0)
    with torch.no_grad():
        for t in st.ema.ema.state_dict().values():
            if t.dtype.is_floating_point:
                t.add_(torch.randn_like(t) * 1e-3)
    state = {k: v.clone() for k, v in st.ema.ema.state_dict().items()}
    ptrs = {k: v.data_ptr() for k, v in st.ema.ema.state_dict().items()}
    results, maps, t = st.validate(_val_loader())
    assert len(results) == 7 and maps.shape == (80,)
    for k, v in st.ema.ema.state_dict().items():
        assert v.data_ptr() == ptrs[k], k
        want = state[k].half().float() if v.dtype.is_floating_point else state[k]
        assert torch.equal(v, want), k


@pytest.mark.parametrize("kind", ["ssod", "burn_in", "sup"])
def test_captured_step_replayed_after_validate_matches_eager(kind):
    """step (graph: the capture), validate(), step (graph: a replay): the state the eager run leaves, within the spread of
    two eager runs.  validate() must neither move the EMA's storage nor free a buffer the graphs read."""
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    us = uw.flip(3).contiguous()
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    loader = _val_loader()
    out = {}
    for mode in ("eager", "eager2", "graph"):
        st = _make(kind, img, bl, bu)
        g = mode == "graph"
        if kind == "ssod":
            f = lambda ni: (st.train_instance_graphed if g else st.train_instance)(imgs, tg, us, uw, None, Ms, ni)  # noqa: E731
        elif kind == "burn_in":
            f = lambda ni: (st.train_without_unlabeled_graphed if g else st.train_without_unlabeled)(imgs, tg, ni)  # noqa: E731
        else:
            f = lambda ni: (st.train_step_graphed if g else st.train_step)(imgs, tg, ni)  # noqa: E731
        emas = [e for e in (st.ema, st.semi_ema) if e is not None]
        f(1)
        ptrs = [t.data_ptr() for e in emas for t in e.ema.state_dict().values()]
        res = st.validate(loader)
        assert len(res) == (5 if kind != "sup" else 3) and st.model.training
        assert [t.data_ptr() for e in emas for t in e.ema.state_dict().values()] == ptrs
        f(3)
        torch.cuda.synchronize()
        out[mode] = dict(weights=_flat(st.model.state_dict().values()), ema=_flat(t for e in emas for t in e.ema.state_dict().values()))
    for what in ("weights", "ema"):
        a, b, c = out["eager"][what], out["graph"][what], out["eager2"][what]
        assert torch.isfinite(b).all(), what
        n = a.norm().clamp_min(1e-30)
        rel, rel_eager = ((a - b).norm() / n).item(), ((a - c).norm() / n).item()
        assert rel <= 3.0 * rel_eager + 2e-3, (kind, what, rel, rel_eager)
