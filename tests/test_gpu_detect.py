"""GPU (H100): batched inference on raw frames -- etb_letterbox_u8 (csrc/letterbox.cu), etb_detect_rescale (csrc/metrics.cu)
and detect.Predictor.

  * the letterbox kernel equals cv2 byte for byte on the sweep of tests/letterbox_port.py, frames of mixed sizes in one
    launch, and the numpy restatement there on every eighth frame (on every frame without cv2);
  * the rescale equals scale_coords(...).round() done with torch ops on the same rows, bit for bit;
  * Predictor equals host letterbox -> the model's engine forward -> nms.non_max_suppression -> torch scale_coords + round,
    rows and counts, on YOLOv5s and YOLOv5l;
  * a call makes a fixed number of library launches per shape group and one host sync;
  * classes=, augment, half and keypoint heads are refused;
  * a captured SSOD step replayed after a Predictor call on its teacher matches the eager step."""
import warnings

import numpy as np
import pytest
import torch

import letterbox_port
import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _frame(r, h0, w0):
    return np.frombuffer(bytearray(r.bytes(h0 * w0 * 3)), np.uint8).reshape(h0, w0, 3)


def test_letterbox_kernel_matches_the_restatement():
    from efficientteacher_b200.detect import letterbox_batch, letterbox_geometry
    try:
        import cv2
    except ImportError:
        cv2 = None
    groups = {}
    for h0, w0, S in letterbox_port.sweep():
        g = letterbox_geometry(h0, w0, S)
        groups.setdefault((S, g[4], g[5]), []).append((h0, w0, g))
    r = np.random.RandomState(2)
    launches = checked = 0
    for (S, H, W), items in groups.items():
        for k in range(0, len(items), 16):                 # at most 16 frames (up to 2000 x 2000) per launch
            part = items[k:k + 16]
            imgs = [_frame(r, h0, w0) for h0, w0, _ in part]
            dev = [torch.from_numpy(im.copy()).to(DEV) for im in imgs]
            out, _ = letterbox_batch(dev, [g for _, _, g in part], H, W)
            out = out.cpu().numpy()
            launches += 1
            for im, (h0, w0, g), got in zip(imgs, part, out):
                checked += 1
                if cv2 is None or checked % 8 == 0:            # the CPU tests show the restatement equals cv2 on the sweep
                    assert np.array_equal(got, letterbox_port.letterbox_chw(im, g)), (h0, w0, S)
                if cv2 is not None:
                    new_h, new_w, top, left = g[:4]
                    want = im if (h0, w0) == (new_h, new_w) else cv2.resize(im, (new_w, new_h), interpolation=cv2.INTER_LINEAR)
                    want = cv2.copyMakeBorder(want, top, H - new_h - top, left, W - new_w - left, cv2.BORDER_CONSTANT,
                                              value=(114, 114, 114))
                    assert np.array_equal(got, want[:, :, ::-1].transpose(2, 0, 1)), (h0, w0, S, "cv2")
    assert launches < len(letterbox_port.sweep()) / 2      # mixed frame sizes do share launches


def _scale_round(rows, H, W, h0, w0):
    from efficientteacher_b200 import val
    d = rows.clone()
    d[:, :4] = val.scale_coords_((H, W), d[:, :4], (h0, w0)).round()
    return d


def _shapes(H, W, sizes):
    out = []
    for h0, w0 in sizes:
        g = min(H / h0, W / w0)
        out.append(((h0, w0), ((g, g), ((W - w0 * g) / 2, (H - h0 * g) / 2))))
    return out


def test_rescale_matches_scale_coords_round():
    from efficientteacher_b200 import detect, val
    B, max_det, H, W = 4, 300, 384, 640
    sizes = [(1080, 1920), (720, 1280), (481, 853), (377, 641)]
    r = np.random.RandomState(5)
    det = torch.zeros((B, max_det, 8), dtype=torch.float32)
    xy = r.uniform(-20, W + 20, (B, max_det, 2)).astype(np.float32)
    wh = r.uniform(0, 200, (B, max_det, 2)).astype(np.float32)
    det[..., :2], det[..., 2:4] = torch.from_numpy(xy), torch.from_numpy(xy + wh)
    det[:, :8, :4] = torch.arange(32, dtype=torch.float32).view(8, 4) + 0.5          # halves: round half to even
    det[..., 4] = torch.from_numpy(r.rand(B, max_det).astype(np.float32))
    det[..., 5] = torch.from_numpy(r.randint(0, 80, (B, max_det)).astype(np.float32))
    det = det.to(DEV)
    cnt = torch.tensor([300, 0, 17, 123], dtype=torch.int32, device=DEV)
    meta = torch.from_numpy(val._image_meta(_shapes(H, W, sizes))).to(DEV)
    got = detect.rescale_rows(det, cnt, meta)
    for b, (h0, w0) in enumerate(sizes):
        n = int(cnt[b])
        assert torch.equal(got[b, :n], _scale_round(det[b, :n, :6], H, W, h0, w0)), b


def _model(size, seed=0):
    """YOLOv5 `size` (Model for s, SupModel for l) whose head keeps classes 0..3 above conf 0.25"""
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.model import Model, SupModel
    torch.manual_seed(seed)
    m = (Model(yolov5_ssod_cfg(size, batch_size=4, img_size=320)) if size == "s" else
         SupModel(yolov5_sup_cfg(size, batch_size=4, img_size=320))).to(DEV)
    with torch.no_grad():
        for h in m.head.m:
            b = h.bias.view(3, -1)
            b[:, 4] += 6.0
            b[:, 5:] = -12.0
            b[:, 5:9] = 1.0
    return m


SIZES = [(480, 640), (720, 1280), (300, 500), (640, 480), (481, 641), (1080, 1920), (200, 200)]


def _composition(model, frames, S):
    from efficientteacher_b200 import nms
    from efficientteacher_b200.detect import letterbox_geometry
    geoms = [letterbox_geometry(f.shape[0], f.shape[1], S) for f in frames]
    groups = {}
    for i, g in enumerate(geoms):
        groups.setdefault(g[4:6], []).append(i)
    out = [None] * len(frames)
    for (H, W), idx in groups.items():
        img = torch.from_numpy(np.stack([letterbox_port.letterbox_chw(frames[i], geoms[i]) for i in idx])).to(DEV)
        with torch.no_grad():
            (pred, _), _ = model.engine().forward(img, with_features=False)
        dets = nms.non_max_suppression(pred, 0.25, 0.45, max_det=1000)
        for i, d in zip(idx, dets):
            out[i] = _scale_round(d, H, W, frames[i].shape[0], frames[i].shape[1])
    return out


@pytest.mark.parametrize("size", ["s", "l"])
def test_predictor_matches_the_composition(size):
    from efficientteacher_b200.detect import Predictor
    model = _model(size)
    r = np.random.RandomState(7)
    frames = [_frame(r, h, w) for h, w in SIZES]
    inputs = [frames[0], torch.from_numpy(frames[1].copy()), torch.from_numpy(frames[2].copy()).to(DEV)] + frames[3:]
    for S in (320, 640):
        got = Predictor(model, img_size=S)(inputs)
        want = _composition(model, frames, S)
        assert sum(w.shape[0] for w in want) > 0
        for i, (g, w) in enumerate(zip(got, want)):
            assert g.shape == w.shape and torch.equal(g, w), (size, S, i, g.shape, w.shape)


def _launches():
    from efficientteacher_b200 import _lib
    torch.cuda.synchronize()
    return int(_lib.lib().etb_launch_count())


def test_one_call_launches_per_group_and_syncs_once():
    from efficientteacher_b200.detect import Predictor
    p = Predictor(_model("s"), img_size=320)
    r = np.random.RandomState(3)
    video = [_frame(r, 360, 640) for _ in range(4)]
    mixed = video[:2] + [_frame(r, 640, 360), _frame(r, 640, 360)]
    p(video), p(mixed)                                     # first calls: allocations of the engine and workspaces
    counts = []
    for frames in (video[:2], video, mixed):
        n0 = _launches()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                p(frames)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counts.append(_launches() - n0)
        syncs = [x for x in w if "synchroniz" in str(x.message)]
        assert len(syncs) == 1, [str(x.message) for x in syncs]
    assert counts[0] == counts[1] > 0 and counts[2] == 2 * counts[0], counts


def test_refusals():
    from efficientteacher_b200.detect import Predictor
    m = _model("s")
    for kw in (dict(classes=[0]), dict(augment=True), dict(half=True), dict(num_points=5)):
        with pytest.raises(NotImplementedError):
            Predictor(m, **kw)
    with pytest.raises(ValueError):
        Predictor(m, img_size=600)
    with pytest.raises(ValueError):
        Predictor(m)([np.zeros((10, 10), np.uint8)])


def _images(seed, n, img):
    return torch.from_numpy(np.random.RandomState(seed).rand(n, 3, img, img).astype(np.float32)).to(DEV)


def _flat(tensors):
    return torch.cat([t.detach().flatten().float() for t in tensors])


def test_captured_ssod_step_replayed_after_predictor_matches_eager():
    """step (graph: the capture), Predictor on the teacher, step (graph: a replay): the state the eager run leaves, within the
    spread of two eager runs.  The Predictor must neither move the teacher's storage nor grow a workspace the graph reads."""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.detect import Predictor
    from efficientteacher_b200.trainer import SSODTrainerStep
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    us = uw.flip(3).contiguous()
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    r = np.random.RandomState(11)
    frames = [_frame(r, 720, 1280) for _ in range(3)] + [_frame(r, 1280, 720)]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        torch.manual_seed(0)
        cfg = yolov5_ssod_cfg('l_shallow', batch_size=bl + bu, img_size=img)
        cfg.hyp.warmup_epochs = 0
        cfg.hyp.burn_epochs = 0
        st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
        with torch.no_grad():
            for mm in (st.model, st.ema.ema, st.semi_ema.ema):
                for h in mm.head.m:
                    h.bias.view(3, -1)[:, 4] += 6.5
                    h.bias.view(3, -1)[:, 5:] += 5.0
        g = mode == "graph"
        f = lambda ni: (st.train_instance_graphed if g else st.train_instance)(imgs, tg, us, uw, None, Ms, ni)  # noqa: E731
        emas = [st.ema, st.semi_ema]
        f(1)
        ptrs = [t.data_ptr() for e in emas for t in e.ema.state_dict().values()]
        dets = Predictor(st.ema.ema, img_size=640, max_det=1000)(frames)
        assert len(dets) == 4 and sum(d.shape[0] for d in dets) > 0 and st.model.training
        assert [t.data_ptr() for e in emas for t in e.ema.state_dict().values()] == ptrs
        f(3)
        torch.cuda.synchronize()
        out[mode] = dict(weights=_flat(st.model.state_dict().values()), ema=_flat(t for e in emas for t in e.ema.state_dict().values()))
    for what in ("weights", "ema"):
        a, b, c = out["eager"][what], out["graph"][what], out["eager2"][what]
        assert torch.isfinite(b).all(), what
        n = a.norm().clamp_min(1e-30)
        rel, rel_eager = ((a - b).norm() / n).item(), ((a - c).norm() / n).item()
        assert rel <= 3.0 * rel_eager + 2e-3, (what, rel, rel_eager)
