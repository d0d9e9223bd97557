"""GPU (H100): the detection confusion matrix on the device -- etb_confusion_matrix (csrc/val.cu),
etb_val_epoch_append_confusion (csrc/metrics.cu), metrics.ConfusionMatrix, ValEpoch / val.run / validate(confusion_matrix=).

  * per-image process_batch equals the live reference's matrices bit for bit (tests/golden/confusion_*.npz), and follows the
    tie rule of tests/confusion_port.py;
  * a validation epoch with a matrix fills it as the per-image restatement does over the same NMS rows (val.py:347-373:
    only images with rows and labels, detections in class 0 under single_cls, labels as they are), and leaves the results
    of the run without one unchanged;
  * ValEpoch.add with a matrix makes no host sync and one launch more per batch;
  * a validation with a matrix between a captured SSOD step and its replay leaves the replay unchanged;
  * a class outside [0, nc) raises IndexError from finish() and from matrix."""
import numpy as np
import pytest
import torch

import confusion_port as cp
import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _launches():
    from efficientteacher_b200 import _lib
    torch.cuda.synchronize()
    return int(_lib.lib().etb_launch_count())


@pytest.mark.parametrize("name", ["nc1", "nc2", "nc8", "nc20", "nc80", "shapes"])
def test_process_batch_matches_reference_golden(golden, name):
    from efficientteacher_b200.metrics import ConfusionMatrix
    nc, images = cp.golden_cases()[name]
    cm = ConfusionMatrix(nc)
    for det, lab in images:
        cm.process_batch(torch.from_numpy(det).to(DEV), torch.from_numpy(lab).to(DEV))
    m = cm.matrix
    assert m.dtype == np.float64 and np.array_equal(m, golden("confusion_" + name)["matrix"]), name
    # fp16 rows widen exactly (val.py's labels are fp32, so torch compares in fp32 too)
    cm.reset()
    for det, lab in images:
        d16 = torch.from_numpy(det).half()
        cm.process_batch(d16.to(DEV), torch.from_numpy(lab).to(DEV))
    assert np.array_equal(cm.matrix, cp.matrix_of(nc, [(d.astype(np.float16).astype(np.float32), l) for d, l in images]))


def test_ties_and_random_images_follow_the_port():
    """exact IoU ties (identical boxes, the multi-label NMS copies) and random images with many pairs, other thresholds"""
    from efficientteacher_b200.metrics import ConfusionMatrix
    r = np.random.RandomState(5)
    nc = 6
    images = []
    for _ in range(40):
        n_lab = r.randint(0, 12)
        boxes = np.round(r.uniform(0, 200, (n_lab, 2)))
        lab = np.concatenate([r.randint(0, nc, (n_lab, 1)), boxes, boxes + np.round(r.uniform(5, 60, (n_lab, 2)))], 1).astype(np.float32)
        rows = []
        for l in range(n_lab):
            for _ in range(r.randint(0, 4)):
                rows.append(np.r_[lab[l, 1:] + np.round(r.uniform(-4, 4, 4)), np.round(r.rand(), 1), r.randint(0, nc)])
        det = np.asarray(rows, np.float32).reshape(-1, 6)
        if len(det):
            det = np.concatenate([det, det[:2] * [1, 1, 1, 1, 1, 0] + [0, 0, 0, 0, 0, r.randint(0, nc)]])   # multi-label copies
        images.append((det, lab))
    assert sum(cp.deciding_ties(d, l) for d, l in images) > 10
    for conf, iou in ((0.25, 0.45), (0.0, 0.3), (0.5, 0.6)):
        cm = ConfusionMatrix(nc, conf=conf, iou_thres=iou)
        for det, lab in images:
            cm.process_batch(torch.from_numpy(det).to(DEV), torch.from_numpy(lab).to(DEV))
        assert np.array_equal(cm.matrix, cp.matrix_of(nc, images, conf, iou)), (conf, iou)


def _epoch_batches(seed, nc, single_cls, n_batches=4):
    """synthetic NMS rows of rect batches (etb_nms_val's layout, some images without rows), Poisson labels (some images
    without labels), loader shapes"""
    r = np.random.RandomState(seed)
    out = []
    for bi in range(n_batches):
        B, (H, W) = 4, ((128, 160), (160, 128), (128, 128), (96, 160))[bi % 4]
        max_det = 40
        nt = r.poisson(4, B)
        nt[bi % B] = 0
        rows = []
        for b in range(B):
            for _ in range(nt[b]):
                rows.append((b, r.randint(0, nc), r.uniform(0.1, 0.9), r.uniform(0.1, 0.9), r.uniform(0.05, 0.4), r.uniform(0.05, 0.4)))
        tg = torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)
        det = torch.zeros((B, max_det, 6))
        cnt = r.randint(1, max_det + 1, B)
        cnt[(bi + 1) % B] = 0
        for b in range(B):
            own = tg[tg[:, 0] == b]
            for k in range(cnt[b]):
                if len(own) and r.rand() < 0.6:
                    t = own[r.randint(len(own))]
                    cx, cy, w, h = (t[2:] * torch.tensor([W, H, W, H])).tolist()
                    cx, cy, w, h = cx + r.uniform(-4, 4), cy + r.uniform(-4, 4), w * r.uniform(0.7, 1.3), h * r.uniform(0.7, 1.3)
                    c = int(t[1]) if r.rand() < 0.7 else r.randint(0, nc)
                else:
                    cx, cy, w, h, c = r.uniform(0, W), r.uniform(0, H), r.uniform(4, 60), r.uniform(4, 60), r.randint(0, nc)
                det[b, k] = torch.tensor([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2, r.rand(), 0 if single_cls else c])
        shapes = []
        for _ in range(B):
            h0, w0 = int(r.randint(H // 2, 3 * H)), int(r.randint(W // 2, 3 * W))
            g = min(H / h0, W / w0)
            shapes.append(((h0, w0), ((g, g), ((W - w0 * g) / 2, (H - h0 * g) / 2))))
        out.append((det.to(DEV), torch.from_numpy(cnt.astype(np.int32)).to(DEV), tg, shapes, (H, W)))
    return out


def _restated(batches, nc, single_cls):
    """val.py:347-373 per image over the same rows: the torch rescale, then the numpy restatement"""
    from efficientteacher_b200 import val
    m = np.zeros((nc + 1, nc + 1))
    for det, cnt, tg, shapes, (H, W) in batches:
        t = tg.to(DEV).clone()
        t[:, 2:6] *= torch.tensor([W, H, W, H], device=DEV, dtype=torch.float32)
        for si in range(det.shape[0]):
            n = int(cnt[si])
            lab = t[t[:, 0] == si, 1:]
            if n == 0 or lab.shape[0] == 0:
                continue
            predn = det[si, :n].clone()
            if single_cls:
                predn[:, 5] = 0
            val.scale_coords_((H, W), predn[:, :4], shapes[si][0], shapes[si][1])
            box = torch.cat((lab[:, 1:3] - lab[:, 3:5] / 2, lab[:, 1:3] + lab[:, 3:5] / 2), 1)
            val.scale_coords_((H, W), box, shapes[si][0], shapes[si][1])
            cp.process_batch(m, predn.cpu().numpy(), torch.cat((lab[:, 0:1], box), 1).cpu().numpy())
    return m


@pytest.mark.parametrize("single_cls", [False, True])
def test_val_epoch_fills_the_matrix_like_the_per_image_restatement(single_cls):
    from efficientteacher_b200 import val
    from efficientteacher_b200.metrics import ConfusionMatrix
    nc = 1 if single_cls else 8
    batches = _epoch_batches(11 + single_cls, 1 if single_cls else nc, single_cls)
    cm = ConfusionMatrix(nc)
    ep, plain = val.ValEpoch(DEV, nc, single_cls=single_cls, confusion_matrix=cm), val.ValEpoch(DEV, nc, single_cls=single_cls)
    for det, cnt, tg, shapes, hw in batches:
        ep.add(det, cnt, tg, shapes, hw)
        plain.add(det, cnt, tg, shapes, hw)
    got, want = ep.finish(), plain.finish()
    assert got[0] == want[0] and np.array_equal(got[1], want[1])
    for a, b in zip(got[2] or (), want[2] or ()):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    m = cm.matrix
    assert np.array_equal(m, _restated(batches, nc, single_cls)) and m.sum() > 50


def _detector(nc=8, seed=0):
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.model import SupModel
    torch.manual_seed(seed)
    cfg = yolov5_sup_cfg('s', batch_size=4, img_size=160)
    cfg.Dataset.nc, cfg.Dataset.names = nc, [str(i) for i in range(nc)]
    m = SupModel(cfg).to(DEV)
    with torch.no_grad():
        for h in m.head.m:
            b = h.bias.view(3, -1)
            b[:, 4] += 6.0
            b[:, 5:] = -12.0
            b[:, 5:8] = 1.0
    return m.eval()


def _val_loader(model, seed=3, single_cls=False):
    """rect batches of uint8 images; labels: Poisson counts of jittered copies of the model's own detections and random
    boxes (some images without labels); single_cls: every label in class 0, as a single_cls dataset gives them"""
    from efficientteacher_b200 import val
    r = np.random.RandomState(seed)
    out = []
    for bi, (B, H, W) in enumerate(((3, 128, 160), (2, 160, 128), (3, 128, 128))):
        img = torch.from_numpy(r.randint(0, 256, (B, 3, H, W)).astype(np.uint8))
        det, cnt = val._nms(val._unwrap(model(img.to(DEV))), 0.001, 0.6, False)
        rows = []
        for b in range(B):
            d = det[b, :int(cnt[b])].cpu().numpy()
            for _ in range(r.poisson(4) if b != 1 else 0):
                if len(d) and r.rand() < 0.7:
                    x1, y1, x2, y2, _, c = d[r.randint(len(d))][:6]
                    j = r.uniform(0.85, 1.15, 4)
                    rows.append((b, c, (x1 + x2) / 2 / W, (y1 + y2) / 2 / H, (x2 - x1) * j[2] / W, (y2 - y1) * j[3] / H))
                else:
                    rows.append((b, r.randint(0, model.nc), r.rand(), r.rand(), r.uniform(0.05, 0.3), r.uniform(0.05, 0.3)))
        tg = torch.tensor(rows, dtype=torch.float32).reshape(-1, 6)
        if single_cls:
            tg[:, 1] = 0
        out.append((img, tg, ["im%d_%d.jpg" % (bi, b) for b in range(B)], _shapes(B, H, W, 10 + bi)))
    return out


def _shapes(B, H, W, seed):
    r = np.random.RandomState(seed)
    out = []
    for _ in range(B):
        h0, w0 = int(r.randint(H // 2, 3 * H)), int(r.randint(W // 2, 3 * W))
        g = min(H / h0, W / w0)
        out.append(((h0, w0), ((g, g), ((W - w0 * g) / 2, (H - h0 * g) / 2))))
    return out


@pytest.mark.parametrize("single_cls", [False, True])
def test_run_with_a_matrix(single_cls):
    """val.run(confusion_matrix=cm): the matrix of the per-image restatement over the same NMS rows, and the results of the
    run without the keyword"""
    from efficientteacher_b200 import val
    from efficientteacher_b200.metrics import ConfusionMatrix
    model = _detector()
    loader = _val_loader(model, single_cls=single_cls)
    nc = 1 if single_cls else model.nc
    plain = val.run({'nc': model.nc}, model=model, dataloader=loader, plots=False, half=False, single_cls=single_cls)
    cm = ConfusionMatrix(nc)
    got = val.run({'nc': model.nc}, model=model, dataloader=loader, plots=False, half=False, single_cls=single_cls,
                  confusion_matrix=cm)
    assert got[0] == plain[0] and np.array_equal(got[1], plain[1])
    batches = []
    for img, tg, _, shapes in loader:
        det, cnt = val._nms(val._unwrap(model(img.to(DEV))), 0.001, 0.6, single_cls)
        batches.append((det, cnt, tg, shapes, tuple(img.shape[2:])))
    m = cm.matrix
    assert np.array_equal(m, _restated(batches, nc, single_cls)) and np.trace(m[:nc, :nc]) > 0


def test_add_with_a_matrix_makes_no_host_sync_and_one_more_launch():
    from efficientteacher_b200 import val
    from efficientteacher_b200.metrics import ConfusionMatrix
    batches = _epoch_batches(21, 8, False)
    tgs = [b[2].to(DEV) for b in batches]
    eps = {"plain": val.ValEpoch(DEV, 8), "cm": val.ValEpoch(DEV, 8, confusion_matrix=ConfusionMatrix(8))}
    for ep in eps.values():
        det, cnt, _, shapes, hw = batches[0]
        ep.add(det, cnt, tgs[0], shapes, hw)            # first call: workspaces
    per_batch = {}
    for k, ep in eps.items():
        n0 = _launches()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for (det, cnt, _, shapes, hw), tg in zip(batches, tgs):
                ep.add(det, cnt, tg, shapes, hw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        per_batch[k] = (_launches() - n0) / len(batches)
    assert per_batch["cm"] == per_batch["plain"] + 1, per_batch
    eps["cm"].finish()


def test_out_of_range_class_raises_index_error():
    from efficientteacher_b200 import val
    from efficientteacher_b200.metrics import ConfusionMatrix
    cm = ConfusionMatrix(4)
    cm.process_batch(torch.tensor([[0, 0, 10, 10, 0.9, 6.0]], device=DEV), torch.tensor([[1.0, 0, 0, 10, 10]], device=DEV))
    with pytest.raises(IndexError):
        cm.matrix
    cm.reset()
    assert not cm.matrix.any()
    # a detection class outside [0, nc): the labels of the epoch are in range, so only the matrix flags it
    det, cnt, tg, shapes, hw = _epoch_batches(31, 4, False, 1)[0]
    det[:, :, 5] = 4.0
    ep = val.ValEpoch(DEV, 4, confusion_matrix=cm)
    ep.add(det, cnt, tg, shapes, hw)
    with pytest.raises(IndexError):
        ep.finish()
    with pytest.raises(IndexError):
        cm.matrix


def test_captured_ssod_step_replayed_after_validate_with_a_matrix():
    """step (graph: the capture), validate(confusion_matrix=), step (graph: a replay) against the eager run"""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.metrics import ConfusionMatrix
    from efficientteacher_b200.trainer import SSODTrainerStep
    img, bl, bu = 256, 2, 2
    r = np.random.RandomState(3)
    imgs = torch.from_numpy(r.rand(bl, 3, img, img).astype(np.float32)).to(DEV)
    uw = torch.from_numpy(r.rand(bu, 3, img, img).astype(np.float32)).to(DEV)
    us = uw.flip(3).contiguous()
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    vr = np.random.RandomState(8)
    loader = [(torch.from_numpy(vr.randint(0, 256, (2, 3, 128, 128)).astype(np.uint8)), torch.from_numpy(synth.make_targets(40 + i, 10, 2)),
               ["a.jpg", "b.jpg"], _shapes(2, 128, 128, 30 + i)) for i in range(2)]
    out, mats = {}, {}
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
        f = st.train_instance_graphed if mode == "graph" else st.train_instance
        f(imgs, tg, us, uw, None, Ms, 1)
        cm = ConfusionMatrix(st.semi_ema.ema.nc)
        res = st.validate(loader, confusion_matrix=cm)
        assert len(res) == 5 and st.model.training
        mats[mode] = cm.matrix
        f(imgs, tg, us, uw, None, Ms, 3)
        torch.cuda.synchronize()
        out[mode] = torch.cat([t.detach().flatten().float() for t in st.model.state_dict().values()])
    assert all(m.sum() > 0 for m in mats.values())
    a, b, c = out["eager"], out["graph"], out["eager2"]
    assert torch.isfinite(b).all()
    n = a.norm().clamp_min(1e-30)
    assert ((a - b).norm() / n).item() <= 3.0 * ((a - c).norm() / n).item() + 2e-3
