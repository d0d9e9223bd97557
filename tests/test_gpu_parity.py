"""GPU (H100): the CUDA kernels, called through the reference-shaped Python mirrors over the C ABI, against the
oracle (oracle/port.py) and the golden vectors of the live reference.  Bit-exact for indices / keep-sets / EMA;
fp32 losses within 1e-4 relative (the tolerance BASELINE.json's north_star states)."""
import math

import numpy as np
import pytest
import torch

import synth
from oracle import port

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LOSS_RTOL = 1e-4


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)


def _assigner():
    from efficientteacher_b200.assigner import YOLOAnchorAssigner
    return YOLOAnchorAssigner(3, 3, torch.from_numpy(synth.ANCHORS_GRID), 4.0, torch.tensor([8., 16., 32.]))


def _zeros_p(B, img=640):
    return [torch.empty(B, 3, ny, nx, 85, device=DEV) for ny, nx in synth.level_shapes(img)]


# ------------------------------------------------------------------------------------------------ assigner
@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_build_targets_bit_exact(golden, name):
    g = golden("assign_" + name)
    B, n = int(g["B"]), int(g["n"])
    t = synth.make_targets(int(g["seed"]), n, B)
    sc = np.random.RandomState(int(g["score_seed"])).uniform(0.1, 1, (n, 1)).astype(np.float32)
    asg = _assigner()
    p = _zeros_p(B)
    for pref, tt, ws in (("bt_", t, False), ("uc_", np.concatenate([t, sc], 1), True)):
        res = asg(p, torch.from_numpy(tt).to(DEV), with_pseudo_score=ws)
        tcls, tbox, indices, anch = res[:4]
        for l in range(3):
            assert np.array_equal(torch.stack(indices[l], 1).cpu().numpy(), g[f"{pref}idx{l}"]), (pref, l)
            assert indices[l][0].dtype == torch.int64 and tcls[l].dtype == torch.int64
            assert np.array_equal(tcls[l].cpu().numpy(), g[f"{pref}tcls{l}"])
            assert np.array_equal(tbox[l].cpu().numpy(), g[f"{pref}tbox{l}"])
            assert np.array_equal(anch[l].cpu().numpy(), g[f"{pref}anch{l}"])
            if ws:
                assert np.array_equal(res[4][l].cpu().numpy(), g[f"{pref}tscore{l}"])


def test_build_targets_empty_and_large():
    asg = _assigner()
    tcls, tbox, indices, anch = asg(_zeros_p(2), torch.zeros(0, 6, device=DEV))
    assert all(len(c) == 0 for c in tcls)
    t = synth.make_targets(99, 4800, 16)                      # 300 pseudo labels x 16 images (maximum size)
    tcls, tbox, indices, anch = asg(_zeros_p(16), torch.from_numpy(t).to(DEV))
    ref = port.build_targets(t, synth.ANCHORS_GRID, synth.level_shapes())
    for l in range(3):
        assert np.array_equal(torch.stack(indices[l], 1).cpu().numpy(), ref[l]["idx"])
        assert np.array_equal(tbox[l].cpu().numpy(), ref[l]["tbox"])


# ------------------------------------------------------------------------------------------------ NMS / pseudo labels
@pytest.mark.parametrize("name", ["a", "dense", "cap", "hi"])
def test_nms_keep_sets_and_pseudo_rows(golden, name):
    from efficientteacher_b200 import nms as N
    from efficientteacher_b200.pseudo_label import FairPseudoLabel
    g = golden("nms_" + name)
    B, P = int(g["B"]), int(g["P"])
    pred = synth.make_teacher_pred(int(g["seed"]), B, P, cand_frac=float(g["frac"]))
    if name == "a":
        pred[2, :, 4] = 0.01
    tp = torch.from_numpy(pred).to(DEV)
    dets = N.non_max_suppression_ssod(tp, float(g["conf_thres"]), float(g["iou_thres"]))
    for b in range(B):
        assert np.array_equal(dets[b].cpu().numpy(), g[f"det{b}"]), (name, b)
    if "val0" in g.files:
        d6 = N.non_max_suppression(tp, 0.25, 0.45)
        for b in range(B):
            assert np.array_equal(d6[b].cpu().numpy(), g[f"val{b}"])

    class Cfg:  # the slice of the yacs tree FairPseudoLabel reads
        class SSOD:
            nms_conf_thres, nms_iou_thres, debug, multi_label = float(g["conf_thres"]), float(g["iou_thres"]), False, False
        class Dataset:
            names, np = [], 0
    fpl = FairPseudoLabel(Cfg)
    imgs = torch.empty(B, 3, 640, 640, device=DEV)
    rows, invalid = fpl.create_pseudo_label_online_with_gt(tp, imgs, torch.from_numpy(g["Ms"]), imgs)
    assert invalid == bool(g["invalid"])
    assert rows.dtype == torch.float64 and rows.device.type == "cpu"
    rows = rows.numpy()
    assert rows.shape == g["rows"].shape
    assert np.array_equal(rows[:, :2], g["rows"][:, :2])                    # image / class / order exact
    np.testing.assert_allclose(rows, g["rows"], rtol=1e-9, atol=1e-9)     # float64 boxes


def test_nms_no_candidates_and_properties_full_size():
    from efficientteacher_b200 import nms as N
    pred = synth.make_teacher_pred(5, 16, 25200)          # BASELINE config #3 size: 16 x 25200 x 85
    tp = torch.from_numpy(pred).to(DEV)
    empty = tp.clone()
    empty[..., 4] = 0.0
    assert all(d.shape == (0, 8) for d in N.non_max_suppression_ssod(empty, 0.1, 0.65))
    dets = N.non_max_suppression_ssod(tp, 0.1, 0.65)
    want = port.nms_ssod(pred, 0.1, 0.65)
    for b, d in enumerate(dets):
        d = d.cpu().numpy()
        assert np.array_equal(d, want[b])
        assert len(d) <= 300 and np.all(np.diff(d[:, 4]) <= 0) and np.all(d[:, 4] > 0.1)
    # idempotence: the kept boxes of an image suppress nothing among themselves
    b0 = dets[0]
    again = torch.zeros(1, len(b0), 85, device=DEV)
    again[0, :, 0] = (b0[:, 0] + b0[:, 2]) / 2; again[0, :, 1] = (b0[:, 1] + b0[:, 3]) / 2
    again[0, :, 2] = b0[:, 2] - b0[:, 0]; again[0, :, 3] = b0[:, 3] - b0[:, 1]
    again[0, :, 4] = 1.0
    again[0, torch.arange(len(b0)), 5 + b0[:, 5].long()] = b0[:, 4]
    d2 = N.non_max_suppression_ssod(again, 0.1, 0.65)[0]
    assert len(d2) == len(b0)


def test_nms_1280_geometry_vs_oracle():
    """BASELINE configs[4]: 1280x1280 -> 102,000 predictions per image; keep-sets and rows bit-exact vs the oracle."""
    from efficientteacher_b200 import nms as N
    pred = synth.make_teacher_pred(11, 3, 102000, img=1280)
    dets = N.non_max_suppression_ssod(torch.from_numpy(pred).to(DEV), 0.1, 0.65)
    want = port.nms_ssod(pred, 0.1, 0.65)
    for b, d in enumerate(dets):
        d = d.cpu().numpy()
        assert np.array_equal(d, want[b])
        assert len(d) <= 300 and np.all(np.diff(d[:, 4]) <= 0)


# ------------------------------------------------------------------------------------------------ select_targets
def _ssod_loss_obj(model_like=None):
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    cfg = ssod_cfg()
    return ComputeStudentMatchLoss(HeadOnlyModel().to(DEV), cfg), cfg


def test_select_targets(golden):
    g = golden("select")
    crit, _ = _ssod_loss_obj()
    crit.ignore_thres_high = list(g["high"])
    crit.ignore_thres_low = list(g["low"])
    rows = synth.make_pseudo_rows(int(g["seed"]), int(g["n"]), int(g["B"]))
    sel = crit.select_targets(torch.from_numpy(rows).to(DEV))
    for i in range(4):
        assert np.array_equal(sel[i].cpu().numpy(), g[f"s{i}"]), i


# ------------------------------------------------------------------------------------------------ CIoU / decode
def test_bbox_ciou(golden):
    from efficientteacher_b200.loss import bbox_iou
    g = golden("ciou")
    c = bbox_iou(torch.from_numpy(g["b1"]).to(DEV).T, torch.from_numpy(g["b2"]).to(DEV), x1y1x2y2=False, CIoU=True)
    np.testing.assert_allclose(c.cpu().numpy(), g["ciou"], rtol=1e-5, atol=1e-6)


def test_detect_decode(golden):
    from efficientteacher_b200.head import decode_levels
    g = golden("decode")
    raw = [torch.from_numpy(g[f"raw{l}"]).to(DEV) for l in range(3)]
    pred = decode_levels(raw, torch.from_numpy(synth.ANCHORS_GRID), synth.STRIDES)
    np.testing.assert_allclose(pred.cpu().numpy(), g["pred"], rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ losses
def _check_grads(g, p):
    for l, pi in enumerate(p):
        gr = pi.grad.cpu().numpy().reshape(-1)
        np.testing.assert_allclose(gr[g[f"g{l}_si"]], g[f"g{l}_sv"], rtol=LOSS_RTOL, atol=1e-7)
        np.testing.assert_allclose(gr[g[f"g{l}_ti"]], g[f"g{l}_tv"], rtol=LOSS_RTOL, atol=1e-7)
        np.testing.assert_allclose(np.abs(gr).sum(dtype=np.float64), float(g[f"g{l}_l1"]), rtol=LOSS_RTOL)
        np.testing.assert_allclose(pi.grad.cpu().numpy()[..., 4].reshape(-1)[::7], g[f"g{l}_obj"], rtol=LOSS_RTOL, atol=1e-8)


def test_compute_loss_sup(golden):
    from efficientteacher_b200.loss import ComputeLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    g = golden("loss_sup")
    B = int(g["B"])
    crit = ComputeLoss(HeadOnlyModel().to(DEV), ssod_cfg())
    p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in synth.make_head_logits(int(g["logit_seed"]), B)]
    tg = synth.make_targets(int(g["target_seed"]), int(g["n"]), B)
    loss, items = crit(p, torch.from_numpy(tg).to(DEV))
    assert loss.shape == (1,) and loss.requires_grad and set(items) == {"box", "obj", "cls", "loss"}
    np.testing.assert_allclose(loss.detach().cpu().numpy(), g["loss"], rtol=LOSS_RTOL)
    for k in ("box", "obj", "cls"):
        np.testing.assert_allclose(items[k].cpu().numpy(), g[k], rtol=LOSS_RTOL)
    loss.backward()
    _check_grads(g, p)


def test_compute_loss_ssod(golden):
    g = golden("loss_ssod")
    B = int(g["B"])
    crit, _ = _ssod_loss_obj()
    p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in synth.make_head_logits(int(g["logit_seed"]), B)]
    rows = synth.make_pseudo_rows(int(g["rows_seed"]), int(g["n"]), B)
    loss, items = crit(p, torch.from_numpy(rows).to(DEV))
    assert set(items) == {"ss_box", "ss_obj", "ss_cls"}
    np.testing.assert_allclose(loss.detach().cpu().numpy(), g["loss"], rtol=LOSS_RTOL)
    for k in ("box", "obj", "cls"):
        np.testing.assert_allclose(items["ss_" + k].cpu().numpy(), g[k], rtol=LOSS_RTOL)
    (loss * 3.0).backward()                 # teacher_loss_weight-style upstream scale
    for pi in p:
        pi.grad /= 3.0
    _check_grads(g, p)


def test_loss_full_size_vs_oracle():
    """BASELINE config #3 size (B=16): fused loss vs the oracle on the same seeded inputs, plus linearity in the
    upstream gradient."""
    from efficientteacher_b200.loss import ComputeLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    B = 16
    crit = ComputeLoss(HeadOnlyModel().to(DEV), ssod_cfg())
    logits = synth.make_head_logits(77, B)
    tg = synth.make_targets(78, 128, B)
    p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in logits]
    loss, items = crit(p, torch.from_numpy(tg).to(DEV))
    loss.backward()
    pc = [torch.from_numpy(x).requires_grad_(True) for x in logits]
    ref, _ = port.det_loss(pc, [port.build_targets(tg, synth.ANCHORS_GRID, synth.level_shapes())], [4.0, 1.0, 0.4], 0.05, 0.7, 0.3)
    ref.backward()
    np.testing.assert_allclose(loss.item(), ref.item(), rtol=LOSS_RTOL)
    for a, b in zip(p, pc):
        ga, gb = a.grad.cpu().numpy(), b.grad.numpy()
        assert np.abs(ga - gb).max() <= 1e-4 * np.abs(gb).max() + 1e-9
    g1 = [a.grad.clone() for a in p]
    for a in p:
        a.grad = None
    loss2, _ = crit(p, torch.from_numpy(tg).to(DEV))
    (loss2 * 2.0).backward()
    for a, b in zip(p, g1):
        torch.testing.assert_close(a.grad, 2.0 * b, rtol=1e-6, atol=1e-9)


# ------------------------------------------------------------------------------------------------ EMA
class Tiny(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Conv2d(3, 7, 3, bias=False)
        self.bn = torch.nn.BatchNorm2d(7)
        self.b = torch.nn.Linear(13, 5)


def _load(mod, g, prefix):
    sd = {k: torch.from_numpy(np.asarray(g[prefix + k])) for k in mod.state_dict()}
    mod.load_state_dict(sd)


def test_ema_bit_exact(golden):
    from efficientteacher_b200.ema import ModelEMA, CosineEMA, SemiSupModelEMA, update_ema_pair
    g = golden("ema")
    src = Tiny()
    _load(src, g, "init_")
    src = src.to(DEV)
    ema, ema_f = ModelEMA(src), ModelEMA(src)
    semi = CosineEMA(ema.ema, decay_start=0.99, decay_end=0.9999, total_epoch=10)
    semi_f = CosineEMA(ema_f.ema, decay_start=0.99, decay_end=0.9999, total_epoch=10)
    semi.update_decay(3); semi_f.update_decay(3)
    assert semi.decay == float(g["semi_decay"])
    ssup = SemiSupModelEMA(src, 0.999)
    assert not ema.ema.training and all(not q.requires_grad for q in ema.ema.parameters())
    for step in range(3):
        with torch.no_grad():
            for k, v in src.state_dict().items():
                v.copy_(torch.from_numpy(np.asarray(g[f"src{step}_{k}"])))
        ema.update(src); semi.update(ema.ema); ssup.update(src)
        update_ema_pair(ema_f, semi_f, src)                      # fused 5-stream variant
        assert ema.updates == step + 1 and ema_f.updates == step + 1
        for name, obj in (("ema", ema), ("semi", semi), ("ssup", ssup), ("ema", ema_f), ("semi", semi_f)):
            for k, v in obj.ema.state_dict().items():
                assert np.array_equal(v.cpu().numpy(), g[f"{name}{step}_{k}"]), (name, step, k)


def test_ema_large_unaligned_vs_two_rounding_formula():
    from efficientteacher_b200.ema import ModelEMA

    class Big(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w1 = torch.nn.Parameter(torch.randn(3_000_001))
            self.w2 = torch.nn.Parameter(torch.randn(4097, 33))
            self.register_buffer("odd", torch.randn(7))
    torch.manual_seed(0)
    m = Big().to(DEV)
    ema = ModelEMA(m, updates=5000)
    before = {k: v.clone() for k, v in ema.ema.state_dict().items()}
    with torch.no_grad():
        for q in m.parameters():
            q.add_(torch.randn_like(q) * 0.01)
    ema.update(m)
    d = 0.9999 * (1 - math.exp(-5001 / 2000))
    for k, v in ema.ema.state_dict().items():
        want = before[k] * np.float32(d) + np.float32(1.0 - d) * m.state_dict()[k]     # torch CUDA: mul, mul, add
        assert torch.equal(v, want), k


# ------------------------------------------------------------------------------------------------ fused SGD
def test_fused_sgd_matches_torch_sgd():
    """FusedSGD (one launch, grads zeroed in the same pass) vs torch.optim.SGD(nesterov) with the reference's three
    parameter groups (bias | conv weights + weight decay | BN weights), trainer/trainer.py:215-217."""
    from efficientteacher_b200.optim import FusedSGD
    torch.manual_seed(0)
    shapes = [(255,), (64, 3, 6, 6), (128, 64, 3, 3), (1024, 1024, 1, 1), (513,), (7,)]
    groups = [[0, 4], [1, 2, 3], [5]]
    mk = lambda: [torch.nn.Parameter(torch.randn(s, generator=torch.Generator().manual_seed(i)).to(DEV)) for i, s in enumerate(shapes)]  # noqa: E731
    pa, pb = mk(), mk()
    oa = FusedSGD([pa[i] for i in groups[0]], lr=0.01, momentum=0.937, nesterov=True)
    ob = torch.optim.SGD([pb[i] for i in groups[0]], lr=0.01, momentum=0.937, nesterov=True)
    for o, ps in ((oa, pa), (ob, pb)):
        o.add_param_group({'params': [ps[i] for i in groups[1]], 'weight_decay': 0.0005})
        o.add_param_group({'params': [ps[i] for i in groups[2]]})
    for step in range(3):
        if step == 2:
            for o in (oa, ob):
                o.param_groups[1]['lr'] = 0.02       # schedule change is picked up
        for i, (a, b) in enumerate(zip(pa, pb)):
            gr = torch.randn(a.shape, generator=torch.Generator().manual_seed(100 * step + i)).to(DEV)
            a.grad = gr.clone() if a.grad is None else a.grad.copy_(gr)
            b.grad = gr.clone()
        oa.step()
        ob.step()
        for a, b in zip(pa, pb):
            torch.testing.assert_close(a.detach(), b.detach(), rtol=2e-6, atol=1e-6)   # fma vs mul+add rounding
            assert float(a.grad.abs().max()) == 0.0          # zeroed by the fused pass
        for a, b in zip(pa, pb):
            torch.testing.assert_close(oa.state[a]["momentum_buffer"], ob.state[b]["momentum_buffer"], rtol=2e-6, atol=1e-6)


def test_fused_sgd_load_state_dict_restores_momentum():
    """resume (trainer/trainer.py:251 optimizer.load_state_dict): the restored momentum buffers must be the ones the fused
    kernel reads -- a step after load_state_dict equals the step of the optimizer the state was saved from"""
    from efficientteacher_b200.optim import FusedSGD
    mk = lambda: [torch.nn.Parameter(torch.randn(s, generator=torch.Generator().manual_seed(i)).to(DEV)) for i, s in enumerate([(33,), (16, 8, 3, 3)])]  # noqa: E731
    pa, pb = mk(), mk()
    grads = [[torch.randn(p.shape, generator=torch.Generator().manual_seed(50 + 10 * k + i)).to(DEV) for i, p in enumerate(pa)] for k in range(3)]

    def step(opt, ps, k):
        for p, g in zip(ps, grads[k]):
            p.grad = g.clone() if p.grad is None else p.grad.copy_(g)
        opt.step()
    oa = FusedSGD(pa, lr=0.01, momentum=0.9, nesterov=True)
    step(oa, pa, 0); step(oa, pa, 1)
    sd = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in oa.state_dict().items()}
    sd["state"] = {k: {"momentum_buffer": v["momentum_buffer"].clone()} for k, v in oa.state_dict()["state"].items()}
    ob = FusedSGD(pb, lr=0.01, momentum=0.9, nesterov=True)
    with torch.no_grad():
        for a, b in zip(pa, pb):
            b.copy_(a)
    step(ob, pb, 2)                      # builds ob's flat buffer (with a wrong history) ...
    with torch.no_grad():
        for a, b in zip(pa, pb):
            b.copy_(a)
    ob.load_state_dict(sd)               # ... which load_state_dict must overwrite
    step(oa, pa, 2); step(ob, pb, 2)
    for a, b in zip(pa, pb):
        assert torch.equal(a.detach(), b.detach())


def test_fused_sgd_load_state_dict_without_momentum_starts_fresh():
    """A torch SGD state dict saved before any step has no momentum buffers.  Loaded into a FusedSGD that has already
    stepped, it must drop the old momentum: the next step equals torch.optim.SGD's first step (buf = grad)."""
    from efficientteacher_b200.optim import FusedSGD
    mk = lambda: [torch.nn.Parameter(torch.randn(s, generator=torch.Generator().manual_seed(i)).to(DEV)) for i, s in enumerate([(33,), (16, 8, 3, 3)])]  # noqa: E731
    pa, pb = mk(), mk()
    grads = [[torch.randn(p.shape, generator=torch.Generator().manual_seed(70 + 10 * k + i)).to(DEV) for i, p in enumerate(pa)] for k in range(2)]

    def step(opt, ps, k):
        for p, g in zip(ps, grads[k]):
            p.grad = g.clone() if p.grad is None else p.grad.copy_(g)
        opt.step()
    ob = torch.optim.SGD(pb, lr=0.01, momentum=0.9, nesterov=True)
    sd = ob.state_dict()                 # saved before any step
    oa = FusedSGD(pa, lr=0.01, momentum=0.9, nesterov=True)
    step(oa, pa, 0)                      # oa's flat momentum buffer now holds a history ...
    with torch.no_grad():
        for a, b in zip(pa, pb):
            a.copy_(b)
    oa.load_state_dict(sd)               # ... which the loaded state does not have
    step(oa, pa, 1); step(ob, pb, 1)
    for a, b in zip(pa, pb):
        torch.testing.assert_close(a.detach(), b.detach(), rtol=2e-6, atol=1e-6)   # fma vs mul+add rounding
        torch.testing.assert_close(oa.state[a]["momentum_buffer"], ob.state[b]["momentum_buffer"], rtol=2e-6, atol=1e-6)


def test_labelmatch_device_path_matches_reference(golden):
    """LabelMatch on the device pipeline: rows, the per-class score lists (async pinned copy + flush) and the epoch thresholds
    against the live-reference fixture (tests/golden/labelmatch.npz)."""
    from types import SimpleNamespace as NS
    from efficientteacher_b200.labelmatch import LabelMatch
    g = golden("labelmatch")
    cfg = NS(SSOD=NS(nms_conf_thres=float(g["nms_conf_thres"]), nms_iou_thres=float(g["nms_iou_thres"]), debug=False, multi_label=False,
                     ignore_thres_low=float(g["ignore_thres_low"]), ignore_thres_high=float(g["ignore_thres_high"]),
                     resample_high_percent=float(g["resample_high_percent"]), resample_low_percent=float(g["resample_low_percent"])),
             Dataset=NS(names=[str(i) for i in range(80)], np=0))
    lm = LabelMatch(cfg, 1000, 7.0, np.full(80, 1.0 / 80))
    for bi in range(2):
        seed, B, P, frac = g[f"b{bi}_meta"]
        pred = torch.from_numpy(synth.make_teacher_pred(int(seed), int(B), int(P), cand_frac=float(frac))).to(DEV)
        Ms = torch.from_numpy(synth.make_Ms(int(seed) + 100, int(B))).to(DEV)
        imgs = torch.zeros(int(B), 3, 640, 640, device=DEV)
        rows, invalid = lm.create_pseudo_label_online_with_gt(pred, imgs, Ms, imgs)
        assert not invalid
        rows = rows.numpy()
        want = g[f"b{bi}_rows"]
        assert rows.shape == want.shape and np.array_equal(rows[:, :2], want[:, :2])
        np.testing.assert_allclose(rows, want, rtol=1e-9, atol=1e-9)
        lm.update(rows, n=int(B), pse_n=int(B))
    lm.flush()
    assert np.array_equal(np.array([len(c) for c in lm.score_list_epoch]), g["epoch_score_lens"])
    assert np.array_equal(np.array([v for c in lm.score_list_epoch for v in c]), g["epoch_scores"])
    lm.update_epoch_cls_thr(0)
    np.testing.assert_allclose(np.array(lm.cls_thr_low), g["thr_low_e0"], rtol=0, atol=0)
    np.testing.assert_allclose(np.array(lm.cls_thr_high), g["thr_high_e0"], rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("name", ["ml_cap", "ml_few", "ml_agn"])
def test_val_nms_multi_label_vs_reference_golden(golden, name):
    """val.py path: non_max_suppression(multi_label=True) on the device (radix top-30000 + shared NMS kernels) against the
    live-reference fixture: keep-sets, order, boxes and scores bit-exact."""
    from efficientteacher_b200 import nms as N
    g = golden("nms_val")
    seed, B, P, frac, conf, iou, ml, agn = g[name + "_meta"]
    pred = synth.make_teacher_pred(int(seed), int(B), int(P), cand_frac=float(frac))
    if name == "ml_agn":
        pred[1, :, 4] = 0.0
    dets = N.non_max_suppression(torch.from_numpy(pred).to(DEV), float(conf), float(iou), multi_label=True, agnostic=bool(agn))
    for b in range(int(B)):
        want = g[f"{name}_det{b}"]
        got = dets[b].cpu().numpy()
        assert got.shape == want.shape, (name, b, got.shape, want.shape)
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("name", ["a", "b", "c", "d"])
def test_val_process_batch_vs_reference_golden(name):
    """val.py:123-145 on the device (etb_val_process_batch) against the live-reference fixture, single image and batched"""
    import os
    from efficientteacher_b200 import val as etb_val
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "val_process_batch.npz"))
    det, lab, want = g[name + "_det"], g[name + "_lab"], g[name + "_correct"]
    iouv = torch.linspace(0.5, 0.95, 10).to(DEV)
    got = etb_val.process_batch(torch.from_numpy(det).to(DEV), torch.from_numpy(lab).to(DEV), iouv)
    assert np.array_equal(got.cpu().numpy(), want)
    # batched: the same image twice plus an empty one, padded rows, per-image counts
    n = det.shape[0]
    pad = torch.zeros((3, n + 5, 6), device=DEV)
    pad[0, :n] = torch.from_numpy(det).to(DEV); pad[2, :n] = torch.from_numpy(det).to(DEV)
    cnt = torch.tensor([n, 0, n], dtype=torch.int32, device=DEV)
    labs = torch.cat([torch.cat([torch.full((len(lab), 1), float(i)), torch.from_numpy(lab)], 1) for i in (0, 2)], 0).to(DEV)
    out = etb_val.process_batch_batched(pad, cnt, labs, iouv).cpu().numpy()
    assert np.array_equal(out[0, :n], want) and np.array_equal(out[2, :n], want) and not out[1].any() and not out[0, n:].any()


def test_extra_teachers_merge_vs_reference_golden():
    """device merge (NMS of every teacher + class remap + class-agnostic etb_nms_boxes per teacher) vs the live-reference fixture"""
    import os
    from efficientteacher_b200.pseudo_label import merge_extra_teacher_detections
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "extra_teachers.npz"))
    B, P = 2, 4000
    mk = lambda s, f: torch.from_numpy(synth.make_teacher_pred(s, B, P, cand_frac=f)).to(DEV)  # noqa: E731
    got = merge_extra_teacher_detections(mk(21, 0.05), [mk(22, 0.04), mk(23, 0.03)], [{3: 70, 5: 1, 7: 7}, {}], float(g["conf"]), float(g["iou"]))
    assert np.array_equal(got[0].cpu().numpy(), g["out0"]) and np.array_equal(got[1].cpu().numpy(), g["out1"])
