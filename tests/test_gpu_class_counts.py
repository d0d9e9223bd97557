"""GPU (H100): the Detect head, decode, NMS, assigner, routing, fused loss and the whole training step at the class counts
of the reference's other datasets -- VOC (nc 20, no 25), Cityscapes (nc 8, anchor_t 5.0), the custom configs (nc 2) and
single_cls (nc 1) -- plus nc 85 (no 90) and nc 128 (no 133) for the Detect backward, whose dy packing once required
no + pad <= 128.  Every native path that branches on no, nc or anchor_t is compared with a float64 (or bit-exact)
oracle here; the rest of the suite runs at nc 80 only."""
import math

import numpy as np
import pytest
import torch

import synth
from oracle import port
from test_oracle_golden_nc import IMG, NCS, SWITCHES, check_loss, loss_prefix

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOSS_RTOL = 1e-4


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _ints(shape, seed, lo=-2, hi=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).float().to(DEV)


# ------------------------------------------------------------------------------------------------ Detect conv
DET_NO = [85, 25, 13, 7, 6, 90, 133]
MAPS = [(20, 20), (11, 7), (1, 1)]


def _det_ref(x, w, b, no):
    """float64 Detect conv in the train layout [N,na,H,W,no]"""
    N, _, H, W = x.shape
    y = torch.einsum("nchw,oc->nohw", x.double(), w.double().flatten(1)) + b.double().view(1, -1, 1, 1)
    return y.view(N, -1, no, H, W).permute(0, 1, 3, 4, 2)


@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("hw", MAPS)
@pytest.mark.parametrize("no", DET_NO)
def test_detect_conv_forward_exact_and_in_bounds(no, hw, N):
    """the fp32 Detect-layout epilogue (EPI 2): every element of [N,na,H,W,no] written once with the float64 value, nothing
    past the end -- the inference path the teacher engine takes (folded bias) on a channel-sliced input"""
    from efficientteacher_b200 import convops as co
    H, W = hw
    na, Cin = 3, 128
    Cout = na * no
    x, w, b = _ints((N, Cin, H, W), 1), _ints((Cout, Cin, 1, 1), 2), _ints((Cout,), 3, -8, 8)
    xw = torch.zeros((N, H, W, Cin + 64), dtype=torch.bfloat16, device=DEV)
    co.to_nhwc_bf16(x, out=xw, coffset=32)
    n_out, guard = N * na * H * W * no, 4096
    buf = torch.full((n_out + guard,), float("nan"), device=DEV)
    out = buf[:n_out].view(N, na, H, W, no)
    co.conv_fwd(xw, co.pack_weight(w), Cin, Cout, 1, 1, 0, None, b, act=None, x_coffset=32, x_cstride=Cin + 64, det_out=out,
                det_no=no)
    assert torch.equal(out.double(), _det_ref(x, w, b, no))
    assert torch.isnan(buf[n_out:]).all()


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("hw", MAPS)
@pytest.mark.parametrize("no", DET_NO)
def test_detect_conv_fn_forward_backward_exact(no, hw, N, accumulate):
    """DetectConvFn (the student's head): forward as above; backward on an integer gradient -- dx (bf16) is the float64
    input gradient rounded once, dW and the bias gradient equal float64, also added into existing .grad tensors"""
    from efficientteacher_b200.autograd_conv import DetectConvFn
    H, W = hw
    na, Cin = 3, 128
    Cout = na * no
    x = _ints((N, Cin, H, W), 4).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = _ints((Cout, Cin, 1, 1), 5).requires_grad_(True)
    b = _ints((Cout,), 6, -8, 8).requires_grad_(True)
    w0, b0 = _ints((Cout, Cin, 1, 1), 7, -64, 64), _ints((Cout,), 8, -64, 64)
    if accumulate:
        w.grad, b.grad = w0.clone(), b0.clone()
    out = DetectConvFn.apply(x, w, b, na, no)
    assert out.shape == (N, na, H, W, no)
    assert torch.equal(out.double(), _det_ref(x.float(), w.detach(), b.detach(), no))
    g = _ints((N, na, H, W, no), 9)
    out.backward(g)
    g2 = g.double().permute(0, 1, 4, 2, 3).reshape(N, Cout, H, W)
    want_dx = torch.einsum("nohw,oc->nchw", g2, w.detach().double().flatten(1))
    want_dw = torch.einsum("nohw,nchw->oc", g2, x.detach().double()).view(Cout, Cin, 1, 1)
    want_db = g2.sum((0, 2, 3))
    if accumulate:
        want_dw, want_db = want_dw + w0.double(), want_db + b0.double()
    assert torch.equal(x.grad.float(), want_dx.to(torch.bfloat16).float())
    assert torch.equal(w.grad.double(), want_dw)
    assert torch.equal(b.grad.double(), want_db)


@pytest.mark.parametrize("no", DET_NO)
def test_detect_dy_pack_zeroes_every_pad_channel(no):
    """the dgrad K padding [na*no, ceil64(na*no)) is zero even where the buffer held NaN; the wgrad / dgrad of DetectConvFn
    read it (up to 53 pad channels at these class counts), and the column sums give the bias gradient"""
    from efficientteacher_b200 import _lib
    from efficientteacher_b200 import convops as co
    N, na, H, W = 2, 3, 13, 11
    C_ = na * no
    cpad = (C_ + 63) // 64 * 64
    g = torch.randn((N, na, H, W, no), generator=torch.Generator().manual_seed(10)).to(DEV)
    dy = torch.full((N, H, W, cpad), float("nan"), dtype=torch.bfloat16, device=DEV)
    rows = int(_lib.lib().etb_detect_dy_rows(N, H, W))
    partials = torch.empty((rows, C_), device=DEV)
    _lib.check(_lib.lib().etb_detect_dy_pack(_lib.ptr(g), _lib.ptr(dy), _lib.ptr(partials), N, na, H, W, no, cpad,
                                             _lib.stream_ptr()), "etb_detect_dy_pack")
    assert torch.equal(dy[..., :C_], g.permute(0, 2, 3, 1, 4).reshape(N, H, W, C_).to(torch.bfloat16))
    assert (dy[..., C_:] == 0).all()
    want = g.double().sum((0, 2, 3)).reshape(-1)
    assert float((co.column_sum(partials).double() - want).abs().max()) <= 1e-5 * float(want.abs().max()) + 1e-5


# ------------------------------------------------------------------------------------------------ decode
@pytest.mark.parametrize("no", [85, 25, 13, 7, 6, 90])
def test_detect_decode_vs_float64(no):
    from efficientteacher_b200.head import decode_levels
    r = np.random.RandomState(no)
    raw = [(r.standard_normal((2, 3, ny, nx, no)) * 2).astype(np.float32) for ny, nx in synth.level_shapes(320)]
    pred = decode_levels([torch.from_numpy(x).to(DEV) for x in raw], torch.from_numpy(synth.ANCHORS_GRID), synth.STRIDES)
    outs = []
    for x, anc, s in zip(raw, synth.ANCHORS_GRID, synth.STRIDES):
        y = 1.0 / (1.0 + np.exp(-x.astype(np.float64)))
        B, na, ny, nx, _ = x.shape
        gy, gx = np.meshgrid(np.arange(ny), np.arange(nx), indexing="ij")
        o = y.copy()
        o[..., 0] = (y[..., 0] * 2 - 0.5 + gx) * s
        o[..., 1] = (y[..., 1] * 2 - 0.5 + gy) * s
        o[..., 2:4] = (y[..., 2:4] * 2) ** 2 * (anc.astype(np.float64) * s).reshape(1, na, 1, 1, 2)
        outs.append(o.reshape(B, -1, no))
    want = np.concatenate(outs, 1)
    assert pred.shape == want.shape
    np.testing.assert_allclose(pred.cpu().numpy(), want, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ NMS / pseudo labels
@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("nc", [20, 8, 2, 1])
def test_nms_ssod_and_pseudo_rows(nc, ties):
    from efficientteacher_b200 import nms as N
    from efficientteacher_b200.pseudo_label import FairPseudoLabel
    B = 3
    pred = synth.make_teacher_pred_ties(20 + nc, B, nc, ties)
    tp = torch.from_numpy(pred).to(DEV)
    dets = N.non_max_suppression_ssod(tp, 0.1, 0.65)
    want = port.nms_ssod(pred, 0.1, 0.65)
    for b in range(B):
        assert np.array_equal(dets[b].cpu().numpy(), want[b]), (nc, b)
        assert len(want[b]) > 0

    class Cfg:  # the slice of the yacs tree FairPseudoLabel reads
        class SSOD:
            nms_conf_thres, nms_iou_thres, debug, multi_label = 0.1, 0.65, False, False
        class Dataset:
            names, np = [str(i) for i in range(nc)], 0
    Ms = synth.make_Ms(30 + nc, B)
    imgs = torch.empty(B, 3, 640, 640, device=DEV)
    rows, _ = FairPseudoLabel(Cfg).create_pseudo_label_online_with_gt(tp, imgs, torch.from_numpy(Ms), imgs)
    rows, want_rows = rows.numpy(), port.pseudo_label_rows(want, Ms, 640, 640)
    assert rows.shape == want_rows.shape and len(rows) > 0
    assert np.array_equal(rows[:, :2], want_rows[:, :2])
    np.testing.assert_allclose(rows, want_rows, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("conf", [0.001, 0.25])
@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("nc", [20, 8, 2, 1])
def test_val_nms_routes(nc, ties, conf):
    """val._nms: etb_nms_val (multi-label) for nc > 1, the best-class pipeline with the class-confidence filter at nc 1;
    single_cls (class-agnostic) at every nc"""
    from efficientteacher_b200 import val
    B = 2
    pred = synth.make_teacher_pred_ties(40 + nc, B, nc, ties, 320)
    tp = torch.from_numpy(pred).to(DEV)
    for agnostic in (False, True):
        det, cnt = val._nms(tp, conf, 0.6, agnostic)
        want = port.nms_val(pred, conf, 0.6, multi_label=True, agnostic=agnostic)
        cnt = cnt.cpu().tolist()
        for b in range(B):
            assert np.array_equal(det[b, :cnt[b], :6].cpu().numpy(), want[b]), (nc, agnostic, b)


# ------------------------------------------------------------------------------------------------ assigner / routing
@pytest.mark.parametrize("anchor_t", [4.0, 5.0])
def test_build_targets_anchor_t(anchor_t):
    from efficientteacher_b200.assigner import YOLOAnchorAssigner
    B, n = 4, 160
    t = synth.make_targets(50, n, B, nc=8)
    t[: n // 8, 4:6] *= 3.0          # wide spread of box-to-anchor ratios: many fall between 4 and 5
    sc = np.random.RandomState(51).uniform(0.1, 1, (n, 1)).astype(np.float32)
    asg = YOLOAnchorAssigner(3, 3, torch.from_numpy(synth.ANCHORS_GRID), anchor_t, torch.tensor([8., 16., 32.]), 8)
    p = [torch.empty(B, 3, ny, nx, 13, device=DEV) for ny, nx in synth.level_shapes(960)]
    for tt, ws in ((t, False), (np.concatenate([t, sc], 1), True)):
        res = asg(p, torch.from_numpy(tt).to(DEV), with_pseudo_score=ws)
        ref = port.build_targets(tt, synth.ANCHORS_GRID, synth.level_shapes(960), anchor_t=anchor_t, with_score=ws)
        for l in range(3):
            assert np.array_equal(torch.stack(res[2][l], 1).cpu().numpy(), ref[l]["idx"]), (ws, l)
            assert np.array_equal(res[0][l].cpu().numpy(), ref[l]["tcls"])
            assert np.array_equal(res[1][l].cpu().numpy(), ref[l]["tbox"])
            assert np.array_equal(res[3][l].cpu().numpy(), ref[l]["anch"])
            if ws:
                assert np.array_equal(res[4][l].cpu().numpy(), ref[l]["tscore"])
    if anchor_t == 5.0:     # the threshold matters for these targets
        ref4 = port.build_targets(t, synth.ANCHORS_GRID, synth.level_shapes(960), anchor_t=4.0)
        assert sum(len(r["idx"]) for r in ref4) < sum(len(r["idx"]) for r in ref)


def test_select_targets_per_class_thresholds():
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    nc = 8
    crit = ComputeStudentMatchLoss(HeadOnlyModel(nc).to(DEV), ssod_cfg(nc))
    crit.ignore_thres_high = [0.6, 0.5, 0.75, 0.9, 0.4, 0.6, 0.55, 0.8]
    crit.ignore_thres_low = [0.1, 0.2, 0.05, 0.3, 0.1, 0.15, 0.25, 0.12]
    rows = synth.make_pseudo_rows(60, 400, 4, nc=nc)
    sel = crit.select_targets(torch.from_numpy(rows).to(DEV))
    want = port.select_targets(rows, crit.ignore_thres_high, crit.ignore_thres_low, True)
    for i in range(4):
        assert np.array_equal(sel[i].cpu().numpy(), want[i]), i
    assert all(len(w) for w in want)


def test_label_class_hist_two_classes():
    from efficientteacher_b200 import _lib
    nc = 2
    t = synth.make_targets(70, 300, 4, nc=nc)
    t[:5, 1] = [-0.5, 1.9, 2.0, -1.0, float("nan")]     # int() truncates: 0, 1; then out of range / NaN -> slot nc
    tt = torch.from_numpy(t).to(DEV)
    hist = torch.zeros(nc + 1, dtype=torch.int32, device=DEV)
    for _ in range(2):       # accumulates
        _lib.check(_lib.lib().etb_label_class_hist(_lib.ptr(tt), None, len(t), len(t), 6, nc, _lib.ptr(hist), _lib.stream_ptr()),
                   "etb_label_class_hist")
    c = t[:, 1]
    ok = (c > -1) & (c < nc)
    want = np.bincount(np.where(ok, np.trunc(np.nan_to_num(c, nan=-9)), nc).astype(np.int64), minlength=nc + 1) * 2
    assert hist.cpu().numpy().tolist() == want.tolist()


# ------------------------------------------------------------------------------------------------ fused loss
def _logits(seed, B, nc, img=320):
    return synth.make_head_logits(seed, B, img=img, no=nc + 5)


def _check_loss(items, loss, p, ref_items, ref_loss, ref_p, nc):
    np.testing.assert_allclose(loss.item(), ref_loss.item(), rtol=LOSS_RTOL)
    for a, b in zip(items, ref_items):
        np.testing.assert_allclose(float(a), float(b.detach()), rtol=LOSS_RTOL, atol=1e-12)
    for a, b in zip(p, ref_p):
        ga, gb = a.grad.double().cpu().numpy(), b.grad.numpy()
        assert np.abs(ga - gb).max() <= 1e-4 * np.abs(gb).max(), (np.abs(ga - gb).max(), np.abs(gb).max())
        if nc == 1:
            assert not a.grad[..., 5].any()


def _sup_targets(nc, B, case):
    t = synth.make_targets(80 + nc, 12 * B, B, nc=nc)
    if case == "empty_level":            # boxes far smaller than every P5 anchor: the last level assigns nothing
        t[:, 4:6] = np.float32(0.02)
    return t


@pytest.mark.parametrize("case", ["dup", "empty_level"])
@pytest.mark.parametrize("smooth", [0.0, 0.1])
@pytest.mark.parametrize("nc", [20, 8, 2, 1])
def test_compute_loss_vs_float64(nc, smooth, case):
    from efficientteacher_b200.loss import ComputeLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    B = 2
    cfg = ssod_cfg(nc)
    cfg.Loss.label_smoothing = smooth
    cfg.single_cls = nc == 1
    anchor_t = 5.0 if nc == 8 else 4.0
    cfg.Loss.anchor_t = anchor_t
    crit = ComputeLoss(HeadOnlyModel(nc).to(DEV), cfg)
    logits = _logits(90 + nc, B, nc)
    tg = _sup_targets(nc, B, case)
    p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in logits]
    loss, items = crit(p, torch.from_numpy(tg).to(DEV))
    loss.backward()
    sets = [port.build_targets(tg, synth.ANCHORS_GRID, synth.level_shapes(320), anchor_t)]
    if case == "empty_level":
        assert len(sets[0][2]["idx"]) == 0 and len(sets[0][0]["idx"]) > 0
    pd = [torch.from_numpy(x).double().requires_grad_(True) for x in logits]
    cp, cn = 1.0 - 0.5 * smooth, 0.5 * smooth
    ref, ref_items = port.det_loss(pd, sets, [4.0, 1.0, 0.4], 0.05, 0.7, 0.3 * nc / 80. * 3. / 3, cp, cn)
    ref.backward()
    _check_loss([items[k] for k in ("box", "obj", "cls")], loss, p, ref_items, ref, pd, nc)
    if nc == 1:
        assert float(items["cls"]) == 0.0


@pytest.mark.parametrize("smooth", [0.0, 0.1])
@pytest.mark.parametrize("ignore_obj,with_bbox,with_cls", [(a, b, c) for a in (False, True) for b in (False, True) for c in (False, True)])
@pytest.mark.parametrize("nc", [20, 8, 2, 1])
def test_student_match_loss_switches_vs_float64(nc, ignore_obj, with_bbox, with_cls, smooth):
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    B = 2
    cfg = ssod_cfg(nc)
    cfg.Loss.label_smoothing = smooth
    cfg.SSOD.ignore_obj, cfg.SSOD.pseudo_label_with_bbox, cfg.SSOD.pseudo_label_with_cls = ignore_obj, with_bbox, with_cls
    anchor_t = 5.0 if nc == 8 else 4.0
    cfg.Loss.anchor_t = anchor_t
    crit = ComputeStudentMatchLoss(HeadOnlyModel(nc).to(DEV), cfg)
    r = np.random.RandomState(nc)
    crit.ignore_thres_high = list(r.uniform(0.4, 0.8, nc))
    crit.ignore_thres_low = list(r.uniform(0.05, 0.3, nc))
    logits = _logits(110 + nc, B, nc)
    rows = synth.make_pseudo_rows_dup(100 + nc, 96, B, nc=nc)     # duplicate cells across the routed sets
    p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in logits]
    loss, items = crit(p, torch.from_numpy(rows).to(DEV))
    (loss * 3.0).backward()      # a non-unit upstream gradient (teacher_loss_weight 3): the backward kernels read its scale
    for pi in p:
        pi.grad /= 3.0
    shapes = synth.level_shapes(320)
    sel = port.select_targets(rows, crit.ignore_thres_high, crit.ignore_thres_low, True)
    assert all(len(s) for s in sel)
    sets = [port.build_targets(sel[0][:, :6], synth.ANCHORS_GRID, shapes, anchor_t)]
    sets += [port.build_targets(s, synth.ANCHORS_GRID, shapes, anchor_t, with_score=True) for s in sel[1:]]
    pd = [torch.from_numpy(x).double().requires_grad_(True) for x in logits]
    cp, cn = 1.0 - 0.5 * smooth, 0.5 * smooth
    ref, ref_items = port.det_loss(pd, sets, [4.0, 1.0, 0.4], 0.05, 0.7, 0.3 * nc / 80. * 3. / 3, cp, cn, ignore_obj=ignore_obj,
                                   with_bbox=with_bbox, with_cls=with_cls)
    ref.backward()
    _check_loss([items["ss_" + k] for k in ("box", "obj", "cls")], loss, p, ref_items, ref, pd, nc)
    if nc == 1:
        assert float(items["ss_cls"]) == 0.0


@pytest.mark.parametrize("nc", [2, 1])
def test_loss_reads_only_the_counted_rows_of_a_padded_buffer(nc):
    """the captured steps hand the losses a label buffer of fixed capacity whose first n_dev rows are the labels: stale rows
    past the count (here in-range classes and boxes that would assign) change nothing, supervised and SSOD"""
    from efficientteacher_b200.loss import ComputeLoss
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    B = 2
    cfg = ssod_cfg(nc)
    cfg.single_cls = nc == 1
    logits = _logits(120 + nc, B, nc)
    tg = synth.make_targets(121 + nc, 20, B, nc=nc)
    rows = synth.make_pseudo_rows_dup(122 + nc, 64, B, nc=nc)
    for crit, lab in ((ComputeLoss(HeadOnlyModel(nc).to(DEV), cfg), tg), (ComputeStudentMatchLoss(HeadOnlyModel(nc).to(DEV), cfg), rows)):
        n = len(lab)
        stale = np.concatenate([lab, lab[::-1]], 0)      # capacity 2n
        stale[n:, 0] = stale[n:, 0][::-1]
        got = []
        for buf, n_dev in ((lab, None), (stale, torch.tensor([n], dtype=torch.int32, device=DEV))):
            p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in logits]
            loss, items = crit(p, torch.from_numpy(np.ascontiguousarray(buf)).to(DEV), n_dev)
            loss.backward()
            got.append((loss.item(), [pi.grad.clone() for pi in p]))
        # equal up to the order of the loss kernels' atomic sums (the assignment buffers are sized by the capacity)
        assert abs(got[0][0] - got[1][0]) <= 1e-6 * abs(got[0][0]), (type(crit).__name__, got[0][0], got[1][0])
        for a, b in zip(got[0][1], got[1][1]):
            assert (a - b).abs().max() <= 1e-6 * a.abs().max()
            if nc == 1:
                assert not a[..., 5].any()


# ------------------------------------------------------------------------------------------------ end to end
def _cfg(kind, nc, anchor_t, img, B, da=False):
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    cfg = (yolov5_ssod_cfg if kind == "ssod" else yolov5_sup_cfg)('l_shallow', batch_size=B, img_size=img)
    cfg.Dataset.nc, cfg.Dataset.names, cfg.Loss.anchor_t = nc, [str(i) for i in range(nc)], anchor_t
    if da:               # the Cityscapes config: domain-adaptation losses of both halves, weight 0.1
        cfg.SSOD.with_da_loss, cfg.SSOD.da_loss_weights = True, 0.1
    return cfg


def _ssod_step(nc, anchor_t, img, B, da):
    from efficientteacher_b200.trainer import SSODTrainerStep
    torch.manual_seed(0)
    cfg = _cfg("ssod", nc, anchor_t, img, B, da)
    st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, amp_dtype=torch.bfloat16)
    assert st.model.head.no == nc + 5
    with torch.no_grad():             # a teacher with candidates: objectness ~0.5, class scores ~0.5
        for mm in (st.model, st.ema.ema, st.semi_ema.ema):
            for h in mm.head.m:
                h.bias.view(3, -1)[:, 4] += 6.5
                h.bias.view(3, -1)[:, 5:] += 5.0
    return st, cfg


def _ssod_batch(nc, img, bl, bu):
    r = np.random.RandomState(3)
    imgs = torch.from_numpy(r.rand(bl, 3, img, img).astype(np.float32))
    uw = torch.from_numpy(r.rand(bu, 3, img, img).astype(np.float32))
    return imgs, synth.make_targets(7, 8 * bl, bl, nc=nc), uw.flip(3).contiguous(), uw, synth.make_Ms(9, bu, img)


# VOC at 640; Cityscapes: nc 8, anchor_t 5.0, 960 input, domain-adaptation losses; the custom configs' nc 2
STEP_CASES = [(20, 4.0, 640, False), (8, 5.0, 960, True), (2, 4.0, 256, False)]


@pytest.mark.parametrize("nc,anchor_t,img,da", STEP_CASES)
def test_ssod_step_matches_cpu_step(nc, anchor_t, img, da):
    from oracle.step_ref import CpuSSODStep
    bl = bu = 2
    st, cfg = _ssod_step(nc, anchor_t, img, bl + bu, da)
    cpu = CpuSSODStep({k: v.cpu() for k, v in st.model.state_dict().items()}, (1, 2, 3, 1), 1, batch_size=bl + bu, nc=nc,
                      anchor_t=anchor_t, da_loss_weight=cfg.SSOD.da_loss_weights if da else 0.0)
    imgs, tg, us, uw, Ms = _ssod_batch(nc, img, bl, bu)
    loss = st.train_instance(imgs.to(DEV), torch.from_numpy(tg).to(DEV), us.to(DEV), uw.to(DEV), None, torch.from_numpy(Ms).to(DEV), 0)
    n_pl = int(st.pseudo_label_creator.last_count_dev.item())
    ref_loss, ref_n = cpu.step(imgs, tg, us, uw, Ms)
    assert torch.isfinite(loss).all()
    assert n_pl > 0 and abs(n_pl - ref_n) <= max(3, 0.1 * ref_n), (n_pl, ref_n)
    assert abs(loss.item() - ref_loss) <= 0.05 * abs(ref_loss), (loss.item(), ref_loss)
    assert math.isfinite(ref_loss) and st.ema.updates == 1


@pytest.mark.parametrize("nc,anchor_t,img,da", [(20, 4.0, 256, False), (8, 5.0, 256, True), (2, 4.0, 256, False)])
def test_graphed_ssod_step_matches_eager(nc, anchor_t, img, da):
    """train_instance_graphed (the captured step training runs) against eager launches, with the yardstick of
    test_gpu_engine.test_graphed_step_matches_eager_step: the spread between two eager runs of the same seed"""
    bl = bu = 2
    imgs, tg, us, uw, Ms = [torch.from_numpy(x).to(DEV) if isinstance(x, np.ndarray) else x.to(DEV)
                            for x in _ssod_batch(nc, img, bl, bu)]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        st, _ = _ssod_step(nc, anchor_t, img, bl + bu, da)
        f = st.train_instance_graphed if mode == "graph" else st.train_instance
        losses = [float(f(imgs, tg, us, uw, None, Ms, i).item()) for i in range(3)]
        out[mode] = (losses, {k: v.clone() for k, v in st.ema.ema.state_dict().items()}, st.ema.updates)
    assert out["eager"][2] == out["graph"][2] == out["eager2"][2] == 3
    for i, (a, b, c) in enumerate(zip(out["eager"][0], out["graph"][0], out["eager2"][0])):
        assert abs(a - b) <= 3.0 * abs(a - c) + (0.01 + 0.02 * i) * abs(a), (out["eager"][0], out["graph"][0], out["eager2"][0])
    ke = [k for k, v in out["eager"][1].items() if v.dtype.is_floating_point and "running" not in k]
    a, b, c = (torch.cat([out[m][1][k].flatten() for k in ke]) for m in ("eager", "graph", "eager2"))
    assert ((a - b).norm() / a.norm()).item() <= 3.0 * ((a - c).norm() / a.norm()).item() + 2e-3


@pytest.mark.parametrize("nc,anchor_t,img", [(20, 4.0, 640), (8, 5.0, 320), (2, 4.0, 256)])
def test_supervised_step_matches_cpu_reference(nc, anchor_t, img):
    """SupTrainerStep at these class counts: the native step's loss against the fp32 CPU trunk and port.det_loss (class-loss
    weight 0.3 * nc / 80, the dataset's anchor_t), then the captured step"""
    from efficientteacher_b200.trainer import SupTrainerStep
    from oracle.trunk_ref import TrunkRef
    B = 2
    torch.manual_seed(0)
    st = SupTrainerStep(_cfg("sup", nc, anchor_t, img, B), torch.device(DEV))
    assert st.model.head.no == nc + 5
    sd = {k: v.detach().cpu().clone() for k, v in st.model.state_dict().items()}
    x = torch.rand(B, 3, img, img, generator=torch.Generator().manual_seed(3))
    tg = synth.make_targets(5, 16, B, nc=nc)
    raw, _ = TrunkRef(sd, (1, 2, 3, 1), 1).forward(x, train=True, with_features=False)
    ref, _ = port.det_loss(raw, [port.build_targets(tg, synth.ANCHORS_GRID, synth.level_shapes(img), anchor_t)], [4.0, 1.0, 0.4],
                           0.05, 0.7, 0.3 * nc / 80. * 3. / 3)
    loss = st.train_step(x.to(DEV), torch.from_numpy(tg).to(DEV), 0)
    assert abs(loss.item() - ref.item()) <= 0.03 * abs(ref.item()), (loss.item(), ref.item())
    loss2 = st.train_step_graphed(x.to(DEV), torch.from_numpy(tg).to(DEV), 1)
    assert torch.isfinite(loss2).all() and st.ema.updates == 2


# ------------------------------------------------------------------------------------------------ reference fixtures
@pytest.mark.parametrize("nc", NCS)
def test_kernels_vs_reference_fixtures(golden, nc):
    """the fixtures of the live reference (tests/golden/make_golden_nc.py) reproduced by the kernels: NMS keep-sets, pseudo-label
    rows and multi-label val NMS with and without ties, ComputeLoss and ComputeStudentMatchLoss at every switch setting"""
    from efficientteacher_b200 import nms as N
    from efficientteacher_b200.loss import ComputeLoss
    from efficientteacher_b200.pseudo_label import FairPseudoLabel
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    g = golden(f"class_counts_nc{nc}")
    cfg = ssod_cfg(nc)
    imgs = torch.empty(2, 3, IMG, IMG, device=DEV)
    for ties in (0, 1):
        tp = torch.from_numpy(synth.make_teacher_pred_ties(20 + nc, 2, nc, ties, IMG)).to(DEV)
        dets = N.non_max_suppression_ssod(tp, 0.1, 0.65)
        val = N.non_max_suppression(tp, 0.05, 0.6, multi_label=True)
        for b in range(2):
            assert np.array_equal(dets[b].cpu().numpy(), g[f"t{ties}_det{b}"]), (ties, b)
            assert np.array_equal(val[b].cpu().numpy(), g[f"t{ties}_val{b}"]), (ties, b)
        rows, _ = FairPseudoLabel(cfg).create_pseudo_label_online_with_gt(tp, imgs, torch.from_numpy(synth.make_Ms(30 + nc, 2, IMG)),
                                                                          imgs)
        want = g[f"t{ties}_rows"]
        assert rows.shape == want.shape and np.array_equal(rows.numpy()[:, :2], want[:, :2])
        np.testing.assert_allclose(rows.numpy(), want, rtol=1e-9, atol=1e-9)
    logits = synth.make_head_logits(90 + nc, 2, img=IMG, no=nc + 5)
    tg = torch.from_numpy(synth.make_targets(80 + nc, 24, 2, nc=nc)).to(DEV)
    srows = torch.from_numpy(synth.make_pseudo_rows_dup(100 + nc, 96, 2, nc=nc)).to(DEV)
    hi, lo = synth.make_class_thresholds(nc)
    cfg.single_cls = nc == 1
    for smooth in (0.0, 0.1):
        cfg.Loss.label_smoothing = smooth
        for sw in [None] + SWITCHES:
            p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in logits]
            if sw is None:
                loss, items = ComputeLoss(HeadOnlyModel(nc).to(DEV), cfg)(p, tg)
                keys = ("box", "obj", "cls")
            else:
                cfg.SSOD.ignore_obj, cfg.SSOD.pseudo_label_with_bbox, cfg.SSOD.pseudo_label_with_cls = sw
                crit = ComputeStudentMatchLoss(HeadOnlyModel(nc).to(DEV), cfg)
                crit.ignore_thres_high, crit.ignore_thres_low = list(hi), list(lo)
                loss, items = crit(p, srows)
                keys = ("ss_box", "ss_obj", "ss_cls")
            loss.backward()
            check_loss(g, loss_prefix(smooth, sw), [float(items[k]) for k in keys] + [float(loss.detach())], [pi.grad.cpu().numpy() for pi in p])
