"""GPU (H100): the YOLOv5 sizes whose widths are not powers of two -- YOLOv5m (48/96/192/384/768) and YOLOv5x
(80/160/320/640/1280) -- and YOLOv5n, on the native training path.

a. Training BatchNorm (stats, finalize, apply with and without the residual, backward reduce / finalize / apply) for
   C/8 not a power of two, each activation, on NaN-filled channel slices, at a small map and at one with many partial
   rows, against float64 with batch statistics; two runs bit-equal.
b. Weight gradient for Cin % 64 != 0 (3x3 s1, 3x3 s2, flat 1x1) with accumulate_into and channel slices; two runs
   bit-equal.
c. The netD tail at C = 1280 (YOLOv5x det_32), forward and backward.
d. ConvBnActFn at YOLOv5m / YOLOv5x layer shapes, and a width-80 Bottleneck with its fused shortcut.
e. Whole models n, m and x: the teacher engine against TrunkRef, the supervised step against its CPU restatement with every
   student Conv on the fused path, the SSOD step against CpuSSODStep, graphed against eager and one burn-in step at
   YOLOv5m width, and one full-depth YOLOv5x SSOD step at 640.
References are float64 on bf16-rounded operands with the tolerances of test_gpu_geometry.py, or the bars of the SiLU
tests in test_gpu_engine.py for the whole-model checks."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_geometry import NAN, _bf, _check_bf16, _check_per_channel, _nchw64, _nhwc, _out_hw, _untouched

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = {"relu": F.relu, "hard_swish": F.hardswish, "silu": F.silu}
M_WIDTHS = [48, 96, 192, 384, 768]
X_WIDTHS = [80, 160, 320, 640, 1280]


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ------------------------------------------------------------------------------------------------- a. BatchNorm kernels
@pytest.mark.parametrize("C_", M_WIDTHS + X_WIDTHS)
@pytest.mark.parametrize("act", ["silu", "relu", "hard_swish"])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("N,H,W", [(2, 11, 20), (4, 40, 64)])
def test_bn_any_width_nan_poisoned_slices(C_, act, residual, N, H, W):
    from efficientteacher_b200 import _lib
    from efficientteacher_b200 import convops as co
    eps, mom = 1e-3, 0.03
    M = N * H * W
    if M > 1000:      # the large map splits the reduction over many blocks: many partial rows for the second stage
        assert _lib.lib().etb_bn_partial_rows(M, C_, 0) >= 8 and _lib.lib().etb_bn_partial_rows(M, C_, 1) >= 8
    y = (_bf((N, C_, H, W), 81, 2.0) + 0.25).to(torch.bfloat16).float()
    r, da = _bf((N, C_, H, W), 82), _bf((N, C_, H, W), 83)
    gamma = torch.rand(C_, generator=torch.Generator().manual_seed(84)) * 3 + 0.5
    beta = torch.randn(C_, generator=torch.Generator().manual_seed(85)) * 0.5
    yo, oo, ro, dao = 8, 16, 24, 8
    ybuf, rbuf, dabuf = _nhwc(y, yo + C_ + 16, yo), _nhwc(r, ro + C_ + 8, ro), _nhwc(da, dao + C_ + 24, dao)
    yv = ybuf[..., yo:yo + C_]
    runs = []
    for _ in range(2):
        obuf = torch.full((N, H, W, oo + C_ + 8), NAN, dtype=torch.bfloat16, device=DEV)
        rm, rv = torch.zeros(C_, device=DEV), torch.ones(C_, device=DEV)
        _, stats = co.bn_forward(yv, C_, gamma.to(DEV), beta.to(DEV), rm, rv, eps, mom, act, y_cstride=ybuf.shape[3],
                                 out=obuf[..., oo:oo + C_], out_cstride=obuf.shape[3],
                                 res=rbuf[..., ro:ro + C_] if residual else None, res_cstride=rbuf.shape[3] if residual else None)
        dybuf = torch.full((N, H, W, C_ + 24), NAN, dtype=torch.bfloat16, device=DEV)
        dy, dg, db = co.bn_backward(dabuf[..., dao:dao + C_], yv, C_, stats, act, da_cstride=dabuf.shape[3],
                                    y_cstride=ybuf.shape[3], out=dybuf)
        runs.append((obuf, dybuf, dg, db, rm, rv, stats))
    for a, b in zip(*runs):                           # fixed reduction order: bit-reproducible
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                           b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))
    obuf, dybuf, dg, db, rm, rv, _ = runs[0]
    y64 = y.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm64, rv64 = torch.zeros(C_, dtype=torch.float64), torch.ones(C_, dtype=torch.float64)
    z = F64[act](F.batch_norm(y64, rm64, rv64, g64, b64, True, mom, eps))
    z.backward(da.double())
    _check_bf16(_nchw64(obuf, oo, C_), z.detach() + (r.double() if residual else 0.0), "bn forward")
    _untouched(obuf, oo, C_, "bn forward")
    _check_bf16(_nchw64(dybuf, 0, C_), y64.grad, "bn backward")
    _untouched(dybuf, 0, C_, "bn backward")
    for got, want, what in ((dg, g64.grad, "dgamma"), (db, b64.grad, "dbeta")):
        d = got.double().cpu()
        assert ((d - want).abs() <= 1e-3 * want.abs().max() + 1e-3 * want.abs()).all(), (what, (d - want).abs().max().item())
    torch.testing.assert_close(rm.double().cpu(), rm64, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(rv.double().cpu(), rv64, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("C_", [8, 2048 + 8])
def test_bn_rejects_widths_outside_the_rule(C_):
    """C/8 <= 256 is the rule: 2056 channels are refused (C = 8 is the smallest accepted width)"""
    from efficientteacher_b200 import _lib
    assert (_lib.lib().etb_bn_partial_rows(1024, C_, 0) > 0) == (C_ == 8)


# ------------------------------------------------------------------------------------------------------ b. weight gradient
def _ref_wgrad(x, dy, Cout, k, s, p):
    return torch.nn.grad.conv2d_weight(x.double(), (Cout, x.shape[1], k, k), dy.double(), stride=s, padding=p)


@pytest.mark.parametrize("Cin", [80, 96, 160, 192, 320])
@pytest.mark.parametrize("k,s", [(3, 1), (3, 2), (1, 1)])
def test_wgrad_partial_channel_chunk(Cin, k, s):
    from efficientteacher_b200 import convops as co
    Cout = {80: 160, 96: 96, 160: 80, 192: 384, 320: 320}[Cin]
    N, H, W, p = 2, 13, 20, k // 2
    Ho, Wo = _out_hw(H, W, k, s, p)
    x = _bf((N, Cin, H, W), 71)
    dy = _bf((N, Cout, Ho, Wo), 72, 0.1)
    xo, do = 16, 8
    xbuf, dybuf = _nhwc(x, xo + Cin + 48, xo), _nhwc(dy, do + Cout + 32, do)
    ref = _ref_wgrad(x, dy, Cout, k, s, p)
    dw1 = co.conv_wgrad(xbuf, dybuf, Cin, Cout, k, s, p, x_coffset=xo, dy_coffset=do)
    dw2 = co.conv_wgrad(xbuf, dybuf, Cin, Cout, k, s, p, x_coffset=xo, dy_coffset=do)
    assert torch.equal(dw1, dw2)
    _check_per_channel(dw1, ref, 5e-4, "wgrad")
    base = _bf((Cout, Cin, k, k), 73).to(DEV)
    g = base.clone()
    out = co.conv_wgrad(xbuf, dybuf, Cin, Cout, k, s, p, x_coffset=xo, dy_coffset=do, accumulate_into=g)
    assert out.data_ptr() == g.data_ptr()
    _check_per_channel(g - base, ref, 5e-4, "wgrad accumulate_into")


# ------------------------------------------------------------------------------------------------------------ c. netD tail
def test_netd_tail_1280_fwd_bwd():
    from efficientteacher_b200 import convops as co
    C_, N, H = 1280, 2, 20
    g = torch.Generator().manual_seed(2)
    hbuf = torch.full((N, H, H, C_ + 16), NAN, dtype=torch.bfloat16, device=DEV)
    hbuf[..., :C_] = torch.relu(torch.randn((N, H, H, C_), generator=g)).to(DEV, torch.bfloat16)
    h = hbuf[..., :C_]
    w2 = (torch.randn((2, C_, 1, 1), generator=g) * C_ ** -0.5).to(DEV)
    o = co.netd_tail_fwd(h, C_, w2, h_cstride=hbuf.shape[3])
    hr = h.double().permute(0, 3, 1, 2).requires_grad_(True)
    w2r = w2.double().requires_grad_(True)
    orf = F.conv2d(hr, w2r)
    torch.testing.assert_close(o.permute(0, 3, 1, 2).double(), orf.detach(), rtol=1e-5, atol=1e-5)
    do = torch.randn((N, H, H, 2), generator=g).to(DEV)
    orf.backward(do.double().permute(0, 3, 1, 2))
    dh, partials = co.netd_tail_bwd(do, h, C_, w2, h_cstride=hbuf.shape[3])
    want_dh = (hr.grad.permute(0, 2, 3, 1) * (h.double() > 0))
    _check_bf16(dh.double(), want_dh, "netD dh")
    dw2 = co.column_sum(partials).view(2, C_)
    torch.testing.assert_close(dw2.double(), w2r.grad.view(2, C_), rtol=1e-4, atol=1e-4)


# --------------------------------------------------------------------------------------- d. ConvBnActFn (training Conv)
def _train_conv(m, Cout, seed, spread=3.0):
    with torch.no_grad():
        m.bn.weight.copy_(torch.rand(Cout, generator=torch.Generator().manual_seed(seed)) * spread + 0.5)
        m.bn.bias.copy_(torch.randn(Cout, generator=torch.Generator().manual_seed(seed + 1)) * 0.5)


# (Cin, Cout, k, s): YOLOv5m stage2_1 / C3 cv1 / cv3 / stage4_1, YOLOv5x stage2_1 / C3 cv1 / Bottleneck cv2 / neck conv1
LAYERS = [(48, 96, 3, 2), (96, 48, 1, 1), (96, 96, 1, 1), (192, 384, 3, 2),
          (80, 160, 3, 2), (160, 80, 1, 1), (80, 80, 3, 1), (1280, 640, 1, 1)]


@pytest.mark.parametrize("Cin,Cout,k,s", LAYERS)
@pytest.mark.parametrize("act", ["silu", "relu"])
def test_conv_bn_act_fn_layer_shapes(Cin, Cout, k, s, act):
    """dW is held to 3e-3 of its channel's largest value, not the wgrad kernel's own 5e-4 (test_wgrad_partial_channel_chunk
    at these Cin): the kernels' BatchNorm input gradient dy is rounded to bf16 from an fp32 computation (and, for SiLU,
    tanh.approx), so a few of its elements land on the neighbouring bf16 value of the float64 reference's, which moves
    the small, cancelling dW channels by up to ~1.5e-3."""
    from efficientteacher_b200.model import Conv
    torch.manual_seed(0)
    m = Conv(Cin, Cout, k, s, act=act).to(DEV).train()
    _train_conv(m, Cout, 3)
    N, H, W = 2, 15, 21
    x64 = _bf((N, Cin, H, W), 5).double()
    x = x64.to(DEV, torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_()
    assert m.fused(x)
    a = m(x)
    da = _bf(tuple(a.shape), 6)
    (a * da.to(DEV, torch.bfloat16)).sum().backward()
    w64 = m.conv.weight.detach().to(torch.bfloat16).double().cpu()
    p = m.conv.padding[0]
    y64 = F.conv2d(x64, w64, None, s, p).to(torch.bfloat16).double().requires_grad_(True)
    g64 = m.bn.weight.detach().double().cpu().requires_grad_(True)
    b64 = m.bn.bias.detach().double().cpu().requires_grad_(True)
    a64 = F64[act](F.batch_norm(y64, None, None, g64, b64, True, 0.0, m.bn.eps))
    a64.backward(da.double())
    dy64 = y64.grad.to(torch.bfloat16).double()
    _check_bf16(a.float(), a64.detach(), "output")
    _check_bf16(x.grad.float(), torch.nn.grad.conv2d_input(tuple(x64.shape), w64, dy64, stride=s, padding=p), "dx")
    _check_per_channel(m.conv.weight.grad, torch.nn.grad.conv2d_weight(x64, tuple(w64.shape), dy64, stride=s, padding=p),
                       3e-3, "dW")
    for got, want, what in ((m.bn.weight.grad, g64.grad, "dgamma"), (m.bn.bias.grad, b64.grad, "dbeta")):
        d = got.double().cpu()
        assert ((d - want).abs() <= 1e-3 * want.abs().max() + 1e-3 * want.abs()).all(), (what, (d - want).abs().max().item())


def test_bottleneck_width_80_fused_shortcut():
    """YOLOv5x's first C3 Bottleneck: cv2's BN apply adds the shortcut, and x's two gradients (cv1 dgrad, shortcut) meet in
    the fan-in of cv1's dgrad epilogue.  Float64 reference through the same bf16 roundings of every stored tensor."""
    from efficientteacher_b200.model import Bottleneck
    C_, N, H, W = 80, 2, 14, 18
    torch.manual_seed(0)
    m = Bottleneck(C_, C_, True, e=1.0).to(DEV).train()
    _train_conv(m.cv1, C_, 11, 1.0)      # gamma <= 1.5: cv1's output feeds a second bf16 conv and BatchNorm
    _train_conv(m.cv2, C_, 13, 1.0)
    x64 = _bf((N, C_, H, W), 7).double()
    x = x64.to(DEV, torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_()
    assert m.cv2.glue(x) and m.add
    a = m(x)
    da = _bf(tuple(a.shape), 8)
    (a * da.to(DEV, torch.bfloat16)).sum().backward()

    def bf16(t):        # the value rounds like the stored bf16 tensor; the gradient passes straight through
        return t + (t.to(torch.bfloat16).double() - t).detach()

    def conv_bn(cv, inp):
        w = cv.conv.weight.detach().to(torch.bfloat16).double().cpu().requires_grad_(True)
        y = bf16(F.conv2d(inp, w, None, 1, cv.conv.padding[0]))       # raw conv output, stored in bf16
        g = cv.bn.weight.detach().double().cpu().requires_grad_(True)
        b = cv.bn.bias.detach().double().cpu().requires_grad_(True)
        return F.silu(F.batch_norm(y, None, None, g, b, True, 0.0, cv.bn.eps)), (w, g, b)

    xr = x64.clone().requires_grad_(True)
    h, p1 = conv_bn(m.cv1, xr)
    out, p2 = conv_bn(m.cv2, bf16(h))
    out = out + xr
    out.backward(da.double())
    _check_bf16(a.float(), out.detach(), "output")
    _check_bf16(x.grad.float(), xr.grad, "dx (fan-in of cv1 dgrad and shortcut)")
    for cv, (w, g, b) in ((m.cv1, p1), (m.cv2, p2)):
        _check_per_channel(cv.conv.weight.grad, w.grad, 2e-2, "dW")
        for got, want, what in ((cv.bn.weight.grad, g.grad, "dgamma"), (cv.bn.bias.grad, b.grad, "dbeta")):
            d, want = got.double().cpu(), want.double()
            assert ((d - want).abs() <= 2e-2 * want.abs().max() + 2e-2 * want.abs()).all(), (what, (d - want).abs().max().item())


# ------------------------------------------------------------------------------------------------------- e. whole models
SIZES = ["n", "m_shallow", "x_shallow"]


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-6)).item()


def _widths(model):
    from efficientteacher_b200.model import Conv
    return {m.conv.out_channels for m in model.modules() if isinstance(m, Conv)}


@pytest.mark.parametrize("size", SIZES)
def test_teacher_engine_vs_trunk_reference(size):
    """criteria of test_teacher_forward_vs_torch_fp32"""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    from oracle import port
    from oracle.trunk_ref import TrunkRef
    import synth
    torch.manual_seed(0)
    m = Model(yolov5_ssod_cfg(size))
    g = torch.Generator().manual_seed(1)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
            mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
            mod.weight.data.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
            mod.bias.data.copy_(torch.randn(mod.bias.shape, generator=g) * 0.1)
    m = m.to(DEV).eval()
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(5)).to(DEV)
    with torch.no_grad():
        (pred, raw), feat = m(x)
        rraw, rfeat = TrunkRef.from_module(m).forward(x, train=False)
    for a, b in zip(raw, rraw):
        assert a.shape == b.shape and a.dtype == torch.float32
        assert _rel(a, b) < 0.05, _rel(a, b)
        assert F.cosine_similarity(a.flatten(), b.flatten(), dim=0).item() > 0.999
    # netD maps: 0.06 of the map's own max|ref|, as in test_teacher_forward_vs_torch_fp32.  A map whose output cancels to
    # under a quarter of the model's largest netD map is held to 0.06 of that largest map instead, plus cosine 0.99: with
    # this seeding YOLOv5x's det_32 (1280 -> 2) peaks at 1.6e-3 while every other map of n / m_shallow / l_shallow /
    # x_shallow peaks at 0.015-0.05, and the pixel-to-pixel spread (~3e-4) -- what the trunk's bf16 error acts on -- is
    # the same in all of them.
    top = max(float(b.abs().max()) for b in rfeat)
    for l, (a, b) in enumerate(zip(feat, rfeat)):
        own = float(b.abs().max())
        err = float((a - b).abs().max())
        cos = F.cosine_similarity(a.flatten(), b.flatten(), dim=0).item()
        scale = own if own >= 0.25 * top else top
        assert a.shape == b.shape and err < 0.06 * scale and cos > 0.99, dict(map=l, err=err, own_max=own, largest_map_max=top, cos=cos)
    want = port.detect_decode([r.cpu() for r in raw], synth.ANCHORS_GRID, synth.STRIDES)
    torch.testing.assert_close(pred.cpu(), want, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("size", SIZES)
def test_supervised_step_all_convs_fused(size, monkeypatch):
    """bar of test_gpu_engine.test_supervised_step_matches_cpu_reference; no student Conv may fall back to the conv-only
    Function plus torch BatchNorm"""
    from efficientteacher_b200.autograd_conv import ConvBnActFn, ConvFn
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.trainer import SupTrainerStep
    from oracle import port
    from oracle.trunk_ref import TrunkRef
    import synth
    B, img = 2, 256
    torch.manual_seed(0)
    st = SupTrainerStep(yolov5_sup_cfg(size, batch_size=B, img_size=img), torch.device(DEV))
    if size != "n":
        assert any((c // 8) & (c // 8 - 1) for c in _widths(st.model))
    calls = {"fused": 0}

    def _unfused(*a, **k):
        raise AssertionError("a student Conv left the fused ConvBnActFn path")

    fused_apply = ConvBnActFn.apply

    def _fused(*a, **k):
        calls["fused"] += 1
        return fused_apply(*a, **k)

    monkeypatch.setattr(ConvFn, "apply", _unfused)
    monkeypatch.setattr(ConvBnActFn, "apply", _fused)
    x = torch.rand(B, 3, img, img, generator=torch.Generator().manual_seed(3))
    tg = synth.make_targets(5, 16, B)
    ref_trunk = TrunkRef.from_module(st.model)
    ref_trunk.sd = {k: v.detach().cpu().clone() for k, v in ref_trunk.sd.items()}
    raw, _ = ref_trunk.forward(x, train=True, with_features=False)
    ref, _ = port.det_loss(raw, [port.build_targets(tg, synth.ANCHORS_GRID, synth.level_shapes(img))], [4.0, 1.0, 0.4], 0.05, 0.7, 0.3)
    loss = st.train_step(x.to(DEV), torch.from_numpy(tg).to(DEV), 0)
    assert calls["fused"] >= len(_convs(st.model))
    assert abs(loss.item() - ref.item()) <= 0.03 * abs(ref.item()), (loss.item(), ref.item())


def _convs(model):
    from efficientteacher_b200.model import Conv
    return [m for m in model.modules() if isinstance(m, Conv)]


def _ssod_step(size, img, bl, bu, burn=0):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep
    cfg = yolov5_ssod_cfg(size, batch_size=bl + bu, img_size=img)
    cfg.hyp.burn_epochs = burn
    st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300)
    with torch.no_grad():          # make the teacher produce candidates: objectness and class scores ~0.5
        for mm in (st.model, st.ema.ema) + ((st.semi_ema.ema,) if st.semi_ema is not None else ()):
            for h in mm.head.m:
                h.bias.view(3, -1)[:, 4] += 6.5
                h.bias.view(3, -1)[:, 5:] += 5.0
    return st


def _ssod_inputs(img, bl, bu):
    import synth
    r = np.random.RandomState(3)
    imgs = torch.from_numpy(r.rand(bl, 3, img, img).astype(np.float32))
    uw = torch.from_numpy(r.rand(bu, 3, img, img).astype(np.float32))
    return imgs, uw.flip(3).contiguous(), uw, synth.make_targets(7, 8 * bl, bl), synth.make_Ms(9, bu, img)


@pytest.mark.parametrize("size", ["m_shallow", "x_shallow"])
def test_ssod_step_matches_cpu_step(size):
    """bar of test_gpu_engine.test_full_ssod_step_runs_and_matches_cpu_step"""
    from oracle.step_ref import CpuSSODStep
    from oracle.trunk_ref import TrunkRef
    img, bl, bu = 256, 2, 2
    torch.manual_seed(0)
    st = _ssod_step(size, img, bl, bu)
    r = TrunkRef.from_module(st.model)
    cpu = CpuSSODStep({k: v.cpu() for k, v in st.model.state_dict().items()}, r.depth, r.neck_depth, batch_size=bl + bu)
    imgs, us, uw, tg, Ms = _ssod_inputs(img, bl, bu)
    loss = st.train_instance(imgs.to(DEV), torch.from_numpy(tg).to(DEV), us.to(DEV), uw.to(DEV), None, torch.from_numpy(Ms).to(DEV), 0)
    n_pl = int(st.pseudo_label_creator.last_count_dev.item())
    ref_loss, ref_n = cpu.step(imgs, tg, us, uw, Ms)
    assert torch.isfinite(loss).all() and st.ema.updates == 1
    assert n_pl > 0 and abs(n_pl - ref_n) <= max(3, 0.1 * ref_n), (n_pl, ref_n)
    assert abs(loss.item() - ref_loss) <= 0.05 * abs(ref_loss), (loss.item(), ref_loss)


def test_graphed_ssod_step_matches_eager_step_yolov5m():
    """test_gpu_engine.test_graphed_step_matches_eager_step at YOLOv5m width: the spread between two eager runs of the
    same seed is the yardstick"""
    img, bl, bu = 256, 2, 2
    imgs, us, uw, tg, Ms = (t.to(DEV) if torch.is_tensor(t) else torch.from_numpy(t).to(DEV) for t in _ssod_inputs(img, bl, bu))
    out = {}
    for run in ("eager", "eager2", "graph"):
        torch.manual_seed(0)
        st = _ssod_step("m_shallow", img, bl, bu)
        f = st.train_instance_graphed if run == "graph" else st.train_instance
        losses = [float(f(imgs, tg, us, uw, None, Ms, i).item()) for i in range(3)]
        out[run] = (losses, {k: v.clone() for k, v in st.ema.ema.state_dict().items()}, st.ema.updates)
    assert out["eager"][2] == out["graph"][2] == out["eager2"][2] == 3
    for i, (a, b, c) in enumerate(zip(out["eager"][0], out["graph"][0], out["eager2"][0])):
        assert abs(a - b) <= 3.0 * abs(a - c) + (0.01 + 0.02 * i) * abs(a), (out["eager"][0], out["graph"][0], out["eager2"][0])
    ke = [k for k, v in out["eager"][1].items() if v.dtype.is_floating_point and "running" not in k]
    a, b, c = (torch.cat([out[r][1][k].flatten() for k in ke]) for r in ("eager", "graph", "eager2"))
    rel, rel_eager = ((a - b).norm() / a.norm()).item(), ((a - c).norm() / a.norm()).item()
    assert rel <= 3.0 * rel_eager + 2e-3, (rel, rel_eager)


def test_burn_in_step_yolov5m_matches_cpu_step():
    """bar of test_gpu_burnin.test_burn_in_step_matches_cpu_step"""
    from burnin_ref import CpuBurnInStep
    from oracle.trunk_ref import TrunkRef
    import synth
    img, bl = 256, 2
    torch.manual_seed(0)
    st = _ssod_step("m_shallow", img, bl, 0, burn=2)
    r = TrunkRef.from_module(st.model)
    cpu = CpuBurnInStep({k: v.detach().cpu().clone() for k, v in st.model.state_dict().items()}, r.depth, r.neck_depth,
                        st.cfg.hyp.burn_epochs, da_loss_weights=st.cfg.SSOD.da_loss_weights, batch_size=st.batch_size,
                        warmup=(st.nw, st.warmup_bias_lr, st.warmup_momentum), fixed_accumulate=False)
    imgs = torch.from_numpy(np.random.RandomState(3).rand(bl, 3, img, img).astype(np.float32))
    tg = synth.make_targets(7, 8 * bl, bl)
    loss = st.train_without_unlabeled(imgs.to(DEV), torch.from_numpy(tg).to(DEV), 0)
    ref = cpu.burn_in_step(imgs, tg, None)
    assert abs(loss.item() - ref) <= 0.03 * abs(ref), (loss.item(), ref)
    assert st.ema.updates == 1 and st.in_burn_in


def test_full_yolov5x_ssod_step_640():
    """the whole YOLOv5x (depth 1.33, width 1.25: det_32 has 1280 channels) at 640, 2 labeled + 2 unlabeled images"""
    img, bl, bu = 640, 2, 2
    torch.manual_seed(0)
    st = _ssod_step("x", img, bl, bu)
    assert st.model.det_32.conv1.weight.shape[0] == 1280
    imgs, us, uw, tg, Ms = (t.to(DEV) if torch.is_tensor(t) else torch.from_numpy(t).to(DEV) for t in _ssod_inputs(img, bl, bu))
    loss = st.train_instance(imgs, tg, us, uw, None, Ms, 0)
    assert torch.isfinite(loss).all() and st.ema.updates == 1
    items = [v for d in (st.last["sup"], st.last["unsup"]) for v in d.values()]
    assert all(bool(torch.isfinite(torch.as_tensor(v)).all()) for v in items), st.last
    assert int(st.pseudo_label_creator.last_count_dev.item()) > 0
    assert all(torch.isfinite(p).all() for p in st.model.parameters())
    loss = st.train_instance(imgs, tg, us, uw, None, Ms, 1, _stop_after_backward=True)
    assert torch.isfinite(loss).all()
    grads = [p.grad for p in st.model.parameters() if p.requires_grad]
    assert all(g is not None for g in grads)
    assert all(torch.isfinite(g).all() for g in grads)
    assert sum(float(g.abs().sum()) > 0 for g in grads) > 0.9 * len(grads)
