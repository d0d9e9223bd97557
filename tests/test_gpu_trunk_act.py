"""GPU (H100): the ReLU and Hardswish YOLOv5 trunks.

a. The training BatchNorm kernels for ReLU and Hardswish, forward and backward, on pre-activations that land exactly on
   -3, 0 and +3 and one bf16 step on either side (scale 1, shift 0: the kernels' own z is the bf16-exact input), with and
   without the Bottleneck residual, on channel slices of NaN-filled wider buffers; and the same through the batch
   statistics of bn_forward / bn_backward.
b. The teacher engine's folded-BN epilogue with Hardswish (EPI 3).
c. ConvBnActFn (the training Conv module) for a 3x3 and a 1x1 layer per activation: output, dx, dW, dgamma, dbeta.
d. Every trunk mode end to end: the teacher engine against the activation-aware fp32 trunk reference, the supervised and
   the SSOD step against their CPU restatements, and the captured SSOD step against eager launches.
References are float64 on bf16-rounded operands with the tolerances of test_gpu_geometry.py, or the bars of the SiLU
tests in test_gpu_engine.py for the whole-model checks."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_geometry import NAN, _bf, _check_bf16, _check_per_channel, _nchw64, _nhwc, _out_hw, _untouched
from trunk_act_ref import ActCpuSSODStep, ActTrunkRef

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ACTS = ("relu", "hard_swish")
F64 = {"relu": F.relu, "hard_swish": F.hardswish, "silu": F.silu}
MODES = {"relu": ("ReLU", "ReLU"), "default": ("LeakyReLU", "ReLU"), "hswish": ("Hardswish", "Hardswish")}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _dact64(z, act):
    """torch's own derivative (threshold_backward / hardswish_backward) in float64"""
    z = z.detach().double().requires_grad_(True)
    F64[act](z).backward(torch.ones_like(z))
    return z.grad


# ---------------------------------------------------------------------------------------- a. BatchNorm kernels at the kinks
KINKS = torch.tensor([-3.0, 0.0, 3.0])


def _kink_input(N, C_, H, W, seed):
    """bf16-exact pre-activations: every third element is a kink (-3, 0, +3) or one bf16 step (1/64 at |z| = 3, 2^-20 at 0)
    below / above one; the rest N(0, 2.5^2)"""
    y = _bf((N, C_, H, W), seed, 2.5).flatten()
    step = torch.tensor([2.0 ** -6, 2.0 ** -20, 2.0 ** -6])
    pts = torch.cat([KINKS - step, KINKS, KINKS + step])
    idx = torch.arange(0, y.numel(), 3)
    y[idx] = pts[torch.arange(idx.numel()) % pts.numel()]
    assert torch.equal(y, y.to(torch.bfloat16).float())
    return y.view(N, C_, H, W)


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("C_", [32, 64])
@pytest.mark.parametrize("residual", [False, True])
def test_bn_kernels_at_the_kinks(act, C_, residual):
    from efficientteacher_b200 import _lib
    from efficientteacher_b200 import convops as co
    N, H, W = 2, 11, 20
    M = N * H * W
    y = _kink_input(N, C_, H, W, 91)
    r, da = _bf((N, C_, H, W), 92), _bf((N, C_, H, W), 93)
    yo, oo, ro, dao = 8, 16, 24, 8
    ybuf, rbuf, dabuf = _nhwc(y, yo + C_ + 16, yo), _nhwc(r, ro + C_ + 8, ro), _nhwc(da, dao + C_ + 24, dao)
    obuf = torch.full((N, H, W, oo + C_ + 8), NAN, dtype=torch.bfloat16, device=DEV)
    # scale 1, shift 0, mean 0, invstd 1: z = xhat = y
    stats = torch.stack([torch.ones(C_), torch.zeros(C_), torch.zeros(C_), torch.ones(C_)]).to(DEV)
    lib = _lib.lib()
    _lib.check(lib.etb_bn_act_apply_res(_lib.ptr(ybuf[..., yo:]), _lib.ptr(stats[0]), _lib.ptr(stats[1]),
                                        _lib.ptr(rbuf[..., ro:]) if residual else None, _lib.ptr(obuf[..., oo:]), M, C_,
                                        ybuf.shape[3], rbuf.shape[3] if residual else 0, obuf.shape[3], co.ACT[act],
                                        _lib.stream_ptr()), "etb_bn_act_apply_res")
    dybuf = torch.full((N, H, W, C_ + 24), NAN, dtype=torch.bfloat16, device=DEV)
    g0, b0 = _bf((C_,), 94).to(DEV), _bf((C_,), 95).to(DEV)
    dg, db = g0.clone(), b0.clone()
    co.bn_backward(dabuf[..., dao:dao + C_], ybuf[..., yo:yo + C_], C_, stats, act, da_cstride=dabuf.shape[3],
                   y_cstride=ybuf.shape[3], out=dybuf, dgamma_into=dg, dbeta_into=db)
    y64, da64 = y.double(), da.double()
    want = F64[act](y64) + (r.double() if residual else 0.0)
    _check_bf16(_nchw64(obuf, oo, C_), want, "forward")
    _untouched(obuf, oo, C_, "forward")
    dz = da64 * _dact64(y64, act)
    k0, k1 = dz.sum((0, 2, 3)), (dz * y64).sum((0, 2, 3))
    dy = dz - k0.view(1, -1, 1, 1) / M - y64 * k1.view(1, -1, 1, 1) / M
    _check_bf16(_nchw64(dybuf, 0, C_), dy, "backward")
    _untouched(dybuf, 0, C_, "backward")
    for got, base, w, what in ((dg, g0, k1, "dgamma"), (db, b0, k0, "dbeta")):
        d = (got - base).double().cpu()
        assert ((d - w).abs() <= 1e-3 * w.abs().max() + 1e-3 * w.abs()).all(), (what, (d - w).abs().max().item())
    # the kink elements on their own: a wrong one-sided derivative there moves dy by |da| / 2
    kink = torch.isin(y, KINKS)
    assert int(kink.sum()) > 100
    got_dy = _nchw64(dybuf, 0, C_)
    err = (got_dy - dy).abs()[kink]
    assert (err <= dy.abs()[kink] * 2.0 ** -7 + 1e-2 * dy.pow(2).mean().sqrt()).all(), err.max().item()


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("C_", [32, 64])
def test_bn_batch_statistics_nan_poisoned_slices(act, C_):
    """the three-kernel forward (stats, finalize, apply + residual) and backward with batch statistics, for ReLU and
    Hardswish, against float64 autograd of F.batch_norm + the activation"""
    from efficientteacher_b200 import convops as co
    N, H, W, eps, mom = 2, 11, 20, 1e-3, 0.03
    y = (_bf((N, C_, H, W), 81, 2.0) + 0.25).to(torch.bfloat16).float()
    r, da = _bf((N, C_, H, W), 82), _bf((N, C_, H, W), 83)
    gamma = torch.rand(C_, generator=torch.Generator().manual_seed(84)) * 3 + 0.5     # z spans both Hardswish kinks
    beta = torch.randn(C_, generator=torch.Generator().manual_seed(85)) * 0.5
    yo, oo, ro, dao = 8, 16, 24, 8
    ybuf, rbuf, dabuf = _nhwc(y, yo + C_ + 16, yo), _nhwc(r, ro + C_ + 8, ro), _nhwc(da, dao + C_ + 24, dao)
    obuf = torch.full((N, H, W, oo + C_ + 8), NAN, dtype=torch.bfloat16, device=DEV)
    rm, rv = torch.zeros(C_, device=DEV), torch.ones(C_, device=DEV)
    yv = ybuf[..., yo:yo + C_]
    _, stats = co.bn_forward(yv, C_, gamma.to(DEV), beta.to(DEV), rm, rv, eps, mom, act, y_cstride=ybuf.shape[3],
                             out=obuf[..., oo:oo + C_], out_cstride=obuf.shape[3], res=rbuf[..., ro:ro + C_], res_cstride=rbuf.shape[3])
    dybuf = torch.full((N, H, W, C_ + 24), NAN, dtype=torch.bfloat16, device=DEV)
    dy, dg, db = co.bn_backward(dabuf[..., dao:dao + C_], yv, C_, stats, act, da_cstride=dabuf.shape[3], y_cstride=ybuf.shape[3],
                                out=dybuf)
    y64 = y.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm64, rv64 = torch.zeros(C_, dtype=torch.float64), torch.ones(C_, dtype=torch.float64)
    z = F64[act](F.batch_norm(y64, rm64, rv64, g64, b64, True, mom, eps))
    z.backward(da.double())
    _check_bf16(_nchw64(obuf, oo, C_), z.detach() + r.double(), "bn forward")
    _untouched(obuf, oo, C_, "bn forward")
    _check_bf16(_nchw64(dybuf, 0, C_), y64.grad, "bn backward")
    _untouched(dybuf, 0, C_, "bn backward")
    for got, want, what in ((dg, g64.grad, "dgamma"), (db, b64.grad, "dbeta")):
        d = got.double().cpu()
        assert ((d - want).abs() <= 1e-3 * want.abs().max() + 1e-3 * want.abs()).all(), (what, (d - want).abs().max().item())
    torch.testing.assert_close(rm.double().cpu(), rm64, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(rv.double().cpu(), rv64, rtol=1e-4, atol=1e-5)


# ---------------------------------------------------------------------------------------- b. teacher epilogue with Hardswish
@pytest.mark.parametrize("Cin,Cout,k,s", [(64, 72, 3, 1), (96, 64, 3, 2), (32, 24, 1, 1), (128, 136, 3, 1)])
@pytest.mark.parametrize("residual", [False, True])
def test_epilogue_hardswish_nan_poisoned_slices(Cin, Cout, k, s, residual):
    from efficientteacher_b200 import convops as co
    N, H, W, p = 2, 11, 20, k // 2
    Ho, Wo = _out_hw(H, W, k, s, p)
    x = _bf((N, Cin, H, W), 51)
    w = _bf((Cout, Cin, k, k), 52, (Cin * k * k) ** -0.5)
    r = _bf((N, Cout, Ho, Wo), 53)
    scale = torch.rand(Cout, generator=torch.Generator().manual_seed(54)) * 3 + 0.5
    bias = torch.randn(Cout, generator=torch.Generator().manual_seed(55))
    xo, yo, ro = 24, 16, 8
    xbuf, rbuf = _nhwc(x, xo + Cin + 40, xo), _nhwc(r, ro + Cout + 16, ro)
    ybuf = torch.full((N, Ho, Wo, yo + Cout + 24), NAN, dtype=torch.bfloat16, device=DEV)
    co.conv_fwd(xbuf, co.pack_weight(w.to(DEV)), Cin, Cout, k, s, p, scale.to(DEV), bias.to(DEV), act="hard_swish", out=ybuf,
                out_coffset=yo, x_coffset=xo, residual=rbuf if residual else None, res_coffset=ro)
    z = F.conv2d(x.double(), w.double(), None, s, p) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    assert (z < -3).any() and (z > 3).any()
    _check_bf16(_nchw64(ybuf, yo, Cout), F.hardswish(z) + (r.double() if residual else 0.0), "EPI 3")
    _untouched(ybuf, yo, Cout, "EPI 3")


# --------------------------------------------------------------------------------------- c. ConvBnActFn (training Conv)
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("Cin,Cout,k,s", [(64, 128, 3, 2), (128, 64, 1, 1)])
def test_conv_bn_act_fn(act, Cin, Cout, k, s):
    from efficientteacher_b200.model import Conv, native_act
    torch.manual_seed(0)
    m = Conv(Cin, Cout, k, s, act=act).to(DEV).train()
    with torch.no_grad():
        m.bn.weight.copy_(torch.rand(Cout, generator=torch.Generator().manual_seed(3)) * 3 + 0.5)
        m.bn.bias.copy_(torch.randn(Cout, generator=torch.Generator().manual_seed(4)) * 0.5)
    assert native_act(m.act) == act
    N, H, W = 2, 15, 21
    x64 = _bf((N, Cin, H, W), 5).double()
    x = x64.to(DEV, torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_()
    assert m.fused(x)
    a = m(x)
    da = _bf(tuple(a.shape), 6)
    (a * da.to(DEV, torch.bfloat16)).sum().backward()
    # float64 reference on the operands the kernels see: bf16 x and W, the conv output stored in bf16 (the BatchNorm input),
    # and the BatchNorm input gradient stored in bf16 (the dgrad / wgrad operand)
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
    _check_per_channel(m.conv.weight.grad, torch.nn.grad.conv2d_weight(x64, tuple(w64.shape), dy64, stride=s, padding=p), 5e-4, "dW")
    for got, want, what in ((m.bn.weight.grad, g64.grad, "dgamma"), (m.bn.bias.grad, b64.grad, "dbeta")):
        d = got.double().cpu()
        assert ((d - want).abs() <= 1e-3 * want.abs().max() + 1e-3 * want.abs()).all(), (what, (d - want).abs().max().item())


# ------------------------------------------------------------------------------------------------ d. every trunk mode
def _cfg(sup, mode, size="l_shallow", **kw):
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    bb, nk = MODES[mode]
    return (yolov5_sup_cfg if sup else yolov5_ssod_cfg)(size, backbone_act=bb, neck_act=nk, **kw)


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-6)).item()


@pytest.mark.parametrize("mode", list(MODES))
def test_teacher_engine_vs_trunk_reference(mode):
    """criteria of test_teacher_forward_vs_torch_fp32"""
    from efficientteacher_b200.model import Model
    from oracle import port
    import synth
    torch.manual_seed(0)
    m = Model(_cfg(False, mode))
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
        rraw, rfeat = ActTrunkRef.for_model(m).forward(x, train=False)
    for a, b in zip(raw, rraw):
        assert a.shape == b.shape and a.dtype == torch.float32
        assert _rel(a, b) < 0.05, _rel(a, b)
        assert F.cosine_similarity(a.flatten(), b.flatten(), dim=0).item() > 0.999
    for a, b in zip(feat, rfeat):
        assert a.shape == b.shape and _rel(a, b) < 0.06
    want = port.detect_decode([r.cpu() for r in raw], synth.ANCHORS_GRID, synth.STRIDES)
    torch.testing.assert_close(pred.cpu(), want, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("mode", list(MODES))
def test_supervised_step_matches_cpu_reference(mode):
    """bar of test_gpu_engine.test_supervised_step_matches_cpu_reference"""
    from efficientteacher_b200.trainer import SupTrainerStep
    from oracle import port
    import synth
    B, img = 2, 256
    torch.manual_seed(0)
    st = SupTrainerStep(_cfg(True, mode, batch_size=B, img_size=img), torch.device(DEV))
    x = torch.rand(B, 3, img, img, generator=torch.Generator().manual_seed(3))
    tg = synth.make_targets(5, 16, B)
    ref_trunk = ActTrunkRef.for_model(st.model)
    ref_trunk.sd = {k: v.detach().cpu().clone() for k, v in ref_trunk.sd.items()}
    raw, _ = ref_trunk.forward(x, train=True, with_features=False)
    ref, _ = port.det_loss(raw, [port.build_targets(tg, synth.ANCHORS_GRID, synth.level_shapes(img))], [4.0, 1.0, 0.4], 0.05, 0.7, 0.3)
    loss = st.train_step(x.to(DEV), torch.from_numpy(tg).to(DEV), 0)
    assert abs(loss.item() - ref.item()) <= 0.03 * abs(ref.item()), (loss.item(), ref.item())
    loss2 = st.train_step_graphed(x.to(DEV), torch.from_numpy(tg).to(DEV), 1)
    assert torch.isfinite(loss2).all() and st.ema.updates == 2


def _ssod_step(mode, img, bl, bu):
    from efficientteacher_b200.trainer import SSODTrainerStep
    st = SSODTrainerStep(_cfg(False, mode, batch_size=bl + bu, img_size=img), torch.device(DEV), epochs=300)
    with torch.no_grad():          # make the teacher produce candidates: objectness and class scores ~0.5
        for mm in (st.model, st.ema.ema, st.semi_ema.ema):
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


@pytest.mark.parametrize("mode", list(MODES))
def test_ssod_step_matches_cpu_step(mode):
    """bar of test_gpu_engine.test_full_ssod_step_runs_and_matches_cpu_step"""
    img, bl, bu = 256, 2, 2
    torch.manual_seed(0)
    st = _ssod_step(mode, img, bl, bu)
    ref_trunk = ActTrunkRef.for_model(st.model)
    cpu = ActCpuSSODStep({k: v.cpu() for k, v in st.model.state_dict().items()}, ref_trunk.depth, ref_trunk.neck_depth,
                         batch_size=bl + bu, acts=ref_trunk.acts)
    imgs, us, uw, tg, Ms = _ssod_inputs(img, bl, bu)
    loss = st.train_instance(imgs.to(DEV), torch.from_numpy(tg).to(DEV), us.to(DEV), uw.to(DEV), None, torch.from_numpy(Ms).to(DEV), 0)
    n_pl = int(st.pseudo_label_creator.last_count_dev.item())
    ref_loss, ref_n = cpu.step(imgs, tg, us, uw, Ms)
    assert torch.isfinite(loss).all() and st.ema.updates == 1
    assert n_pl > 0 and abs(n_pl - ref_n) <= max(3, 0.1 * ref_n), (n_pl, ref_n)
    assert abs(loss.item() - ref_loss) <= 0.05 * abs(ref_loss), (loss.item(), ref_loss)


def test_graphed_ssod_step_matches_eager_step():
    """test_gpu_engine.test_graphed_step_matches_eager_step on the reference's default trunk (Hardswish backbone, ReLU
    neck): the spread between two eager runs of the same seed is the yardstick"""
    img, bl, bu = 256, 2, 2
    imgs, us, uw, tg, Ms = (t.to(DEV) if torch.is_tensor(t) else torch.from_numpy(t).to(DEV) for t in _ssod_inputs(img, bl, bu))
    out = {}
    for run in ("eager", "eager2", "graph"):
        torch.manual_seed(0)
        st = _ssod_step("default", img, bl, bu)
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
