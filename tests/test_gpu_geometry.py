"""GPU (H100): the wgmma convolution (forward EPI 0/1/2, dgrad, wgrad), the training BatchNorm kernels, the teacher engine
and the validation batch on the geometries the square, even, contiguous cases of test_gpu_conv.py / test_gpu_engine.py
leave out: non-square maps and their transposes, odd inputs to stride-2 convs, maps of 1-4 pixels, Cout values that leave
dead accumulator columns, a persistent grid that wraps with a partial last round, operands that are channel slices of
wider NaN-filled buffers, and letterboxed (non-square) batches through the engine and val_batch.

One reference discipline: operands are rounded to bf16 first and the reference is the same operation in float64 on the
CPU.  Tolerances are per element: bf16 outputs must satisfy |got - ref| <= 2^-7 |ref| + 1e-2 rms(ref) (bf16 rounding plus
a floor far below one missing filter tap); fp32 weight gradients are checked per output channel against that channel's
max |ref|."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAN = float("nan")


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)
    # the torch trunk reference of the engine tests runs on the GPU in fp32: keep cuDNN / cuBLAS off TF32 for this module
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---------------------------------------------------------------------------------------------------------------- helpers
def _bf(shape, seed, scale=1.0):
    """bf16-exact fp32 CPU tensor"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).float()


def _nhwc(x_nchw, width=None, coffset=0, fill=NAN):
    """[N,C,H,W] bf16-exact -> NHWC bf16 on the GPU, channels [coffset, coffset+C) of a `width`-channel buffer whose other
    channels hold `fill`"""
    N, C_, H, W = x_nchw.shape
    width = C_ if width is None else width
    buf = torch.full((N, H, W, width), fill, dtype=torch.bfloat16, device=DEV)
    buf[..., coffset:coffset + C_] = x_nchw.permute(0, 2, 3, 1).to(DEV, torch.bfloat16)
    return buf


def _nan_nhwc(N, H, W, C_):
    return torch.full((N, H, W, C_), NAN, dtype=torch.bfloat16, device=DEV)


def _nchw64(buf, coffset, C_):
    return buf[..., coffset:coffset + C_].permute(0, 3, 1, 2).double().cpu()


def _check_bf16(got, ref, what=""):
    """per element: |got - ref| <= 2^-7 |ref| + 1e-2 rms(ref); got must be finite"""
    got, ref = got.double().cpu(), ref.double().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    rms = ref.pow(2).mean().sqrt().item()
    tol = ref.abs() * 2.0 ** -7 + 1e-2 * rms
    err = (got - ref).abs()
    bad = ~(err <= tol)                     # NaN / Inf count as bad
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        pytest.fail("%s: %d/%d elements off, first at %s: got %r want %r (rms %.3g)" % (
            what, int(bad.sum()), bad.numel(), i, got[i].item(), ref[i].item(), rms))


def _check_per_channel(got, ref, tol, what=""):
    """fp32 result: every element within tol * max|ref| of its output channel (dim 0)"""
    got, ref = got.double().cpu(), ref.double().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), what
    scale = ref.abs().flatten(1).amax(1).clamp_min(1e-30).view(-1, *([1] * (ref.dim() - 1)))
    rel = ((got - ref).abs() / scale).flatten(1).amax(1)
    worst = int(rel.argmax())
    assert rel.max().item() <= tol, (what, "channel", worst, rel.max().item())


def _untouched(buf, coffset, C_, what=""):
    """every channel of buf outside [coffset, coffset+C) is still NaN"""
    keep = torch.ones(buf.shape[3], dtype=torch.bool, device=buf.device)
    keep[coffset:coffset + C_] = False
    assert torch.isnan(buf[..., keep].float()).all(), what + ": a channel outside the written slice was overwritten"


def _out_hw(H, W, k, s, p):
    return (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1


def _ref_fwd(x, w, s, p):
    return F.conv2d(x.double(), w.double(), None, s, p)


# -------------------------------------------------------------------------------------------------- a. forward geometry
FWD_CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 48, 80, 72, 3, 1, 1),      # 10 x 3 tiles of 8x16: tiles_w != tiles_h
    (2, 64, 80, 48, 136, 3, 1, 1),     # transpose; Cout 136 = one full + one 8-wide BN=128 tile
    (2, 32, 12, 20, 24, 3, 1, 1),
    (2, 96, 20, 12, 8, 3, 1, 1),       # Cout 8: 56 dead columns of a BN=64 tile
    (2, 64, 7, 11, 136, 3, 1, 1),
    (2, 128, 11, 7, 72, 3, 1, 1),      # Cout 72: BN switches to 128, 56 dead columns
    (2, 64, 11, 20, 64, 3, 1, 1),
    (2, 32, 20, 11, 24, 3, 1, 1),
    (3, 64, 1, 5, 72, 3, 1, 1),
    (3, 64, 5, 1, 8, 3, 1, 1),
    (2, 128, 1, 1, 136, 3, 1, 1),
    (2, 64, 2, 2, 64, 3, 1, 1),
    (2, 64, 3, 1, 24, 3, 1, 1),
    (2, 64, 15, 21, 72, 3, 2, 1),      # odd input, stride 2 -> 8 x 11
    (2, 32, 21, 15, 136, 3, 2, 1),     # -> 11 x 8
    (2, 64, 3, 3, 64, 3, 2, 1),        # -> 2 x 2
    (2, 128, 1, 1, 8, 3, 2, 1),        # -> 1 x 1
    (3, 96, 7, 11, 72, 1, 1, 0),       # flat pointwise, 231 pixels: ragged last 128-row tile
    (4, 64, 90, 100, 136, 1, 1, 0),    # flat: 282 x 2 = 564 tiles on a 132-CTA persistent grid, partial last round
    (3, 32, 96, 160, 24, 3, 1, 1),     # 3 x 120 = 360 tiles of 4x32: the ring wraps, 360 % 132 != 0
]


def _fwd_tiles(N, H, W, Cout, k, s, p):
    """tile count of the forward launch (pick_tile restated): used to assert the wrap cases really wrap"""
    Ho, Wo = _out_hw(H, W, k, s, p)
    bn = 128 if Cout > 64 else 64
    ntiles = -(-Cout // bn)
    if k == 1 and s == 1 and p == 0:
        return -(-(N * H * W) // 128) * ntiles
    best, tiles = -1.0, None
    for tw in range(1, 129):
        if tw > Wo and tw != 1:
            break
        th = min(128 // tw, Ho)
        t = -(-Wo // tw) * -(-Ho // th)
        eff = Wo * Ho / (t * 128.0)
        if eff > best + 1e-9:
            best, tiles = eff, t
    return tiles * N * ntiles


def test_forward_cases_wrap_the_persistent_grid():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    wraps = [c for c in FWD_CASES if _fwd_tiles(c[0], c[2], c[3], c[4], c[5], c[6], c[7]) > 2 * sms
             and _fwd_tiles(c[0], c[2], c[3], c[4], c[5], c[6], c[7]) % sms]
    assert len(wraps) >= 2, [(c, _fwd_tiles(c[0], c[2], c[3], c[4], c[5], c[6], c[7])) for c in FWD_CASES]


@pytest.mark.parametrize("case", FWD_CASES)
def test_forward_geometry(case):
    """EPI 0 (raw bf16) and EPI 1 (folded BN scale/bias -> SiLU -> + residual) on the same operands"""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = _out_hw(H, W, k, s, p)
    x = _bf((N, Cin, H, W), 1)
    w = _bf((Cout, Cin, k, k), 2, (Cin * k * k) ** -0.5)
    r = _bf((N, Cout, Ho, Wo), 3)
    scale = torch.rand(Cout, generator=torch.Generator().manual_seed(4)) + 0.5
    bias = torch.randn(Cout, generator=torch.Generator().manual_seed(5)) * 0.1
    xb, wp = _nhwc(x), co.pack_weight(w.to(DEV))
    acc = _ref_fwd(x, w, s, p)
    # outputs start as NaN, so a pixel the kernel never stores cannot pass by holding a stale copy of the right value
    y0 = co.conv_fwd(xb, wp, Cin, Cout, k, s, p, None, None, act=None, out=_nan_nhwc(N, Ho, Wo, Cout))
    _check_bf16(_nchw64(y0, 0, Cout), acc, "EPI 0")
    y1 = co.conv_fwd(xb, wp, Cin, Cout, k, s, p, scale.to(DEV), bias.to(DEV), act="silu", residual=_nhwc(r), out=_nan_nhwc(N, Ho, Wo, Cout))
    z = acc * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    _check_bf16(_nchw64(y1, 0, Cout), F.silu(z) + r.double(), "EPI 1")


@pytest.mark.parametrize("N,Cin,H,W", [(3, 128, 11, 20), (2, 64, 20, 11), (1, 256, 7, 5)])
def test_detect_scatter_non_square(N, Cin, H, W):
    """EPI 2: 1x1 conv + bias scattered as fp32 [N, 3, ny, nx, 85] with ny != nx (yolov5_head.py:66)"""
    from efficientteacher_b200 import convops as co
    no = 85
    x = _bf((N, Cin, H, W), 6)
    w = _bf((3 * no, Cin, 1, 1), 7, Cin ** -0.5)
    b = torch.randn(3 * no, generator=torch.Generator().manual_seed(8))
    out = torch.full((N, 3, H, W, no), NAN, dtype=torch.float32, device=DEV)
    co.conv_fwd(_nhwc(x), co.pack_weight(w.to(DEV)), Cin, 3 * no, 1, 1, 0, None, b.to(DEV), act=None, det_out=out, det_no=no)
    ref = (_ref_fwd(x, w, 1, 0) + b.double().view(1, -1, 1, 1)).view(N, 3, no, H, W).permute(0, 1, 3, 4, 2)
    got = out.double().cpu()
    assert torch.isfinite(got).all()
    tol = 1e-5 * ref.abs() + 1e-5 * ref.pow(2).mean().sqrt()
    assert ((got - ref).abs() <= tol).all(), (got - ref).abs().max().item()


# ------------------------------------------------------------------------------------------------------------- b. dgrad
DGRAD_CASES = [
    # N, Cin, H, W, Cout, k, s, p   (Cin = channels of dx, Cout = the dgrad reduction)
    (2, 64, 48, 80, 72, 3, 1, 1),
    (2, 72, 80, 48, 64, 3, 1, 1),
    (2, 32, 11, 20, 24, 3, 1, 1),
    (2, 64, 7, 11, 8, 3, 1, 1),
    (2, 64, 2, 2, 64, 3, 1, 1),
    (2, 64, 15, 21, 64, 3, 2, 1),      # odd H and W: parity classes of 8x11, 8x10, 7x11, 7x10 pixels
    (2, 136, 21, 15, 32, 3, 2, 1),
    (2, 64, 1, 5, 64, 3, 2, 1),        # H = 1: the ph = 1 classes are empty
    (2, 64, 5, 1, 128, 3, 2, 1),       # W = 1: the pw = 1 classes are empty
    (2, 64, 1, 1, 64, 3, 2, 1),        # one pixel: only class (0,0)
    (2, 24, 3, 3, 64, 3, 2, 1),
    (2, 64, 12, 20, 96, 3, 2, 1),      # even, non-square
    (3, 96, 7, 11, 72, 1, 1, 0),       # flat
]


@pytest.mark.parametrize("case", DGRAD_CASES)
def test_dgrad_geometry(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = _out_hw(H, W, k, s, p)
    dy = _bf((N, Cout, Ho, Wo), 21)
    w = _bf((Cout, Cin, k, k), 22, (Cout * k * k) ** -0.5)
    base = _bf((N, Cin, H, W), 23)
    wd = co.pack_weight_dgrad(w.to(DEV), s, p)
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), stride=s, padding=p)
    dx = co.conv_dgrad(_nhwc(dy), wd, N, H, W, Cin, Cout, k, s, p, out=_nan_nhwc(N, H, W, Cin))
    _check_bf16(_nchw64(dx, 0, Cin), ref, "dgrad")
    buf = _nhwc(base)
    co.conv_dgrad(_nhwc(dy), wd, N, H, W, Cin, Cout, k, s, p, out=buf, accumulate=True)
    _check_bf16(_nchw64(buf, 0, Cin), ref + base.double(), "dgrad accumulate")


# ------------------------------------------------------------------------------------------------------------- c. wgrad
WGRAD_CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 48, 80, 72, 3, 1, 1),
    (2, 32, 80, 48, 24, 3, 1, 1),
    (2, 128, 11, 20, 136, 3, 1, 1),
    (2, 64, 7, 11, 8, 3, 1, 1),
    (2, 64, 15, 21, 64, 3, 2, 1),
    (2, 32, 21, 15, 128, 3, 2, 1),
    (3, 64, 7, 11, 72, 1, 1, 0),       # flat, ragged
    # output maps of at most 3 pixels: the K-tile plan's fallback box
    (2, 64, 1, 1, 64, 3, 1, 1),        # 1x1
    (2, 128, 2, 2, 72, 3, 2, 1),       # 3x3 s2 on a 2x2 map -> 1x1
    (2, 64, 4, 2, 64, 3, 2, 1),        # Wo x Ho = 1x2
    (2, 32, 5, 1, 24, 3, 2, 1),        # 1x3
    (2, 64, 2, 4, 64, 3, 2, 1),        # 2x1
    (2, 64, 1, 3, 136, 3, 1, 1),       # 3x1
]


def _ref_wgrad(x, dy, Cout, k, s, p):
    return torch.nn.grad.conv2d_weight(x.double(), (Cout, x.shape[1], k, k), dy.double(), stride=s, padding=p)


@pytest.mark.parametrize("case", WGRAD_CASES)
def test_wgrad_geometry(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = _out_hw(H, W, k, s, p)
    x = _bf((N, Cin, H, W), 31)
    dy = _bf((N, Cout, Ho, Wo), 32, 0.1)
    ref = _ref_wgrad(x, dy, Cout, k, s, p)
    xb, dyb = _nhwc(x), _nhwc(dy, (Cout + 7) // 8 * 8, 0, 0.0)
    dw = co.conv_wgrad(xb, dyb, Cin, Cout, k, s, p)
    _check_per_channel(dw, ref, 5e-4, "wgrad")
    base = _bf((Cout, Cin, k, k), 33).to(DEV)
    g = base.clone()
    out = co.conv_wgrad(xb, dyb, Cin, Cout, k, s, p, accumulate_into=g)
    assert out.data_ptr() == g.data_ptr()
    _check_per_channel(g - base, ref, 5e-4, "wgrad accumulate_into")


def test_wgrad_non_square_deterministic():
    """the split-K partials are summed in a fixed order: two runs agree bit for bit (non-square 11x20 map, wide layer)"""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = 4, 256, 11, 20, 256, 3, 1, 1
    x, dy = _bf((N, Cin, H, W), 41), _bf((N, Cout, H, W), 42, 0.1)
    xb, dyb = _nhwc(x), _nhwc(dy)
    dw1 = co.conv_wgrad(xb, dyb, Cin, Cout, k, s, p)
    dw2 = co.conv_wgrad(xb, dyb, Cin, Cout, k, s, p)
    assert torch.equal(dw1, dw2)
    _check_per_channel(dw1, _ref_wgrad(x, dy, Cout, k, s, p), 5e-4, "wgrad")


# ---------------------------------------------------------------------------------------- d. NaN-poisoned channel slices
# every operand lives in a channel slice of a wider buffer whose other channels are NaN: a box that read past the logical
# channel count would multiply NaN by the zero-padded weights; a store outside the slice would overwrite a NaN
@pytest.mark.parametrize("Cin,Cout,k,s", [(64, 72, 3, 1), (96, 64, 3, 2), (32, 24, 1, 1), (128, 136, 3, 1)])
def test_forward_nan_poisoned_slices(Cin, Cout, k, s):
    from efficientteacher_b200 import convops as co
    N, H, W, p = 2, 11, 20, k // 2
    Ho, Wo = _out_hw(H, W, k, s, p)
    x = _bf((N, Cin, H, W), 51)
    w = _bf((Cout, Cin, k, k), 52, (Cin * k * k) ** -0.5)
    r = _bf((N, Cout, Ho, Wo), 53)
    scale = torch.rand(Cout, generator=torch.Generator().manual_seed(54)) + 0.5
    bias = torch.randn(Cout, generator=torch.Generator().manual_seed(55)) * 0.1
    xo, yo, ro = 24, 16, 8
    xbuf = _nhwc(x, xo + Cin + 40, xo)
    rbuf = _nhwc(r, ro + Cout + 16, ro)
    wp = co.pack_weight(w.to(DEV))
    acc = _ref_fwd(x, w, s, p)
    for epi in (0, 1):
        ybuf = torch.full((N, Ho, Wo, yo + Cout + 24), NAN, dtype=torch.bfloat16, device=DEV)
        if epi == 0:
            co.conv_fwd(xbuf, wp, Cin, Cout, k, s, p, None, None, act=None, out=ybuf, out_coffset=yo, x_coffset=xo)
            ref = acc
        else:
            co.conv_fwd(xbuf, wp, Cin, Cout, k, s, p, scale.to(DEV), bias.to(DEV), act="silu", out=ybuf, out_coffset=yo, x_coffset=xo,
                        residual=rbuf, res_coffset=ro)
            ref = F.silu(acc * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)) + r.double()
        _check_bf16(_nchw64(ybuf, yo, Cout), ref, "EPI %d" % epi)
        _untouched(ybuf, yo, Cout, "EPI %d" % epi)


@pytest.mark.parametrize("Cin,Cout,k,s", [(64, 64, 3, 2), (32, 96, 3, 1), (136, 128, 1, 1), (72, 32, 3, 2)])
def test_dgrad_nan_poisoned_slices(Cin, Cout, k, s):
    from efficientteacher_b200 import convops as co
    N, H, W, p = 2, 15, 20, k // 2
    Ho, Wo = _out_hw(H, W, k, s, p)
    dy = _bf((N, Cout, Ho, Wo), 61)
    w = _bf((Cout, Cin, k, k), 62, (Cout * k * k) ** -0.5)
    do, xo = 8, 16
    dybuf = _nhwc(dy, do + Cout + 24, do)
    dxbuf = torch.full((N, H, W, xo + Cin + 8), NAN, dtype=torch.bfloat16, device=DEV)
    co.conv_dgrad(dybuf, co.pack_weight_dgrad(w.to(DEV), s, p), N, H, W, Cin, Cout, k, s, p, out=dxbuf, out_coffset=xo, dy_coffset=do)
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), stride=s, padding=p)
    _check_bf16(_nchw64(dxbuf, xo, Cin), ref, "dgrad")
    _untouched(dxbuf, xo, Cin, "dgrad")


@pytest.mark.parametrize("Cin,Cout,k,s", [(64, 72, 3, 1), (128, 64, 3, 2), (32, 24, 3, 1), (32, 136, 1, 1)])
def test_wgrad_nan_poisoned_slices(Cin, Cout, k, s):
    from efficientteacher_b200 import convops as co
    N, H, W, p = 2, 11, 20, k // 2
    Ho, Wo = _out_hw(H, W, k, s, p)
    x = _bf((N, Cin, H, W), 71)
    dy = _bf((N, Cout, Ho, Wo), 72, 0.1)
    xo, do = 16, 8
    xbuf, dybuf = _nhwc(x, xo + Cin + 48, xo), _nhwc(dy, do + Cout + 32, do)
    dw = co.conv_wgrad(xbuf, dybuf, Cin, Cout, k, s, p, x_coffset=xo, dy_coffset=do)
    _check_per_channel(dw, _ref_wgrad(x, dy, Cout, k, s, p), 5e-4, "wgrad")


@pytest.mark.parametrize("C_", [32, 64])
def test_bn_nan_poisoned_slices(C_):
    """training BatchNorm + SiLU forward (y / out / residual slices) and backward (da / y slices, dy into a wider buffer,
    dgamma / dbeta added into existing gradients) against float64 autograd of F.batch_norm"""
    from efficientteacher_b200 import convops as co
    N, H, W, eps, mom = 2, 11, 20, 1e-3, 0.03
    y = _bf((N, C_, H, W), 81, 2.0) + 0.25
    y = y.to(torch.bfloat16).float()
    r, da = _bf((N, C_, H, W), 82), _bf((N, C_, H, W), 83)
    gamma = torch.rand(C_, generator=torch.Generator().manual_seed(84)) + 0.5
    beta = torch.randn(C_, generator=torch.Generator().manual_seed(85)) * 0.1
    yo, oo, ro, dao = 8, 16, 24, 8
    ybuf, rbuf, dabuf = _nhwc(y, yo + C_ + 16, yo), _nhwc(r, ro + C_ + 8, ro), _nhwc(da, dao + C_ + 24, dao)
    obuf = torch.full((N, H, W, oo + C_ + 8), NAN, dtype=torch.bfloat16, device=DEV)
    rm, rv = torch.zeros(C_, device=DEV), torch.ones(C_, device=DEV)
    yv = ybuf[..., yo:yo + C_]
    a, stats = co.bn_forward(yv, C_, gamma.to(DEV), beta.to(DEV), rm, rv, eps, mom, "silu", y_cstride=ybuf.shape[3],
                             out=obuf[..., oo:oo + C_], out_cstride=obuf.shape[3], res=rbuf[..., ro:ro + C_], res_cstride=rbuf.shape[3])
    dybuf = torch.full((N, H, W, C_ + 24), NAN, dtype=torch.bfloat16, device=DEV)
    g0, b0 = _bf((C_,), 86).to(DEV), _bf((C_,), 87).to(DEV)
    dg, db = g0.clone(), b0.clone()
    out, none1, none2 = co.bn_backward(dabuf[..., dao:dao + C_], yv, C_, stats, "silu", da_cstride=dabuf.shape[3], y_cstride=ybuf.shape[3],
                                       out=dybuf, dgamma_into=dg, dbeta_into=db)
    assert out.data_ptr() == dybuf.data_ptr() and none1 is None and none2 is None
    # float64 reference
    y64 = y.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    rm64, rv64 = torch.zeros(C_, dtype=torch.float64), torch.ones(C_, dtype=torch.float64)
    z = F.silu(F.batch_norm(y64, rm64, rv64, g64, b64, True, mom, eps))
    z.backward(da.double())
    _check_bf16(_nchw64(obuf, oo, C_), z.detach() + r.double(), "bn forward")
    _untouched(obuf, oo, C_, "bn forward")
    _check_bf16(_nchw64(dybuf, 0, C_), y64.grad, "bn backward")
    _untouched(dybuf, 0, C_, "bn backward")
    for got, base, want, what in ((dg, g0, g64.grad, "dgamma"), (db, b0, b64.grad, "dbeta")):
        d = (got - base).double().cpu()
        assert torch.isfinite(d).all(), what
        assert ((d - want).abs() <= 1e-3 * want.abs().max() + 1e-3 * want.abs()).all(), (what, (d - want).abs().max().item())
    torch.testing.assert_close(rm.double().cpu(), rm64, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(rv.double().cpu(), rv64, rtol=1e-4, atol=1e-5)


# -------------------------------------------------------------------------------- e. teacher engine on letterboxed batches
def _model(size, seed=0, obj_bias=0.0, cls_bias=0.0):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(seed)
    m = Model(yolov5_ssod_cfg(size))
    g = torch.Generator().manual_seed(seed + 1)
    for mod in m.modules():          # non-trivial BN statistics so the folding is exercised
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
            mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
            mod.weight.data.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
            mod.bias.data.copy_(torch.randn(mod.bias.shape, generator=g) * 0.1)
    with torch.no_grad():
        for h in m.head.m:
            h.bias.view(3, -1)[:, 4] += obj_bias
            h.bias.view(3, -1)[:, 5:] += cls_bias
    return m.to(DEV).eval()


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-6)).item()


@pytest.mark.parametrize("size", ["l_shallow", "s"])
@pytest.mark.parametrize("H,W", [(224, 352), (352, 224)])
def test_teacher_engine_letterboxed(size, H, W):
    """maps 28x44 / 14x22 / 7x11 and their transposes; same criteria as test_teacher_forward_vs_torch_fp32"""
    from oracle.trunk_ref import TrunkRef
    from oracle import port
    import synth
    m = _model(size)
    x = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(5)).to(DEV)
    with torch.no_grad():
        (pred, raw), feat = m(x)
        rraw, rfeat = TrunkRef.from_module(m).forward(x, train=False)
    for a, b, st in zip(raw, rraw, synth.STRIDES):
        assert a.shape == b.shape == (2, 3, H // st, W // st, 85) and a.dtype == torch.float32
        assert _rel(a, b) < 0.05, _rel(a, b)
        cos = F.cosine_similarity(a.flatten(), b.flatten(), dim=0).item()
        assert cos > 0.999, cos
    for a, b in zip(feat, rfeat):
        assert a.shape == b.shape and _rel(a, b) < 0.06
    want = port.detect_decode([r.cpu() for r in raw], synth.ANCHORS_GRID, synth.STRIDES)
    assert pred.shape == want.shape
    torch.testing.assert_close(pred.cpu(), want, rtol=1e-5, atol=1e-4)


# ------------------------------------------------------------------------------------------ f. val_batch end to end
def _scale_coords(img1_shape, coords, img0_shape, ratio_pad):
    """utils/general.py:702-715 semantics on an fp32 [n,4] xyxy tensor: remove the letterbox pad, divide by the gain,
    clip x to [0, w0] and y to [0, h0]"""
    gain, pad = ratio_pad[0][0], ratio_pad[1]
    c = coords.clone()
    c[:, 0] -= pad[0]; c[:, 2] -= pad[0]
    c[:, 1] -= pad[1]; c[:, 3] -= pad[1]
    c /= gain
    c[:, 0].clamp_(0, img0_shape[1]); c[:, 2].clamp_(0, img0_shape[1])
    c[:, 1].clamp_(0, img0_shape[0]); c[:, 3].clamp_(0, img0_shape[0])
    return c


def test_val_batch_letterboxed():
    """val.val_batch on a 224x352 batch with per-image (ratio, pad) letterboxes, against the same pipeline assembled from
    the oracle on the engine's own predictions: port.nms_val -> scale_coords -> port.process_batch.  correct, conf,
    predicted class and target classes must be identical per image."""
    from efficientteacher_b200 import val as etb_val
    from oracle import port
    B, H, W = 3, 224, 352
    m = _model("l_shallow", obj_bias=5.0, cls_bias=1.0)
    img = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(9)).to(DEV)
    # (shape0 = native (h0, w0), (ratio, pad = (dw, dh))) as the rect letterbox loader makes them (val.py:300-372)
    shapes = [((306, 500), ((0.704, 0.704), (0.0, 4.5))),
              ((200, 330), ((1.0, 1.0), (11.0, 12.0))),
              ((450, 700), ((0.5, 0.5), (1.0, 0.5)))]
    with torch.no_grad():
        pred0 = m(img)[0][0]
        pred = m(img)[0][0]
    assert torch.equal(pred0, pred)          # the engine forward is deterministic: val_batch sees these predictions
    iouv = torch.linspace(0.5, 0.95, 10)
    dets = port.nms_val(pred.cpu().numpy(), 0.001, 0.6, multi_label=True)
    assert all(len(d) > 0 for d in dets)
    # targets: a few of each image's own top detections (jittered, so the IoU ladder splits) plus random boxes and classes
    rng = np.random.RandomState(11)
    rows = []
    for si, d in enumerate(dets):
        for j in range(min(6, len(d))):
            x1, y1, x2, y2, _, c = d[j * 7 % len(d)]
            jit = 1.0 + 0.08 * rng.standard_normal(4)
            cx, cy, bw, bh = (x1 + x2) / 2 * jit[0], (y1 + y2) / 2 * jit[1], (x2 - x1) * jit[2], (y2 - y1) * jit[3]
            rows.append([si, c, cx / W, cy / H, abs(bw) / W, abs(bh) / H])
        for _ in range(3):
            rows.append([si, rng.randint(0, 80), *rng.uniform(0.2, 0.8, 2), *rng.uniform(0.05, 0.3, 2)])
    targets = torch.tensor(rows, dtype=torch.float32)
    stats = etb_val.val_batch(m, img, targets.to(DEV), shapes, iouv=iouv.to(DEV))
    assert len(stats) == B
    # the restatement runs its fp32 ops on the device val_batch uses, so the rescaled boxes are the same floats
    tg = targets.to(DEV)
    tg[:, 2:6] *= torch.tensor([W, H, W, H], dtype=torch.float32, device=DEV)
    n_correct = 0
    for si, d in enumerate(dets):
        pn = _scale_coords((H, W), torch.from_numpy(d[:, :4].copy()).to(DEV), shapes[si][0], shapes[si][1])
        lab = tg[tg[:, 0] == si, 1:]
        tb = torch.cat((lab[:, 1:3] - lab[:, 3:5] / 2, lab[:, 1:3] + lab[:, 3:5] / 2), 1)       # xywh -> xyxy
        tb = _scale_coords((H, W), tb, shapes[si][0], shapes[si][1])
        detn = np.concatenate([pn.cpu().numpy(), d[:, 4:6]], 1)
        want = port.process_batch(detn, torch.cat((lab[:, 0:1], tb), 1).cpu().numpy(), iouv.numpy())
        correct, conf, pcls, tcls = stats[si]
        assert np.array_equal(correct.cpu().numpy(), want), si
        assert np.array_equal(conf.cpu().numpy(), d[:, 4]) and np.array_equal(pcls.cpu().numpy(), d[:, 5]), si
        assert tcls == lab[:, 0].tolist(), si
        n_correct += int(want.sum())
    assert n_correct > 0            # the matching path is exercised, not just the empty case
