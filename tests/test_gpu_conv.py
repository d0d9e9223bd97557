"""GPU (H100): the wgmma implicit-GEMM convolution and the trunk helpers against a plain PyTorch fp32 reference
of the same op on bf16-rounded operands (floating-point kernel => torch reference, tolerance = bf16 output rounding)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(DEV)


def _bf(x):
    return x.to(torch.bfloat16).float()


def _check(got, want, tol=2e-2):
    err = (got - want).abs().max().item()
    ref = want.abs().max().item()
    assert err <= tol * max(ref, 1.0), (err, ref)


CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 16, 16, 64, 1, 1, 0),      # flat pointwise, BN=64
    (2, 128, 20, 20, 128, 1, 1, 0),    # flat, ragged M (800 px), BN=128
    (1, 256, 8, 8, 512, 1, 1, 0),      # flat, BN=256 x2 N-tiles, M < 128
    (2, 64, 16, 16, 64, 3, 1, 1),      # 3x3 s1 exact tiles
    (2, 64, 20, 20, 128, 3, 1, 1),     # 3x3 s1 ragged tiles (20x20)
    (1, 128, 40, 40, 256, 3, 1, 1),    # 3x3 s1 40x40, BN=256
    (2, 64, 32, 32, 128, 3, 2, 1),     # 3x3 s2 (TMA element strides)
    (1, 128, 40, 40, 128, 3, 2, 1),    # 3x3 s2 -> 20x20
    # YOLOv5s widths: channel counts that are not a multiple of the 64-channel K block (TMA clips the box, packs are padded)
    (2, 32, 16, 16, 64, 3, 2, 1),      # Cin = 32, stride 2 (stage2_1 of v5s)
    (2, 32, 20, 20, 32, 3, 1, 1),      # Cin = Cout = 32 (Bottleneck of the first C3)
    (2, 64, 20, 20, 32, 1, 1, 0),      # pointwise to 32 channels
    (2, 96, 16, 16, 32, 1, 1, 0),      # Cin = 96: 1.5 K blocks
    # YOLOv5m widths (48 / 96 / 192 ...): the last 32-channel epilogue chunk is partial
    (2, 48, 20, 20, 48, 3, 1, 1),
    (2, 96, 16, 16, 192, 1, 1, 0),
    # real YOLOv5l shapes at the bench batch
    (32, 64, 160, 160, 64, 3, 1, 1),   # first C3's Bottleneck conv: 160x160 maps, batch 32
    (32, 2048, 20, 20, 1024, 1, 1, 0), # SPPF cv2: K = 2048
    (32, 128, 160, 160, 256, 3, 2, 1), # stage3_1
]


@pytest.mark.parametrize("case", CASES)
def test_conv_bn_silu(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    x = _rand((N, Cin, H, W), 1)
    w = _rand((Cout, Cin, k, k), 2, scale=(Cin * k * k) ** -0.5)
    scale = torch.rand(Cout, device=DEV) + 0.5
    bias = torch.randn(Cout, device=DEV) * 0.1
    y = co.conv_fwd(co.to_nhwc_bf16(x), co.pack_weight(w), Cin, Cout, k, s, p, scale, bias, act="silu")
    got = co.to_nchw_f32(y)
    ref = F.conv2d(_bf(x), _bf(w), None, s, p) * scale.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)
    _check(got, F.silu(ref))


def test_conv_residual_and_concat_slices():
    from efficientteacher_b200 import convops as co
    N, C_, H, W = 2, 64, 16, 16
    x = _rand((N, C_, H, W), 3)
    r = _rand((N, C_, H, W), 4)
    w = _rand((C_, C_, 3, 3), 5, scale=(C_ * 9) ** -0.5)
    # input lives in channels [64,128) of a 192-wide buffer, output goes to [128,192), residual read from [0,64)
    buf = torch.zeros((N, H, W, 192), dtype=torch.bfloat16, device=DEV)
    co.to_nhwc_bf16(r, out=buf, coffset=0)
    co.to_nhwc_bf16(x, out=buf, coffset=64)
    co.conv_fwd(buf, co.pack_weight(w), C_, C_, 3, 1, 1, None, None, act="silu", out=buf, out_coffset=128, x_coffset=64,
                residual=buf, res_coffset=0)
    got = co.to_nchw_f32(buf, C_, 128)
    _check(got, F.silu(F.conv2d(_bf(x), _bf(w), None, 1, 1)) + _bf(r))
    assert torch.equal(co.to_nchw_f32(buf, C_, 64), _bf(x))       # neighbours untouched


def test_conv_residual_partial_chunk():
    """Cout = 48 (YOLOv5m Bottleneck width): the shortcut must also be added in the last, partial 32-channel chunk."""
    from efficientteacher_b200 import convops as co
    N, C_, H, W = 2, 48, 20, 20
    x, r = _rand((N, C_, H, W), 3), _rand((N, C_, H, W), 4)
    w = _rand((C_, C_, 3, 3), 5, scale=(C_ * 9) ** -0.5)
    y = co.conv_fwd(co.to_nhwc_bf16(x), co.pack_weight(w), C_, C_, 3, 1, 1, None, None, act="silu", residual=co.to_nhwc_bf16(r))
    _check(co.to_nchw_f32(y), F.silu(F.conv2d(_bf(x), _bf(w), None, 1, 1)) + _bf(r))


def test_detect_head_layout():
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, no = 2, 128, 20, 20, 85
    x = _rand((N, Cin, H, W), 6)
    w = _rand((3 * no, Cin, 1, 1), 7, scale=Cin ** -0.5)
    b = _rand((3 * no,), 8)
    out = torch.empty((N, 3, H, W, no), dtype=torch.float32, device=DEV)
    co.conv_fwd(co.to_nhwc_bf16(x), co.pack_weight(w), Cin, 3 * no, 1, 1, 0, None, b, act=None, det_out=out, det_no=no)
    ref = F.conv2d(_bf(x), _bf(w), b).view(N, 3, no, H, W).permute(0, 1, 3, 4, 2).contiguous()   # yolov5_head.py:66
    _check(out, ref, tol=1e-3)


def test_stem_im2col_conv():
    from efficientteacher_b200 import convops as co
    x = torch.rand((2, 3, 64, 64), generator=torch.Generator().manual_seed(9)).to(DEV) * 255.0
    w = _rand((64, 3, 6, 6), 10, scale=108 ** -0.5)
    col = co.stem_im2col_parts([x], 255.0)
    y = co.conv_fwd(col, co.pack_stem_weight(w), 128, 64, 1, 1, 0, None, None, act="silu")
    ref = F.silu(F.conv2d(_bf(x / 255), _bf(w), None, 2, 2))
    _check(co.to_nchw_f32(y), ref)


def test_sppf_and_upsample():
    from efficientteacher_b200 import convops as co
    x = _rand((2, 64, 20, 20), 11)
    buf = torch.zeros((2, 20, 20, 256), dtype=torch.bfloat16, device=DEV)
    co.to_nhwc_bf16(x, out=buf, coffset=0)
    co.sppf_pool(buf, 64)
    y1 = F.max_pool2d(_bf(x), 5, 1, 2); y2 = F.max_pool2d(y1, 5, 1, 2); y3 = F.max_pool2d(y2, 5, 1, 2)
    assert torch.equal(co.to_nchw_f32(buf, 256, 0), torch.cat([_bf(x), y1, y2, y3], 1))     # common.py:702-708
    up = torch.zeros((2, 40, 40, 128), dtype=torch.bfloat16, device=DEV)
    co.upsample2x(buf, 64, up, 64, x_coffset=0)
    assert torch.equal(co.to_nchw_f32(up, 64, 64), F.interpolate(_bf(x), scale_factor=2, mode="nearest"))


DGRAD_CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 16, 16, 128, 1, 1, 0),
    (2, 128, 20, 20, 64, 3, 1, 1),
    (1, 64, 40, 40, 128, 3, 1, 1),
    (2, 64, 32, 32, 128, 3, 2, 1),     # stride 2: four parity-class launches
    (1, 128, 40, 40, 256, 3, 2, 1),
    (2, 32, 16, 16, 64, 3, 2, 1),      # v5s: dgrad K = Cout = 64, 32 output channels
    (2, 32, 20, 20, 32, 3, 1, 1),      # v5s: K = 32 (half a K block, zero-filled by TMA)
    (2, 64, 20, 20, 32, 1, 1, 0),
    # YOLOv5m widths: Cin (= dgrad output channels) not a multiple of 32 -> partial epilogue chunk, incl. the fan-in accumulate
    (2, 48, 16, 16, 96, 1, 1, 0),
    (2, 96, 20, 20, 48, 3, 1, 1),
    (2, 48, 20, 20, 48, 3, 1, 1),
    # real YOLOv5l shapes at the bench batch
    (32, 64, 160, 160, 64, 3, 1, 1),
    (32, 2048, 20, 20, 1024, 1, 1, 0),
    (32, 128, 160, 160, 256, 3, 2, 1),
]


@pytest.mark.parametrize("case", DGRAD_CASES)
def test_conv_dgrad(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy = _rand((N, Cout, Ho, Wo), 21)
    w = _rand((Cout, Cin, k, k), 22, scale=(Cout * k * k) ** -0.5)
    dx = co.conv_dgrad(co.to_nhwc_bf16(dy), co.pack_weight_dgrad(w, s, p), N, H, W, Cin, Cout, k, s, p)
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), _bf(w), _bf(dy), stride=s, padding=p)
    _check(co.to_nchw_f32(dx), ref)
    # accumulate into an existing gradient (tensors with two consumers)
    base = _rand((N, Cin, H, W), 23)
    buf = co.to_nhwc_bf16(base)
    co.conv_dgrad(co.to_nhwc_bf16(dy), co.pack_weight_dgrad(w, s, p), N, H, W, Cin, Cout, k, s, p, out=buf, accumulate=True)
    _check(co.to_nchw_f32(buf), ref + _bf(base))


WGRAD_CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 16, 16, 128, 1, 1, 0),     # flat, single K block per split
    (4, 128, 20, 20, 255, 1, 1, 0),    # Detect head shape (Cout not a multiple of 64/128), ragged pixel count
    (2, 64, 16, 16, 64, 3, 1, 1),      # 9 taps, Cout < 128 (zero-filled M half)
    (2, 128, 20, 20, 128, 3, 1, 1),    # 20x20: K tiles with out-of-image rows
    (2, 64, 32, 32, 128, 3, 2, 1),     # stride 2
    (8, 256, 40, 40, 256, 3, 1, 1),    # split-K
    (2, 32, 16, 16, 64, 3, 2, 1),      # v5s: Cin = 32 (half-filled ci tile), 9 taps
    (2, 32, 20, 20, 32, 3, 1, 1),
    (2, 64, 20, 20, 32, 1, 1, 0),
    (2, 32, 20, 20, 64, 1, 1, 0),
    # real YOLOv5l shapes at the bench batch (deep split-K)
    (32, 64, 160, 160, 64, 3, 1, 1),   # 819,200 pixels reduced per tap
    (32, 2048, 20, 20, 1024, 1, 1, 0),
    (32, 256, 40, 40, 256, 3, 1, 1),
    (32, 128, 160, 160, 256, 3, 2, 1),
    # wide layers (Cout >= 256, Cin >= 128): tails in co / ci, several ci tiles
    (4, 512, 20, 20, 512, 3, 1, 1),
    (2, 1024, 20, 20, 512, 1, 1, 0),   # 8 ci tiles
    (2, 128, 16, 16, 320, 1, 1, 0),    # co tail: 256 + 64
    (2, 192, 16, 16, 256, 3, 1, 1),    # ci tail: 128 + 64
    (2, 640, 12, 12, 256, 1, 1, 0),    # 5 ci tiles
    (3, 256, 24, 24, 512, 3, 2, 1),    # stride 2
]


def _wgrad_inputs(case, seed):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x = _rand((N, Cin, H, W), seed)
    dy = _rand((N, Cout, Ho, Wo), seed + 1, scale=0.1)
    return x, dy, co.to_nhwc_bf16(x), co.to_nhwc_bf16(dy)


# The two tests below keep the names (and parameter ids) of the tests these wide shapes were written for, which drove a
# Blackwell-only 2-CTA weight-gradient kernel; on Hopper every shape runs wgrad_kernel, and the tests check what their
# docstrings say.
@pytest.mark.parametrize("case", [c for c in WGRAD_CASES if c[4] >= 256 and c[1] >= 128])
def test_conv_wgrad_2sm_kernel(case):
    """Wide-layer weight gradients are deterministic: the split-K partial tiles are summed in a fixed order (no atomics), so
    two runs on the same inputs agree bit for bit -- and agree with torch."""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    x, dy, xb, dyb = _wgrad_inputs(case, 71)
    dw1 = co.conv_wgrad(xb, dyb, Cin, Cout, k, s, p)
    dw2 = co.conv_wgrad(xb, dyb, Cin, Cout, k, s, p)
    assert torch.equal(dw1, dw2)
    ref = torch.nn.grad.conv2d_weight(_bf(x), (Cout, Cin, k, k), _bf(dy), stride=s, padding=p)
    err = (dw1 - ref).abs().max().item()
    assert err <= 2e-3 * max(ref.abs().max().item(), 1.0), (err, ref.abs().max().item())


WGRAD2_WIDE_CASES = [c for c in WGRAD_CASES if c[4] >= 256 and c[1] % 256 == 0] + [
    (2, 256, 16, 16, 256, 1, 1, 0),
    (2, 512, 12, 12, 320, 1, 1, 0),    # co tail 256 + 64
    (2, 768, 12, 12, 256, 1, 1, 0),
    (2, 256, 20, 20, 256, 3, 1, 1),    # K tiles with out-of-image rows
    (2, 256, 16, 16, 512, 3, 2, 1),    # stride 2, two 256-wide co groups
    (32, 512, 20, 20, 512, 3, 1, 1),   # real shape, deep split-K
    (32, 512, 40, 40, 256, 1, 1, 0),
]


@pytest.mark.parametrize("case", WGRAD2_WIDE_CASES)
def test_conv_wgrad_2sm_wide_kernel(case):
    """Wide layers with Cin % 256 == 0, up to real shapes with a deep split-K: the weight gradient accumulated into an
    existing gradient (the split-K reduce adds to the arena) equals existing + torch's weight gradient."""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    x, dy, xb, dyb = _wgrad_inputs(case, 81)
    base = _rand((Cout, Cin, k, k), 83)
    g = base.clone()
    out = co.conv_wgrad(xb, dyb, Cin, Cout, k, s, p, accumulate_into=g)
    assert out.data_ptr() == g.data_ptr()
    ref = torch.nn.grad.conv2d_weight(_bf(x), (Cout, Cin, k, k), _bf(dy), stride=s, padding=p)
    err = (g - base - ref).abs().max().item()
    assert err <= 2e-3 * max(ref.abs().max().item(), 1.0), (err, ref.abs().max().item())


@pytest.mark.parametrize("case", WGRAD_CASES)
def test_conv_wgrad(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x = _rand((N, Cin, H, W), 31)
    dy = _rand((N, Cout, Ho, Wo), 32, scale=0.1)
    dyp = torch.zeros((N, Ho, Wo, (Cout + 7) // 8 * 8), dtype=torch.bfloat16, device=DEV)
    co.to_nhwc_bf16(dy, out=dyp, coffset=0)
    dw = co.conv_wgrad(co.to_nhwc_bf16(x), dyp, Cin, Cout, k, s, p)
    ref = torch.nn.grad.conv2d_weight(_bf(x), (Cout, Cin, k, k), _bf(dy), stride=s, padding=p)
    err = (dw - ref).abs().max().item()
    assert err <= 2e-3 * max(ref.abs().max().item(), 1.0), (err, ref.abs().max().item())


def test_stem_wgrad():
    from efficientteacher_b200 import convops as co
    x = torch.rand((2, 3, 64, 64), generator=torch.Generator().manual_seed(41)).to(DEV)
    dy = _rand((2, 64, 32, 32), 42, scale=0.1)
    col = co.stem_im2col_parts([x])
    dw = co.conv_wgrad(col, co.to_nhwc_bf16(dy), 128, 64, 1, 1, 0, stem=True)
    ref = torch.nn.grad.conv2d_weight(_bf(x), (64, 3, 6, 6), _bf(dy), stride=2, padding=2)
    err = (dw - ref).abs().max().item()
    assert err <= 2e-3 * max(ref.abs().max().item(), 1.0), (err, ref.abs().max().item())


@pytest.mark.parametrize("C_,H,act", [(64, 16, "silu"), (256, 20, "silu"), (1024, 8, "silu"), (128, 12, "relu"), (64, 160, "silu"), (2048, 4, "silu")])
def test_fused_bn_act_forward_backward(C_, H, act):
    """Training-mode BatchNorm+activation kernels (statistics, finalize, apply; forward and backward) vs torch (fp32 math
    on the same bf16 inputs), incl. running stats."""
    from efficientteacher_b200 import convops as co
    N = 4
    y = _rand((N, C_, H, H), 51) * 2.0 + 0.3
    da = _rand((N, C_, H, H), 52)
    gamma = torch.rand(C_, device=DEV) + 0.5
    beta = torch.randn(C_, device=DEV) * 0.1
    rm, rv = torch.zeros(C_, device=DEV), torch.ones(C_, device=DEV)
    yb, dab = co.to_nhwc_bf16(y), co.to_nhwc_bf16(da)
    a, stats = co.bn_forward(yb, C_, gamma, beta, rm, rv, 1e-3, 0.03, act)
    dy, dg, db = co.bn_backward(dab, yb, C_, stats, act)
    yr = _bf(y).requires_grad_(True)
    g2, b2 = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rm2, rv2 = torch.zeros(C_, device=DEV), torch.ones(C_, device=DEV)
    z = F.batch_norm(yr, rm2, rv2, g2, b2, True, 0.03, 1e-3)
    ar = F.silu(z) if act == "silu" else F.relu(z)
    ar.backward(_bf(da))
    _check(co.to_nchw_f32(a), ar.detach(), tol=1e-2)
    _check(co.to_nchw_f32(dy), yr.grad, tol=2e-2)
    torch.testing.assert_close(dg, g2.grad, rtol=2e-2, atol=2e-2 * g2.grad.abs().max().item())
    torch.testing.assert_close(db, b2.grad, rtol=2e-2, atol=2e-2 * b2.grad.abs().max().item())
    torch.testing.assert_close(rm, rm2, rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(rv, rv2, rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("case", [(4, 128, 20, 20, 256, 1, 1, 0), (2, 256, 16, 16, 256, 3, 1, 1), (2, 512, 8, 8, 512, 1, 1, 0)])
def test_conv_wgrad_accumulates_into_existing_grad(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    x = _rand((N, Cin, H, W), 61)
    dy = _rand((N, Cout, H, W), 62, scale=0.1)
    base = _rand((Cout, Cin, k, k), 63)
    g = base.clone()
    out = co.conv_wgrad(co.to_nhwc_bf16(x), co.to_nhwc_bf16(dy), Cin, Cout, k, s, p, accumulate_into=g)
    assert out.data_ptr() == g.data_ptr()
    ref = base + torch.nn.grad.conv2d_weight(_bf(x), (Cout, Cin, k, k), _bf(dy), stride=s, padding=p)
    err = (g - ref).abs().max().item()
    assert err <= 2e-3 * max(ref.abs().max().item(), 1.0), err


# ---------------------------------------------------------------- training-side glue (csrc/glue.cu)
def _cl(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def test_maxpool5_fwd_bwd_vs_torch():
    from efficientteacher_b200 import convops as co
    N, C_, H, W = 2, 64, 20, 20
    x = _cl(_rand((N, C_, H, W), 11))
    xb = x.permute(0, 2, 3, 1)
    y = torch.empty((N, H, W, C_), dtype=torch.bfloat16, device=DEV)
    idx = torch.empty((N, H, W, C_), dtype=torch.uint8, device=DEV)
    co.maxpool5_fwd(xb, C_, C_, y, C_, idx)
    xr = x.float().requires_grad_(True)
    yr = F.max_pool2d(xr, 5, 1, 2)
    assert torch.equal(y.permute(0, 3, 1, 2).float(), yr.detach())          # max of bf16 values is exact
    g = _cl(_rand((N, C_, H, W), 12))
    add = _cl(_rand((N, C_, H, W), 13))
    yr.backward(g.float())
    out = torch.empty((N, H, W, C_), dtype=torch.bfloat16, device=DEV)
    co.maxpool5_bwd(g.permute(0, 2, 3, 1), C_, idx, add.permute(0, 2, 3, 1), C_, out, C_, C_)
    want = xr.grad + add.float()
    # ties inside a window (bf16 has few distinct values) are routed to the first maximum by both implementations
    _check(out.permute(0, 3, 1, 2).float(), want, tol=1e-2)
    out2 = torch.empty_like(out)
    co.maxpool5_bwd(g.permute(0, 2, 3, 1), C_, idx, None, C_, out2, C_, C_)
    _check(out2.permute(0, 3, 1, 2).float(), xr.grad, tol=1e-2)


def test_upsample_bwd_and_slice_copy():
    from efficientteacher_b200 import convops as co
    N, C_, H, W = 2, 64, 10, 12
    big = _cl(_rand((N, 2 * C_, 2 * H, 2 * W), 21))                       # dy lives in a channel slice of a wider gradient
    gb = big.permute(0, 2, 3, 1)[..., C_:]
    dx = torch.empty((N, H, W, C_), dtype=torch.bfloat16, device=DEV)
    co.upsample2x_bwd(gb, 2 * C_, dx, C_)
    want = F.avg_pool2d(big[:, C_:].float(), 2) * 4.0
    _check(dx.permute(0, 3, 1, 2).float(), want, tol=1e-2)
    dst = torch.zeros((N, 2 * H, 2 * W, 3 * C_), dtype=torch.bfloat16, device=DEV)
    co.copy_slice(gb, 2 * C_, dst[..., C_:2 * C_], 3 * C_, N * 4 * H * W, C_)
    assert torch.equal(dst[..., C_:2 * C_], gb) and float(dst[..., :C_].abs().max()) == 0 and float(dst[..., 2 * C_:].abs().max()) == 0


@pytest.mark.parametrize("n,shortcut", [(2, True), (1, False)])
def test_c3_concat_by_offset_matches_torch_glue(n, shortcut):
    """C3 with the fused glue (outputs written into concat slices, shortcut add inside the BN apply) against the same
    native convs glued by torch.cat / torch add: outputs and every gradient must agree to bf16 rounding."""
    from efficientteacher_b200.model import C3, Conv
    torch.manual_seed(3)
    m = C3(128, 128, n, shortcut, 1, 0.5, "silu").to(DEV).train()
    x0 = _cl(_rand((2, 128, 20, 20), 31))
    res = {}
    for glue in (True, False):
        Conv.FUSED_GLUE = glue
        try:
            m.zero_grad(set_to_none=True)
            for mod in m.modules():
                if isinstance(mod, torch.nn.BatchNorm2d):
                    mod.reset_running_stats()
            x = x0.clone().requires_grad_(True)
            y = m(x)
            (y.float() * torch.linspace(-1, 1, y.numel(), device=DEV).reshape(y.shape)).sum().backward()
            res[glue] = (y.detach().float(), x.grad.float(), {k: p.grad.float().clone() for k, p in m.named_parameters()})
        finally:
            Conv.FUSED_GLUE = True
    ya, xa, pa = res[True]
    yb, xb_, pb = res[False]
    _check(ya, yb, tol=2e-2)
    cos = lambda a, b: float((a * b).sum() / (a.norm() * b.norm() + 1e-12))  # noqa: E731
    assert cos(xa, xb_) > 0.999, cos(xa, xb_)
    for k in pa:
        assert cos(pa[k], pb[k]) > 0.995, (k, cos(pa[k], pb[k]))


def test_sppf_and_neck_fused_glue_match_torch_glue():
    """SPPF + neck with the fused glue vs the same native convs glued by torch ops.  Yardstick: the torch-glue path run
    twice -- the BN statistics are summed with atomics, so two runs of the SAME path already differ by flipped bf16
    roundings that compound over the neck's ~15 BN layers; the fused path must sit within 3x of that noise."""
    from efficientteacher_b200.model import SPPF, Conv, YoloV5Neck
    from efficientteacher_b200.config import yolov5_ssod_cfg
    torch.manual_seed(5)
    cos = lambda a, b: float((a * b).sum() / (a.norm() * b.norm() + 1e-12))  # noqa: E731
    rel = lambda a, b: float((a - b).norm() / (b.norm() + 1e-12))  # noqa: E731
    sp = SPPF(256, 256, 5, "silu").to(DEV).train()
    neck = YoloV5Neck(yolov5_ssod_cfg("l_shallow")).to(DEV).train()
    x0 = _cl(_rand((2, 256, 10, 10), 41))
    feats0 = [_cl(_rand((4, 256, 32, 32), 42)), _cl(_rand((4, 512, 16, 16), 43)), _cl(_rand((4, 1024, 8, 8), 44))]
    res = []
    for glue in (True, False, False):
        Conv.FUSED_GLUE = glue
        try:
            for mod in (sp, neck):
                mod.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(True)
            y = sp(x)
            (y.float() * torch.linspace(-1, 1, y.numel(), device=DEV).reshape(y.shape)).sum().backward()
            feats = [f.clone().requires_grad_(True) for f in feats0]
            outs = neck(feats)
            sum((o.float() * torch.linspace(-1, 1, o.numel(), device=DEV).reshape(o.shape)).sum() for o in outs).backward()
            res.append(([y.detach().float()] + [o.detach().float() for o in outs], [x.grad.float()] + [f.grad.float() for f in feats],
                        {("sp." if mod is sp else "neck.") + k: p.grad.float().clone() for mod in (sp, neck) for k, p in mod.named_parameters()}))
        finally:
            Conv.FUSED_GLUE = True
    fused, t1, t2 = res
    # SPPF forward has a single BN before the pools: tight
    _check(fused[0][0], t1[0][0], tol=2e-2)
    for i in range(len(fused[0])):
        noise = rel(t2[0][i], t1[0][i])
        assert rel(fused[0][i], t1[0][i]) <= max(3 * noise, 4e-3), (i, rel(fused[0][i], t1[0][i]), noise)
    for i in range(len(fused[1])):
        noise = 1 - cos(t2[1][i], t1[1][i])
        assert 1 - cos(fused[1][i], t1[1][i]) <= max(3 * noise, 2e-3), (i, cos(fused[1][i], t1[1][i]), noise)
    for k in fused[2]:
        noise = 1 - cos(t2[2][k], t1[2][k])
        assert 1 - cos(fused[2][k], t1[2][k]) <= max(3 * noise, 1e-2), (k, cos(fused[2][k], t1[2][k]), noise)


def test_fanin_epilogue_accumulation_matches_autograd_adds():
    """Gradient fan-in (C3 input -> cv1 + cv2, Bottleneck input -> cv1 + shortcut) accumulated inside the dgrad epilogue
    vs autograd's add kernels: same forward, so the input gradient may differ only by bf16 rounding of the partial sums."""
    from efficientteacher_b200.model import C3, Conv
    torch.manual_seed(7)
    m = C3(128, 128, 3, True, 1, 0.5, "silu").to(DEV).train()
    x0 = _cl(_rand((2, 128, 24, 24), 51))
    res = {}
    for fan in (True, False):
        Conv.FUSED_FANIN = fan
        try:
            m.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(True)
            y = m(x)
            (y.float() * torch.linspace(-1, 1, y.numel(), device=DEV).reshape(y.shape)).sum().backward()
            res[fan] = (y.detach().float(), x.grad.float(), {k: p.grad.float().clone() for k, p in m.named_parameters()})
        finally:
            Conv.FUSED_FANIN = True
    assert torch.equal(res[True][0], res[False][0])          # forward is untouched (and deterministic)
    cos = lambda a, b: float((a * b).sum() / (a.norm() * b.norm() + 1e-12))  # noqa: E731
    assert cos(res[True][1], res[False][1]) > 0.9995
    _check(res[True][1], res[False][1], tol=3e-2)
    for k in res[True][2]:
        assert cos(res[True][2][k], res[False][2][k]) > 0.999, (k, cos(res[True][2][k], res[False][2][k]))
