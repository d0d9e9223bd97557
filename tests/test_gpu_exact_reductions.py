"""GPU (H100): the weight-gradient convolution, the training BatchNorm reductions and the SPPF / neck glue kernels, exact, at
every layer shape the five YOLOv5 sizes train at (batch 32, 640x640: test_exact_reduction_shapes).

Integer operands make the fp32 sums exact whatever the split-K, tiling or summation order:
  * weight gradient: x in {-1,0,1}, dy in {-2..2}: every partial sum is an integer of magnitude <= 2 * pixels
    <= 2 * 3,276,800 (the stem's flat K=128 GEMM) < 2^24, so dW must equal the float64 result exactly;
  * BatchNorm: y, da in {-2..2}: sum y, sum y^2 and sum da are integers < 2^24 at every layer, so etb_bn_stats_sums and
    dbeta must equal the float64 sums exactly; the rest of the statistics are checked against bounds derived from the fp32
    rounding steps the kernels take;
  * glue: max, 2x2 block sums and copies of small integers are exact in bf16.
A row, K block, split slice or tap lost or counted twice moves a result by one part in ~1/pixels: invisible to a relative
tolerance at these sizes, an exact mismatch here.  The float64 references run on the GPU (cuDNN off: im2col + DGEMM, whose
integer partial sums stay exact)."""

import pytest
import torch
import torch.nn.functional as F

from test_exact_reduction_shapes import all_bn_cases, all_stem_cases, all_wgrad_cases, glue_cases, wgrad_splits
from test_gpu_geometry import _check_bf16

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24          # unit roundoff of fp32
EPS, MOM = 1e-3, 0.03   # the trunk's BatchNorm settings
F32 = lambda v: float(torch.tensor(v, dtype=torch.float32))  # noqa: E731  (a Python float as the kernels see it)


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)
    saved = torch.backends.cudnn.enabled
    torch.backends.cudnn.enabled = False
    yield
    torch.backends.cudnn.enabled = saved


def _ints(shape, lo, hi, seed, dtype=torch.bfloat16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV, dtype=torch.int32).to(dtype)


def _slice(t, off, width, fill):
    """t [..., C] placed at channels [off, off + C) of a `width`-channel buffer whose other channels hold `fill`"""
    buf = torch.full((*t.shape[:-1], width), fill, dtype=t.dtype, device=DEV)
    buf[..., off:off + t.shape[-1]] = t
    return buf


def _id(case):
    return "x".join(str(v) for v in case)


# ------------------------------------------------------------------------------------------------------ weight gradient
def _wgrad_operands(case, seed):
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x = _ints((N, H, W, Cin), -1, 1, seed)
    dy = _ints((N, Ho, Wo, Cout), -2, 2, seed + 1)
    ref = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2).double(), (Cout, Cin, k, k), dy.permute(0, 3, 1, 2).double(), s, p)
    assert torch.equal(ref, ref.round())
    return x, dy, ref.float()


@pytest.mark.parametrize("case", all_wgrad_cases(), ids=_id)
def test_wgrad_exact(case):
    """dense operands (dy padded to a multiple of 8 channels, as the Detect head's 255 -> 256), channel-sliced operands whose
    other channels hold non-zero integers, and accumulate_into an integer-valued gradient: all exact"""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    x, dy, want = _wgrad_operands(case, 1)
    c8 = (Cout + 7) // 8 * 8
    dyd = _slice(dy, 0, c8, 0.0)
    assert torch.equal(co.conv_wgrad(x, dyd, Cin, Cout, k, s, p), want), "dense"
    xs, dys = _slice(x, 16, Cin + 40, 1.0), _slice(dy, 8, c8 + 24, -2.0)
    assert torch.equal(co.conv_wgrad(xs, dys, Cin, Cout, k, s, p, x_coffset=16, dy_coffset=8), want), "channel slices"
    base = _ints((Cout, Cin, k, k), -1000, 1000, 3, torch.float32)
    g = base.clone()
    out = co.conv_wgrad(xs, dys, Cin, Cout, k, s, p, x_coffset=16, dy_coffset=8, accumulate_into=g)
    assert out.data_ptr() == g.data_ptr()
    assert torch.equal(g, base + want), "accumulate_into"


@pytest.mark.parametrize("case", all_stem_cases(), ids=_id)
def test_wgrad_stem_exact(case):
    """the stem's K=128 GEMM over a 32x320x320 im2col buffer: exact, and the 20 pad slots (k >= 108), filled with non-zero
    values here, never reach the [Cout,3,6,6] gradient"""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout = case[:5]
    x = _ints((N, H, W, 128), -1, 1, 5)
    x[..., 108:] = 1.0
    dy = _ints((N, H, W, Cout), -2, 2, 6)
    ref = (dy.view(-1, Cout).double().t() @ x[..., :108].reshape(-1, 108).double()).view(Cout, 3, 6, 6)
    want = ref.float()
    assert torch.equal(co.conv_wgrad(x, dy, 128, Cout, 1, 1, 0, stem=True), want)
    base = _ints((Cout, 3, 6, 6), -1000, 1000, 7, torch.float32)
    g = base.clone()
    co.conv_wgrad(x, dy, 128, Cout, 1, 1, 0, stem=True, accumulate_into=g)
    assert torch.equal(g, base + want)


# pointwise model layers whose plan runs each instance of wgrad_reduce_kernel (SG = 1, 4, 16)
MISALIGNED = [((32, 1024, 20, 20, 512, 1, 1, 0), (2, 5)), ((32, 512, 20, 20, 256, 1, 1, 0), (6, 31)),
              ((32, 128, 40, 40, 64, 1, 1, 0), (32, 512))]


@pytest.mark.parametrize("case,splits", MISALIGNED, ids=[_id(c) for c, _ in MISALIGNED])
def test_wgrad_accumulate_into_misaligned_view(case, splits):
    """accumulate_into a view that starts 4 bytes past a 16-byte boundary: the kk = 1 reduce takes its scalar path (the
    gradient arena aligns every view, so training never runs it); the floats around the view stay untouched"""
    from efficientteacher_b200 import _lib
    from efficientteacher_b200 import convops as co
    assert case in all_wgrad_cases()
    assert splits[0] <= wgrad_splits(_lib, case) <= splits[1]
    N, Cin, H, W, Cout, k, s, p = case
    x, dy, want = _wgrad_operands(case, 9)
    n = Cout * Cin
    store = torch.full((n + 8,), 5.0, device=DEV)
    g = store[1:1 + n].view(Cout, Cin, 1, 1)
    assert g.data_ptr() % 16 == 4
    base = _ints((Cout, Cin, 1, 1), -1000, 1000, 10, torch.float32)
    g.copy_(base)
    co.conv_wgrad(x, dy, Cin, Cout, k, s, p, accumulate_into=g)
    assert torch.equal(g, base + want)
    assert store[0].item() == 5.0 and (store[1 + n:] == 5.0).all()


# ------------------------------------------------------------------------------------------------------------ BatchNorm
def _bn_chain_depth(lib, M, C_, which):
    """an upper bound on the number of fp32 additions any one row's term goes through in a channel_reduce +
    reduce_partials sum: rows per thread, the PL lanes of a block, the partial rows per reduce thread, the fixed tree"""
    rows = int(lib.etb_bn_partial_rows(M, C_, which))
    PL = 256 // (C_ // 8)
    GR = 128 if C_ <= 256 else 32
    return -(-M // (rows * PL)) + PL + -(-rows // GR) + 24


def _chain_bound(n, size):
    """worst-case error of a sum whose every term goes through at most n fp32 roundings: n u / (1 - n u) * sum |term|"""
    return n * U / (1 - n * U) * size


@pytest.mark.parametrize("case", all_bn_cases(), ids=_id)
def test_bn_reductions_exact(case):
    from efficientteacher_b200 import _lib
    from efficientteacher_b200 import convops as co
    lib = _lib.lib()
    M, C_ = case
    width, off = C_ + 16, 8
    y = _ints((M, C_), -2, 2, 11)
    ybuf = _slice(y, off, width, 1.0).view(1, 1, M, width)
    yv = ybuf[..., off:off + C_]
    y64 = y.double()
    S1, S2 = y64.sum(0), (y64 * y64).sum(0)
    # etb_bn_stats_sums: [sum y, sum y^2, M] in fp64 from the fp32 totals -- the integers themselves
    rows = int(lib.etb_bn_partial_rows(M, C_, 0))
    partials = torch.empty((rows, 2, C_), dtype=torch.float32, device=DEV)
    sums = torch.empty(2 * C_ + 1, dtype=torch.float64, device=DEV)
    _lib.check(lib.etb_bn_stats_sums(_lib.ptr(yv), M, C_, width, _lib.ptr(partials), rows, _lib.ptr(sums), _lib.stream_ptr()))
    assert torch.equal(sums[:C_], S1) and torch.equal(sums[C_:2 * C_], S2) and sums[2 * C_].item() == M
    # etb_bn_finalize, through bn_forward: mean, invstd and the running statistics against the fp32 steps of the kernel
    gamma = torch.rand(C_, device=DEV) + 0.5
    beta = torch.randn(C_, device=DEV) * 0.1
    rm0, rv0 = torch.randn(C_, device=DEV) * 0.1, torch.rand(C_, device=DEV) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    _, stats = co.bn_forward(yv, C_, gamma, beta, rm, rv, EPS, MOM, "none", y_cstride=width)
    mean_k, invstd_k = stats[2].double(), stats[3].double()
    m, e2 = S1 / M, S2 / M
    var = e2 - m * m
    # mean = fl(S1 * fl(1/M)); q = fl(S2 * fl(1/M)); var = fl(q - mean^2) (one FMA), clamped at 0
    err_mean = m.abs() * (2 * U + U * U)
    assert ((mean_k - m).abs() <= err_mean).all(), "mean"
    err_var = (e2 * (2 * U + U * U) + m * m * (4 * U + 7 * U * U) + U * var) / (1 - U)
    # invstd = rsqrtf(fl(var + eps)): rsqrtf is within 2 ulp (4u relative)
    t = var + F32(EPS)
    dt = (err_var + U * (t + err_var)) / t
    is_true = t.rsqrt()
    assert ((invstd_k - is_true).abs() <= is_true * (0.5 * dt * (1 + dt) + 4 * U) * (1 + 4 * U)).all(), "invstd"
    # running stats: fmaf(mom, x - r0, r0) with x = mean, and x = fl(var * fl(M / (M - 1))) (torch's unbiased variance)
    mom = F32(MOM)
    r0m, r0v = rm0.double(), rv0.double()
    want_rm = r0m + mom * (m - r0m)
    assert ((rm.double() - want_rm).abs() <= mom * err_mean + mom * U * (mean_k - r0m).abs() + U * rm.double().abs() * (1 + U)).all()
    ratio = M / (M - 1)
    unb = var * ratio
    err_unb = ratio * (err_var + (var + err_var) * (2 * U + U * U))
    want_rv = r0v + mom * (unb - r0v)
    assert ((rv.double() - want_rv).abs() <= mom * err_unb + mom * U * ((unb - r0v).abs() + err_unb)
            + U * rv.double().abs() * (1 + U)).all(), "running_var"
    # backward with act none: dz = da (an integer), so dbeta = sum da exactly, written and accumulated
    da = _ints((M, C_), -2, 2, 12)
    dabuf = _slice(da, off, width, -1.0).view(1, 1, M, width)
    dav = dabuf[..., off:off + C_]
    _, dgamma, dbeta = co.bn_backward(dav, yv, C_, stats, "none", da_cstride=width, y_cstride=width)
    da64 = da.double()
    assert torch.equal(dbeta.double(), da64.sum(0)), "dbeta"
    # dgamma = sum da * xhat with xhat = fmaf(y, invstd, fl(-mean * invstd)) exactly as the kernel forms it: the only
    # error left is the summation, bounded by the depth of its chain
    mu = (-stats[2] * stats[3]).double()
    xh = (y64 * invstd_k + mu).float().double()
    terms = da64 * xh
    want_dg = terms.sum(0)
    err_dg = _chain_bound(_bn_chain_depth(lib, M, C_, 1), terms.abs().sum(0))
    assert ((dgamma.double() - want_dg).abs() <= err_dg).all(), "dgamma"
    gb, bb = _ints((C_,), -1000, 1000, 13, torch.float32), _ints((C_,), -1000, 1000, 14, torch.float32)
    dg, db = gb.clone(), bb.clone()
    co.bn_backward(dav, yv, C_, stats, "none", da_cstride=width, y_cstride=width, dgamma_into=dg, dbeta_into=db)
    assert torch.equal(db.double(), bb.double() + da64.sum(0)), "dbeta_into"
    acc = gb.double() + want_dg
    assert ((dg.double() - acc).abs() <= err_dg + U * acc.abs() * (1 + U) + U * err_dg).all(), "dgamma_into"


def _offset_channels(M, C_, seed):
    """bf16 [M, C]: channel c has mean/std ratio R = (0, 8, 32)[c % 4] with std (0.25, 1, 4)[(c // 4) % 3]; every channel
    with c % 4 == 3 is constant (dead), at (0, 1.5, -0.75, 2)[(c // 4) % 4]"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = torch.arange(C_, device=DEV)
    R = torch.tensor([0.0, 8.0, 32.0, 0.0], device=DEV)[c % 4]
    sd = torch.tensor([0.25, 1.0, 4.0], device=DEV)[(c // 4) % 3]
    y = (torch.randn((M, C_), generator=g, device=DEV) + R) * sd
    dead = c % 4 == 3
    y[:, dead] = torch.tensor([0.0, 1.5, -0.75, 2.0], device=DEV)[(c // 4) % 4][dead]
    return y.to(torch.bfloat16), dead


@pytest.mark.parametrize("M", [32 * 160 * 160, 32 * 320 * 320])
def test_bn_offset_means_and_dead_channels(M):
    """precision, not exactness: mean/std ratios up to 32 and constant channels through var = E[y^2] - mean^2 in fp32"""
    from efficientteacher_b200 import convops as co
    C_ = 64
    y, dead = _offset_channels(M, C_, 21)
    gamma = torch.rand(C_, device=DEV) + 0.5
    beta = (torch.rand(C_, device=DEV) * 0.5 + 0.25) * torch.where(torch.arange(C_, device=DEV) % 8 < 4, 1.0, -1.0)
    width, off = C_ + 8, 8
    ybuf = _slice(y, off, width, 0.0).view(1, 1, M, width)
    a, stats = co.bn_forward(ybuf[..., off:off + C_], C_, gamma, beta, torch.zeros(C_, device=DEV), torch.ones(C_, device=DEV),
                             EPS, MOM, "silu", y_cstride=width)
    y64 = y.double()
    mean = y64.mean(0)
    var = (y64 - mean).pow(2).mean(0)
    is_ref = (var + F32(EPS)).rsqrt()
    rel = (stats[3].double() - is_ref).abs() / is_ref
    assert rel.max().item() <= 2.0 ** -9, ("invstd", int(rel.argmax()), rel.max().item())
    ref = F.silu((y64 - mean) * is_ref * gamma.double() + beta.double())
    a = a.view(M, C_)
    live = ~dead
    _check_bf16(a[:, live], ref[:, live], "live channels")
    # a constant channel normalises to 0: its output is act(beta) to within one bf16 ulp
    want = F.silu(beta.double())[dead]
    ulp = torch.exp2(torch.floor(torch.log2(want.abs())) - 7)
    assert ((a[:, dead].double() - want).abs() <= ulp).all(), "dead channels"


# ----------------------------------------------------------------------------------------------- glue (SPPF and the neck)
POOL, UP, CAT = glue_cases()


@pytest.mark.parametrize("case", POOL, ids=_id)
def test_sppf_maxpool_exact(case):
    """SPPF at every size: the three maxpool5_fwd of SppfPoolFn (slice k -> slice k + 1 of the 4C concat buffer, argmax),
    maxpool5_bwd fused with the add of the next slice's gradient, and the teacher's sppf_pool.  Integer data puts ties in
    every window: the argmax must be ATen's (first maximum in scan order)."""
    from efficientteacher_b200 import convops as co
    N, C_, H, W = case
    x = _ints((N, H, W, C_), -2, 2, 31)
    width = 4 * C_
    buf = _slice(x, 0, width, -7.0)
    idx = torch.empty((3, N, H, W, C_), dtype=torch.uint8, device=DEV)
    for k in range(3):
        co.maxpool5_fwd(buf[..., k * C_:], C_, width, buf[..., (k + 1) * C_:], width, idx[k])
    src = x.permute(0, 3, 1, 2).double()
    hh = torch.arange(H, device=DEV).view(H, 1)
    ww = torch.arange(W, device=DEV).view(1, W)
    for k in range(3):
        y, i = F.max_pool2d(src, 5, 1, 2, return_indices=True)
        assert torch.equal(buf[..., (k + 1) * C_:(k + 2) * C_], y.permute(0, 2, 3, 1).to(torch.bfloat16)), "pool %d" % k
        pos = ((i // W - hh + 2) * 5 + (i % W - ww + 2)).permute(0, 2, 3, 1)
        assert torch.equal(idx[k].long(), pos), "argmax %d" % k
        src = y
    # teacher: the same three pools in one kernel, on a buffer with a wider channel stride
    tb = _slice(x, 0, width + 16, -7.0)
    co.sppf_pool(tb, C_)
    assert torch.equal(tb[..., C_:4 * C_], buf[..., C_:]) and (tb[..., 4 * C_:] == -7.0).all()
    # backward: out = add + pool5_bwd(src) through the argmax, src and add channel slices of the concat gradient
    g = _ints((N, H, W, width), -2, 2, 32)
    t2 = _slice(torch.zeros((N, H, W, C_), dtype=torch.bfloat16, device=DEV), 8, C_ + 16, 3.0)
    co.maxpool5_bwd(g[..., 3 * C_:], width, idx[2], g[..., 2 * C_:], width, t2[..., 8:], C_ + 16, C_)
    gs = g[..., 3 * C_:].permute(0, 3, 1, 2).double()
    y1 = F.max_pool2d(F.max_pool2d(x.permute(0, 3, 1, 2).double(), 5, 1, 2), 5, 1, 2).requires_grad_(True)
    F.max_pool2d(y1, 5, 1, 2).backward(gs)
    want = y1.grad + g[..., 2 * C_:3 * C_].permute(0, 3, 1, 2).double()
    assert torch.equal(t2[..., 8:8 + C_], want.permute(0, 2, 3, 1).to(torch.bfloat16)), "maxpool5_bwd"
    assert (t2[..., :8] == 3.0).all() and (t2[..., 8 + C_:] == 3.0).all()


@pytest.mark.parametrize("case", UP, ids=_id)
def test_upsample2x_bwd_exact(case):
    """the neck's upsample backward: 2x2 block sums of the upsampled slice of the concat gradient"""
    from efficientteacher_b200 import convops as co
    N, C_, H, W = case
    width = 2 * C_ + 8
    g = _ints((N, 2 * H, 2 * W, width), -2, 2, 41)
    dx = torch.full((N, H, W, C_), 7.0, dtype=torch.bfloat16, device=DEV)
    co.upsample2x_bwd(g[..., 8:], width, dx, C_)
    want = g[..., 8:8 + C_].double().view(N, H, 2, W, 2, C_).sum((2, 4))
    assert torch.equal(dx, want.to(torch.bfloat16))


@pytest.mark.parametrize("case", CAT, ids=_id)
def test_copy_slice_exact(case):
    """the neck's concat: the lateral copied into its channel slice; the slice before it and the pixels after are kept"""
    from efficientteacher_b200 import convops as co
    N, H, W, C_, off, width = case
    M = N * H * W
    lat = _slice(_ints((M, C_), -100, 100, 51), 8, C_ + 24, 9.0)
    out = torch.full((M + 5, width), -3.0, dtype=torch.bfloat16, device=DEV)
    co.copy_slice(lat[:, 8:], C_ + 24, out[:, off:], width, M, C_)
    assert torch.equal(out[:M, off:off + C_], lat[:, 8:8 + C_])
    assert (out[:M, :off] == -3.0).all() and (out[M:] == -3.0).all()
