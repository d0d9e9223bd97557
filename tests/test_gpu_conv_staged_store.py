"""GPU (H100): the staged store of the raw-output conv epilogue (EPI 0: the student's training forward and every dgrad).
Storage order does not change values:
* forward: the staged raw output equals, bit for bit, the output of the direct-from-register epilogue (the folded-BN
  instance with scale 1, no bias, no activation) on the same operands, also written into a channel slice of a wider
  buffer whose other channels stay untouched;
* forward and dgrad (stride 1 and 2, with and without accumulation, into a channel slice of a wider buffer) on
  integer-valued operands whose fp32 sums are exact: the output is the float64 result rounded once to bf16."""
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


def _ints(shape, seed, lo=-2, hi=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).float().to(DEV)


CASES = [
    # N, Cin, H, W, Cout, k, s, p, x_cwidth (pixel stride of the input buffer; Cin is read at channel offset 16 if wider)
    (2, 64, 20, 20, 64, 1, 1, 0, 64),        # 1x1 flat, BN = 64
    (2, 64, 20, 20, 128, 3, 1, 1, 64),       # 3x3 s1
    (2, 64, 32, 32, 256, 3, 2, 1, 64),       # 3x3 s2, two N tiles
    (1, 256, 8, 8, 1024, 1, 1, 0, 256),      # Cout 1024: eight N tiles
    (2, 48, 20, 20, 96, 3, 1, 1, 48),        # YOLOv5m width: the second column half lies past Cout
    (2, 96, 16, 16, 192, 1, 1, 0, 96),       # YOLOv5m width, flat
    (2, 32, 16, 16, 36, 1, 1, 0, 32),        # Cout % 8 != 0: a partial last group of 8 channels
    (2, 64, 12, 12, 128, 3, 1, 1, 192),      # channel-sliced input (x_cstride > Cin)
    (2, 64, 1, 1, 64, 3, 1, 1, 64),          # 1x1 map
    (2, 64, 2, 3, 128, 3, 1, 1, 64),         # 2x3 map
    (3, 64, 5, 7, 128, 3, 2, 1, 64),         # 5x7 map, stride 2
    (2, 64, 5, 7, 64, 1, 1, 0, 64),          # 5x7 map, flat (ragged last M tile)
    (32, 128, 80, 80, 128, 3, 1, 1, 128),    # YOLOv5l batch 32: many tiles per persistent CTA
]


@pytest.mark.parametrize("case", CASES)
def test_staged_store_equals_direct_store(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p, xw = case
    xb = torch.zeros((N, H, W, xw), dtype=torch.bfloat16, device=DEV)
    xo = 16 if xw > Cin else 0
    co.to_nhwc_bf16(_rand((N, Cin, H, W), 1), out=xb, coffset=xo)
    wp = co.pack_weight(_rand((Cout, Cin, k, k), 2, scale=(Cin * k * k) ** -0.5))
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    cw = (Cout + 7) // 8 * 8
    run = lambda out, **kw: co.conv_fwd(xb, wp, Cin, Cout, k, s, p, x_coffset=xo, x_cstride=xw, bias=None, act=None, out=out, **kw)  # noqa: E731
    y = run(torch.full((N, Ho, Wo, cw), 9.0, dtype=torch.bfloat16, device=DEV), scale=None)
    direct = run(torch.full((N, Ho, Wo, cw), 9.0, dtype=torch.bfloat16, device=DEV), scale=torch.ones(Cout, device=DEV))
    assert torch.equal(y[..., :Cout], direct[..., :Cout])
    assert (y[..., Cout:] == 9).all()
    wide = torch.full((N, Ho, Wo, cw + 64), 7.0, dtype=torch.bfloat16, device=DEV)
    run(wide, scale=None, out_coffset=32)
    assert torch.equal(wide[..., 32:32 + Cout], y[..., :Cout])
    assert (wide[..., :32] == 7).all() and (wide[..., 32 + Cout:] == 7).all()
    assert torch.equal(run(torch.empty_like(y), scale=None)[..., :Cout], y[..., :Cout])     # reproducible


def test_stem_staged_store():
    from efficientteacher_b200 import convops as co
    x = torch.rand((2, 3, 64, 96), generator=torch.Generator().manual_seed(9)).to(DEV) * 255.0
    col = co.stem_im2col_parts([x], 255.0)
    wp = co.pack_stem_weight(_rand((64, 3, 6, 6), 10, scale=108 ** -0.5))
    y = co.conv_fwd(col, wp, 128, 64, 1, 1, 0, None, None, act=None)
    assert torch.equal(y, co.conv_fwd(col, wp, 128, 64, 1, 1, 0, torch.ones(64, device=DEV), None, act=None))


DGRAD_CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 20, 20, 128, 3, 1, 1),
    (2, 64, 20, 20, 128, 3, 2, 1),     # four parity lattices
    (2, 96, 13, 11, 64, 3, 2, 1),      # odd map, dx width 96 (second column half past the end)
    (2, 128, 16, 16, 64, 1, 1, 0),     # flat
    (2, 64, 5, 7, 64, 3, 1, 1),
]


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("case", DGRAD_CASES)
def test_dgrad_staged_store_exact(case, accumulate):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy, w = _ints((N, Cout, Ho, Wo), 5), _ints((Cout, Cin, k, k), 6)
    prev = _ints((N, Cin, H, W), 7, -8, 8)
    width, off = Cin + 64, 32
    dx = torch.full((N, H, W, width), 3.0, dtype=torch.bfloat16, device=DEV)
    co.to_nhwc_bf16(prev, out=dx, coffset=off)
    co.conv_dgrad(co.to_nhwc_bf16(dy), co.pack_weight_dgrad(w, s, p), N, H, W, Cin, Cout, k, s, p, out=dx, out_coffset=off,
                  accumulate=accumulate)
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), s, p)
    if accumulate:
        ref = ref + prev.double()
    assert torch.equal(dx[..., off:off + Cin], ref.permute(0, 2, 3, 1).to(torch.bfloat16))
    assert (dx[..., :off] == 3).all() and (dx[..., off + Cin:] == 3).all()


def test_forward_staged_store_exact():
    """Forward into a channel slice, on integer operands: exact sums rounded once."""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout = 2, 64, 9, 13, 192
    x, w = _ints((N, Cin, H, W), 8), _ints((Cout, Cin, 3, 3), 9)
    y = torch.full((N, H, W, Cout + 64), 5.0, dtype=torch.bfloat16, device=DEV)
    co.conv_fwd(co.to_nhwc_bf16(x), co.pack_weight(w), Cin, Cout, 3, 1, 1, None, None, act=None, out=y, out_coffset=64)
    want = F.conv2d(x.double(), w.double(), None, 1, 1).permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(y[..., 64:], want) and (y[..., :64] == 5).all()
