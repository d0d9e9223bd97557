"""GPU (H100): the raw-output conv epilogue (EPI 0) stores each tile by TMA from the store warp and, for a gradient fan-in
(dgrad with accumulate), TMA-loads the tile's existing output into the staged tile while the K loop runs.  On
integer-valued operands, whose fp32 sums are exact, the output is the float64 result (+ the existing value) rounded once
to bf16.  Every case writes into a channel slice of a wider buffer that has sentinel pixels after its last pixel: the
neighbouring channels and the trailing pixels keep their sentinels, which checks the tensor map's clipping at Cout, at
the edges of the output lattice (odd maps, stride-2 parity lattices, empty lattices) and at the last pixel."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENT = 3.0
TAIL = 37          # sentinel pixels after the output's last pixel
OFF = 32           # channel offset of the output slice


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _ints(shape, seed, lo=-2, hi=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).float().to(DEV)


def _sliced_out(N, H, W, C):
    """(whole buffer, [N,H,W,width] view) of a sentinel-filled buffer with TAIL extra pixels; the output goes to channels
    [OFF, OFF + C) of the view, whose pixel stride is width = C + OFF + 24 (a multiple of 8)"""
    width = (C + OFF + 24 + 7) // 8 * 8
    buf = torch.full(((N * H * W + TAIL) * width,), SENT, dtype=torch.bfloat16, device=DEV)
    return buf, buf[:N * H * W * width].view(N, H, W, width)


def _check_sentinels(buf, view, C):
    assert (view[..., :OFF] == SENT).all() and (view[..., OFF + C:] == SENT).all(), "a neighbouring channel was written"
    assert (buf[view.numel():] == SENT).all(), "a pixel past the output was written"


FWD_CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 20, 20, 128, 1, 1, 0),     # flat 1x1 tiling
    (2, 64, 13, 11, 128, 3, 1, 1),     # odd map
    (2, 64, 13, 11, 192, 3, 2, 1),     # stride 2, odd map, BN = 128 with a last N tile of one region
    (2, 32, 9, 7, 36, 1, 1, 0),        # Cout % 8 != 0 (stored from registers: TMA writes whole 16 B channel groups), flat
    (2, 64, 9, 7, 36, 3, 1, 1),        # Cout % 8 != 0, odd map
    (3, 64, 1, 1, 64, 3, 1, 1),        # 1x1 map
    (3, 64, 1, 1, 128, 3, 2, 1),       # 1x1 map, stride 2
    (2, 64, 1, 9, 64, 3, 2, 1),        # one-row map, stride 2
    (32, 128, 80, 80, 128, 1, 1, 0),   # YOLOv5l batch 32, flat: every persistent CTA walks ~12 tiles
    (32, 64, 40, 40, 256, 3, 1, 1),    # batch 32, 3x3: many tiles per CTA, two N tiles
]


@pytest.mark.parametrize("case", FWD_CASES)
def test_forward_tma_store_exact(case):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x, w = _ints((N, Cin, H, W), 11), _ints((Cout, Cin, k, k), 12)
    xb, wp = co.to_nhwc_bf16(x), co.pack_weight(w)
    buf, y = _sliced_out(N, Ho, Wo, Cout)
    co.conv_fwd(xb, wp, Cin, Cout, k, s, p, None, None, act=None, out=y, out_coffset=OFF)
    want = F.conv2d(x.double(), w.double(), None, s, p).permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(y[..., OFF:OFF + Cout], want)
    _check_sentinels(buf, y, Cout)
    buf2, y2 = _sliced_out(N, Ho, Wo, Cout)
    co.conv_fwd(xb, wp, Cin, Cout, k, s, p, None, None, act=None, out=y2, out_coffset=OFF)
    assert torch.equal(buf, buf2), "two runs differ"


DGRAD_CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 128, 16, 16, 64, 1, 1, 0),     # flat, BN = 128
    (2, 64, 13, 11, 128, 3, 1, 1),     # odd map, BN = 64
    (2, 64, 13, 11, 128, 3, 2, 1),     # four parity lattices of an odd map
    (2, 96, 7, 9, 64, 3, 2, 1),        # dx width 96: the second region of the only N tile is partial
    (2, 64, 1, 7, 64, 3, 2, 1),        # H = 1: the two odd-row lattices are empty
    (2, 64, 9, 1, 64, 3, 2, 1),        # W = 1: the two odd-column lattices are empty
    (3, 64, 1, 1, 64, 3, 2, 1),        # 1x1 map: three empty lattices
    (3, 128, 1, 1, 64, 3, 1, 1),       # 1x1 map, stride 1
    (32, 128, 80, 80, 128, 1, 1, 0),   # batch 32, flat: many tiles per CTA (staged-tile reuse with the accumulate prefetch)
    (32, 128, 40, 40, 128, 3, 2, 1),   # batch 32, stride 2: many tiles per CTA in every parity lattice
]


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("case", DGRAD_CASES)
def test_dgrad_tma_store_exact(case, accumulate):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    dy, w = _ints((N, Cout, Ho, Wo), 13), _ints((Cout, Cin, k, k), 14)
    prev = _ints((N, Cin, H, W), 15, -8, 8)
    dyb, wd = co.to_nhwc_bf16(dy), co.pack_weight_dgrad(w, s, p)

    def run():
        buf, dx = _sliced_out(N, H, W, Cin)
        co.to_nhwc_bf16(prev, out=dx, coffset=OFF)
        co.conv_dgrad(dyb, wd, N, H, W, Cin, Cout, k, s, p, out=dx, out_coffset=OFF, accumulate=accumulate)
        return buf, dx

    buf, dx = run()
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), s, p)
    if accumulate:
        ref = ref + prev.double()
    assert torch.equal(dx[..., OFF:OFF + Cin], ref.permute(0, 2, 3, 1).to(torch.bfloat16))
    _check_sentinels(buf, dx, Cin)
    assert torch.equal(buf, run()[0]), "two runs differ"


def test_dgrad_accumulate_rounds_once():
    """old + acc is rounded once: operands whose sum needs more than bf16's 8 significant bits would differ by one ulp if
    acc were rounded to bf16 before the add (or if the add were a bf16 reduction)."""
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout = 2, 64, 12, 12, 64
    dy = _ints((N, Cout, H, W), 16, 0, 1)
    w = torch.full((Cout, Cin, 1, 1), 1.0, device=DEV)
    w[::2] = 0.0078125       # 2^-7: dy sums to values with fractional bits at 2^-7
    prev = _ints((N, Cin, H, W), 17, 100, 140)
    buf, dx = _sliced_out(N, H, W, Cin)
    co.to_nhwc_bf16(prev, out=dx, coffset=OFF)
    co.conv_dgrad(co.to_nhwc_bf16(dy), co.pack_weight_dgrad(w, 1, 0), N, H, W, Cin, Cout, 1, 1, 0, out=dx, out_coffset=OFF,
                  accumulate=True)
    acc = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), 1, 0)
    want = (acc + prev.to(torch.bfloat16).double()).permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(dx[..., OFF:OFF + Cin], want)
    _check_sentinels(buf, dx, Cin)
