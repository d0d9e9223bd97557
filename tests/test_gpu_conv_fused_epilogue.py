"""GPU (H100): the fused conv epilogues of the teacher's forward (EPI 1: folded BN -> SiLU/ReLU -> + shortcut; EPI 3: the
same with Hardswish) stage the tile in shared memory and store it by TMA, with the shortcut TMA-loaded into the staged tile
while the K loop runs.  On integer-valued operands the accumulator is exact; with power-of-two scales and dyadic biases so
is act(v*scale + bias) + shortcut for no activation and ReLU, so the output is the float64 result rounded once to bf16
(tolerance 0).  SiLU (tanh.approx) and Hardswish are held to the tolerance of the other fused-conv tests.  Every case
writes into a channel slice of a wider buffer with sentinels around it and after its last pixel, and the shortcut may be
a channel slice of a wider buffer too.  Outputs with Cout % 8 != 0 store from registers; they are checked the same way."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_conv import _check
from test_gpu_conv_tma_epilogue import OFF, _check_sentinels, _ints, _sliced_out

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RES_OFF = 24       # channel offset of a shortcut that is a slice of a wider buffer
EXACT = ("none", "relu")


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _fold(Cout, seed):
    """power-of-two scales and biases on a 1/4 grid: v*scale + bias is exact in fp32 for the integer accumulators here"""
    g = torch.Generator().manual_seed(seed)
    scale = 2.0 ** torch.randint(-2, 2, (Cout,), generator=g).float()
    bias = torch.randint(-8, 9, (Cout,), generator=g).float() / 4
    return scale.to(DEV), bias.to(DEV)


def _act(z, act):
    return {"none": lambda t: t, "relu": F.relu, "silu": F.silu, "hard_swish": F.hardswish}[act](z)


def _shortcut(N, Ho, Wo, Cout, mode, seed):
    """(float64 NCHW shortcut or None, bf16 NHWC tensor for conv_fwd, res_coffset)"""
    if mode is None:
        return None, None, 0
    r = _ints((N, Cout, Ho, Wo), seed, -3, 3)
    if mode == "own":
        return r.double(), r.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16), 0
    wide = torch.full((N, Ho, Wo, Cout + RES_OFF + 16), -5.0, dtype=torch.bfloat16, device=DEV)
    wide[..., RES_OFF:RES_OFF + Cout] = r.permute(0, 2, 3, 1).to(torch.bfloat16)
    return r.double(), wide, RES_OFF


def _run_and_check(case, act, mode, seed=0):
    from efficientteacher_b200 import convops as co
    N, Cin, H, W, Cout, k, s, p = case
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    x, w = _ints((N, Cin, H, W), 21 + seed, -1, 1), _ints((Cout, Cin, k, k), 22 + seed, -1, 1)
    scale, bias = _fold(Cout, 23 + seed)
    r64, rb, rco = _shortcut(N, Ho, Wo, Cout, mode, 24 + seed)
    xb, wp = co.to_nhwc_bf16(x), co.pack_weight(w)

    def run():
        buf, y = _sliced_out(N, Ho, Wo, Cout)
        co.conv_fwd(xb, wp, Cin, Cout, k, s, p, scale, bias, act, out=y, out_coffset=OFF, residual=rb, res_coffset=rco)
        return buf, y

    buf, y = run()
    z = F.conv2d(x.double(), w.double(), None, s, p) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    want = _act(z, act)
    if r64 is not None:
        want = want + r64
    got = y[..., OFF:OFF + Cout]
    if act in EXACT:
        assert torch.equal(got, want.permute(0, 2, 3, 1).to(torch.bfloat16))
    else:
        _check(got.permute(0, 3, 1, 2).float(), want.float())
    _check_sentinels(buf, y, Cout)
    assert torch.equal(buf, run()[0]), "two runs differ"


CASES = [
    # N, Cin, H, W, Cout, k, s, p
    (2, 64, 20, 20, 128, 1, 1, 0),     # flat 1x1 tiling
    (2, 64, 13, 11, 128, 3, 1, 1),     # odd map
    (2, 64, 13, 11, 192, 3, 2, 1),     # stride 2, odd map, BN = 128 with a last N tile of one region
    (3, 64, 1, 1, 64, 3, 1, 1),        # 1x1 map
    (3, 64, 1, 1, 128, 3, 2, 1),       # 1x1 map, stride 2
    (2, 64, 1, 9, 64, 3, 2, 1),        # one-row map, stride 2
    (2, 32, 20, 20, 32, 3, 1, 1),      # YOLOv5s Bottleneck width: TMA clips the shortcut load and the store at Cout = 32
    (2, 48, 13, 11, 48, 3, 1, 1),      # YOLOv5m width 48, odd map
    (2, 96, 16, 16, 48, 1, 1, 0),      # width 48, flat
]


@pytest.mark.parametrize("mode", [None, "own", "slice"])
@pytest.mark.parametrize("act", ["none", "relu", "silu", "hard_swish"])
@pytest.mark.parametrize("case", CASES)
def test_fused_epilogue(case, act, mode):
    _run_and_check(case, act, mode)


BATCH32 = [
    (32, 64, 40, 40, 64, 3, 1, 1),     # the Bottleneck 3x3 at batch 32: every persistent CTA walks ~60 tiles, so each
    (32, 128, 80, 80, 128, 1, 1, 0),   # reuse of the staged tile alternates with the next tile's shortcut prefetch
]


@pytest.mark.parametrize("act,mode", [("relu", "own"), ("silu", "slice"), ("hard_swish", "own"), ("silu", None)])
@pytest.mark.parametrize("case", BATCH32)
def test_fused_epilogue_many_tiles(case, act, mode):
    _run_and_check(case, act, mode, seed=1)


@pytest.mark.parametrize("act", ["none", "relu", "silu", "hard_swish"])
@pytest.mark.parametrize("case", [(2, 32, 9, 7, 36, 1, 1, 0), (2, 64, 9, 7, 36, 3, 1, 1), (2, 64, 13, 11, 2, 1, 1, 0)])
def test_fused_epilogue_cout_not_multiple_of_8(case, act):
    """Cout % 8 != 0 (no shortcut is allowed there) stores from registers, channel by channel"""
    _run_and_check(case, act, None)


@pytest.mark.parametrize("act", ["relu", "silu"])
def test_fused_epilogue_slices_of_one_buffer(act):
    """input, output and shortcut in disjoint channel slices of one buffer: the shortcut map and the output map cover
    the same allocation"""
    from efficientteacher_b200 import convops as co
    N, C_, H, W = 2, 64, 17, 13
    x, r = _ints((N, C_, H, W), 31, -1, 1), _ints((N, C_, H, W), 32, -3, 3)
    w = _ints((C_, C_, 3, 3), 33, -1, 1)
    scale, bias = _fold(C_, 34)
    buf = torch.full((N, H, W, 200), 7.0, dtype=torch.bfloat16, device=DEV)   # [0,64) shortcut, [64,128) x, [128,192) y
    co.to_nhwc_bf16(r, out=buf, coffset=0)
    co.to_nhwc_bf16(x, out=buf, coffset=64)
    co.conv_fwd(buf, co.pack_weight(w), C_, C_, 3, 1, 1, scale, bias, act, out=buf, out_coffset=128, x_coffset=64,
                residual=buf, res_coffset=0)
    z = F.conv2d(x.double(), w.double(), None, 1, 1) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    want = (_act(z, act) + r.double()).permute(0, 2, 3, 1)
    got = buf[..., 128:192]
    if act in EXACT:
        assert torch.equal(got, want.to(torch.bfloat16))
    else:
        _check(got.float(), want.float())
    assert torch.equal(buf[..., :64], r.permute(0, 2, 3, 1).to(torch.bfloat16)), "the shortcut was written"
    assert torch.equal(buf[..., 64:128], x.permute(0, 2, 3, 1).to(torch.bfloat16)), "the input was written"
    assert (buf[..., 192:] == 7.0).all(), "channels past the output were written"
