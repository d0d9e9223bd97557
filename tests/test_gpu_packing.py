"""GPU (H100): the bf16 GEMM operands of convops.pack_weight / pack_stem_weight / pack_weight_dgrad (etb_pack_multi) equal,
bit for bit, the operands built in plain torch from the layouts the convolution kernels read (include/etb200.h)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _ceil64(c):
    return (c + 63) // 64 * 64


def _weight(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g).to(DEV)


def _fwd_ref(w):
    """[Cout][kh][kw][ceil64(Cin)], pads zero"""
    Cout, Cin, k, _ = w.shape
    out = torch.zeros((Cout, k, k, _ceil64(Cin)), dtype=torch.bfloat16, device=DEV)
    out[..., :Cin] = w.permute(0, 2, 3, 1).to(torch.bfloat16)
    return out.reshape(Cout, -1)


def _dgrad_ref(w, s, p):
    """per parity class (ph outer, pw inner) [Cin][ntaps][ceil64(Cout)], pads zero, classes concatenated"""
    from efficientteacher_b200.packing import dgrad_classes
    Cout, Cin, k, _ = w.shape
    blocks = []
    for khs, kws in dgrad_classes(k, s, p):
        blk = torch.zeros((Cin, len(khs), _ceil64(Cout)), dtype=torch.bfloat16, device=DEV)
        blk[..., :Cout] = w[:, :, khs, kws].permute(1, 2, 0).to(torch.bfloat16)
        blocks.append(blk.reshape(-1))
    return torch.cat(blocks)


@pytest.mark.parametrize("k,s", [(1, 1), (1, 2), (3, 1), (3, 2)])
@pytest.mark.parametrize("Cin,Cout", [(32, 48), (48, 255), (255, 32)])
def test_pack_weight_and_dgrad_match_torch_layout(k, s, Cin, Cout):
    from efficientteacher_b200 import convops as co
    p = k // 2
    w = _weight((Cout, Cin, k, k), 1000 * k + 100 * s + Cin + Cout)
    assert torch.equal(co.pack_weight(w), _fwd_ref(w))
    assert torch.equal(co.pack_weight_dgrad(w, s, p), _dgrad_ref(w, s, p))
    assert torch.equal(co.pack_weight_dgrad(w, s, p, negate=True), _dgrad_ref(-w, s, p))


@pytest.mark.parametrize("Cout", [32, 48])
def test_pack_stem_weight_matches_torch_layout(Cout):
    """[Cout][128]: the OIHW row (c,kh,kw) in K 0..107 -- the stem_im2col_parts K order -- and zeros above"""
    from efficientteacher_b200 import convops as co
    w = _weight((Cout, 3, 6, 6), Cout)
    want = torch.zeros((Cout, 128), dtype=torch.bfloat16, device=DEV)
    want[:, :108] = w.reshape(Cout, 108).to(torch.bfloat16)
    assert torch.equal(co.pack_stem_weight(w), want)
