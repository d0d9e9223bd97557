"""GPU (H100): the autograd bridge of the student's training step.

a. The conv-only path of the Conv module (native conv under torch BatchNorm, taken by widths the fused BatchNorm kernels
   do not cover, e.g. YOLOv5m's 48 / 96): output, dx and dW against float64 on bf16-rounded operands, with the tolerances
   of test_gpu_geometry.py, both with the operands of Model.pack_weights() and standalone.
b. The gradient arena and the weight-gradient side stream change no bit: a trunk piece that runs every native Function
   (C3 with shortcut, SPPF, the neck's concat/upsample glue, Detect, netD with the folded GradReverse) gives identical
   input and parameter gradients under plain .backward() and under autograd_conv.backward() into a zeroed GradArena."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_gpu_geometry import _bf, _check_bf16, _check_per_channel

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _conv_only(conv):
    """the Conv module's own convolution: BatchNorm and activation replaced by identities (the widths used here keep the
    module off the fused ConvBnActFn path either way)"""
    conv.bn, conv.act = nn.Identity(), nn.Identity()
    return conv


def _check_conv(conv, x, x64, needs_dx):
    """x: what the module receives; x64: the bf16-exact image / feature it stands for (CPU float64)"""
    w = conv.conv.weight
    w64 = w.detach().to(torch.bfloat16).double().cpu()
    s, p = conv.conv.stride[0], conv.conv.padding[0]
    ref = F.conv2d(x64, w64, None, s, p)
    y = conv(x)
    _check_bf16(y.float(), ref, "output")
    dy = _bf(tuple(ref.shape), 7, 0.1)
    w.grad = None
    # dy reaches the conv through a torch op, as through the module's BatchNorm in training: an autograd worker thread has
    # no current CUDA context before its first runtime call, and the wgrad's tensor-map encode needs one
    (y * dy.to(DEV, torch.bfloat16)).sum().backward()
    _check_per_channel(w.grad, torch.nn.grad.conv2d_weight(x64, tuple(w.shape), dy.double(), stride=s, padding=p), 5e-4, "dW")
    if needs_dx:
        _check_bf16(x.grad.float(), torch.nn.grad.conv2d_input(tuple(x64.shape), w64, dy.double(), stride=s, padding=p), "dx")


def _feature(N, C_, H, W, seed):
    x64 = _bf((N, C_, H, W), seed).double()
    x = x64.to(DEV, torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_()
    return x, x64


def test_conv_only_with_packed_operands():
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(0)
    m = Model(yolov5_ssod_cfg('m')).to(DEV).train()
    m.pack_weights()
    stem, conv = _conv_only(m.backbone.stage1), _conv_only(m.backbone.stage2_1)
    assert (stem.conv.out_channels, conv.conv.in_channels, conv.conv.out_channels) == (48, 48, 96)
    g = torch.Generator().manual_seed(1)
    parts = [torch.randint(0, 256, (1, 3, 20, 28), generator=g, dtype=torch.uint8) for _ in range(2)]
    img64 = (torch.cat(parts).double() / 255).to(torch.bfloat16).double()
    _check_conv(stem, m._stem_input([q.to(DEV) for q in parts]), img64, False)    # uint8 batch parts, as the loaders give them
    _check_conv(conv, *_feature(2, 48, 15, 21, 2), True)


def test_conv_only_standalone():
    from efficientteacher_b200.model import Conv
    torch.manual_seed(0)
    stem = _conv_only(Conv(3, 48, 6, 2, 2)).to(DEV).train()
    stem.is_stem = True
    img64 = _bf((2, 3, 20, 28), 3).abs().clamp(max=1.0).double()
    _check_conv(stem, img64.float().to(DEV), img64, False)
    _check_conv(_conv_only(Conv(48, 96, 3, 2)).to(DEV).train(), *_feature(2, 48, 15, 21, 4), True)
    _check_conv(_conv_only(Conv(64, 48, 1, 1)).to(DEV).train(), *_feature(2, 64, 11, 17, 5), True)


def test_arena_and_side_stream_gradients_are_bit_identical():
    from efficientteacher_b200 import autograd_conv as ac
    from efficientteacher_b200 import model as M
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.parallel import GradArena
    torch.manual_seed(0)
    m = M.Model(yolov5_ssod_cfg('l_shallow')).to(DEV).train()
    b = m.backbone

    def objective(x):
        """a fixed linear function of the head and netD outputs, from the stride-4 feature x onwards"""
        aux = m.pack_weights()
        c3 = b.stage3_2(b.stage3_1(b.stage2_2(x)))
        c4 = b.stage4_2(b.stage4_1(M._fan_out(c3)))
        f = m.neck((c3, c4, b.sppf(b.stage5_2(b.stage5_1(M._fan_out(c4))))))
        outs = m.head(f, aux.get("head")) + [getattr(m, d)(fi, True, aux.get(d)) for d, fi in zip(("det_8", "det_16", "det_32"), f)]
        g = torch.Generator().manual_seed(7)
        return sum((o * torch.randn(o.shape, generator=g).to(DEV)).sum() for o in outs)

    params = [p for p in m.parameters() if p.requires_grad]
    for p in params:
        p.grad = None
    xa = _feature(2, b.stage2_1.conv.out_channels, 32, 40, 6)[0]
    objective(xa).backward()
    want = [None if p.grad is None else p.grad.clone() for p in params]
    assert sum(w is not None for w in want) > 100

    arena = GradArena(m.parameters(), DEV, reverse=True)
    arena.zero()
    xb = _feature(2, b.stage2_1.conv.out_channels, 32, 40, 6)[0]
    ac.backward(objective(xb), side=True)
    assert torch.equal(xb.grad, xa.grad)
    for i, (p, w) in enumerate(zip(params, want)):
        assert torch.equal(p.grad, torch.zeros_like(p) if w is None else w), (i, tuple(p.shape))
