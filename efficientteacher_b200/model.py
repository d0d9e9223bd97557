"""YOLOv5 detector with the reference's module tree, attribute names and state_dict keys
(models/detector/yolo_ssod.py:44-118, models/detector/yolo.py:45-110, models/backbone/yolov5_backbone.py:26-88,
models/neck/yolov5_neck.py:6-109, models/head/yolov5_head.py:7-87, models/backbone/common.py Conv/Bottleneck/C3/SPPF),
so reference checkpoints / EMA deep copies / optimizer param grouping keep working (SURVEY.md section 8b).

Execution:
  * eval / no-grad forward (the teacher-EMA pass of trainer/ssod_trainer.py:595-599) runs on the native engine
    (engine.TrunkEngine: wgmma implicit-GEMM convs, NHWC bf16, BN folded, concat-by-offset, fused Detect).
  * training forward/backward: torch autograd only sequences the graph; every node is a native Function
    (autograd_conv.ConvBnActFn = wgmma conv + fused BatchNorm(train)+activation(+shortcut), JoinFn / SppfPoolFn /
    UpsampleIntoFn = concat-by-offset glue of csrc/glue.cu, DetectConvFn), tensors stay NHWC bf16 and are exposed to
    torch as channels_last views.
There is no CPU path: forward raises without a CUDA device + libetb200.so.
"""
import itertools
import math

import torch
import torch.nn as nn

from . import _lib
from .head import decode_levels
from .parallel import BnSync

_BN = nn.modules.batchnorm._BatchNorm      # nn.BatchNorm2d and nn.SyncBatchNorm (convert_sync_batchnorm)


def make_divisible(x, divisor):
    return math.ceil(x / divisor) * divisor


def autopad(k, p=None):
    return k // 2 if p is None else p


# activation module -> convops.ACT key of the native kernels (the modules get_activation of common.py:28-47 builds)
NATIVE_ACTS = ((nn.SiLU, "silu"), (nn.ReLU, "relu"), (nn.Hardswish, "hard_swish"))


def native_act(m):
    """convops.ACT key of activation module m; None (no activation) for nn.Identity or any other module"""
    return next((name for t, name in NATIVE_ACTS if isinstance(m, t)), None)


def trunk_acts(activation):
    """(CONV_ACT, C_ACT) of a cfg.Model.{Backbone,Neck}.activation string (yolov5_backbone.py:47-55, yolov5_neck.py:48-56):
    'SiLU' and 'ReLU' run everywhere; any other string selects Hardswish for the plain convs and SPPF and the mixed
    'relu_hswish' C3."""
    if activation == 'SiLU':
        return 'silu', 'silu'
    if activation == 'ReLU':
        return 'relu', 'relu'
    return 'hard_swish', 'relu_hswish'


def _split_act(act):
    """C3 / SPPF (common.py:566-592, 682-700): 'relu_hswish' = ReLU in the inner convs, Hardswish in the last one"""
    return ('relu', 'hard_swish') if act == 'relu_hswish' else (act, act)


class Conv(nn.Module):
    """conv2d(bias=False) + BatchNorm2d(eps 1e-3, momentum 0.03) + SiLU / ReLU / Hardswish   (common.py:471-484,
    torch_utils.py:168-169)"""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, act=True):
        super().__init__()
        assert g == 1
        self.conv = nn.Conv2d(c1, c2, k, s, autopad(k, p), groups=g, bias=False)
        self.bn = nn.BatchNorm2d(c2, eps=1e-3, momentum=0.03)
        if act is True or act == "silu":
            self.act = nn.SiLU()
        elif act == "relu":
            self.act = nn.ReLU(inplace=True)
        elif act == "hard_swish":
            self.act = nn.Hardswish(inplace=True)
        elif isinstance(act, str):
            raise NotImplementedError("activation %r is not on the hot path" % act)
        else:
            self.act = nn.Identity()
        self.act_name = act if act in ("relu", "hard_swish") else None

    # `_packed` aliases the owning model's packer buffers and `bn_sync` holds a process group: copies start without them
    def __deepcopy__(self, memo):
        from copy import deepcopy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k not in ("_packed", "bn_sync"):
                new.__dict__[k] = deepcopy(v, memo)
        return new

    def __getstate__(self):
        s = dict(self.__dict__)
        s.pop("_packed", None)
        s.pop("bn_sync", None)
        return s

    NATIVE = True        # training convs on the wgmma fwd/dgrad/wgrad kernels (False: torch/cuDNN scaffold)
    FUSED_BN = True      # BatchNorm(train)+activation forward/backward on the fused kernels of csrc/bn.cu (False: torch ops)
    FUSED_GLUE = True    # concat-by-offset / fused shortcut add / native pool+upsample (csrc/glue.cu) instead of torch ops
    FUSED_FANIN = True   # gradient fan-in (C3 input, shortcut, backbone feature) accumulated in the dgrad epilogue
    is_stem = False
    bn_sync = None       # parallel.BnSync forced on the fused BatchNorm (Model.set_bn_sync); else a SyncBatchNorm's own group

    def _sync(self):
        """The BnSync of the fused BatchNorm: the forced one, else -- for a torch.nn.SyncBatchNorm (convert_sync_batchnorm)
        -- its process group's when torch's module would synchronise too; None: per-rank statistics."""
        if self.bn_sync is not None:
            return self.bn_sync
        return BnSync.of_module(self.bn) if isinstance(self.bn, nn.SyncBatchNorm) else None

    def fused(self, x):
        """True when this Conv runs as ONE ConvBnActFn (and can therefore write into a CatBuf slice / add a shortcut)."""
        c = self.conv.out_channels
        bn_ok = c % 8 == 0 and c // 8 <= 256       # csrc/bn.cu bn_c_ok: one thread owns 8 channels, C/8 <= 256 per block
        return (Conv.NATIVE and Conv.FUSED_BN and bn_ok and x.is_cuda and self.training
                and native_act(self.act) is not None)

    def glue(self, x):
        return Conv.FUSED_GLUE and self.fused(x) and self.conv.out_channels % 8 == 0

    def forward(self, x, res=None, dest=None, coff=0):
        """res: shortcut added after the activation; dest/coff: autograd_conv.CatBuf slice to write the output into
        (both only on the fused path -- callers check `glue(x)` first)."""
        if Conv.NATIVE and x.is_cuda:
            from .autograd_conv import ConvBnActFn, ConvFn
            w, s, p = self.conv.weight, self.conv.stride[0], self.conv.padding[0]
            # operands prepared by Model.pack_weights() (one launch per training step)
            pc = getattr(self, "_packed", None) if Conv.FUSED_BN and self.training else None
            wp, wd = (None, None) if pc is None else (pc.fwd, pc.dgrad)
            if self.fused(x):
                bn = self.bn
                return ConvBnActFn.apply(x, w, bn.weight, bn.bias, bn.running_mean, bn.running_var, s, p, bn.eps, bn.momentum,
                                         native_act(self.act),
                                         self.is_stem, wp, wd, res, dest, coff, self._sync())
            assert dest is None
            y = self.act(self.bn(ConvFn.apply(x, w, s, p, self.is_stem, wp, wd)))
            return y if res is None else res + y
        assert dest is None
        y = self.act(self.bn(self.conv(x)))
        return y if res is None else res + y


def _fan_out(x):
    """Mark activation x as having several native consumers (autograd_conv.FanIn): their gradients are accumulated inside
    the dgrad epilogues instead of by autograd's add kernels.  No-op when x needs no gradient or is already marked."""
    if Conv.FUSED_FANIN and x.requires_grad and getattr(x, "_etb_fan", None) is None:
        from .autograd_conv import FanIn
        x._etb_fan = FanIn()
    return x


class Bottleneck(nn.Module):
    def __init__(self, c1, c2, shortcut=True, g=1, k=(1, 3), e=0.5, act=True):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, k[0], 1, act=act)
        self.cv2 = Conv(c_, c2, k[1], 1, g=g, act=act)
        self.add = shortcut and c1 == c2

    def forward(self, x, dest=None, coff=0):
        if self.cv2.glue(x):      # shortcut add fused into cv2's BN+SiLU apply; output optionally straight into a concat slice
            if self.add:
                _fan_out(x)       # x feeds cv1 and the shortcut: their gradients meet in cv1's dgrad epilogue, not in an ATen add
            return self.cv2(self.cv1(x), x if self.add else None, dest, coff)
        assert dest is None
        return x + self.cv2(self.cv1(x)) if self.add else self.cv2(self.cv1(x))


class C3(nn.Module):
    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5, act=True):
        super().__init__()
        c_ = int(c2 * e)
        act, last_act = _split_act(act)
        self.cv1 = Conv(c1, c_, 1, 1, act=act)
        self.cv2 = Conv(c1, c_, 1, 1, act=act)
        self.cv3 = Conv(2 * c_, c2, 1, act=last_act)
        self.m = nn.Sequential(*[Bottleneck(c_, c_, shortcut, g, e=1.0, act=act) for _ in range(n)])

    def forward(self, x):
        if self.cv1.glue(x) and self.cv2.glue(x) and len(self.m) > 0:
            from .autograd_conv import CatBuf, JoinFn
            c_ = self.cv1.conv.out_channels
            N, _, H, W = x.shape
            cb = CatBuf(N, 2 * c_, H, W, x.device)          # [ m(cv1(x)) | cv2(x) ] written in place by their producers
            _fan_out(x)                                     # x feeds cv1 and cv2: the second dgrad accumulates into the first's output
            a = self.cv1(x)
            for i, b in enumerate(self.m):
                a = b(a, cb, 0) if i == len(self.m) - 1 else b(a)
            b2 = self.cv2(x, None, cb, c_)
            return self.cv3(JoinFn.apply(cb, (False, False), a, b2))
        return self.cv3(torch.cat((self.m(self.cv1(x)), self.cv2(x)), dim=1))


class SPPF(nn.Module):
    def __init__(self, c1, c2, k=5, act=True):
        super().__init__()
        c_ = c1 // 2
        act, last_act = _split_act(act)
        self.cv1 = Conv(c1, c_, 1, 1, act=act)
        self.cv2 = Conv(c_ * 4, c2, 1, 1, act=last_act)
        self.m = nn.MaxPool2d(kernel_size=k, stride=1, padding=k // 2)

    def forward(self, x):
        if self.cv1.glue(x) and self.m.kernel_size == 5:
            from .autograd_conv import CatBuf, SppfPoolFn
            c_ = self.cv1.conv.out_channels
            N, _, H, W = x.shape
            cb = CatBuf(N, 4 * c_, H, W, x.device)
            return self.cv2(SppfPoolFn.apply(self.cv1(x, None, cb, 0), cb))
        x = self.cv1(x)
        y1 = self.m(x)
        y2 = self.m(y1)
        return self.cv2(torch.cat([x, y1, y2, self.m(y2)], 1))


class Concat(nn.Module):
    def __init__(self, dimension=1):
        super().__init__()
        self.d = dimension

    def forward(self, x):
        return torch.cat(x, self.d)


class YoloV5BackBone(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.gd, self.gw = cfg.Model.depth_multiple, cfg.Model.width_multiple
        w = lambda n: make_divisible(n * self.gw, 8)  # noqa: E731
        d = lambda n: max(round(n * self.gd), 1) if n > 1 else n  # noqa: E731
        act, c_act = trunk_acts(cfg.Model.Backbone.activation)
        c1, c2, c3, c4, c5 = w(64), w(128), w(256), w(512), w(1024)
        self.stage1 = Conv(3, c1, 6, 2, 2, 1, act)
        self.stage1.is_stem = True
        self.stage2_1 = Conv(c1, c2, 3, 2, None, 1, act)
        self.stage2_2 = C3(c2, c2, d(3), True, 1, 0.5, c_act)
        self.stage3_1 = Conv(c2, c3, 3, 2, None, 1, act)
        self.stage3_2 = C3(c3, c3, d(6), True, 1, 0.5, c_act)
        self.stage4_1 = Conv(c3, c4, 3, 2, None, 1, act)
        self.stage4_2 = C3(c4, c4, d(9), True, 1, 0.5, c_act)
        self.stage5_1 = Conv(c4, c5, 3, 2, None, 1, act)
        self.stage5_2 = C3(c5, c5, d(3), True, 1, 0.5, c_act)
        self.sppf = SPPF(c5, c5, 5, act)
        self.out_shape = {'C3_size': c3, 'C4_size': c4, 'C5_size': c5}

    def forward(self, x):
        x = self.stage2_2(self.stage2_1(self.stage1(x)))
        c3 = self.stage3_2(self.stage3_1(x))
        if self.stage4_1.glue(c3):
            _fan_out(c3)          # consumed by stage4_1 and by the neck's concat (JoinFn lateral)
        c4 = self.stage4_2(self.stage4_1(c3))
        if self.stage5_1.glue(c4):
            _fan_out(c4)
        return c3, c4, self.sppf(self.stage5_2(self.stage5_1(c4)))


class YoloV5Neck(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.gd, self.gw = cfg.Model.depth_multiple, cfg.Model.width_multiple
        w = lambda n: make_divisible(n * self.gw, 8)  # noqa: E731
        d = lambda n: max(round(n * self.gd), 1) if n > 1 else n  # noqa: E731
        ip3, ip4, ip5 = [w(c) for c in cfg.Model.Neck.in_channels]
        op3, op4, op5 = [w(c) for c in cfg.Model.Neck.out_channels]
        self.input_p3, self.input_p4, self.input_p5 = ip3, ip4, ip5
        self.output_p3, self.output_p4, self.output_p5 = op3, op4, op5
        act, c_act = trunk_acts(cfg.Model.Neck.activation)
        self.conv1 = Conv(ip5, int(ip5 / 2), 1, 1, None, 1, act)
        self.upsample1 = nn.Upsample(scale_factor=2, mode="nearest")
        self.C1 = C3(int(ip5 / 2) + ip4, ip4, d(3), False, 1, 0.5, c_act)
        self.conv2 = Conv(ip4, ip3, 1, 1, None, 1, act)
        self.upsample2 = nn.Upsample(scale_factor=2, mode="nearest")
        self.C2 = C3(ip3 + ip3, op3, d(3), False, 1, 0.5, c_act)
        self.conv3 = Conv(op3, op3, 3, 2, None, 1, act)
        self.C3 = C3(op3 + ip3, op4, d(3), False, 1, 0.5, c_act)
        self.conv4 = Conv(op4, op4, 3, 2, None, 1, act)
        self.C4 = C3(op4 + int(ip5 / 2), op5, d(3), False, 1, 0.5, c_act)
        self.concat = Concat()

    def _up_cat(self, x, lateral):
        """cat([upsample2x(x), lateral], 1) by offset: the upsample writes its slice, the lateral is copied into its own."""
        from .autograd_conv import CatBuf, JoinFn, UpsampleIntoFn
        N, C_, H, W = x.shape
        cb = CatBuf(N, C_ + lateral.shape[1], 2 * H, 2 * W, x.device)
        return JoinFn.apply(cb, (False, True), UpsampleIntoFn.apply(x, cb, 0), lateral)

    def _down_cat(self, conv, x, lateral):
        """cat([conv(x), lateral], 1): the stride-2 Conv writes its slice in place."""
        from .autograd_conv import CatBuf, JoinFn
        N, _, H, W = lateral.shape
        C_ = conv.conv.out_channels
        cb = CatBuf(N, C_ + lateral.shape[1], H, W, x.device)
        return JoinFn.apply(cb, (False, True), conv(x, None, cb, 0), lateral)

    def forward(self, inputs):
        P3, P4, P5 = inputs
        xp_1 = self.conv1(P5)
        if self.conv3.glue(P5) and all(t.shape[1] % 8 == 0 for t in (xp_1, P4, P3)):
            x1 = self.C1(self._up_cat(xp_1, P4))
            xp_2 = self.conv2(x1)
            # the three outputs feed the Detect conv, netD (SSOD) and -- x2, x3 -- the next stride-2 conv: their gradients meet
            # in the dgrad epilogues (FanIn) instead of in autograd's add kernels
            x2 = _fan_out(self.C2(self._up_cat(xp_2, P3)))
            x3 = _fan_out(self.C3(self._down_cat(self.conv3, x2, xp_2)))
            x4 = _fan_out(self.C4(self._down_cat(self.conv4, x3, xp_1)))
            return x2, x3, x4
        x1 = self.C1(self.concat([self.upsample1(xp_1), P4]))
        xp_2 = self.conv2(x1)
        x2 = self.C2(self.concat([self.upsample2(xp_2), P3]))
        x3 = self.C3(self.concat([self.conv3(x2), xp_2]))
        x4 = self.C4(self.concat([self.conv4(x3), xp_1]))
        return x2, x3, x4


class Detect(nn.Module):
    """models/head/yolov5_head.py:7-87.  Train: list of [B,na,ny,nx,no]; eval: (pred [B,P,no], list)."""
    stride = None

    def __init__(self, cfg):
        super().__init__()
        self.nc = cfg.Dataset.nc
        self.num_keypoints = cfg.Dataset.np
        if self.num_keypoints:
            raise NotImplementedError("keypoint heads are out of scope")
        anchors = cfg.Model.anchors
        ch = [int(c * cfg.Model.width_multiple) for c in cfg.Model.Neck.out_channels]
        self.no = self.nc + 5
        self.nl = len(anchors)
        self.na = len(anchors[0]) // 2
        self.register_buffer('anchors', torch.tensor(anchors).float().view(self.nl, -1, 2))
        self.m = nn.ModuleList(nn.Conv2d(x, self.no * self.na, 1) for x in ch)
        self.stride = cfg.Model.Head.strides
        self.export = False

    def initialize_biases(self, cf=None):
        for mi, s in zip(self.m, self.stride):
            b = mi.bias.view(self.na, -1)
            b.data[:, 4] += math.log(8 / (640 / s) ** 2)
            b.data[:, 5:] += math.log(0.6 / (self.nc - 0.99)) if cf is None else torch.log(cf / cf.sum())
            mi.bias = torch.nn.Parameter(b.view(-1), requires_grad=True)

    def forward(self, x, packed=None):
        """packed: optional list of packing.PackedConv (Model.pack_weights(): forward + K-padded dgrad operand per level)"""
        x = list(x)
        for i in range(self.nl):
            if Conv.NATIVE and x[i].is_cuda:
                from .autograd_conv import DetectConvFn
                pc = packed[i] if (packed is not None and self.training) else None
                x[i] = DetectConvFn.apply(x[i], self.m[i].weight, self.m[i].bias, self.na, self.no,
                                          None if pc is None else pc.fwd, None if pc is None else pc.dgrad)
                continue
            x[i] = self.m[i](x[i])
            bs, _, ny, nx = x[i].shape
            x[i] = x[i].view(bs, self.na, self.no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
        if self.training:
            return x
        raw = [xi.float() for xi in x]
        return decode_levels(raw, self.anchors, [float(s) for s in self.stride]), x


class GradReverse(torch.autograd.Function):  # yolo_ssod.py:158-172
    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return -g


class netD(nn.Module):  # yolo_ssod.py:224-238
    def __init__(self, channel, ratio, context=False):
        super().__init__()
        self.ratio = ratio
        c = int(channel * ratio)
        self.conv1 = nn.Conv2d(c, c, 1, 1, 0, bias=False)
        self.conv2 = nn.Conv2d(c, 2, 1, 1, 0, bias=False)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x, reverse=False, packed=None):
        """reverse=True: x is the feature itself and the GradReverse of yolo_ssod.py:111-113 is folded into this module's
        backward (NetDFn runs conv1's dgrad on the negated operand); otherwise the caller applied GradReverse.
        packed: optional packing.PackedConv of conv1 (forward + negated dgrad operand)."""
        if Conv.NATIVE and x.is_cuda and reverse:
            from .autograd_conv import NetDFn
            pc = packed if self.training else None
            return NetDFn.apply(x, self.conv1.weight, self.conv2.weight, None if pc is None else pc.fwd, None if pc is None else pc.dgrad)
        if reverse:
            x = GradReverse.apply(x)
        return self.conv2(self.relu(self.conv1(x)))


def _check_head(model, cfg):
    m = model.head
    s = 256
    m.inplace = model.inplace
    # the reference discovers the strides with a 256x256 dummy forward (yolo_ssod.py:76-78); the YOLOv5 trunk
    # halves the resolution 3/4/5 times before the three heads, so they are 8/16/32 by construction.
    m.stride = torch.tensor([float(x) for x in cfg.Model.Head.strides])
    assert [s / (s // int(t)) for t in m.stride] == [8.0, 16.0, 32.0]
    m.anchors /= m.stride.view(-1, 1, 1)
    a = m.anchors.prod(-1).view(-1)
    if (a[-1] - a[0]).sign() != (m.stride[-1] - m.stride[0]).sign():
        m.anchors[:] = m.anchors.flip(0)
    model.stride = m.stride
    m.initialize_biases()


class _ModelBase(nn.Module):
    def _init_common(self, cfg):
        self.cfg = cfg
        self.backbone = YoloV5BackBone(cfg)
        self.neck = YoloV5Neck(cfg)
        self.head = Detect(cfg)
        self.names = cfg.Dataset.names
        self.nc = cfg.Dataset.nc
        self.inplace = cfg.Model.inplace
        self.model_type = 'yolov5'
        self.export = False
        self._engine = None
        self._packer = self._packer_aux = None
        self._state_fp32 = None

    def _require(self, x):
        _lib.require_cuda(*(x if isinstance(x, (list, tuple)) else (x,)))
        _lib.lib()

    def _apply(self, fn, *args, **kwargs):
        self._state_fp32 = None       # .half() / .float() / .to(): the next forward outside the engine checks the dtypes again
        return super()._apply(fn, *args, **kwargs)

    def _require_fp32(self):
        """The native training forward reads the parameters and the BatchNorm state as fp32 (the student trains in fp32).
        A model after .half() / .bfloat16() runs eval() under no_grad only, on the engine; anything else raises here,
        before a launch.  The scan runs once after every conversion (_apply), not per step."""
        if getattr(self, "_state_fp32", None):
            return
        for name, t in itertools.chain(self.named_parameters(), self.named_buffers()):
            if t.is_floating_point() and t.dtype != torch.float32:
                raise NotImplementedError("%s is %s: the native training forward needs an fp32 model (a .half() or .bfloat16() "
                                          "model runs in eval() under torch.no_grad())" % (name, t.dtype))
        self._state_fp32 = True

    def _stem_input(self, x):
        """x: the reference's contract (one fp32 [N,3,H,W] tensor in [0,1]) or, for the native stem, a uint8 tensor / a list of
        tensors to be concatenated along the batch (the loaders' raw batches: trainer/ssod_trainer.py:620,694-696).  On the
        native path this becomes an autograd_conv.StemInput (no cat, no fp32 image); otherwise a plain fp32 tensor."""
        parts = list(x) if isinstance(x, (list, tuple)) else [x]
        native = Conv.NATIVE and self.training and all(p.is_cuda for p in parts)
        if native and (len(parts) > 1 or parts[0].dtype == torch.uint8):
            from .autograd_conv import StemInput
            return StemInput(parts)
        if len(parts) == 1 and parts[0].dtype != torch.uint8:
            return parts[0]
        div = 255.0 if parts[0].dtype == torch.uint8 else 1.0
        t = torch.cat([p.float() for p in parts], 0)
        return t / div if div != 1.0 else t

    def pack_weights(self):
        """bf16 GEMM operands (forward + dgrad) of every Conv for this training step, in ONE launch (packing.WeightPacker);
        the Conv modules pick them up through `_packed`, the head / netD convs through the returned dict."""
        if not (Conv.NATIVE and Conv.FUSED_BN and self.training):
            return {}
        dev = next(self.parameters()).device
        pk = getattr(self, "_packer", None)
        if pk is None or pk.device != dev:
            from .packing import WeightPacker
            pk = WeightPacker(dev)
            for name, m in self.named_modules():
                if isinstance(m, Conv):
                    m._packed = pk.add(m.conv.weight, m.conv.stride[0], m.conv.padding[0], want_dgrad=not m.is_stem, stem=m.is_stem,
                                       name=name + ".conv.weight")
            aux = {"head": [pk.add(m.weight, 1, 0, want_dgrad=True, name="head.m.%d.weight" % i)      # dgrad operand K-padded (255 -> 256)
                            for i, m in enumerate(self.head.m)]}
            for d in ("det_8", "det_16", "det_32"):      # netD.conv1 behind GradReverse: dgrad operand negated (pack mode 3)
                if hasattr(self, d):
                    aux[d] = pk.add(getattr(self, d).conv1.weight, 1, 0, want_dgrad=True, negate_dgrad=True, name=d + ".conv1.weight")
            self._packer, self._packer_aux = pk, aux
        pk.run()
        return self._packer_aux

    def _count_bn_batches(self):
        """BatchNorm2d.num_batches_tracked += 1 for every BN (what nn.BatchNorm2d does per training forward), as ONE
        multi-tensor op; the fused BN kernels update running_mean / running_var themselves."""
        if Conv.NATIVE and Conv.FUSED_BN and self.training:
            if getattr(self, "_nbt", None) is None:
                self._nbt = [m.num_batches_tracked for m in self.modules() if isinstance(m, _BN)]
            torch._foreach_add_(self._nbt, 1)

    def sync_batchnorm(self, process_group=None):
        """torch.nn.SyncBatchNorm.convert_sync_batchnorm on every BatchNorm of the model, in place (the module objects that
        hold them, their parameters and their buffers stay the same).  Training forwards then normalise with the statistics
        of the global batch whenever torch's SyncBatchNorm would: a process group of more than one rank.  Returns self."""
        for name, m in list(self.named_children()):
            setattr(self, name, nn.SyncBatchNorm.convert_sync_batchnorm(m, process_group))
        self._nbt = None
        return self

    def set_bn_sync(self, sync):
        """Force parallel.BnSync `sync` (None: back to the default) on the fused BatchNorm of every Conv -- e.g.
        BnSync(loopback=True), the synced kernels at world 1.  Layers on torch's BatchNorm keep their module."""
        for m in self.modules():
            if isinstance(m, Conv):
                m.bn_sync = sync

    def engine(self):
        from .engine import TrunkEngine
        if self._engine is None:
            self._engine = TrunkEngine(self)
        return self._engine

    def __deepcopy__(self, memo):  # the engine holds raw device pointers: EMA / checkpoint copies rebuild their own
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        from copy import deepcopy
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k in ("_engine", "_nbt", "_packer", "_packer_aux") else deepcopy(v, memo)
        return new

    def __getstate__(self):
        s = dict(self.__dict__)
        s["_engine"] = None
        s["_nbt"] = None
        s["_packer"] = None
        s["_packer_aux"] = None
        return s


class Model(_ModelBase):
    """SSOD detector (models/detector/yolo_ssod.py:44-118): forward -> (head_out, [d8, d16, d32])."""

    def __init__(self, cfg):
        super().__init__()
        self._init_common(cfg)
        oc = cfg.Model.Neck.out_channels
        self.det_8 = netD(oc[0], cfg.Model.width_multiple)
        self.det_16 = netD(oc[1], cfg.Model.width_multiple)
        self.det_32 = netD(oc[2], cfg.Model.width_multiple)
        _check_head(self, cfg)

    def forward(self, x, augment=False, profile=False, visualize=False):
        self._require(x)
        if not self.training and not torch.is_grad_enabled():
            return self.engine().forward(x, with_features=True)
        self._require_fp32()
        self._count_bn_batches()
        aux = self.pack_weights()
        f = self.neck(self.backbone(self._stem_input(x)))
        out = self.head(f, aux.get("head"))
        f8, f16, f32 = f
        feature = [self.det_8(f8, True, aux.get("det_8")), self.det_16(f16, True, aux.get("det_16")), self.det_32(f32, True, aux.get("det_32"))]
        return out, feature


class SupModel(_ModelBase):
    """Supervised detector (models/detector/yolo.py:45-110): forward -> head_out."""

    def __init__(self, cfg):
        super().__init__()
        self._init_common(cfg)
        _check_head(self, cfg)

    def forward(self, x, augment=False, profile=False, visualize=False):
        self._require(x)
        if not self.training and not torch.is_grad_enabled():
            return self.engine().forward(x, with_features=False)[0]
        self._require_fp32()
        self._count_bn_batches()
        aux = self.pack_weights()
        f = self.neck(self.backbone(self._stem_input(x)))
        return self.head(f, aux.get("head"))
