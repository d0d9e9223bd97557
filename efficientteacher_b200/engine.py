"""Native inference engine for the YOLOv5 trunk + Detect head: the teacher-EMA forward of the SSOD step
(trainer/ssod_trainer.py:595-599 -> models/detector/yolo_ssod.py:105-118) on hand-written sm_90a kernels.

Data layout: every activation is NHWC bf16 in HBM.  torch.cat never happens: producers write straight into the
channel slice of the consumer's concat buffer (C3's [m(cv1(x)), cv2(x)], SPPF's [x,y1,y2,y3], the PANet concats),
and the 2x nearest upsample writes into its slice too.  BatchNorm (eval) is folded into a per-channel scale/bias
applied, with the activation (SiLU, ReLU or Hardswish) and the Bottleneck shortcut, in the convolution epilogue.  The Detect 1x1 convs write fp32
logits directly in the [B,na,ny,nx,no] layout, and the eval decode writes the concatenated [B,P,no] prediction.
"""
import torch

from . import _lib
from . import convops as co
from .head import decode_levels
from .model import native_act


class _ConvParams:
    """Packed bf16 weights + folded BN of one Conv (refreshed on demand from the nn.Parameters: fp32, or fp16 / bf16 after
    model.half() / model.bfloat16())."""

    def __init__(self, mod, stem=False, name=""):
        self.mod, self.stem, self.name = mod, stem, name
        conv = mod.conv if hasattr(mod, "conv") else mod
        self.conv = conv
        self.bn = getattr(mod, "bn", None)
        self.Cout, self.Cin = conv.weight.shape[0], conv.weight.shape[1]
        self.k, self.s, self.p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        self.act = native_act(getattr(mod, "act", None))
        self.w = self.scale = self.bias = None
        self._pb = None

    def register(self, packer):
        cname = self.name + ".conv" if hasattr(self.mod, "conv") else self.name
        pc = packer.add(self.conv.weight, self.s, self.p, want_dgrad=False, stem=self.stem, name=cname + ".weight")
        self.w = pc.fwd
        if self.bn is not None:
            packer.add_fold(self.bn, pc, name=self.name + ".bn")
            self.scale, self.bias = pc.scale, pc.bias
        elif self.conv.bias is not None:
            self._pb = packer.add_bias(self.conv, name=cname + ".bias")
        self._pc = pc

    def refresh_bias(self):
        """the epilogue reads an fp32 bias: the parameter itself, or the copy the pack launch made of an fp16 / bf16 one"""
        if self.bn is None and self.conv.bias is not None:
            b = self.conv.bias.detach()
            self.scale, self.bias = None, (b if b.dtype == torch.float32 else self._pb.fp32)


class TrunkEngine:
    def __init__(self, model):
        self.model = model
        self.ssod = hasattr(model, "det_8")
        self.params = {}
        for name, mod in model.named_modules():
            if hasattr(mod, "conv") and hasattr(mod, "bn"):
                self.params[name] = _ConvParams(mod, stem=(name == "backbone.stage1"), name=name)
        for i, m in enumerate(model.head.m):
            self.params["head.m.%d" % i] = _ConvParams(m, name="head.m.%d" % i)
        if self.ssod:
            for d in ("det_8", "det_16", "det_32"):
                self.params[d + ".conv1"] = _ConvParams(getattr(model, d).conv1, name=d + ".conv1")
                self.params[d + ".conv2"] = _ConvParams(getattr(model, d).conv2, name=d + ".conv2")
            for d in ("det_8", "det_16", "det_32"):
                self.params[d + ".conv1"].act = "relu"
        for q in self.params.values():
            if q.Cin % 8 != 0 and not q.stem:
                raise NotImplementedError("wgmma conv path needs Cin %% 8 == 0 (16 B rows; got %d)" % q.Cin)
        self.launches = 0
        self.packer = None

    # -- helpers ------------------------------------------------------------------------------------------
    def refresh(self):
        """Re-pack weights / re-fold BN from the current parameters (the EMA teacher changes every step).  fp32, fp16 and
        bf16 state is read as stored; any other dtype raises NotImplementedError before anything is launched."""
        if self.packer is None or self.packer.device != next(self.model.parameters()).device:
            from .packing import WeightPacker
            self.packer = WeightPacker(next(self.model.parameters()).device)
            for q in self.params.values():
                q.register(self.packer)
        self.packer.run()                      # ONE pack launch + ONE BN-fold launch for the whole model
        for q in self.params.values():
            q.refresh_bias()
        self.launches += 2

    def _conv(self, name, x, x_coffset=0, out=None, out_coffset=0, residual=None, res_coffset=0, cin=None):
        q = self.params[name]
        self.launches += 1
        k, st, pd = (1, 1, 0) if q.stem else (q.k, q.s, q.p)   # the stem runs as a pointwise GEMM over its im2col buffer
        return co.conv_fwd(x, q.w, q.Cin if cin is None else cin, q.Cout, k, st, pd, q.scale, q.bias, q.act, out=out,
                           out_coffset=out_coffset, x_coffset=x_coffset, residual=residual, res_coffset=res_coffset)

    def _c3(self, prefix, x, x_coffset, c_in, out=None, out_coffset=0):
        """C3 (common.py:566-592): cv3(cat(m(cv1(x)), cv2(x))).  x logical channels [x_coffset, x_coffset+c_in)."""
        mod = self.model.get_submodule(prefix)
        c_ = mod.cv1.conv.weight.shape[0]
        N, H, W, _ = x.shape
        cat = co.nhwc_empty(N, H, W, 2 * c_, x.device)
        self._conv(prefix + ".cv2", x, x_coffset, out=cat, out_coffset=c_)
        n = len(mod.m)
        t = self._conv(prefix + ".cv1", x, x_coffset, out=(cat if n == 0 else None), out_coffset=0)
        for i, b in enumerate(mod.m):
            u = self._conv("%s.m.%d.cv1" % (prefix, i), t)
            last = (i == n - 1)
            dst = cat if last else co.nhwc_empty(N, H, W, c_, x.device)
            self._conv("%s.m.%d.cv2" % (prefix, i), u, out=dst, out_coffset=0, residual=(t if b.add else None), res_coffset=0)
            t = dst
        return self._conv(prefix + ".cv3", cat, out=out, out_coffset=out_coffset)

    # -- forward ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x, with_features=True, refresh=True, decode=True):
        """x [N,3,H,W] fp32 or fp16 (already /255) or uint8 -> ((pred [N,P,no], [raw levels]), features) like Model.forward
        in eval.  The outputs are fp32 whatever the model's and the image's dtype."""
        _lib.require_cuda(x)
        m = self.model
        if refresh:
            self.refresh()
        N, _, H, W = x.shape
        assert H % 32 == 0 and W % 32 == 0
        dev = x.device
        bb, nk = m.backbone, m.neck
        c3c, c4c, c5c = bb.out_shape['C3_size'], bb.out_shape['C4_size'], bb.out_shape['C5_size']
        half5 = nk.conv1.conv.weight.shape[0]
        ip3 = nk.conv2.conv.weight.shape[0]
        # concat buffers that receive producers from far away
        cat1 = co.nhwc_empty(N, H // 16, W // 16, half5 + c4c, dev)   # [up(xp_1), P4]      yolov5_neck.py:93
        cat2 = co.nhwc_empty(N, H // 8, W // 8, ip3 + c3c, dev)       # [up(xp_2), P3]      :98
        cat3 = co.nhwc_empty(N, H // 16, W // 16, nk.output_p3 + ip3, dev)   # [conv3(x2), xp_2]   :102
        cat4 = co.nhwc_empty(N, H // 32, W // 32, nk.output_p4 + half5, dev)  # [conv4(x3), xp_1]   :106
        # backbone (yolov5_backbone.py:76-88)
        # uint8 = the loaders' raw batch (value / 255 inside the im2col kernel); fp32 = the reference contract (already scaled);
        # fp16 = val.py's `img.half() / 255` with a .half() model, read as stored
        col = co.stem_im2col_parts([x], 255.0 if x.dtype == torch.uint8 else 1.0)
        self.launches += 1
        x1 = self._conv("backbone.stage1", col, cin=128)
        x21 = self._conv("backbone.stage2_1", x1)
        x22 = self._c3("backbone.stage2_2", x21, 0, x21.shape[3])
        x31 = self._conv("backbone.stage3_1", x22)
        self._c3("backbone.stage3_2", x31, 0, x31.shape[3], out=cat2, out_coffset=ip3)           # P3 lives in cat2
        x41 = self._conv("backbone.stage4_1", cat2, x_coffset=ip3)
        self._c3("backbone.stage4_2", x41, 0, x41.shape[3], out=cat1, out_coffset=half5)         # P4 lives in cat1
        x51 = self._conv("backbone.stage5_1", cat1, x_coffset=half5)
        x5 = self._c3("backbone.stage5_2", x51, 0, x51.shape[3])
        cq = bb.sppf.cv1.conv.weight.shape[0]
        sp = co.nhwc_empty(N, H // 32, W // 32, 4 * cq, dev)
        self._conv("backbone.sppf.cv1", x5, out=sp, out_coffset=0)
        co.sppf_pool(sp, cq)
        self.launches += 1
        p5 = self._conv("backbone.sppf.cv2", sp)
        # neck (yolov5_neck.py:88-109)
        self._conv("neck.conv1", p5, out=cat4, out_coffset=nk.output_p4)                         # xp_1
        co.upsample2x(cat4, half5, cat1, 0, x_coffset=nk.output_p4)
        n1 = self._c3("neck.C1", cat1, 0, cat1.shape[3])
        self._conv("neck.conv2", n1, out=cat3, out_coffset=nk.output_p3)                         # xp_2
        co.upsample2x(cat3, ip3, cat2, 0, x_coffset=nk.output_p3)
        self.launches += 2
        f8 = self._c3("neck.C2", cat2, 0, cat2.shape[3])
        self._conv("neck.conv3", f8, out=cat3, out_coffset=0)
        f16 = self._c3("neck.C3", cat3, 0, cat3.shape[3])
        self._conv("neck.conv4", f16, out=cat4, out_coffset=0)
        f32_ = self._c3("neck.C4", cat4, 0, cat4.shape[3])
        feats = (f8, f16, f32_)
        # Detect (yolov5_head.py:47-87): 1x1 conv + bias written as fp32 [N,na,ny,nx,no]
        head = m.head
        raw = []
        for i, f in enumerate(feats):
            q = self.params["head.m.%d" % i]
            out = torch.empty((N, head.na, f.shape[1], f.shape[2], head.no), dtype=torch.float32, device=dev)
            co.conv_fwd(f, q.w, q.Cin, q.Cout, 1, 1, 0, None, q.bias, None, det_out=out, det_no=head.no)
            self.launches += 1
            raw.append(out)
        pred = None
        if decode:
            pred = decode_levels(raw, head.anchors, [float(s) for s in head.stride])
            self.launches += len(raw)
        if not (self.ssod and with_features):
            return (pred, raw), None
        feature = []
        for d, f in zip(("det_8", "det_16", "det_32"), feats):   # netD on the (gradient-reversed) features
            h = self._conv(d + ".conv1", f)
            o8 = co.nhwc_empty(N, f.shape[1], f.shape[2], 8, dev)
            q = self.params[d + ".conv2"]
            co.conv_fwd(h, q.w, q.Cin, q.Cout, 1, 1, 0, None, None, None, out=o8, out_coffset=0)
            self.launches += 2
            feature.append(co.to_nchw_f32(o8, 2, 0))
        return (pred, raw), feature
