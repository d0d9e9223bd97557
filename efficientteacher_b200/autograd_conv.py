"""torch.autograd bridge for the wgmma convolutions: forward = implicit-GEMM conv, backward = dgrad (same kernel,
transposed taps) + wgrad (pixel-reduction GEMM).  Tensors stay NHWC bf16 in HBM and are exposed to torch as
channels_last NCHW views (zero copy), so torch's BatchNorm/SiLU/cat/upsample/maxpool can sit between the convs while
the dense contractions (97% of the step's FLOPs, SURVEY.md 8a a1) run on the hand-written kernels.

Replaces cuDNN fprop/dgrad/wgrad behind Conv.forward (reference models/backbone/common.py:480-481), the Detect 1x1
convs (models/head/yolov5_head.py:55) and netD.conv1 (models/detector/yolo_ssod.py:228).
"""
import torch

from . import convops as co


# Optional side stream for the weight-gradient branch.  In backward, wgrad (+ its split-K reduce) of a layer depends only on
# that layer's dy and feeds nothing but the gradient arena, while the critical path continues dgrad -> previous layer's BN
# backward -> ...  With the branch on its own stream the tails of the persistent conv kernels and the many tiny launches
# (BN finalize, reduces) overlap with wgrad CTAs instead of leaving SMs idle; inside a captured CUDA graph the fork/join
# events become parallel graph branches.  Only the trainer turns it on (it joins before the all-reduce / optimizer);
# operands are kept alive until the join so the caching allocator cannot hand their memory out early.
WGRAD_SIDE = {"on": False, "stream": None, "keep": [], "dirty": False}


def wgrad_side_run(fn, keep):
    S = WGRAD_SIDE
    cur = torch.cuda.current_stream()
    if S["stream"] is None or S["stream"].device != cur.device:
        S["stream"] = torch.cuda.Stream(cur.device)
    ev = torch.cuda.Event()
    ev.record(cur)
    S["stream"].wait_event(ev)
    with torch.cuda.stream(S["stream"]):
        fn()
    S["keep"].append(keep)
    S["dirty"] = True


def backward(loss, side=True):
    """loss.backward() with the weight-gradient branch on the side stream, joined before returning"""
    WGRAD_SIDE["on"] = bool(side)
    try:
        loss.backward()
    finally:
        WGRAD_SIDE["on"] = False
        wgrad_side_join()


def wgrad_side_join():
    S = WGRAD_SIDE
    if S["dirty"]:
        ev = torch.cuda.Event()
        ev.record(S["stream"])
        torch.cuda.current_stream().wait_event(ev)
        S["keep"].clear()
        S["dirty"] = False


def _inplace_nhwc(t, C_):
    """(NHWC view, pixel stride) of a bf16 NCHW-shaped tensor that is physically NHWC (possibly a channel slice), else None"""
    N, C2, H, W = t.shape
    if t.dtype != torch.bfloat16 or C2 != C_:
        return None
    sN, sC, sH, sW = t.stride()
    if sC == 1 and sW >= C_ and sW % 8 == 0 and sH == W * sW and sN == H * W * sW and t.data_ptr() % 16 == 0:
        return t.permute(0, 2, 3, 1), sW
    return None


def _as_nhwc(t, C_):
    """(view [N,H,W,C] bf16 whose channel stride may exceed C, channel_stride) for an NCHW-shaped tensor; copies only if
    the layout is not NHWC.  A channel-slice of a channels_last tensor (what torch.cat's backward hands out) is used in
    place: the kernels take the pixel stride separately and never touch channels outside the slice."""
    N, C2, H, W = t.shape
    assert C2 == C_
    t = t.to(torch.bfloat16)
    v = _inplace_nhwc(t, C_)
    if v is None:
        t = t.contiguous(memory_format=torch.channels_last)
        if t.stride() != (H * W * C_, 1, W * C_, C_):     # degenerate shapes (H=W=1 ...): force the NHWC strides
            t = t.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
        v = t.permute(0, 2, 3, 1), C_
    return v


def _empty_cl(N, C_, H, W, device):
    """NCHW-shaped bf16 tensor with channels_last strides (physically NHWC); returned from the Functions as a real
    tensor (not a view) so downstream in-place ops (ReLU(inplace)) are legal."""
    return torch.empty((N, C_, H, W), dtype=torch.bfloat16, device=device, memory_format=torch.channels_last)


def _nhwc_of(t):
    """dense NHWC view of a tensor from _empty_cl"""
    v = _inplace_nhwc(t, t.shape[1])
    if v is None or v[1] != t.shape[1]:
        raise RuntimeError("unexpected channels_last strides %s for %s" % (t.stride(), tuple(t.shape)))
    return v[0]


class StemInput:
    """The student's input batch as the stem sees it: one or several [n_i,3,H,W] tensors (uint8 straight from the loaders,
    or fp32 already scaled) that are logically concatenated along the batch (trainer/ssod_trainer.py:620 torch.cat) and
    divided by `div` (:694-696 `.float() / 255`).  Deliberately NOT a tensor: the stem's Function receives it as an opaque argument
    and the im2col kernel reads every part in place -- neither the cat nor the fp32 image is ever materialised."""

    def __init__(self, parts, div=None):
        self.parts = [p for p in parts]
        self.div = float(div) if div is not None else (255.0 if self.parts[0].dtype == torch.uint8 else 1.0)
        self.is_cuda = all(p.is_cuda for p in self.parts)
        self.device = self.parts[0].device
        n = sum(int(p.shape[0]) for p in self.parts)
        self.shape = (n,) + tuple(self.parts[0].shape[1:])
        self.requires_grad = False

    def im2col(self):
        return co.stem_im2col_parts(self.parts, self.div)


class GradSlot:
    """Lazily allocated gradient buffer shared by the outputs of SplitBatchFn: the consumers' backward kernels write their
    gradients straight into batch slices of ONE buffer, so the split's backward is a no-op instead of zeros + 2 copies."""

    def __init__(self, like):
        self.like, self.buf = like, None

    def get(self):
        if self.buf is None:
            self.buf = torch.empty_like(self.like)       # same strides (dense): batch slices are contiguous runs
        return self.buf


def grad_buffer_for(t):
    """gradient destination for tensor t inside a native backward: its slice of a GradSlot when t came out of SplitBatchFn,
    else a fresh tensor"""
    hint = getattr(t, "_etb_gslot", None)
    if hint is None:
        return torch.empty_like(t)
    slot, a, b = hint
    return slot.get()[a:b]


class SplitBatchFn(torch.autograd.Function):
    """(t[:n], t[n:]) -- trainer/ssod_trainer.py:568-585 split_predict_and_feature -- whose backward hands the two gradients
    back as ONE tensor without copying when the consumers wrote them into the shared GradSlot (grad_buffer_for)."""

    stats = {"zero_copy": 0, "copied": 0}      # diagnostics (tests assert that the step takes the zero-copy path)

    @staticmethod
    def forward(ctx, t, n, slot):
        ctx.n, ctx.slot, ctx.like = n, slot, t
        return t[:n], t[n:]

    @staticmethod
    def backward(ctx, ga, gb):
        n, slot = ctx.n, ctx.slot
        buf = slot.buf
        if buf is not None and ga is not None and gb is not None and ga.data_ptr() == buf[:n].data_ptr() and gb.data_ptr() == buf[n:].data_ptr() \
                and ga.stride() == buf[:n].stride() and gb.stride() == buf[n:].stride():
            slot.buf = None
            SplitBatchFn.stats["zero_copy"] += 1
            return buf, None, None
        SplitBatchFn.stats["copied"] += 1
        like = ctx.like
        za = ga if ga is not None else torch.zeros_like(like[:n])
        zb = gb if gb is not None else torch.zeros_like(like[n:])
        return torch.cat([za, zb], 0), None, None


def split_batch(t, n):
    """t[:n], t[n:] with the zero-copy backward above (falls back to plain slicing for tensors that need no gradient)"""
    if not (torch.is_tensor(t) and t.requires_grad and t.is_cuda):
        return t[:n], t[n:]
    slot = GradSlot(t)
    a, b = SplitBatchFn.apply(t, n, slot)
    a._etb_gslot, b._etb_gslot = (slot, 0, n), (slot, n, t.shape[0])
    return a, b


class ZeroTermFn(torch.autograd.Function):
    """0 * (t_0.mean() + t_1.mean() + ...) for finite t_i (trainer/ssod_trainer.py:516 keeps the unlabeled Detect outputs in
    the graph that way): value 0, gradient exact zeros.  The zeros are written into each tensor's grad_buffer_for
    destination, so a batch half that came out of split_batch keeps SplitBatchFn's zero-copy backward."""

    @staticmethod
    def forward(ctx, *ts):
        ctx.ts = ts          # the tensors themselves: grad_buffer_for reads their split_batch tag
        return torch.zeros(1, dtype=torch.float32, device=ts[0].device)

    @staticmethod
    def backward(ctx, g):
        return tuple(grad_buffer_for(t).zero_() for t in ctx.ts)


class CatBuf:
    """A concat buffer [N, Ct, H, W] (channels_last = NHWC in memory).  Producers write their outputs straight into
    channel slices of `buf` (concat-by-offset, the training-side twin of engine.TrunkEngine's layout) and JoinFn turns
    the filled buffer into the autograd node the consumer sees -- torch.cat and its backward copies never run.
    Deliberately NOT a tensor: the Functions below receive it as an opaque argument, so the slice views they return
    are plain tensors to autograd (no view/in-place bookkeeping; the kernels write through raw pointers)."""

    def __init__(self, N, Ct, H, W, device):
        self.buf = _empty_cl(N, Ct, H, W, device)
        self.Ct = Ct

    def slice(self, coff, C_):
        return self.buf[:, coff:coff + C_]


class FanIn:
    """Gradient fan-in of an activation that has several native consumers (C3 input -> cv1 and cv2; Bottleneck input ->
    cv1 and the shortcut; backbone feature -> next stage and the neck's concat).  Autograd would sum the consumers'
    gradients with one ATen add per extra consumer (3 passes over the tensor each).  Instead every participating
    consumer registers in forward (`n`), and in backward the first contribution becomes the accumulation buffer, later
    convolutions ADD their dgrad into it in the kernel epilogue (etb_conv_dgrad accumulate: 1 extra read), and only the
    last participant hands the buffer to autograd -- the others return None.  Consumers that do not participate (torch
    ops) are still summed by the engine, so the result is exact in every mix."""
    __slots__ = ("n", "k", "buf")

    def __init__(self):
        self.n, self.k, self.buf = 0, 0, None

    @staticmethod
    def of(x):
        """the FanIn attached to tensor x by its producer module (None if x has a single consumer)"""
        return getattr(x, "_etb_fan", None) if x.requires_grad else None

    @staticmethod
    def join(x):
        """register a native consumer of x in forward; returns x's FanIn (None if x has a single consumer)"""
        f = FanIn.of(x)
        if f is not None:
            f.n += 1
        return f

    def done(self):
        self.k += 1
        if self.k < self.n:
            return None
        buf, self.buf = self.buf, None
        return buf

    def put(self, g):
        """pass-through contribution (shortcut / concat slice): g becomes, or is added to, the buffer"""
        self.buf = g if self.buf is None else self.buf + g
        return self.done()

    def add_dgrad(self, run, N, C_, H, W, device):
        """convolution contribution: run(out_nhwc, out_cstride, accumulate) launches the dgrad"""
        if self.buf is None:
            self.buf = input_grad(None, run, N, C_, H, W, device)
        else:
            v = _inplace_nhwc(self.buf, C_)
            if v is None:                      # layout the kernel cannot address in place: out-of-place fallback
                self.buf = self.buf + input_grad(None, run, N, C_, H, W, device)
            else:
                run(v[0], v[1], True)
        return self.done()


def input_grad(fan, run, N, C_, H, W, device):
    """the input gradient a native backward hands to autograd, from the dgrad launcher run(out_nhwc, out_cstride,
    accumulate): a fresh tensor, or -- when the input's gradient fans in -- this contribution to the FanIn buffer"""
    if fan is not None:
        return fan.add_dgrad(run, N, C_, H, W, device)
    dx = _empty_cl(N, C_, H, W, device)
    run(_nhwc_of(dx), C_, False)
    return dx


def _arena_grad(p):
    """p.grad when it is the contiguous fp32 gradient-arena view the kernels may accumulate into, else None"""
    g = p.grad
    return g if (g is not None and g.dtype == torch.float32 and g.is_contiguous()) else None


def weight_grad(p, fn, keep=None):
    """the gradient of parameter p a native backward hands to autograd, from the launcher fn(accumulate_into).  When p.grad
    is a gradient-arena view (trainer.GradArena) the result is added into it in place and autograd gets None (no separate
    AccumulateGrad pass, no temporary).  keep: the operands of a weight-gradient conv; with the side stream on, an
    in-place launch goes there and they stay alive until the join.  Launchers without `keep` stay on the current stream."""
    tgt = _arena_grad(p)
    if tgt is None:
        return fn(None)
    if keep is not None and WGRAD_SIDE["on"]:
        wgrad_side_run(lambda: fn(tgt), keep)
    else:
        fn(tgt)
    return None


def _slice_nhwc(dest, coff, C_):
    """(NHWC view of the channel slice, its pixel stride)"""
    return dest.slice(coff, C_).permute(0, 2, 3, 1), dest.Ct


class JoinFn(torch.autograd.Function):
    """torch.cat(parts, 1) where the parts with copy flag False already live in their slices of dest.buf (written by
    ConvBnActFn / UpsampleIntoFn); parts with flag True are copied in by one strided-copy kernel.  Backward hands every
    part its channel slice of the incoming gradient as a view (no copies)."""

    @staticmethod
    def forward(ctx, dest, copy_flags, *parts):
        off, splits = 0, []
        ctx.fans = []
        for p, cp in zip(parts, copy_flags):
            ctx.fans.append(FanIn.join(p) if cp else None)      # a copied-in part (backbone feature, lateral) may have other consumers
            C_ = p.shape[1]
            if cp:
                pb, pcs = _as_nhwc(p, C_)
                N, H, W, _ = pb.shape
                co.copy_slice(pb, pcs, _slice_nhwc(dest, off, C_)[0], dest.Ct, N * H * W, C_)
            splits.append(C_)
            off += C_
        assert off == dest.Ct
        ctx.splits = splits
        return dest.buf

    @staticmethod
    def backward(ctx, g):
        outs, off = [], 0
        for C_, fan in zip(ctx.splits, ctx.fans):
            gs = g[:, off:off + C_]
            outs.append(gs if fan is None else fan.put(gs))
            off += C_
        return (None, None, *outs)


class UpsampleIntoFn(torch.autograd.Function):
    """nn.Upsample(scale_factor=2, 'nearest') (models/neck/yolov5_neck.py:38,46) written into a CatBuf slice; backward =
    2x2 block sums."""

    @staticmethod
    def forward(ctx, x, dest, coff):
        N, C_, H, W = x.shape
        xb, xcs = _as_nhwc(x, C_)
        co.upsample2x(xb, C_, dest.buf.permute(0, 2, 3, 1), coff, x_cstride=xcs)
        ctx.geom = (N, C_, H, W)
        return dest.slice(coff, C_)

    @staticmethod
    def backward(ctx, g):
        N, C_, H, W = ctx.geom
        gb, gcs = _as_nhwc(g, C_)
        dx = _empty_cl(N, C_, H, W, g.device)
        co.upsample2x_bwd(gb, gcs, _nhwc_of(dx), C_)
        return dx, None, None


class SppfPoolFn(torch.autograd.Function):
    """SPPF's three cascaded MaxPool2d(5,1,2) + concat (models/backbone/common.py:702-708): x already sits in slice 0 of
    dest.buf (written by cv1); the pools fill slices 1..3 and keep their uint8 argmax; returns the whole buffer.
    Backward runs the three pool backwards in gather form, each fused with the add of the next slice's gradient."""

    @staticmethod
    def forward(ctx, x, dest):
        N, C_, H, W = x.shape
        assert dest.Ct == 4 * C_
        idx = torch.empty((3, N, H, W, C_), dtype=torch.uint8, device=x.device)
        for k in range(3):
            co.maxpool5_fwd(_slice_nhwc(dest, k * C_, C_)[0], C_, dest.Ct, _slice_nhwc(dest, (k + 1) * C_, C_)[0], dest.Ct, idx[k])
        ctx.save_for_backward(idx)
        ctx.geom = (N, C_, H, W)
        return dest.buf

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        N, C_, H, W = ctx.geom
        gb, gcs = _as_nhwc(g, 4 * C_)
        gs = [gb[..., k * C_:(k + 1) * C_] for k in range(4)]
        t2 = torch.empty((N, H, W, C_), dtype=torch.bfloat16, device=g.device)
        co.maxpool5_bwd(gs[3], gcs, idx[2], gs[2], gcs, t2, C_, C_)
        t1 = torch.empty((N, H, W, C_), dtype=torch.bfloat16, device=g.device)
        co.maxpool5_bwd(t2, C_, idx[1], gs[1], gcs, t1, C_, C_)
        dx = _empty_cl(N, C_, H, W, g.device)
        co.maxpool5_bwd(t1, C_, idx[0], gs[0], gcs, _nhwc_of(dx), C_, C_)
        return dx, None


def _conv_forward(ctx, x, weight, stride, pad, is_stem, wp, wd):
    """The convolution shared by ConvFn and ConvBnActFn: (operand saved for backward, raw output y as a channels_last
    [N,Cout,Ho,Wo] bf16 tensor).  The stem (6x6 s2 p2 on the image, a StemInput or an fp32 tensor) runs as im2col (K=108
    padded to 128) + pointwise GEMM and saves the im2col instead of the image.  wp / wd: operands from
    Model.pack_weights(), else packed here."""
    Cout = weight.shape[0]
    if is_stem:
        xs = x.im2col() if isinstance(x, StemInput) else co.stem_im2col_parts([x], 255.0 if x.dtype == torch.uint8 else 1.0)
        xb, xcs, Cin, k, st, pd = xs, 128, 128, 1, 1, 0
        wp = co.pack_stem_weight(weight) if wp is None else wp
    else:
        xs, Cin, k, st, pd = x, weight.shape[1], weight.shape[2], stride, pad
        xb, xcs = _as_nhwc(x, Cin)
        wp = co.pack_weight(weight) if wp is None else wp
    N, H, W = xb.shape[:3]
    y = _empty_cl(N, Cout, (H + 2 * pd - k) // st + 1, (W + 2 * pd - k) // st + 1, xb.device)
    co.conv_fwd(xb, wp, Cin, Cout, k, st, pd, None, None, None, x_cstride=xcs, out=_nhwc_of(y))
    ctx.conv = (stride, pad, is_stem, wd)
    return xs, y


def _conv_backward(ctx, xs, weight, dy, dycs, fan):
    """(dx, dW) of the convolution from dy [N,Ho,Wo,*] bf16 NHWC (pixel stride dycs): dgrad, then wgrad.  The image
    needs no gradient: the stem runs only the wgrad, on the saved im2col."""
    stride, pad, is_stem, wd = ctx.conv
    Cout = weight.shape[0]
    dx = dw = None
    if is_stem:
        xb, xcs, Cin, k, stride, pad = xs, 128, 128, 1, 1, 0
    else:
        Cin, k = weight.shape[1], weight.shape[2]
        if ctx.needs_input_grad[0]:
            N, _, H, W = xs.shape
            wd = co.pack_weight_dgrad(weight, stride, pad) if wd is None else wd
            dx = input_grad(fan, lambda o, ocs, acc: co.conv_dgrad(dy, wd, N, H, W, Cin, Cout, k, stride, pad, out=o, out_cstride=ocs,
                                                                   accumulate=acc, dy_cstride=dycs), N, Cin, H, W, dy.device)
        xb, xcs = _as_nhwc(xs, Cin)
    if ctx.needs_input_grad[1]:
        dw = weight_grad(weight, lambda into: co.conv_wgrad(xb, dy, Cin, Cout, k, stride, pad, stem=is_stem, x_cstride=xcs,
                                                            dy_cstride=dycs, accumulate_into=into), (xs, xb, dy))
    return dx, dw


class ConvFn(torch.autograd.Function):
    """y = conv2d(x, w) (no bias, no activation), bf16 channels_last out: the Conv modules whose BatchNorm width the fused
    kernels do not cover run it under torch BatchNorm + activation."""

    @staticmethod
    def forward(ctx, x, weight, stride, pad, is_stem, wp=None, wd=None):
        xs, y = _conv_forward(ctx, x, weight, stride, pad, is_stem, wp, wd)
        ctx.save_for_backward(xs, weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        xs, weight = ctx.saved_tensors
        dyb, dycs = _as_nhwc(dy, weight.shape[0])
        dx, dw = _conv_backward(ctx, xs, weight, dyb, dycs, None)
        return dx, dw, None, None, None, None, None


class ConvBnActFn(torch.autograd.Function):
    """a = act(BatchNorm_train(conv2d(x, w))) -- the whole Conv module (common.py:480-481) in training mode:
    wgmma conv -> per-channel batch statistics -> fused normalise+activation; backward = fused act'/BN backward (2 passes)
    -> dgrad + wgrad.  Saves x, the raw conv output and [4,C] statistics (not the normalised tensor)."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, stride, pad, eps, momentum, act, is_stem,
                wp=None, wd=None, res=None, dest=None, coff=0, sync=None):
        """res: optional shortcut tensor added after the activation (Bottleneck, common.py:499); dest/coff: optional
        CatBuf slice the activation is written into (the returned tensor is then that slice).  sync: parallel.BnSync for
        SyncBatchNorm (statistics of the global batch; their all-reduced vector, with the global count, is saved for the
        backward)."""
        ctx.fan = FanIn.join(x)
        ctx.res_fan = FanIn.join(res) if res is not None else None
        ctx.has_res = res is not None
        xs, y = _conv_forward(ctx, x, weight, stride, pad, is_stem, wp, wd)
        y = _nhwc_of(y)
        N, Ho, Wo, Cout = y.shape
        if dest is None:
            a = _empty_cl(N, Cout, Ho, Wo, y.device)
            ab, acs = _nhwc_of(a), Cout
        else:
            a = dest.slice(coff, Cout)
            ab, acs = _slice_nhwc(dest, coff, Cout)
        rb, rcs = _as_nhwc(res, Cout) if res is not None else (None, None)
        r = co.bn_forward(y, Cout, gamma.detach(), beta.detach(), running_mean, running_var, eps, momentum, act, out=ab,
                          out_cstride=acs, res=rb, res_cstride=rcs, sync=sync)
        stats = r[1]
        ctx.sync = sync
        ctx.save_for_backward(xs, weight, y, stats, r[2] if sync is not None else None)
        ctx.act = act
        ctx.bn_params = (gamma, beta)        # for their .grad (gradient arena): dgamma / dbeta are accumulated in place
        return a

    @staticmethod
    def backward(ctx, da):
        xs, weight, y, stats, global_sums = ctx.saved_tensors
        Cout = weight.shape[0]
        dab, dacs = _as_nhwc(da, Cout)
        gamma, beta = ctx.bn_params
        dy, dgamma, dbeta = co.bn_backward(dab, y, Cout, stats, ctx.act, da_cstride=dacs, dgamma_into=_arena_grad(gamma),
                                           dbeta_into=_arena_grad(beta), sync=ctx.sync, global_sums=global_sums)
        dx, dw = _conv_backward(ctx, xs, weight, dy, Cout, ctx.fan)
        dres = None
        if ctx.has_res:
            dres = da if ctx.res_fan is None else ctx.res_fan.put(da)
        return (dx, dw, dgamma, dbeta, None, None, None, None, None, None, None, None, None, None, dres, None, None, None)


class DetectConvFn(torch.autograd.Function):
    """Detect's 1x1 conv + bias, emitting fp32 logits directly in the train layout [N,na,ny,nx,no]
    (the view/permute/contiguous of models/head/yolov5_head.py:66 is fused into the epilogue).  Backward is native too:
    etb_detect_dy_pack turns the loss gradient into the bf16 NHWC operand (+ bias-gradient partials) in one pass, dgrad runs
    on the K-padded operand and joins the feature's gradient fan-in (neck conv, netD), wgrad / bias gradient are added
    into the gradient arena."""

    @staticmethod
    def forward(ctx, x, weight, bias, na, no, wp=None, wd=None):
        Cout, Cin = weight.shape[0], weight.shape[1]
        xb, xcs = _as_nhwc(x, Cin)
        N, H, W, _ = xb.shape
        out = torch.empty((N, na, H, W, no), dtype=torch.float32, device=x.device)
        co.conv_fwd(xb, wp if wp is not None else co.pack_weight(weight), Cin, Cout, 1, 1, 0, None, bias.detach().float().contiguous(), None,
                    x_cstride=xcs, det_out=out, det_no=no)
        ctx.save_for_backward(x, weight)
        ctx.meta = (na, no)
        ctx.wd, ctx.bias = wd, bias
        ctx.fan = FanIn.join(x)
        return out

    @staticmethod
    def backward(ctx, g):
        x, weight = ctx.saved_tensors
        na, no = ctx.meta
        Cout, Cin = weight.shape[0], weight.shape[1]
        N, _, H, W, _ = g.shape
        if g.dtype != torch.float32 or not g.is_contiguous():
            g = g.float().contiguous()
        kpad = (Cout + 63) // 64 * 64          # dgrad contracts over K = Cout: padded to the 64-channel K block
        dyb, partials = co.detect_dy_pack(g, kpad)
        dx = dw = db = None
        if ctx.needs_input_grad[2]:
            db = weight_grad(ctx.bias, lambda into: co.column_sum(partials, out=into, accumulate=True))
        if ctx.needs_input_grad[0]:
            wd = ctx.wd if ctx.wd is not None else co.pack_weight_dgrad(weight, 1, 0)    # Cout zero-padded to kpad
            dx = input_grad(ctx.fan, lambda o, ocs, acc: co.conv_dgrad(dyb, wd, N, H, W, Cin, kpad, 1, 1, 0, out=o, out_cstride=ocs,
                                                                       accumulate=acc), N, Cin, H, W, g.device)
        if ctx.needs_input_grad[1]:
            xb, xcs = _as_nhwc(x, Cin)
            dw = weight_grad(weight, lambda into: co.conv_wgrad(xb, dyb, Cin, Cout, 1, 1, 0, x_cstride=xcs, accumulate_into=into),
                             (x, xb, dyb))
        return dx, dw, db, None, None, None, None


class NetDFn(torch.autograd.Function):
    """netD behind GradReverse (models/detector/yolo_ssod.py:105-118,158-172,224-238): o = conv2(relu(conv1(x))) with the
    gradient of x negated.  conv1 = wgmma GEMM with the ReLU in its epilogue; conv2 (C -> 2) = etb_netd_tail_fwd; the map is
    returned as an NCHW-shaped view [N,2,H,W] of the fp32 [N,H,W,2] buffer.  Backward: etb_netd_tail_bwd (dh with the ReLU
    mask, dW2 partials), conv1 wgrad into the arena, and conv1 dgrad on the NEGATED operand (pack mode 3) so the sign flip
    of GradReverse costs nothing and the result joins the feature's gradient fan-in."""

    @staticmethod
    def forward(ctx, x, w1, w2, wp1=None, wd1n=None):
        C_ = w1.shape[0]
        xb, xcs = _as_nhwc(x, C_)
        N, H, W, _ = xb.shape
        h = torch.empty((N, H, W, C_), dtype=torch.bfloat16, device=x.device)
        co.conv_fwd(xb, wp1 if wp1 is not None else co.pack_weight(w1), C_, C_, 1, 1, 0, None, None, "relu", x_cstride=xcs, out=h)
        w2f = w2.detach().float().contiguous()
        o = co.netd_tail_fwd(h, C_, w2f)
        ctx.save_for_backward(x, w1, w2, h)
        ctx.wd1n = wd1n
        ctx.fan = FanIn.join(x)
        return o.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, g):
        x, w1, w2, h = ctx.saved_tensors
        C_ = w1.shape[0]
        N, H, W, _ = h.shape
        do = g.permute(0, 2, 3, 1)
        if do.dtype != torch.float32 or not do.is_contiguous():
            do = do.float().contiguous()
        dh, partials = co.netd_tail_bwd(do, h, C_, w2.detach().float().contiguous())
        dx = dw1 = dw2 = None
        if ctx.needs_input_grad[2]:
            dw2 = weight_grad(w2, lambda into: co.column_sum(partials, out=into, accumulate=True).view_as(w2))
        if ctx.needs_input_grad[0]:
            wd = ctx.wd1n if ctx.wd1n is not None else co.pack_weight_dgrad(w1, 1, 0, negate=True)
            dx = input_grad(ctx.fan, lambda o, ocs, acc: co.conv_dgrad(dh, wd, N, H, W, C_, C_, 1, 1, 0, out=o, out_cstride=ocs,
                                                                       accumulate=acc), N, C_, H, W, g.device)
        if ctx.needs_input_grad[1]:
            xb, xcs = _as_nhwc(x, C_)
            dw1 = weight_grad(w1, lambda into: co.conv_wgrad(xb, dh, C_, C_, 1, 1, 0, x_cstride=xcs, accumulate_into=into), (x, xb, dh))
        return dx, dw1, dw2, None, None
