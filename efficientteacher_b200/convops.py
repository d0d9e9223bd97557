"""Thin Python wrappers over the wgmma convolution and the trunk layout kernels (NHWC bf16 tensors)."""
import ctypes as C

import torch

from . import _lib
from ._lib import EtbConvParams
from .packing import WeightPacker

# activation codes of the conv epilogue and the BatchNorm kernels (include/etb200.h); 3 is not a code
ACT = {None: 0, "none": 0, "silu": 1, "relu": 2, "hard_swish": 4}


def nhwc_empty(N, H, W, C, device):
    return torch.empty((N, H, W, C), dtype=torch.bfloat16, device=device)


def to_nhwc_bf16(x_nchw, out=None, coffset=0, mul=1.0):
    _lib.require_cuda(x_nchw)
    x = x_nchw.float().contiguous()
    N, Cc, H, W = x.shape
    if out is None:
        out = nhwc_empty(N, H, W, Cc, x.device)
    _lib.check(_lib.lib().etb_nchw_f32_to_nhwc_bf16(_lib.ptr(x), _lib.ptr(out), N, Cc, H, W, out.shape[3], coffset,
                                                    float(mul), _lib.stream_ptr()), "etb_nchw_f32_to_nhwc_bf16")
    return out


def to_nchw_f32(x_nhwc, C_=None, coffset=0):
    N, H, W, cs = x_nhwc.shape
    Cc = cs - coffset if C_ is None else C_
    y = torch.empty((N, Cc, H, W), dtype=torch.float32, device=x_nhwc.device)
    _lib.check(_lib.lib().etb_nhwc_bf16_to_nchw_f32(_lib.ptr(x_nhwc), _lib.ptr(y), N, Cc, H, W, cs, coffset,
                                                    _lib.stream_ptr()), "etb_nhwc_bf16_to_nchw_f32")
    return y


def _pack_one(w_oihw, stride=1, pad=0, stem=False, dgrad=False, negate=False):
    """packing.PackedConv of one weight, from a one-shot WeightPacker (the etb_pack_multi layouts).  The packer uploads its
    descriptor table, which a stream capture does not allow: captured steps take their operands from Model.pack_weights."""
    assert not torch.cuda.is_current_stream_capturing(), "one-shot weight packing inside a stream capture"
    w = w_oihw.detach().float().contiguous()
    pk = WeightPacker(w.device)
    pc = pk.add(w, stride, pad, want_dgrad=dgrad, stem=stem, negate_dgrad=negate)
    pk.run()
    return pc


def pack_weight(w_oihw):
    """[Cout,Cin,k,k] -> forward operand [Cout][k*k*ceil64(Cin)] bf16: every tap padded to the 64-channel K block"""
    return _pack_one(w_oihw).fwd


def pack_stem_weight(w_oihw):
    """[Cout,3,6,6] -> stem operand [Cout][128] bf16 in the stem_im2col_parts K order"""
    assert tuple(w_oihw.shape[1:]) == (3, 6, 6)
    return _pack_one(w_oihw, stem=True).fwd


def _conv_params(N, H, W, Cin, Cout, k, stride, pad, **fields):
    """EtbConvParams of a k x k convolution; `fields` sets the remaining members (pixel strides, offsets, act, det_no)"""
    return EtbConvParams(N=N, H=H, W=W, Cin=Cin, Cout=Cout, kh=k, kw=k, stride=stride, pad=pad, **fields)


def conv_fwd(x, w_packed, Cin, Cout, k, stride, pad, scale=None, bias=None, act="silu", out=None, out_coffset=0,
             x_coffset=0, residual=None, res_coffset=0, det_out=None, det_no=0, x_cstride=None):
    """x: [N,H,W,Cs] bf16 NHWC (logical channels [x_coffset, x_coffset+Cin)).  Returns `out` (bf16 NHWC, written at
    channel offset out_coffset) or det_out (fp32 [N,na,Ho,Wo,det_no])."""
    _lib.require_cuda(x, w_packed)
    N, H, W, cs = x.shape
    if x_cstride is not None:     # x is a strided channel-slice view: pixel stride given explicitly
        cs = x_cstride
    Ho = (H + 2 * pad - k) // stride + 1
    Wo = (W + 2 * pad - k) // stride + 1
    cp = _conv_params(N, H, W, Cin, Cout, k, stride, pad, x_cstride=cs, act=ACT[act], det_no=det_no)
    xp = x.data_ptr() + 2 * x_coffset
    if det_out is None:
        if out is None:
            out = nhwc_empty(N, Ho, Wo, Cout, x.device)
        assert tuple(out.shape[:3]) == (N, Ho, Wo)
        cp.y_cstride, cp.y_coffset = out.shape[3], out_coffset
    if residual is not None:
        cp.res_cstride, cp.res_coffset = residual.shape[3], res_coffset
    _lib.check(_lib.lib().etb_conv_fwd(C.c_void_p(xp), _lib.ptr(w_packed), _lib.ptr(scale), _lib.ptr(bias), _lib.ptr(residual),
                                       _lib.ptr(out) if det_out is None else C.c_void_p(0), _lib.ptr(det_out), C.byref(cp),
                                       _lib.stream_ptr()), "etb_conv_fwd")
    return out if det_out is None else det_out


def sppf_pool(buf, Cq):
    N, H, W, cs = buf.shape
    _lib.check(_lib.lib().etb_sppf_pool(_lib.ptr(buf), N, H, W, Cq, cs, _lib.stream_ptr()), "etb_sppf_pool")
    return buf


def upsample2x(x, Cc, out, out_coffset, x_coffset=0, x_cstride=None):
    N, H, W, cs = x.shape
    if x_cstride is not None:     # x is a strided channel-slice view: pixel stride given explicitly
        cs = x_cstride
    _lib.check(_lib.lib().etb_upsample2x_nhwc(_lib.ptr(x), _lib.ptr(out), N, H, W, Cc, cs, x_coffset, out.shape[3], out_coffset,
                                              _lib.stream_ptr()), "etb_upsample2x_nhwc")
    return out


def pack_weight_dgrad(w_oihw, stride, pad, negate=False):
    """[Cout,Cin,k,k] -> the etb_conv_dgrad operand: per parity class (packing.dgrad_classes) a [Cin][ntaps][ceil64(Cout)]
    bf16 block, concatenated (Cin*k*k*ceil64(Cout) elements).  negate: the operand of -W (a conv behind GradReverse)."""
    return _pack_one(w_oihw, stride, pad, dgrad=True, negate=negate).dgrad


def conv_dgrad(dy, wd_packed, N, H, W, Cin, Cout, k, stride, pad, out=None, out_coffset=0, dy_coffset=0, accumulate=False,
               dy_cstride=None, out_cstride=None):
    """dy: [N,Ho,Wo,Cs] bf16 NHWC (channels [dy_coffset, +Cout)) -> dx [N,H,W,*] bf16 at channel offset out_coffset."""
    _lib.require_cuda(dy, wd_packed)
    if out is None:
        out = nhwc_empty(N, H, W, Cin, dy.device)
    cp = _conv_params(N, H, W, Cin, Cout, k, stride, pad, x_cstride=dy.shape[3] if dy_cstride is None else dy_cstride,
                      y_cstride=out.shape[3] if out_cstride is None else out_cstride, y_coffset=out_coffset)
    _lib.check(_lib.lib().etb_conv_dgrad(C.c_void_p(dy.data_ptr() + 2 * dy_coffset), _lib.ptr(wd_packed), _lib.ptr(out), C.byref(cp),
                                         int(accumulate), _lib.stream_ptr()), "etb_conv_dgrad")
    return out


def conv_wgrad(x, dy, Cin, Cout, k, stride, pad, x_coffset=0, dy_coffset=0, stem=False, x_cstride=None, dy_cstride=None,
               accumulate_into=None):
    """x [N,H,W,*] bf16, dy [N,Ho,Wo,*] bf16 -> dW [Cout,Cin,k,k] fp32 (parameter layout).
    accumulate_into: an existing contiguous fp32 gradient of that shape (the arena view p.grad): dW is ADDED into it and
    returned (saves the separate AccumulateGrad pass)."""
    _lib.require_cuda(x, dy)
    N, H, W, xcs = x.shape
    cp = _conv_params(N, H, W, Cin, Cout, k, stride, pad, x_cstride=xcs if x_cstride is None else x_cstride,
                      y_cstride=dy.shape[3] if dy_cstride is None else dy_cstride)
    lib = _lib.lib()
    xp, dyp = C.c_void_p(x.data_ptr() + 2 * x_coffset), C.c_void_p(dy.data_ptr() + 2 * dy_coffset)
    acc = accumulate_into
    if acc is not None and not (acc.is_contiguous() and acc.dtype == torch.float32):
        acc = None
    shape = (Cout, 3, 6, 6) if stem else (Cout, Cin, k, k)
    out = acc if acc is not None else torch.empty(shape, dtype=torch.float32, device=x.device)
    ws = torch.empty(int(lib.etb_conv_wgrad_workspace_bytes(C.byref(cp))), dtype=torch.uint8, device=x.device)
    flags = (1 if stem else 0) | (2 if acc is not None else 0)
    _lib.check(lib.etb_conv_wgrad(xp, dyp, _lib.ptr(out), C.byref(cp), flags, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "etb_conv_wgrad")
    return out


# ---- training-mode BatchNorm + activation around the convs (csrc/bn.cu) ----


def bn_forward(y, C_, gamma, beta, running_mean, running_var, eps, momentum, act, y_cstride=None, out=None, out_cstride=None,
               res=None, res_cstride=None, sync=None):
    """y [N,H,W,*] bf16 raw conv output -> (a bf16 same geometry, stats [4,C] fp32 = scale, shift, mean, invstd).
    `out` may be a channel slice of a wider NHWC buffer (pass its pixel stride as out_cstride); `res` (same for
    res_cstride) is added after the activation (Bottleneck shortcut).
    sync (parallel.BnSync): SyncBatchNorm -- the statistics are those of the global batch (etb_bn_stats_sums, SUM
    all-reduce of [2C+1] fp64, etb_bn_finalize_global) and the result is (a, stats, global_sums): bn_backward reads the
    global count from global_sums on the device."""
    N, H, W, cs = y.shape
    if y_cstride is not None:
        cs = y_cstride
    M = N * H * W
    lib = _lib.lib()
    rows = int(lib.etb_bn_partial_rows(M, C_, 0))
    partials = torch.empty((rows, 2, C_), dtype=torch.float32, device=y.device)
    stats = torch.empty((4, C_), dtype=torch.float32, device=y.device)
    st_ptrs = (_lib.ptr(stats[0]), _lib.ptr(stats[1]), _lib.ptr(stats[2]), _lib.ptr(stats[3]))
    if sync is None:
        _lib.check(lib.etb_bn_stats(_lib.ptr(y), M, C_, cs, _lib.ptr(partials), rows, _lib.stream_ptr()), "etb_bn_stats")
        _lib.check(lib.etb_bn_finalize(_lib.ptr(partials), rows, M, C_, _lib.ptr(gamma), _lib.ptr(beta), float(eps), float(momentum),
                                       _lib.ptr(running_mean), _lib.ptr(running_var), *st_ptrs, _lib.stream_ptr()), "etb_bn_finalize")
    else:
        sums = torch.empty(2 * C_ + 1, dtype=torch.float64, device=y.device)
        _lib.check(lib.etb_bn_stats_sums(_lib.ptr(y), M, C_, cs, _lib.ptr(partials), rows, _lib.ptr(sums), _lib.stream_ptr()),
                   "etb_bn_stats_sums")
        sync.all_reduce(sums)
        _lib.check(lib.etb_bn_finalize_global(_lib.ptr(sums), C_, _lib.ptr(gamma), _lib.ptr(beta), float(eps), float(momentum),
                                              _lib.ptr(running_mean), _lib.ptr(running_var), *st_ptrs, _lib.stream_ptr()),
                   "etb_bn_finalize_global")
    if out is None:
        out = nhwc_empty(N, H, W, C_, y.device)
    ocs = out.shape[3] if out_cstride is None else out_cstride
    _lib.check(lib.etb_bn_act_apply_res(_lib.ptr(y), _lib.ptr(stats[0]), _lib.ptr(stats[1]), None if res is None else _lib.ptr(res),
                                        _lib.ptr(out), M, C_, cs, 0 if res is None else (res.shape[3] if res_cstride is None else res_cstride),
                                        ocs, ACT[act], _lib.stream_ptr()), "etb_bn_act_apply_res")
    return (out, stats) if sync is None else (out, stats, sums)


def bn_backward(da, y, C_, stats, act, da_cstride=None, y_cstride=None, out=None, dgamma_into=None, dbeta_into=None, sync=None,
                global_sums=None):
    """da, y [N,H,W,*] bf16 -> (dy_raw bf16 [N,H,W,C], dgamma [C], dbeta [C]).  With dgamma_into / dbeta_into (the
    parameters' fp32 .grad in the gradient arena) the two sums are ADDED in place by the finalize kernel and
    (dy, None, None) is returned -- no AccumulateGrad add kernels.
    sync / global_sums (the BnSync and the all-reduced [2C+1] of the synced forward): the sums [2C] are SUM all-reduced
    before the apply, which divides by the global count global_sums[2C]; dgamma / dbeta stay this rank's own (torch's
    SyncBatchNorm returns them so, and the gradient all-reduce sums them)."""
    N, H, W, ycs = y.shape
    if y_cstride is not None:
        ycs = y_cstride
    dacs = da.shape[3] if da_cstride is None else da_cstride
    M = N * H * W
    lib = _lib.lib()
    rows = int(lib.etb_bn_partial_rows(M, C_, 1))
    partials = torch.empty((rows, 2, C_), dtype=torch.float32, device=y.device)
    _lib.check(lib.etb_bn_act_bwd_reduce(_lib.ptr(da), _lib.ptr(y), _lib.ptr(stats[0]), _lib.ptr(stats[1]), _lib.ptr(stats[2]),
                                         _lib.ptr(stats[3]), M, C_, dacs, ycs, ACT[act], _lib.ptr(partials), rows, _lib.stream_ptr()),
               "etb_bn_act_bwd_reduce")
    sums = torch.empty(2 * C_, dtype=torch.float32, device=y.device)
    acc = dgamma_into is not None and dbeta_into is not None
    dgb = None if acc else torch.empty((2, C_), dtype=torch.float32, device=y.device)
    _lib.check(lib.etb_bn_act_bwd_finalize(_lib.ptr(partials), rows, C_, _lib.ptr(sums), _lib.ptr(dgamma_into if acc else dgb[0]),
                                           _lib.ptr(dbeta_into if acc else dgb[1]), 1 if acc else 0, _lib.stream_ptr()),
               "etb_bn_act_bwd_finalize")
    if out is None:
        out = nhwc_empty(N, H, W, C_, y.device)
    if sync is None:
        _lib.check(lib.etb_bn_act_bwd_apply(_lib.ptr(da), _lib.ptr(y), _lib.ptr(stats[0]), _lib.ptr(stats[1]), _lib.ptr(stats[2]),
                                            _lib.ptr(stats[3]), _lib.ptr(sums), M, C_, dacs, ycs, out.shape[3], ACT[act], _lib.ptr(out),
                                            _lib.stream_ptr()), "etb_bn_act_bwd_apply")
    else:
        sync.all_reduce(sums)
        _lib.check(lib.etb_bn_act_bwd_apply_global(_lib.ptr(da), _lib.ptr(y), _lib.ptr(stats[0]), _lib.ptr(stats[1]), _lib.ptr(stats[2]),
                                                   _lib.ptr(stats[3]), _lib.ptr(sums), _lib.ptr(global_sums), M, C_, dacs, ycs,
                                                   out.shape[3], ACT[act], _lib.ptr(out), _lib.stream_ptr()), "etb_bn_act_bwd_apply_global")
    return (out, None, None) if acc else (out, dgb[0], dgb[1])


def maxpool5_fwd(x, C_, x_cstride, y, y_cstride, idx):
    """5x5 s1 p2 max pool of the NHWC slice x (pixel stride x_cstride) into the slice y; idx [N,H,W,C] uint8 argmax."""
    N, H, W, _ = x.shape
    _lib.check(_lib.lib().etb_maxpool5_fwd(_lib.ptr(x), _lib.ptr(y), _lib.ptr(idx), N, H, W, C_, x_cstride, y_cstride, _lib.stream_ptr()),
               "etb_maxpool5_fwd")


def maxpool5_bwd(src, src_cstride, idx, add, add_cstride, out, out_cstride, C_):
    """out = add + maxpool5-backward(src) through idx (gather form); add may be None."""
    N, H, W, _ = src.shape
    _lib.check(_lib.lib().etb_maxpool5_bwd(_lib.ptr(src), _lib.ptr(idx), None if add is None else _lib.ptr(add), _lib.ptr(out), N, H, W, C_,
                                           src_cstride, add_cstride if add is not None else 8, out_cstride, _lib.stream_ptr()),
               "etb_maxpool5_bwd")


def upsample2x_bwd(dy, dy_cstride, dx, C_):
    """dx [N,H,W,C] = 2x2 block sums of dy [N,2H,2W,*]."""
    N, H, W, _ = dx.shape
    _lib.check(_lib.lib().etb_upsample2x_bwd(_lib.ptr(dy), _lib.ptr(dx), N, H, W, C_, dy_cstride, dx.shape[3], _lib.stream_ptr()),
               "etb_upsample2x_bwd")


def copy_slice(x, x_cstride, y, y_cstride, M, C_):
    _lib.check(_lib.lib().etb_copy_slice_nhwc(_lib.ptr(x), _lib.ptr(y), M, C_, x_cstride, y_cstride, _lib.stream_ptr()),
               "etb_copy_slice_nhwc")


# ---- the tail of the student's step (csrc/tail.cu) ----
def stem_im2col_parts(parts, div=1.0):
    """im2col of the stem over the batch-concatenation of `parts` ([n_i,3,H,W] uint8, fp32 or fp16 tensors, read as they
    are; any other dtype goes through .float()) WITHOUT materialising torch.cat: every part is written into its image slots
    of one [sum n_i, H/2, W/2, 128] buffer.  Values are x / div."""
    _lib.require_cuda(*parts)
    H, W = parts[0].shape[2:]
    n_tot = sum(int(p.shape[0]) for p in parts)
    out = nhwc_empty(n_tot, H // 2, W // 2, 128, parts[0].device)
    off = 0
    for p in parts:
        assert p.shape[1] == 3 and tuple(p.shape[2:]) == (H, W)
        if p.dtype not in _lib.ETB_STEM_SRC:
            p = p.float()
        p = p.contiguous()
        if p.shape[0]:
            _lib.check(_lib.lib().etb_stem_im2col_into(_lib.ptr(p), _lib.ETB_STEM_SRC[p.dtype], _lib.ptr(out), int(p.shape[0]), H, W, off,
                                                       float(div), _lib.stream_ptr()), "etb_stem_im2col_into")
        off += int(p.shape[0])
    return out


def detect_dy_pack(g, cpad):
    """g fp32 [N,na,H,W,no] (contiguous) -> (dy bf16 [N,H,W,cpad], partials [rows, na*no]) -- see include/etb200.h"""
    N, na, H, W, no = g.shape
    lib = _lib.lib()
    rows = int(lib.etb_detect_dy_rows(N, H, W))
    dy = torch.empty((N, H, W, cpad), dtype=torch.bfloat16, device=g.device)
    partials = torch.empty((rows, na * no), dtype=torch.float32, device=g.device)
    _lib.check(lib.etb_detect_dy_pack(_lib.ptr(g), _lib.ptr(dy), _lib.ptr(partials), N, na, H, W, no, cpad, _lib.stream_ptr()), "etb_detect_dy_pack")
    return dy, partials


def column_sum(partials, out=None, accumulate=False):
    rows, Cc = partials.shape[0], int(partials.numel() // partials.shape[0])
    if out is None:
        out = torch.empty(Cc, dtype=torch.float32, device=partials.device)
        accumulate = False
    _lib.check(_lib.lib().etb_column_sum(_lib.ptr(partials), rows, Cc, _lib.ptr(out), int(accumulate), _lib.stream_ptr()), "etb_column_sum")
    return out


def netd_tail_fwd(h, C_, w2, h_cstride=None):
    """h [N,H,W,*] bf16 (relu(conv1(x))), w2 [2,C,1,1] fp32 -> o fp32 [N,H,W,2]"""
    N, H, W, cs = h.shape
    o = torch.empty((N, H, W, 2), dtype=torch.float32, device=h.device)
    _lib.check(_lib.lib().etb_netd_tail_fwd(_lib.ptr(h), N * H * W, C_, cs if h_cstride is None else h_cstride, _lib.ptr(w2), _lib.ptr(o),
                                            _lib.stream_ptr()), "etb_netd_tail_fwd")
    return o


def netd_tail_bwd(do, h, C_, w2, h_cstride=None):
    """do fp32 [N,H,W,2] contiguous -> (dh bf16 [N,H,W,C] with the ReLU mask applied, partials [rows, 2*C] of dW2)"""
    N, H, W, cs = h.shape
    M = N * H * W
    lib = _lib.lib()
    rows = int(lib.etb_netd_tail_rows(M))
    dh = nhwc_empty(N, H, W, C_, h.device)
    partials = torch.empty((rows, 2 * C_), dtype=torch.float32, device=h.device)
    _lib.check(lib.etb_netd_tail_bwd(_lib.ptr(do), _lib.ptr(h), M, C_, cs if h_cstride is None else h_cstride, _lib.ptr(w2), _lib.ptr(dh),
                                     _lib.ptr(partials), rows, _lib.stream_ptr()), "etb_netd_tail_bwd")
    return dh, partials
