"""ctypes binding of libetb200.so (the C ABI declared in include/etb200.h).

There is no CPU fallback: importing works anywhere (so the host logic can be unit-tested), but every
compute call raises if the shared library or a CUDA device is missing.
"""
import ctypes as C
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libetb200.so")

ETB_MAX_LEVELS = 3
ETB_NA = 3
ETB_CHUNK = 4096

c_f32p = C.POINTER(C.c_float)
c_i32p = C.POINTER(C.c_int32)
c_f64p = C.POINTER(C.c_double)
vp = C.c_void_p


class EtbChunk(C.Structure):
    _fields_ = [("t", vp * 4), ("n", C.c_int32), ("group", C.c_int32)]


class EtbNmsParams(C.Structure):
    _fields_ = [("B", C.c_int32), ("P", C.c_int32), ("no", C.c_int32), ("conf_thres", C.c_float),
                ("iou_thres", C.c_float), ("max_nms", C.c_int32), ("max_det", C.c_int32), ("max_wh", C.c_float),
                ("need_cls_conf", C.c_int32), ("img_h", C.c_int32), ("img_w", C.c_int32)]


class EtbAssignLevels(C.Structure):
    _fields_ = [("nl", C.c_int32), ("nx", C.c_int32 * ETB_MAX_LEVELS), ("ny", C.c_int32 * ETB_MAX_LEVELS),
                ("anchors", (C.c_float * (ETB_NA * 2)) * ETB_MAX_LEVELS), ("anchor_t", C.c_float)]


class EtbAssignOut(C.Structure):
    _fields_ = [("idx", vp * ETB_MAX_LEVELS), ("tbox", vp * ETB_MAX_LEVELS), ("anch", vp * ETB_MAX_LEVELS),
                ("tcls", vp * ETB_MAX_LEVELS), ("tscore", vp * ETB_MAX_LEVELS), ("cnt", vp), ("cap", C.c_int32)]


class EtbLossParams(C.Structure):
    _fields_ = [("nl", C.c_int32), ("B", C.c_int32), ("na", C.c_int32), ("no", C.c_int32),
                ("nx", C.c_int32 * ETB_MAX_LEVELS), ("ny", C.c_int32 * ETB_MAX_LEVELS),
                ("balance", C.c_float * ETB_MAX_LEVELS), ("box_w", C.c_float), ("obj_w", C.c_float),
                ("cls_w", C.c_float), ("cp", C.c_float), ("cn", C.c_float), ("nsets", C.c_int32),
                ("ignore_obj", C.c_int32), ("with_bbox", C.c_int32), ("with_cls", C.c_int32),
                ("cls_pw", C.c_float), ("obj_pw", C.c_float), ("fl_gamma", C.c_float), ("ssi", C.c_int32),
                ("balance_state", vp)]


class EtbPackDesc(C.Structure):
    _fields_ = [("w", vp), ("out", vp), ("elems", C.c_int64), ("Cout", C.c_int32), ("Cin", C.c_int32), ("k", C.c_int32),
                ("mode", C.c_int32), ("ntaps", C.c_int32), ("out_ld", C.c_int32), ("dtype", C.c_int32), ("kh", C.c_int8 * 12),
                ("kw", C.c_int8 * 12)]


class EtbFoldDesc(C.Structure):
    _fields_ = [("gamma", vp), ("beta", vp), ("mean", vp), ("var", vp), ("scale", vp), ("bias", vp), ("C", C.c_int32),
                ("eps", C.c_float), ("dtype", C.c_int32)]


ETB_PACK_CHUNK = 4096
# ETB_DT_*: the element types the weight packer and the BatchNorm fold read
ETB_DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
# ETB_STEM_SRC_*: the image element types etb_stem_im2col_into reads
ETB_STEM_SRC = {torch.float32: 0, torch.uint8: 1, torch.float16: 2}


class EtbFocalParams(C.Structure):
    _fields_ = [("x", vp * ETB_MAX_LEVELS), ("dx", vp * ETB_MAX_LEVELS), ("M", C.c_int64 * ETB_MAX_LEVELS), ("nl", C.c_int32),
                ("label", C.c_int32)]


class EtbV8Levels(C.Structure):
    _fields_ = [("nl", C.c_int32), ("h", C.c_int32 * ETB_MAX_LEVELS), ("w", C.c_int32 * ETB_MAX_LEVELS),
                ("stride", C.c_float * ETB_MAX_LEVELS)]


class EtbLetterboxFrame(C.Structure):
    _fields_ = [("src", vp), ("h0", C.c_int32), ("w0", C.c_int32), ("new_h", C.c_int32), ("new_w", C.c_int32), ("top", C.c_int32),
                ("left", C.c_int32)]


class EtbConvParams(C.Structure):
    _fields_ = [("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32),
                ("kh", C.c_int32), ("kw", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32),
                ("x_cstride", C.c_int32), ("y_cstride", C.c_int32), ("y_coffset", C.c_int32),
                ("res_cstride", C.c_int32), ("res_coffset", C.c_int32), ("act", C.c_int32), ("det_no", C.c_int32)]


_SIGS = {
    "etb_version": (C.c_int, []),
    "etb_last_error": (C.c_char_p, []),
    "etb_launch_count": (C.c_longlong, []),
    "etb_ema_update": (C.c_int, [vp, C.c_int64, vp, vp]),
    "etb_sgd_step": (C.c_int, [vp, C.c_int64, vp, C.c_int32, vp]),
    "etb_adamw_step": (C.c_int, [vp, C.c_int64, vp, C.c_int32, vp]),
    "etb_detect_decode": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_int32, c_f32p, C.c_float, vp]),
    "etb_nms_workspace_bytes": (C.c_size_t, [C.POINTER(EtbNmsParams)]),
    "etb_nms_ssod": (C.c_int, [vp, C.POINTER(EtbNmsParams), vp, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "etb_nms_val_workspace_bytes": (C.c_size_t, [C.POINTER(EtbNmsParams)]),
    "etb_nms_val": (C.c_int, [vp, C.POINTER(EtbNmsParams), vp, vp, vp, C.c_size_t, vp]),
    "etb_select_targets": (C.c_int, [vp, vp, C.c_int32, C.c_int32, vp, vp, C.c_int32, C.c_int32, vp, vp, vp]),
    "etb_build_targets": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.POINTER(EtbAssignLevels),
                                    C.POINTER(EtbAssignOut), vp]),
    "etb_label_class_hist": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, vp]),
    "etb_bbox_ciou": (C.c_int, [vp, vp, C.c_int32, vp, vp]),
    "etb_loss_workspace_bytes": (C.c_size_t, [C.POINTER(EtbLossParams), C.c_int32]),
    "etb_loss_forward": (C.c_int, [C.POINTER(vp), C.POINTER(EtbLossParams), C.POINTER(EtbAssignOut), vp, vp,
                                   C.c_size_t, vp]),
    "etb_loss_backward": (C.c_int, [C.POINTER(vp), C.POINTER(vp), C.POINTER(EtbLossParams),
                                    C.POINTER(EtbAssignOut), vp, vp, C.c_size_t, vp]),
    "etb_conv_fwd": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.POINTER(EtbConvParams), vp]),
    "etb_conv_dgrad": (C.c_int, [vp, vp, vp, C.POINTER(EtbConvParams), C.c_int32, vp]),
    "etb_conv_wgrad_workspace_bytes": (C.c_size_t, [C.POINTER(EtbConvParams)]),
    "etb_conv_wgrad": (C.c_int, [vp, vp, vp, C.POINTER(EtbConvParams), C.c_int32, vp, C.c_size_t, vp]),
    "etb_bn_partial_rows": (C.c_int32, [C.c_int64, C.c_int32, C.c_int32]),
    "etb_bn_stats": (C.c_int, [vp, C.c_int64, C.c_int32, C.c_int32, vp, C.c_int32, vp]),
    "etb_bn_finalize": (C.c_int, [vp, C.c_int32, C.c_int64, C.c_int32, vp, vp, C.c_float, C.c_float, vp, vp, vp, vp, vp, vp, vp]),
    "etb_bn_stats_sums": (C.c_int, [vp, C.c_int64, C.c_int32, C.c_int32, vp, C.c_int32, vp, vp]),
    "etb_bn_finalize_global": (C.c_int, [vp, C.c_int32, vp, vp, C.c_float, C.c_float, vp, vp, vp, vp, vp, vp, vp]),
    "etb_bn_act_apply_res": (C.c_int, [vp, vp, vp, vp, vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_maxpool5_fwd": (C.c_int, [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_maxpool5_bwd": (C.c_int, [vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_upsample2x_bwd": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_copy_slice_nhwc": (C.c_int, [vp, vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_bn_act_bwd_reduce": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.c_int32, vp]),
    "etb_bn_act_bwd_finalize": (C.c_int, [vp, C.c_int32, C.c_int32, vp, vp, vp, C.c_int32, vp]),
    "etb_bn_act_bwd_apply": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       vp, vp]),
    "etb_bn_act_bwd_apply_global": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_int32, vp, vp]),
    "etb_nchw_f32_to_nhwc_bf16": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                            C.c_float, vp]),
    "etb_nhwc_bf16_to_nchw_f32": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_sppf_pool": (C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_upsample2x_nhwc": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, vp]),
    "etb_pack_multi": (C.c_int, [vp, vp, C.c_int32, vp]),
    "etb_fold_bn_multi": (C.c_int, [vp, C.c_int32, vp]),
    "etb_detect_dy_rows": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "etb_detect_dy_pack": (C.c_int, [vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "etb_column_sum": (C.c_int, [vp, C.c_int64, C.c_int32, vp, C.c_int32, vp]),
    "etb_netd_tail_rows": (C.c_int32, [C.c_int64]),
    "etb_netd_tail_fwd": (C.c_int, [vp, C.c_int64, C.c_int32, C.c_int32, vp, vp, vp]),
    "etb_netd_tail_bwd": (C.c_int, [vp, vp, C.c_int64, C.c_int32, C.c_int32, vp, vp, vp, C.c_int32, vp]),
    "etb_domain_focal_workspace_bytes": (C.c_int64, []),
    "etb_domain_focal_fwd": (C.c_int, [C.POINTER(EtbFocalParams), vp, vp, C.c_int64, vp]),
    "etb_domain_focal_bwd": (C.c_int, [C.POINTER(EtbFocalParams), vp, vp]),
    "etb_val_process_batch": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, C.c_int32, vp, C.c_int32, vp, vp, vp]),
    "etb_nms_boxes": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_float, vp, vp, vp]),
    "etb_val_epoch_append_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "etb_val_epoch_append": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       vp, C.c_int32, C.c_int32, vp, vp, vp, C.c_int64, vp, vp, vp, vp, C.c_size_t, vp]),
    "etb_val_epoch_append_confusion": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, C.c_int32, C.c_int32, C.c_int32,
                                                 C.c_int32, vp, C.c_int32, C.c_int32, vp, vp, vp, C.c_int64, vp, vp, vp, C.c_int32,
                                                 C.c_float, C.c_float, vp, vp, vp, C.c_size_t, vp]),
    "etb_confusion_matrix": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, C.c_int32, C.c_int32, C.c_float, C.c_float, vp, vp,
                                       vp]),
    "etb_ap_per_class_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int32]),
    "etb_ap_per_class": (C.c_int, [vp, vp, vp, C.c_int64, C.c_int32, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp, vp, vp,
                                   C.c_size_t, vp]),
    "etb_stem_im2col_into": (C.c_int, [vp, C.c_int32, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, vp]),
    "etb_tal_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "etb_tal_assign": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                C.c_float, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "etb_v8_decode": (C.c_int, [vp, vp, C.POINTER(EtbV8Levels), C.c_int32, C.c_int32, C.c_int32, C.c_float, vp, vp, vp, vp, vp]),
    "etb_pl_quality_workspace_bytes": (C.c_size_t, []),
    "etb_pl_quality": (C.c_int, [vp, vp, C.c_int32, vp, vp, C.c_int32, vp, vp, C.c_int32, vp, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_int32, vp, vp, vp, C.c_size_t, vp]),
    "etb_meter_update": (C.c_int, [vp, C.c_int32, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32, vp]),
    "etb_letterbox_u8": (C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, vp, vp]),
    "etb_detect_rescale": (C.c_int, [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp]),
}

_lib = None


def exported_symbols():
    """Names the header declares (used by the CPU test that checks the .so exports all of them)."""
    return sorted(_SIGS)


def register(name, restype, argtypes):
    _SIGS[name] = (restype, argtypes)
    if _lib is not None:
        fn = getattr(_lib, name)
        fn.restype, fn.argtypes = restype, argtypes


def lib():
    """Load libetb200.so (no compute is run).  Raises loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libetb200.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU/PyTorch fallback for the native kernels)" % LIB_PATH)
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(_lib, name)
            fn.restype, fn.argtypes = res, args
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().etb_last_error()
        raise RuntimeError("libetb200 %s failed (%d): %s" % (what, rc, msg.decode() if msg else ""))


def require_cuda(*tensors):
    if not torch.cuda.is_available():
        raise RuntimeError("efficientteacher_b200 needs a CUDA (sm_90a) device: there is no CPU fallback")
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("expected a CUDA tensor, got %s" % (t.device,))


def stream_ptr(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def upload(host, device):
    """A ctypes array or numpy array -> a uint8 tensor on `device` holding the same bytes (a descriptor table for a
    kernel).  Not inside a stream capture: the copy from host memory would not be part of the graph."""
    assert not torch.cuda.is_current_stream_capturing(), "descriptor table upload inside a stream capture"
    return torch.from_numpy(np.frombuffer(host, dtype=np.uint8).copy()).to(device)


def chunk_key(streams):
    """The data pointers a chunk table of `streams` holds (see chunk_table); a different key means the table is stale."""
    return tuple(t.data_ptr() if t is not None else 0 for ts in streams for t in ts)


def chunk_table(streams, groups=None):
    """The EtbChunk table of one multi-tensor update (etb_ema_update, etb_sgd_step, etb_adamw_step).

    streams: per tensor of the list, a tuple of up to four same-size contiguous fp32 CUDA tensors in the order of the
    kernel's EtbChunk.t (None for an unused stream); groups: per tensor, the index of its scalars in hyper_dev (default
    0).  Returns (device table, chunk count, chunk_key(streams))."""
    for ts in streams:
        n = ts[0].numel()
        if not all(t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == n) for t in ts):
            raise RuntimeError("chunk_table expects same-size contiguous fp32 CUDA tensors per entry")
    numel = np.array([ts[0].numel() for ts in streams], dtype=np.int64)
    ptrs = np.array([[t.data_ptr() if t is not None else 0 for t in ts] + [0] * (4 - len(ts)) for ts in streams],
                    dtype=np.uint64).reshape(-1, 4)
    counts = (numel + ETB_CHUNK - 1) // ETB_CHUNK
    owner = np.repeat(np.arange(len(streams)), counts)                    # the tensor each chunk belongs to
    start = (np.arange(len(owner)) - np.repeat(np.cumsum(counts) - counts, counts)) * ETB_CHUNK   # its first element
    tab = np.zeros(len(owner), dtype=np.dtype(EtbChunk))
    tab["t"] = np.where(ptrs[owner] != 0, ptrs[owner] + (4 * start).astype(np.uint64)[:, None], 0)
    tab["n"] = np.minimum(numel[owner] - start, ETB_CHUNK)
    tab["group"] = 0 if groups is None else np.asarray(groups, dtype=np.int32)[owner]
    dev = next(t for t in streams[0] if t is not None).device if streams else "cuda"
    return upload(tab, dev), len(tab), chunk_key(streams)
