"""Detect head pieces with the reference's surface (models/head/yolov5_head.py)."""
import ctypes as C

import torch

from . import _lib


_ANCHOR_CACHE = {}


def decode_levels(levels, anchors_grid, strides):
    """Eval-mode decode of Detect (yolov5_head.py:66-78): list of logits [B,na,ny,nx,no] -> pred [B,P,no].
    One elementwise launch per level, written straight into the concatenated output (no torch.cat copy)."""
    _lib.require_cuda(*levels)
    B, na, _, _, no = levels[0].shape
    P = sum(int(x.shape[1] * x.shape[2] * x.shape[3]) for x in levels)
    pred = torch.empty((B, P, no), dtype=torch.float32, device=levels[0].device)
    key = (anchors_grid.data_ptr(), anchors_grid._version, anchors_grid.dtype)   # model.half() gives the buffer new storage
    anc = _ANCHOR_CACHE.get(key)
    if anc is None:                       # one D2H per anchor tensor version, not per call (keeps the step sync-free)
        anc = _ANCHOR_CACHE[key] = anchors_grid.detach().float().cpu().contiguous()
    row0 = 0
    lib = _lib.lib()
    for l, x in enumerate(levels):
        x = x.float().contiguous()
        ny, nx = int(x.shape[2]), int(x.shape[3])
        a = (C.c_float * (na * 2))(*[float(v) for v in anc[l].reshape(-1)])
        _lib.check(lib.etb_detect_decode(_lib.ptr(x), _lib.ptr(pred), B, na, ny, nx, no, P, row0, a, float(strides[l]),
                                         _lib.stream_ptr()), "etb_detect_decode")
        row0 += na * ny * nx
    return pred
