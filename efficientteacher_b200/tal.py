"""Anchor-free (YOLOv8) operators of the reference, on the native kernels of csrc/tal.cu (SURVEY.md section 8f row 5).

Mirrors, with the reference's names and call contracts:
  * `TaskAlignedAssigner`            models/assigner/tal_assigner.py:13-158           -> etb_tal_assign
  * `generate_anchors`               models/module/nanodet_utils.py:135-182           (constant tables, built once per shape)
  * `decode_eval(cls, reg, ...)`     models/head/yolov8_head.py:169-220 (eval branch after the convolutions)  -> etb_v8_decode
  * `assigner_inputs(cls, reg, ...)` models/loss/tal_loss.py:88-95,150-156 (pred_bboxes, pd_scores, pd_bboxes) -> etb_v8_decode

The reference defines no end-to-end training step for this head (`models/loss/tal_loss.py` imports two modules that do not exist
and `SSODTrainer.train_instance` raises for it), so these are standalone operators; the YOLOv8 trunk itself is not built (its
channel widths -- 68, 192, 576 ... -- break the 8-channel vector contract of the wgmma conv kernels, DESIGN.md section 9).
There is no CPU fallback: every call needs libetb200.so and CUDA tensors.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._lib import EtbV8Levels, check, lib, ptr, require_cuda, stream_ptr


def _f32c(t):
    return t.detach().to(torch.float32).contiguous()


class TaskAlignedAssigner(nn.Module):
    """models/assigner/tal_assigner.py:13-80.  forward(pd_scores [B,A,nc] (sigmoid), pd_bboxes [B,A,4] xyxy, anc_points [A,2],
    gt_labels [B,M,1], gt_bboxes [B,M,4] xyxy, mask_gt [B,M,1]) -> (target_labels [B,A] int64, target_bboxes [B,A,4],
    target_scores [B,A,nc], fg_mask [B,A] bool).  Computes in fp32 (float64 ground truth, which the reference's
    `preprocess` happens to produce, is cast); ties inside the top-k go to the lowest anchor index."""

    def __init__(self, top_k=13, num_classes=80, alpha=1.0, beta=6.0, eps=1e-9):
        super().__init__()
        self.topk = top_k
        self.num_classes = num_classes
        self.bg_idx = num_classes
        self.alpha = alpha
        self.beta = beta
        self.eps = eps

    @torch.no_grad()
    def forward(self, pd_scores, pd_bboxes, anc_points, gt_labels, gt_bboxes, mask_gt):
        require_cuda(pd_scores, pd_bboxes, anc_points, gt_labels, gt_bboxes, mask_gt)
        L = lib()
        self.bs = pd_scores.size(0)
        self.n_max_boxes = gt_bboxes.size(1)
        if self.n_max_boxes == 0:       # :53-58 -- float labels filled with bg_idx and a float (not bool) mask: the reference's own early return
            return (torch.full_like(pd_scores[..., 0], self.bg_idx), torch.zeros_like(pd_bboxes), torch.zeros_like(pd_scores),
                    torch.zeros_like(pd_scores[..., 0]))
        B, A, nc = pd_scores.shape
        M = self.n_max_boxes
        if nc != self.num_classes:
            raise ValueError("pd_scores has %d classes, the assigner was built for %d" % (nc, self.num_classes))
        if tuple(pd_bboxes.shape) != (B, A, 4) or tuple(anc_points.shape) != (A, 2) or gt_labels.numel() != B * M or mask_gt.numel() != B * M:
            raise ValueError("TaskAlignedAssigner: inconsistent shapes")
        dev = pd_scores.device
        sc, bx, an = _f32c(pd_scores), _f32c(pd_bboxes), _f32c(anc_points)
        gl, gb, mg = _f32c(gt_labels).view(B, M), _f32c(gt_bboxes), _f32c(mask_gt).view(B, M)
        t_labels = torch.empty((B, A), dtype=torch.int64, device=dev)
        t_bboxes = torch.empty((B, A, 4), dtype=torch.float32, device=dev)
        t_scores = torch.empty((B, A, nc), dtype=torch.float32, device=dev)
        fg = torch.empty((B, A), dtype=torch.bool, device=dev)
        nbytes = L.etb_tal_workspace_bytes(B, A, M)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        check(L.etb_tal_assign(ptr(sc), ptr(bx), ptr(an), ptr(gl), ptr(gb), ptr(mg), B, A, M, nc, int(self.topk), float(self.alpha),
                               float(self.beta), float(self.eps), ptr(t_labels), ptr(t_bboxes), ptr(t_scores), ptr(fg), ptr(ws), nbytes,
                               stream_ptr(dev)), "etb_tal_assign")
        return t_labels, t_bboxes.to(gt_bboxes.dtype), t_scores, fg


_ANCHOR_CACHE = {}


def generate_anchors(feats, fpn_strides, grid_cell_size=5.0, grid_cell_offset=0.5, device='cpu', is_eval=False):
    """models/module/nanodet_utils.py:135-182 (same signature and return values).  The tables only depend on the level shapes:
    they are built once per (shapes, strides, offset, device, dtype) and cached."""
    shapes = tuple((int(f.shape[-2]), int(f.shape[-1])) for f in feats)
    strides = tuple(float(s) for s in fpn_strides)
    dtype = feats[0].dtype if torch.is_tensor(feats[0]) and feats[0].is_floating_point() else torch.float32
    key = (shapes, strides, float(grid_cell_size), float(grid_cell_offset), str(device), bool(is_eval), dtype)
    hit = _ANCHOR_CACHE.get(key)
    if hit is not None:
        return hit
    anchors, pts, st, counts = [], [], [], []
    for (h, w), s in zip(shapes, strides):
        sx = torch.arange(w, device=device, dtype=torch.float32) + grid_cell_offset
        sy = torch.arange(h, device=device, dtype=torch.float32) + grid_cell_offset
        if not is_eval:
            sx, sy = sx * s, sy * s
        yy, xx = torch.meshgrid(sy, sx, indexing="ij")
        pts.append(torch.stack([xx, yy], -1).reshape(-1, 2))
        st.append(torch.full((h * w, 1), s, dtype=torch.float32, device=device))
        if not is_eval:
            half = grid_cell_size * s * 0.5
            anchors.append(torch.stack([xx - half, yy - half, xx + half, yy + half], -1).reshape(-1, 4).to(dtype))
            counts.append(h * w)
    if is_eval:
        out = (torch.cat(pts), torch.cat(st))
    else:
        out = (torch.cat(anchors), torch.cat(pts).to(dtype), counts, torch.cat(st).to(dtype))
    _ANCHOR_CACHE[key] = out
    return out


def _levels(shapes, strides):
    if not 1 <= len(shapes) <= _lib.ETB_MAX_LEVELS or len(strides) != len(shapes):
        raise ValueError("1..%d levels expected" % _lib.ETB_MAX_LEVELS)
    lv = EtbV8Levels()
    lv.nl = len(shapes)
    for i, ((h, w), s) in enumerate(zip(shapes, strides)):
        lv.h[i], lv.w[i], lv.stride[i] = int(h), int(w), float(s)
    return lv, sum(int(h) * int(w) for h, w in shapes)


def _decode(cls, reg, shapes, strides, reg_max, grid_cell_offset, want_pred, want_grid, want_pix, want_scores):
    require_cuda(reg, cls)
    L = lib()
    lv, A = _levels(shapes, strides)
    B = reg.shape[0]
    R = reg_max + 1
    if tuple(reg.shape) != (B, A, 4 * R):
        raise ValueError("reg_distri must be [B,%d,%d], got %s" % (A, 4 * R, tuple(reg.shape)))
    dev = reg.device
    reg = _f32c(reg)
    nc = 1
    if cls is not None:
        if cls.shape[0] != B or cls.shape[1] != A:
            raise ValueError("cls_score must be [B,%d,nc]" % A)
        nc = cls.shape[2]
        cls = _f32c(cls)
    elif want_pred or want_scores:
        raise ValueError("class logits are needed for pred / scores")
    new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)  # noqa: E731
    pred = new(B, A, 5 + nc) if want_pred else None
    bg = new(B, A, 4) if want_grid else None
    bp = new(B, A, 4) if want_pix else None
    sc = new(B, A, nc) if want_scores else None
    check(L.etb_v8_decode(ptr(cls), ptr(reg), C.byref(lv), B, nc, int(reg_max), float(grid_cell_offset), ptr(pred), ptr(bg), ptr(bp), ptr(sc),
                          stream_ptr(dev)), "etb_v8_decode")
    return pred, bg, bp, sc


def decode_eval(cls_score_list, reg_distri_list, shapes, strides, reg_max=16, grid_cell_offset=0.5):
    """The eval branch of YoloV8Detect.forward after the convolutions (models/head/yolov8_head.py:169-220, use_dfl=True):
    cls_score_list [B,A,nc], reg_distri_list [B,A,4*(reg_max+1)] -> pred [B,A,5+nc] = (xywh in pixels, 1, sigmoid scores)."""
    return _decode(cls_score_list, reg_distri_list, shapes, strides, reg_max, grid_cell_offset, True, False, False, False)[0]


def assigner_inputs(pred_scores, pred_distri, shapes, strides, reg_max=16, grid_cell_offset=0.5):
    """What ComputeTalLoss.__call__ builds before calling the assigner (models/loss/tal_loss.py:88-101), in one pass:
    returns (pred_bboxes [B,A,4] xyxy in grid units = bbox_decode(anchor_points / stride, pred_distri),
             pd_scores   [B,A,nc] = pred_scores.sigmoid(),
             pd_bboxes   [B,A,4]  = pred_bboxes * stride_tensor)."""
    _, bg, bp, sc = _decode(pred_scores, pred_distri, shapes, strides, reg_max, grid_cell_offset, False, True, True, True)
    return bg, sc, bp


def bbox_decode(pred_dist, shapes, strides, reg_max=16, grid_cell_offset=0.5):
    """ComputeTalLoss.bbox_decode(anchor_points / stride_tensor, pred_dist) (models/loss/tal_loss.py:150-156): xyxy, grid units."""
    return _decode(None, pred_dist, shapes, strides, reg_max, grid_cell_offset, False, True, False, False)[1]
