"""non_max_suppression_ssod / non_max_suppression with the reference's surface (utils/general.py:887-1098),
backed by the batched on-device pipeline of csrc/nms.cu (all images per launch, no per-image host sync).

Deliberate deviation: the reference's 10 s wall-clock bail-out that silently drops the remaining images
(general.py:988-990) is not replicated (SURVEY.md section 5: nondeterministic).
"""
import ctypes as C

import torch

from . import _lib, _ws
from ._lib import EtbNmsParams

MAX_WH = 7680.0   # general.py:910 / :1013
MAX_NMS = 30000   # general.py:911 / :1014


def _run(prediction, conf_thres, iou_thres, agnostic, max_det, need_cls_conf, Ms=None, img_hw=(0, 0), ws_name="nms"):
    """ws_name: the cached workspace to use.  A captured training step bakes the pointer of "nms" into its graph, so a
    caller with other batch shapes (validation) passes its own name: growing "nms" would free the captured buffer."""
    assert 0 <= conf_thres <= 1, f'Invalid Confidence threshold {conf_thres}, valid values are between 0.0 and 1.0'
    assert 0 <= iou_thres <= 1, f'Invalid IoU {iou_thres}, valid values are between 0.0 and 1.0'
    _lib.require_cuda(prediction)
    pred = prediction
    if pred.dtype != torch.float32:
        pred = pred.float()
    if not pred.is_contiguous():
        pred = pred.contiguous()
    B, P, no = pred.shape
    p = EtbNmsParams()
    p.B, p.P, p.no = B, P, no
    p.conf_thres, p.iou_thres = float(conf_thres), float(iou_thres)
    p.max_nms, p.max_det = MAX_NMS, int(max_det)
    p.max_wh = 0.0 if agnostic else MAX_WH
    p.need_cls_conf = int(need_cls_conf)
    p.img_h, p.img_w = int(img_hw[0]), int(img_hw[1])
    lib = _lib.lib()
    dev = pred.device
    ws = _ws.workspace(ws_name, lib.etb_nms_workspace_bytes(C.byref(p)), dev)
    det = torch.empty((B, max_det, 8), dtype=torch.float32, device=dev)
    det_cnt = torch.empty((B,), dtype=torch.int32, device=dev)
    pl_rows = pl_cnt = None
    if Ms is not None:
        pl_rows = torch.empty((B * max_det, 9), dtype=torch.float64, device=dev)
        pl_cnt = torch.empty((1,), dtype=torch.int32, device=dev)
    _lib.check(lib.etb_nms_ssod(_lib.ptr(pred), C.byref(p), _lib.ptr(det), _lib.ptr(det_cnt), _lib.ptr(Ms),
                                _lib.ptr(pl_rows), _lib.ptr(pl_cnt), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
               "etb_nms_ssod")
    return det, det_cnt, pl_rows, pl_cnt


def _unsupported(classes, multi_label, labels, nc, allow_multi_label=False):
    if classes is not None or (multi_label and nc > 1 and not allow_multi_label) or (labels and len(labels)):
        raise NotImplementedError("efficientteacher_b200 NMS implements classes=None, labels=(); multi_label only through "
                                  "non_max_suppression (the val.py path, SURVEY.md 8f #2)")


def _run_val(prediction, conf_thres, iou_thres, agnostic, max_det):
    """non_max_suppression(multi_label=True): every (row, class) pair above conf, top-30000 by an exact radix select,
    then the shared rank + greedy-NMS kernels (csrc/nms.cu, etb_nms_val)."""
    assert 0 <= conf_thres <= 1 and 0 <= iou_thres <= 1
    _lib.require_cuda(prediction)
    pred = prediction.float().contiguous()
    B, P, no = pred.shape
    p = EtbNmsParams()
    p.B, p.P, p.no = B, P, no
    p.conf_thres, p.iou_thres = float(conf_thres), float(iou_thres)
    p.max_nms, p.max_det = MAX_NMS, int(max_det)
    p.max_wh = 0.0 if agnostic else MAX_WH
    p.need_cls_conf = 1
    lib = _lib.lib()
    ws = _ws.workspace("nms_val", lib.etb_nms_val_workspace_bytes(C.byref(p)), pred.device)
    det = torch.empty((B, max_det, 8), dtype=torch.float32, device=pred.device)
    det_cnt = torch.empty((B,), dtype=torch.int32, device=pred.device)
    _lib.check(lib.etb_nms_val(_lib.ptr(pred), C.byref(p), _lib.ptr(det), _lib.ptr(det_cnt), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
               "etb_nms_val")
    return det, det_cnt


def non_max_suppression_ssod(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False, num_points=0,
                             multi_label=False, labels=(), max_det=300):
    """-> list (one per image) of [k,8] tensors [xyxy, conf, cls, obj_conf, cls_conf] in score order."""
    if num_points:
        raise NotImplementedError("keypoint heads are out of scope")
    _unsupported(classes, multi_label, labels, prediction.shape[2] - 5)
    det, det_cnt, _, _ = _run(prediction, conf_thres, iou_thres, agnostic, max_det, need_cls_conf=False)
    cnt = det_cnt.cpu().tolist()  # the reference-shaped return value needs the sizes on the host
    return [det[b, :cnt[b]] for b in range(det.shape[0])]


def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False, multi_label=False,
                        labels=(), max_det=300):
    """-> list (one per image) of [k,6] tensors [xyxy, conf, cls].  multi_label=True (nc > 1) is the val.py variant."""
    nc = prediction.shape[2] - 5
    _unsupported(classes, multi_label, labels, nc, allow_multi_label=True)
    if multi_label and nc > 1:
        det, det_cnt = _run_val(prediction, conf_thres, iou_thres, agnostic, max_det)
    else:
        det, det_cnt, _, _ = _run(prediction, conf_thres, iou_thres, agnostic, max_det, need_cls_conf=True)
    cnt = det_cnt.cpu().tolist()
    return [det[b, :cnt[b], :6] for b in range(det.shape[0])]
