"""TEST INFRASTRUCTURE ONLY -- CPU restatement (torch-CPU / numpy) of the reference's pseudo-label quality statistics, the
checker of efficientteacher_b200.pl_quality and of the SSOD step's meter (as tests/ap_port.py is for ap_per_class).  Pinned
against the live, unmodified reference by the golden vectors tests/golden/plq_*.npz (tests/golden/make_golden_plq.py).
Every function cites the reference file:line it follows (paths relative to the reference root)."""
import numpy as np
import torch

F32 = np.float32


# ---------------------------------------------------------------------------------------------------------
# pseudo-label quality -- utils/self_supervised_utils.py:456-479 (select_targets), :481-587 (check_pseudo_label_with_gt),
# :589-606 (check_pseudo_label); utils/general.py:630-637 (xywh2xyxy); utils/metrics.py:252-273 (box_iou)
# ---------------------------------------------------------------------------------------------------------
def _plq_select(rows, thr_low, thr_high):
    """:456-479: per row, conf >= thr_high[int(cls)] -> reliable, elif conf >= thr_low[int(cls)] -> uncertain (float64
    compares); both sets cast to fp32"""
    c = rows[:, 1].astype(np.int64)
    rel = rows[:, 6] >= np.asarray(thr_high, dtype=np.float64)[c]
    unc = ~rel & (rows[:, 6] >= np.asarray(thr_low, dtype=np.float64)[c])
    return rows[rel].astype(F32), rows[unc].astype(F32)


def _plq_xyxy_offset(boxes, img):
    """:521-524: xywh * 640 -> xyxy -> + img * 640 on all four coordinates, in the boxes' dtype"""
    b = boxes * 640
    w2, h2 = b[:, 2] / 2, b[:, 3] / 2
    return torch.stack((b[:, 0] - w2, b[:, 1] - h2, b[:, 0] + w2, b[:, 1] + h2), 1) + (img * 640)[:, None]


def _plq_set_count(mask, iou):
    """:538-570: the matches [label, detection, iou] of one set, sorted by IoU descending, np.unique on the detection, then
    on the label; the number of detections marked.  A stable sort, so IoU ties keep torch.where's (label-major) order
    reversed: the later label wins (csrc/val.cu's rule).  numpy's own argsort is not stable on every CPU, so the reference's
    choice between tied labels depends on the machine; the golden vectors avoid cases where that changes a count."""
    li, di = torch.where(mask)
    if li.numel() == 0:
        return 0
    m = torch.cat((torch.stack((li, di), 1), iou[li, di][:, None]), 1).numpy()
    if li.numel() > 1:
        m = m[np.argsort(m[:, 2], kind="stable")[::-1]]
        m = m[np.unique(m[:, 1], return_index=True)[1]]
        m = m[np.unique(m[:, 0], return_index=True)[1]]
    return int(np.unique(m[:, 1].astype(np.int64)).size)


def pl_quality_counts(detections, labels, iouv=(0.5,), ignore_thres_low=None, ignore_thres_high=None):
    """check_pseudo_label_with_gt's counts: (n_uc, tp [T], fp_cls [T], fp_loc [T]) int.  detections [N,9], labels [M,6]
    (img, cls, x, y, w, h normalised).  Without thresholds every row is scored in its own dtype (float64 rows: the IoU is
    float64, with fp32 gt areas, as torch promotes box_iou's mixed operands)."""
    det = torch.as_tensor(np.asarray(detections)).reshape(-1, 9)
    if ignore_thres_low is not None:
        det = torch.from_numpy(_plq_select(det.double().numpy(), ignore_thres_low, ignore_thres_high)[1])
    lab = torch.as_tensor(np.asarray(labels, dtype=F32)).reshape(-1, 6)
    thr = torch.as_tensor(iouv)
    if thr.dtype not in (torch.float32, torch.float64):
        thr = thr.float()
    gt = _plq_xyxy_offset(lab[:, 2:6], lab[:, 0])
    pseudo = _plq_xyxy_offset(det[:, 2:6], det[:, 0])
    area1 = (gt[:, 2] - gt[:, 0]) * (gt[:, 3] - gt[:, 1])
    area2 = (pseudo[:, 2] - pseudo[:, 0]) * (pseudo[:, 3] - pseudo[:, 1])
    inter = (torch.min(gt[:, None, 2:], pseudo[:, 2:]) - torch.max(gt[:, None, :2], pseudo[:, :2])).clamp(0).prod(2)
    iou = inter / (area1[:, None] + area2 - inter)
    same_cls = lab[:, 1:2] == det[:, 1]
    same_img = lab[:, 0:1] == det[:, 0]
    T = thr.numel()
    tp, fp_cls, fp_loc = (np.zeros(T, np.int64) for _ in range(3))
    for i in range(T):
        tp[i] = _plq_set_count((iou >= thr[i]) & same_cls & same_img, iou)
        fp_cls[i] = _plq_set_count((iou >= thr[i]) & ~same_cls & same_img, iou)
        fp_loc[i] = _plq_set_count((iou < thr[i]) & (iou > torch.tensor(0.01)) & same_img, iou)
    return int(det.shape[0]), tp, fp_cls, fp_loc


def check_pseudo_label_with_gt(detections, labels, iouv=(0.5,), ignore_thres_low=None, ignore_thres_high=None, batch_size=1):
    """:481-587 -> (tp_rate, fp_cls_rate, fp_loc_rate, pse_num, gt_num): float64 arrays [T] (int 0 when no row is scored),
    floats.  Leaves `labels` as it was (the reference scales its box columns in place)."""
    n_uc, tp, fp_cls, fp_loc = pl_quality_counts(detections, labels, iouv, ignore_thres_low, ignore_thres_high)
    rates = (0, 0, 0) if n_uc == 0 else tuple(c * 1.0 / n_uc for c in (tp, fp_cls, fp_loc))
    return rates + (n_uc / batch_size, np.asarray(labels).reshape(-1, 6).shape[0] / batch_size)


def check_pseudo_label(detections, ignore_thres_low=None, ignore_thres_high=None, batch_size=1):
    """:589-606 -> (precision, recall, pse_num, reliable_num)"""
    rows = np.asarray(detections, dtype=np.float64).reshape(-1, 9)
    rel, unc = _plq_select(rows, ignore_thres_low, ignore_thres_high)
    reliable_num, uncertain_num = rel.shape[0] / batch_size, unc.shape[0] / batch_size
    denorm = reliable_num + uncertain_num
    precision_rate = 0 if denorm == 0 else reliable_num / denorm
    recall_rate = 0 if rows.shape[0] == 0 else (reliable_num + uncertain_num) * batch_size / rows.shape[0]
    return precision_rate, recall_rate, reliable_num + uncertain_num, reliable_num


def hit_values(rows, gt, thr_low, thr_high, batch_size, with_gt, iouv=(0.5,)):
    """The five values trainer/ssod_trainer.py:655-672 logs for one step (tp fp_cls fp_loc pse_num gt_num), at the first
    IoU threshold; no rows: the invalid step's zeros"""
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, 9)
    if rows.shape[0] == 0:
        return [0.0] * 5
    if with_gt:
        tp, fpc, fpl, pse, gtn = check_pseudo_label_with_gt(rows, gt, iouv, thr_low, thr_high, batch_size)
        return [float(np.asarray(v).reshape(-1)[0]) for v in (tp, fpc, fpl)] + [pse, gtn]
    tp, fpl, pse, gtn = check_pseudo_label(rows, thr_low, thr_high, batch_size)
    return [float(tp), 0.0, float(fpl), pse, gtn]
