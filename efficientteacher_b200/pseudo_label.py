"""FairPseudoLabel with the reference's surface (utils/self_supervised_utils.py:54-245).

create_pseudo_label_online_with_gt keeps the reference's return contract -- (CPU float64 [N,9] tensor, invalid
flag) because trainer/ssod_trainer.py:618,640,645,663-669 consumes it on the host -- but the whole chain
(candidate filter -> NMS -> xyxy2xywh -> affine warp to the strong-aug frame -> box_candidates -> normalise ->
flips) runs on the device in one batch of launches; the single D2H copy is the final [N,9] rows.  A
device-resident twin (`last_rows_dev`, `last_count_dev`) is cached for the fused SSOD loss so the step itself
never waits on that copy.
"""
import torch

from . import _lib
from .nms import _run


class FairPseudoLabel:
    def __init__(self, cfg):
        self.nms_conf_thres = cfg.SSOD.nms_conf_thres
        self.nms_iou_thres = cfg.SSOD.nms_iou_thres
        self.debug = cfg.SSOD.debug
        self.multi_label = cfg.SSOD.multi_label
        self.names = cfg.Dataset.names
        self.num_points = cfg.Dataset.np
        if self.multi_label or self.num_points:
            raise NotImplementedError("SSOD.multi_label / keypoints are not on the hot path")
        self.last_rows_dev = None
        self.last_count_dev = None
        self.last_det = None

    def create_pseudo_label_device(self, out, M_s, height, width):
        """Device-only variant: returns (rows float64 [B*300,9] CUDA, count int32[1] CUDA); no host sync."""
        Ms = M_s.to(device=out.device, dtype=torch.float64, non_blocking=True).contiguous()
        assert Ms.shape == (out.shape[0], 13), "M_s must be [B,13] = [img, M(9), s, ud, lr]"
        det, det_cnt, rows, cnt = _run(out, self.nms_conf_thres, self.nms_iou_thres, False, 300, False, Ms=Ms,
                                       img_hw=(height, width))
        self.last_rows_dev, self.last_count_dev, self.last_det = rows, cnt, (det, det_cnt)
        return rows, cnt

    def create_pseudo_label_online_with_gt(self, out, target_imgs, M_s, target_imgs_ori, gt=None, RANK=-2):
        n_img, _, height, width = target_imgs.shape
        rows, cnt = self.create_pseudo_label_device(out.detach(), M_s, height, width)
        n = int(cnt.item())
        if n == 0:
            return [], True
        return rows[:n].cpu(), False


def merge_extra_teacher_detections(out, extra_teacher_outs, extra_teacher_class_idxs, conf_thres, iou_thres):
    """The detection-merging part of FairPseudoLabel.create_pseudo_label_online_with_extra_teachers
    (utils/self_supervised_utils.py:256-274): NMS of the main teacher's predictions and of every extra teacher's, class
    indices of the extra teachers remapped through their dict, and -- teacher after teacher, per image -- a class-agnostic
    NMS over the concatenation.  All on the device (etb_nms_ssod-family kernels + etb_nms_boxes); returns a list (one per
    image) of [k,6] tensors [x1,y1,x2,y2,conf,cls] like the reference's `out` after the loop.

    The rest of that reference method cannot run: it feeds these 6-column rows to output_to_target_ssod, which unpacks 8
    columns (utils/plots.py:488) and raises for any non-empty detection list -- a dead branch of the reference (every shipped
    config has SSOD.extra_teachers == []).  Parity of this function is pinned up to that point (tests/golden/extra_teachers.npz,
    generated from the live reference with output_to_target_ssod intercepted)."""
    from . import nms as etb_nms
    cur = etb_nms.non_max_suppression(out, conf_thres, iou_thres)
    B = len(cur)
    dev = out.device
    lib = _lib.lib()
    for t_idx, t_out in enumerate(extra_teacher_outs):
        t_det = etb_nms.non_max_suppression(t_out, conf_thres, iou_thres)
        cmap = extra_teacher_class_idxs[t_idx]
        lut = None
        if len(cmap):
            nc = int(t_out.shape[2] - 5)
            lut = torch.arange(max(nc, max(cmap) + 1), dtype=torch.float32, device=dev)
            for k, v in cmap.items():
                lut[int(k)] = float(v)
        nmax = max(max(c.shape[0] + d.shape[0] for c, d in zip(cur, t_det)), 1)
        if nmax > 1024:
            raise NotImplementedError("extra-teachers merge: more than 1024 detections per image (etb_nms_boxes limit)")
        rows = torch.zeros((B, nmax, 6), dtype=torch.float32, device=dev)
        cnt = torch.zeros(B, dtype=torch.int32, device=dev)
        for i in range(B):
            d = t_det[i]
            if lut is not None and d.shape[0]:
                d = d.clone()
                d[:, 5] = lut[d[:, 5].long()]
            x = torch.cat([cur[i], d], 0)
            rows[i, :x.shape[0]] = x
            cnt[i] = x.shape[0]
        kept = torch.empty_like(rows)
        kcnt = torch.empty_like(cnt)
        _lib.check(lib.etb_nms_boxes(_lib.ptr(rows), _lib.ptr(cnt), B, nmax, 6, float(iou_thres), _lib.ptr(kept), _lib.ptr(kcnt),
                                     _lib.stream_ptr()), "etb_nms_boxes")
        kc = kcnt.cpu().tolist()
        cur = [kept[i, :kc[i]] for i in range(B)]
    return cur
