"""ComputeStudentMatchLoss (the Pseudo Label Assigner) with the reference's surface
(models/loss/ssod/ssod_loss.py:26-295), backed by etb_select_targets + 4x etb_build_targets + the fused loss.

The reference's select_targets does one `.cpu()` per pseudo-label row (ssod_loss.py:141) and the four
assigner calls each synchronise; here the routing, the four assignments and the loss run back to back on the
stream with every count kept on the device.
"""
import torch

from . import _lib
from .assigner import YOLOAnchorAssigner, AssignBuffers
from .ema import is_parallel
from .loss import smooth_BCE, make_loss_params, _FusedDetLoss, _prep_p


class ComputeStudentMatchLoss:
    """cfg.Loss.cls_pw / obj_pw weight the class and objectness BCE as in the reference (ssod_loss.py:32-38); Loss.fl_gamma
    is not read there, and Loss.autobalance only sets `ssi`, so neither changes this loss."""

    def __init__(self, model, cfg):
        if cfg.SSOD.focal_loss > 0:
            raise NotImplementedError("SSOD.focal_loss > 0 fails in the reference: ssod_loss.py:40-41 wraps the objectness "
                                      "criterion in FocalLoss, which that module never imports (NameError)")
        if cfg.SSOD.use_ota:
            raise NotImplementedError("SSOD.use_ota=True is broken in the reference (SURVEY.md Appendix C #4) and "
                                      "not on the hot path")
        self.cp, self.cn = smooth_BCE(eps=cfg.Loss.label_smoothing)
        self.cls_pw, self.obj_pw = float(cfg.Loss.cls_pw), float(cfg.Loss.obj_pw)
        det = model.module.head if is_parallel(model) else model.head
        self.balance = {3: [4.0, 1.0, 0.4]}.get(det.nl, [4.0, 1.0, 0.25, 0.06, .02])
        self.autobalance = bool(cfg.Loss.autobalance)
        self.ssi = [float(s) for s in det.stride].index(16.0) if self.autobalance else 0
        self.gr = 1.0
        self.box_w = cfg.SSOD.box_loss_weight
        self.obj_w = cfg.SSOD.obj_loss_weight
        self.cls_w = cfg.SSOD.cls_loss_weight * cfg.Dataset.nc / 80. * 3. / det.nl
        self.anchor_t = cfg.Loss.anchor_t
        self.ignore_thres_high = [cfg.SSOD.ignore_thres_high] * cfg.Dataset.nc
        self.ignore_thres_low = [cfg.SSOD.ignore_thres_low] * cfg.Dataset.nc
        self.uncertain_aug = cfg.SSOD.uncertain_aug
        self.use_ota = False
        self.ignore_obj = cfg.SSOD.ignore_obj
        self.pseudo_label_with_obj = cfg.SSOD.pseudo_label_with_obj
        self.pseudo_label_with_bbox = cfg.SSOD.pseudo_label_with_bbox
        self.pseudo_label_with_cls = cfg.SSOD.pseudo_label_with_cls
        self.num_keypoints = cfg.Dataset.np
        # uncertain_aug=False only asks for a single-target assigner (ssod_loss.py:65-67), whose flag the reference's
        # assigner never reads: both settings assign identically
        self.single_targets = not self.uncertain_aug
        for k in 'na', 'nc', 'nl', 'anchors', 'stride':
            setattr(self, k, getattr(det, k))
        self.assigner = YOLOAnchorAssigner(self.na, self.nl, self.anchors, self.anchor_t, det.stride, self.nc,
                                           self.num_keypoints, single_targets=self.single_targets, ota=False)
        self._thr_cache = None

    def _thresholds(self, device):
        key = (tuple(self.ignore_thres_high), tuple(self.ignore_thres_low), str(device))
        if self._thr_cache is None or self._thr_cache[0] != key:
            hi = torch.tensor(self.ignore_thres_high, dtype=torch.float64, device=device)
            lo = torch.tensor(self.ignore_thres_low, dtype=torch.float64, device=device)
            self._thr_cache = (key, hi, lo)
        return self._thr_cache[1], self._thr_cache[2]

    def _select_device(self, targets, n_dev=None):
        """targets [N,9] float64 CUDA -> (out[4,cap,7] fp32, cnt[4] int32), all on the device."""
        _lib.require_cuda(targets)
        t = targets.double().contiguous()
        if t.shape[1] != 9:
            raise RuntimeError("pseudo-label rows must be [N,9] (img,cls,x,y,w,h,conf,obj,cls_conf)")
        cap = max(int(t.shape[0]), 1)
        hi, lo = self._thresholds(t.device)
        out = torch.empty((4, cap, 7), dtype=torch.float32, device=t.device)
        cnt = torch.zeros(4, dtype=torch.int32, device=t.device)
        _lib.check(_lib.lib().etb_select_targets(_lib.ptr(t), _lib.ptr(n_dev), int(t.shape[0]), cap, _lib.ptr(hi),
                                                 _lib.ptr(lo), self.nc, int(self.pseudo_label_with_obj), _lib.ptr(out),
                                                 _lib.ptr(cnt), _lib.stream_ptr()), "etb_select_targets")
        return out, cnt

    def select_targets(self, targets):
        """Reference-shaped result: 4 tensors [n_i,7] fp32 (one D2H read of the 4 counts)."""
        out, cnt = self._select_device(targets)
        c = cnt.cpu().tolist()
        return tuple(out[s, :c[s]] for s in range(4))

    def default_loss(self, p, targets, n_dev=None):
        p = _prep_p(p)
        targets = targets.to(p[0].device)
        if targets.shape[1] > 6:
            sel, cnt = self._select_device(targets, n_dev)
            cap = sel.shape[1]
            sets = [self.assigner.assign(p, sel[0, :, :6], nt_dev=cnt[0:1], cap_rows=cap)]
            for s in (1, 2, 3):
                sets.append(self.assigner.assign(p, sel[s], nt_dev=cnt[s:s + 1], cap_rows=cap, with_pseudo_score=True))
            nsets = 4
        else:
            sets = [self.assigner.assign(p, targets)]
            nsets = 1
        lp = make_loss_params(p, self.na, self.balance, self.box_w, self.obj_w, self.cls_w, self.cp, self.cn,
                              nsets=nsets, ignore_obj=self.ignore_obj, with_bbox=self.pseudo_label_with_bbox,
                              with_cls=self.pseudo_label_with_cls, cls_pw=self.cls_pw, obj_pw=self.obj_pw)
        out4 = _FusedDetLoss.apply(lp, sets, "ssod", *p)
        loss = out4[3:4]
        return loss, dict(ss_box=out4[0:1].detach(), ss_obj=out4[1:2].detach(), ss_cls=out4[2:3].detach())

    def __call__(self, p, targets, n_dev=None):
        return self.default_loss(p, targets, n_dev)
