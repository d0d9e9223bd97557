"""LabelMatch pseudo-label creator (reference utils/labelmatch.py:57-354; selected by SSOD.pseudo_label_type == 'LabelMatch',
trainer/ssod_trainer.py:69-71) -- SURVEY.md 8f rank 3.

Per step it is the FairPseudoLabel pipeline (same NMS, same affine transform: the reference's two creators return identical
rows, pinned in tests/golden/labelmatch.npz), so the device work is inherited unchanged from pseudo_label.FairPseudoLabel
(etb_nms_ssod: candidate filter -> NMS -> transform, one batch of launches).  What LabelMatch adds is host-side bookkeeping:
the confidence of every NMS detection is filed under its class for the running epoch (labelmatch.py:289-297), and once per
epoch the per-class thresholds are re-estimated -- low = the score at the resample_low_percent position (capped by the
running mean number of boxes per epoch), high = a 2-component Gaussian-mixture split of the epoch's scores
(labelmatch.py:126-187, 190-239).  The mixture fit stays on the CPU (sklearn, once per epoch), as in the reference.

The detections are copied device -> pinned host asynchronously and folded into the lists lazily (flush()), so the training
step itself still never waits on the host."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .pseudo_label import FairPseudoLabel


class LabelMatch(FairPseudoLabel):
    def __init__(self, cfg, target_data_len, label_num_per_img, cls_ratio_gt):
        super().__init__(cfg)
        self.nc = int(np.asarray(cls_ratio_gt).shape[0])
        self.cls_ratio_gt = cls_ratio_gt
        self.ignore_thres_low, self.ignore_thres_high = cfg.SSOD.ignore_thres_low, cfg.SSOD.ignore_thres_high
        self.cls_thr_high = [self.ignore_thres_high] * self.nc
        self.cls_thr_low = [self.ignore_thres_low] * self.nc
        self.resample_high_percent = cfg.SSOD.resample_high_percent
        self.resample_low_percent = cfg.SSOD.resample_low_percent
        self.max_cls_per_img = 10
        self.target_data_len = target_data_len
        self.anno_num_per_img = label_num_per_img * 3
        self.score_list_epoch = [[] for _ in range(self.nc)]
        self.cls_tmp = np.zeros(self.nc)
        self.cls_num_total = np.zeros(self.nc)
        self.count = 0
        self.pse_count = 0
        self._pending = []          # (det pinned [B,max_det,8], det_cnt pinned [B], event) not yet folded into the lists
        self._hist = None           # int32 [nc + 1] device class histogram of the labeled targets (class_hist())

    # ---- per step -------------------------------------------------------------------------------------------------
    def record_detections(self, det, det_cnt):
        """File conf under cls for every detection, images in order, detections in NMS (descending score) order --
        the loop of labelmatch.py:289-297.  det [B,max_det,8] rows [x1,y1,x2,y2,conf,cls,obj,cls_score], det_cnt [B]."""
        det = np.asarray(det)
        for b, n in enumerate(np.asarray(det_cnt).tolist()):
            for k in range(int(n)):
                self.score_list_epoch[int(det[b, k, 5])].append(float(det[b, k, 4]))

    def create_pseudo_label_device(self, out, M_s, height, width):
        rows, cnt = super().create_pseudo_label_device(out, M_s, height, width)
        if not torch.cuda.is_current_stream_capturing():     # inside a captured step the trainer stages after the replay
            self.stage_detections()
        return rows, cnt

    def stage_detections(self):
        """enqueue the device -> pinned-host copy of the last step's detections (async; folded in by flush())"""
        if self.last_det is None:
            return
        det, det_cnt = self.last_det
        h_det = torch.empty(det.shape, dtype=det.dtype, pin_memory=True)
        h_cnt = torch.empty(det_cnt.shape, dtype=det_cnt.dtype, pin_memory=True)
        h_det.copy_(det, non_blocking=True)
        h_cnt.copy_(det_cnt, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(det.device))
        self._pending.append((h_det, h_cnt, ev))

    def class_hist(self, device):
        """the device accumulator of update_device: int32 [nc + 1], the last slot counting classes outside [0, nc);
        allocated once, so a captured step adds into the same memory on every replay"""
        if self._hist is None:
            self._hist = torch.zeros(self.nc + 1, dtype=torch.int32, device=device)
        return self._hist

    def update_device(self, targets, n_dev=None):
        """`update(targets, n_img, n_pse_img)`'s class histogram without a host sync (etb_label_class_hist): the classes
        of the labeled targets [n,6] are added into class_hist() and folded into cls_tmp by flush().  n_dev (int32[1]
        CUDA): targets is a buffer whose first n_dev rows are the labels; the rows past them are not counted."""
        t = targets if targets.is_cuda else targets.to(torch.cuda.current_device())
        t = t.float().contiguous()
        _lib.require_cuda(t, n_dev)
        hist = self.class_hist(t.device)
        cap = int(t.shape[0])
        _lib.check(_lib.lib().etb_label_class_hist(_lib.ptr(t) if cap else C.c_void_p(0), _lib.ptr(n_dev),
                                                   0 if n_dev is not None else cap, cap, int(t.shape[1]), self.nc,
                                                   _lib.ptr(hist), _lib.stream_ptr(t.device)), "etb_label_class_hist")

    def flush(self):
        """fold every finished device->host copy into the epoch's score lists (in step order), and the device class
        histogram into cls_tmp (the accumulator is zeroed, stream-ordered).  A labeled class outside [0, nc) raises
        IndexError, as the reference's `cls_tmp[int(l[1:2])] += 1` does."""
        for h_det, h_cnt, ev in self._pending:
            ev.synchronize()
            self.record_detections(h_det.numpy(), h_cnt.numpy())
        self._pending = []
        if self._hist is not None:
            h = self._hist.cpu().numpy()
            self._hist.zero_()
            if h[self.nc]:
                raise IndexError("LabelMatch: %d labeled target(s) with a class outside [0, %d)" % (int(h[self.nc]), self.nc))
            self.cls_tmp += h[:self.nc]

    def update(self, labels, n=1, pse_n=1):
        """labelmatch.py:114-124: image / pseudo-label counters and the per-class histogram of the rows handed to the loss"""
        self.count += n
        self.pse_count += pse_n
        for row in labels:
            self.cls_tmp[int(row[1])] += 1

    # ---- per epoch ------------------------------------------------------------------------------------------------
    @staticmethod
    def gmm_policy(scores, given_gt_thr=0.5, policy='high'):
        """labelmatch.py:126-187: split the scores with a 2-component 1-D Gaussian mixture (components initialised at the
        min and the max score); 'high': threshold = lowest score of the positive component that is at least as large as the
        positive component's most likely score; 'middle': lowest score assigned to the positive component."""
        import sklearn.mixture as skm
        if len(scores) < 4:
            return given_gt_thr
        if isinstance(scores, torch.Tensor):
            scores = scores.cpu().numpy()
        scores = np.asarray(scores)
        if scores.ndim == 1:
            scores = scores[:, None]
        assert policy in ('middle', 'high')
        gmm = skm.GaussianMixture(2, weights_init=[0.5, 0.5], means_init=[[np.min(scores)], [np.max(scores)]],
                                  precisions_init=[[[1.0]], [[1.0]]])
        gmm.fit(scores)
        assign = gmm.predict(scores)
        if not (assign == 1).any():
            return given_gt_thr
        if policy == 'high':
            loglik = gmm.score_samples(scores)
            loglik[assign == 0] = -np.inf
            peak = np.argmax(loglik, axis=0)
            pos = (assign == 1) & (scores >= scores[peak]).squeeze()
            thr = float(scores[pos].min())
        else:
            thr = float(scores[assign == 1].min())
        return max(given_gt_thr, thr)

    def update_epoch_cls_thr(self, epoch):
        """labelmatch.py:190-239: new per-class thresholds from the epoch's scores, then reset the epoch state"""
        self.flush()
        for c in range(self.nc):
            s = self.score_list_epoch[c]
            s.sort(reverse=True)
            self.cls_num_total[c] += len(s)
            cap = int(self.cls_num_total[c] / (epoch + 1))
            if not s:
                self.cls_thr_high[c], self.cls_thr_low[c] = self.ignore_thres_high, self.ignore_thres_low
                continue
            pos_low = min(cap, int(len(s) * self.resample_low_percent))
            self.cls_thr_high[c] = self.gmm_policy(np.array(s), given_gt_thr=0.0, policy='high')
            self.cls_thr_low[c] = max(self.ignore_thres_low, s[pos_low])
        self.score_list_epoch = [[] for _ in range(self.nc)]
        self.cls_tmp = np.zeros(self.nc)
        self.count = 0
        self.pse_count = 0
