"""YOLOAnchorAssigner with the reference's surface (models/assigner/yolo_anchor_assigner.py:12-51), backed by
etb_build_targets: one launch for all levels, order-preserving, integer-exact with the CPU oracle.

`forward(p, targets, with_pseudo_score=False)` returns the reference's tuple of per-level lists
(tcls, tbox, indices, anch[, tscore]) -- that costs one D2H read of the per-level counts.  The fused losses
call `assign()` instead and keep everything (counts included) on the device.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import EtbAssignLevels, EtbAssignOut, ETB_MAX_LEVELS


class AssignBuffers:
    """Device buffers of one etb_build_targets call (capacity `cap` rows per level)."""

    def __init__(self, nl, cap, device, with_score):
        self.nl, self.cap, self.with_score = nl, cap, with_score
        c = max(cap, 1)
        self.idx = torch.empty((nl, c, 4), dtype=torch.int32, device=device)
        self.tbox = torch.empty((nl, c, 4), dtype=torch.float32, device=device)
        self.anch = torch.empty((nl, c, 2), dtype=torch.float32, device=device)
        self.tcls = torch.empty((nl, c), dtype=torch.int32, device=device)
        self.tscore = torch.empty((nl, c), dtype=torch.float32, device=device)
        self.cnt = torch.zeros((ETB_MAX_LEVELS,), dtype=torch.int32, device=device)
        self.struct = EtbAssignOut()
        for l in range(nl):
            self.struct.idx[l] = self.idx[l].data_ptr()
            self.struct.tbox[l] = self.tbox[l].data_ptr()
            self.struct.anch[l] = self.anch[l].data_ptr()
            self.struct.tcls[l] = self.tcls[l].data_ptr()
            self.struct.tscore[l] = self.tscore[l].data_ptr()
        self.struct.cnt = self.cnt.data_ptr()
        self.struct.cap = cap


class YOLOAnchorAssigner:
    def __init__(self, na, nl, anchors, anchor_t, stride, nc=80, num_keypoints=0, single_targets=False, ota=False,
                 top_k=10):
        if num_keypoints or ota:
            raise NotImplementedError("efficientteacher_b200: only build_targets / build_uc_targets_aug are on the "
                                      "hot path (SURVEY.md section 8 a9); OTA / keypoint assigners are out of scope")
        # single_targets is stored and never read, as in the reference (yolo_anchor_assigner.py:34-51): its
        # build_single_targets is unreachable, so single_targets=True assigns exactly as the default does
        self.single_targets = single_targets
        self.na, self.nl, self.anchors, self.anchor_t = na, nl, anchors, anchor_t
        self.nc, self.np, self.stride, self.ota, self.top_k = nc, num_keypoints, stride, ota, top_k
        assert na == 3 and 1 <= nl <= ETB_MAX_LEVELS
        self._levels = None

    def _level_struct(self, p):
        shapes = tuple((int(pi.shape[2]), int(pi.shape[3])) for pi in p)  # (ny, nx)
        if self._levels is None or self._levels[0] != shapes:
            lv = EtbAssignLevels()
            lv.nl = self.nl
            anc = self.anchors.detach().float().cpu()
            for l, (ny, nx) in enumerate(shapes):
                lv.nx[l], lv.ny[l] = nx, ny
                for k in range(6):
                    lv.anchors[l][k] = float(anc[l].reshape(-1)[k])
            lv.anchor_t = float(self.anchor_t)
            self._levels = (shapes, lv)
        return self._levels[1]

    def assign(self, p, targets, nt_dev=None, cap_rows=None, with_pseudo_score=False):
        """Device-resident assignment.  targets [nt, 6|7] fp32 CUDA; nt may live on the device (nt_dev int32[1])."""
        _lib.require_cuda(targets)
        tstride = 7 if with_pseudo_score else 6
        t = targets[:, :tstride].contiguous().float() if targets.shape[1] != tstride or targets.dtype != torch.float32 \
            or not targets.is_contiguous() else targets
        nt = int(t.shape[0]) if cap_rows is None else int(cap_rows)
        out = AssignBuffers(self.nl, 15 * nt, t.device, with_pseudo_score)
        lv = self._level_struct(p)
        _lib.check(_lib.lib().etb_build_targets(_lib.ptr(t) if t.numel() else C.c_void_p(0),
                                                _lib.ptr(nt_dev), 0 if nt_dev is not None else int(t.shape[0]), tstride,
                                                C.byref(lv), C.byref(out.struct), _lib.stream_ptr()),
                   "etb_build_targets")
        out._keep = t
        return out

    @torch.no_grad()
    def forward(self, p, targets, with_pseudo_score=False):
        out = self.assign(p, targets, with_pseudo_score=with_pseudo_score)
        cnt = out.cnt.cpu().tolist()
        tcls, tbox, indices, anch, tscore = [], [], [], [], []
        for l in range(self.nl):
            n = cnt[l]
            idx = out.idx[l, :n].long()
            indices.append((idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]))
            tbox.append(out.tbox[l, :n])
            anch.append(out.anch[l, :n])
            tcls.append(out.tcls[l, :n].long())
            tscore.append(out.tscore[l, :n])
        if with_pseudo_score:
            return tcls, tbox, indices, anch, tscore
        return tcls, tbox, indices, anch

    __call__ = forward
