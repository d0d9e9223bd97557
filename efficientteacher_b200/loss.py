"""ComputeLoss with the reference's surface (models/loss/loss.py:93-309, default_loss branch), backed by the
fused forward/backward kernels of csrc/loss.cu.  `bbox_iou` mirrors utils/metrics.py:207-249 (CIoU, xywh).

Call contract kept: ComputeLoss(model, cfg)(p, targets[nt,6]) -> (loss[1] requiring grad, dict(box,obj,cls,loss)).
"""
import ctypes as C

import torch

from . import _lib, _ws
from ._lib import EtbLossParams, EtbAssignOut, ETB_MAX_LEVELS
from .assigner import YOLOAnchorAssigner
from .ema import is_parallel


def smooth_BCE(eps=0.1):  # reference models/loss/loss.py:16-18
    return 1.0 - 0.5 * eps, 0.5 * eps


def bbox_iou(box1, box2, x1y1x2y2=True, GIoU=False, DIoU=False, CIoU=False, eps=1e-7):
    """CIoU of box1 [4,n] vs box2 [n,4] (centre/size), the only branch on the hot path."""
    if x1y1x2y2 or not CIoU or GIoU or DIoU or eps != 1e-7:
        raise NotImplementedError("efficientteacher_b200.bbox_iou implements the hot-path branch only: "
                                  "x1y1x2y2=False, CIoU=True (reference utils/metrics.py:207-249)")
    _lib.require_cuda(box1, box2)
    b1 = box1.t().contiguous().float()
    b2 = box2.contiguous().float()
    out = torch.empty((b1.shape[0],), dtype=torch.float32, device=b1.device)
    _lib.check(_lib.lib().etb_bbox_ciou(_lib.ptr(b1), _lib.ptr(b2), b1.shape[0], _lib.ptr(out), _lib.stream_ptr()),
               "etb_bbox_ciou")
    return out


def make_loss_params(p, na, balance, box_w, obj_w, cls_w, cp, cn, nsets=1, ignore_obj=False, with_bbox=False,
                     with_cls=False, cls_pw=1.0, obj_pw=1.0, fl_gamma=0.0, balance_state=None, ssi=0):
    """balance_state: float64 [nl] CUDA tensor (autobalance) that the forward reads and advances, or None"""
    lp = EtbLossParams()
    lp.nl = len(p)
    lp.B, lp.na, lp.no = int(p[0].shape[0]), na, int(p[0].shape[-1])
    for l, pi in enumerate(p):
        assert pi.shape[1] == na
        lp.ny[l], lp.nx[l] = int(pi.shape[2]), int(pi.shape[3])
        lp.balance[l] = float(balance[l])
    lp.box_w, lp.obj_w, lp.cls_w, lp.cp, lp.cn = float(box_w), float(obj_w), float(cls_w), float(cp), float(cn)
    lp.nsets, lp.ignore_obj, lp.with_bbox, lp.with_cls = nsets, int(ignore_obj), int(with_bbox), int(with_cls)
    lp.cls_pw, lp.obj_pw, lp.fl_gamma, lp.ssi = float(cls_pw), float(obj_pw), float(fl_gamma), int(ssi)
    lp.balance_state = balance_state.data_ptr() if balance_state is not None else None
    return lp


class _FusedDetLoss(torch.autograd.Function):
    """out4 = [lbox, lobj, lcls, loss*B]; only d(out4[3]) is propagated (the dict entries are logging values)."""

    @staticmethod
    def forward(ctx, lp, sets, tag, *p):
        lib = _lib.lib()
        dev = p[0].device
        nl = len(p)
        cap = sets[0].cap
        nbytes = lib.etb_loss_workspace_bytes(C.byref(lp), cap)
        # the backward re-reads this workspace, so it is private to the call
        ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
        out4 = torch.empty(4, dtype=torch.float32, device=dev)
        parr = (C.c_void_p * nl)(*[t.data_ptr() for t in p])
        sarr = (EtbAssignOut * len(sets))(*[s.struct for s in sets])
        _lib.check(lib.etb_loss_forward(parr, C.byref(lp), sarr, _lib.ptr(out4), _lib.ptr(ws), ws.numel(),
                                        _lib.stream_ptr()), "etb_loss_forward")
        ctx.lp, ctx.sets, ctx.ws, ctx.p = lp, sets, ws, p
        return out4

    @staticmethod
    def backward(ctx, g4):
        lib = _lib.lib()
        p, lp, sets = ctx.p, ctx.lp, ctx.sets
        nl = len(p)
        from .autograd_conv import grad_buffer_for
        grads = [grad_buffer_for(t) for t in p]      # batch slices of one buffer when p came out of split_batch
        gscale = g4[3:4].contiguous().float()
        parr = (C.c_void_p * nl)(*[t.data_ptr() for t in p])
        garr = (C.c_void_p * nl)(*[t.data_ptr() for t in grads])
        sarr = (EtbAssignOut * len(sets))(*[s.struct for s in sets])
        _lib.check(lib.etb_loss_backward(parr, garr, C.byref(lp), sarr, _lib.ptr(gscale), _lib.ptr(ctx.ws),
                                         ctx.ws.numel(), _lib.stream_ptr()), "etb_loss_backward")
        return (None, None, None) + tuple(grads)


def _prep_p(p):
    out = []
    for pi in p:
        if pi.dtype != torch.float32:
            pi = pi.float()
        if not pi.is_contiguous():
            pi = pi.contiguous()
        out.append(pi)
    return out


class ComputeLoss:
    """cfg.Loss.cls_pw / obj_pw (BCE positive weights), fl_gamma (focal loss) and autobalance as the reference applies
    them (models/loss/loss.py:98-124,191-197).  With autobalance the balance lives on the device as float64 and the loss
    kernel advances it on every call, captured replays included; `balance` reads it back (one host sync) and assigning
    a list to it uploads in place."""

    def __init__(self, model, cfg):
        self.sort_obj_iou = False
        if cfg.Loss.assigner_type == 'SimOTA':
            raise NotImplementedError("OTA loss is not on the hot path (use_ota=False in every shipped config)")
        self.cp, self.cn = smooth_BCE(eps=cfg.Loss.label_smoothing)
        self.cls_pw, self.obj_pw, self.fl_gamma = float(cfg.Loss.cls_pw), float(cfg.Loss.obj_pw), float(cfg.Loss.fl_gamma)
        det = model.module.head if is_parallel(model) else model.head
        self.gr, self.autobalance = 1.0, bool(cfg.Loss.autobalance)
        balance = {3: [4.0, 1.0, 0.4]}.get(det.nl, [4.0, 1.0, 0.25, 0.06, .02])
        if self.autobalance:
            self.ssi = [float(s) for s in det.stride].index(16.0)      # stride 16 index
            dev = det.anchors.device
            self.balance_state = torch.tensor(balance[:det.nl], dtype=torch.float64, device=dev)
        else:
            self.ssi = 0
            self.balance_state = None
            self._balance = balance
        nl = det.nl
        nc = 1 if cfg.single_cls else cfg.Dataset.nc
        self.box_w = cfg.Loss.box * 3.0 / nl
        self.obj_w = cfg.Loss.obj
        self.cls_w = cfg.Loss.cls * nc / 80. * 3. / nl
        self.anchor_t = cfg.Loss.anchor_t
        self.single_targets = cfg.Loss.single_targets
        for k in 'na', 'nc', 'nl', 'num_keypoints', 'anchors':
            setattr(self, k, getattr(det, k))
        if self.num_keypoints:
            raise NotImplementedError("keypoint loss is out of scope")
        self.ota = False
        self.assigner = YOLOAnchorAssigner(self.na, self.nl, self.anchors, self.anchor_t, det.stride, self.nc,
                                           self.num_keypoints, single_targets=self.single_targets, ota=False)

    def default_loss(self, p, targets, n_dev=None):
        """n_dev (int32[1] CUDA): targets is a buffer of capacity targets.shape[0] whose first n_dev rows are the labels --
        the label count stays on the device, so one captured graph serves batches with any number of labels."""
        p = _prep_p(p)
        targets = targets.to(p[0].device)
        if n_dev is None:
            sets = [self.assigner.assign(p, targets)]
        else:
            sets = [self.assigner.assign(p, targets, nt_dev=n_dev, cap_rows=targets.shape[0])]
        if self.balance_state is not None and self.balance_state.device != p[0].device:
            self.balance_state = self.balance_state.to(p[0].device)
        bal = self._balance if self.balance_state is None else [0.0] * self.nl
        lp = make_loss_params(p, self.na, bal, self.box_w, self.obj_w, self.cls_w, self.cp, self.cn,
                              cls_pw=self.cls_pw, obj_pw=self.obj_pw, fl_gamma=self.fl_gamma,
                              balance_state=self.balance_state, ssi=self.ssi)
        out4 = _FusedDetLoss.apply(lp, sets, "sup", *p)
        lbox, lobj, lcls = out4[0:1].detach(), out4[1:2].detach(), out4[2:3].detach()
        loss = out4[3:4]
        return loss, dict(box=lbox, obj=lobj, cls=lcls, loss=loss)

    def __call__(self, p, targets, n_dev=None):
        return self.default_loss(p, targets, n_dev)

    @property
    def balance(self):
        """The per-level objectness balance: a plain list, or with autobalance the device state read back as floats"""
        if self.balance_state is None:
            return self._balance
        return self.balance_state.tolist()

    @balance.setter
    def balance(self, values):
        if self.balance_state is None:
            self._balance = list(values)
        else:
            with torch.no_grad():      # in place: a captured step keeps reading and advancing the same tensor
                self.balance_state.copy_(torch.tensor(list(values), dtype=torch.float64))
