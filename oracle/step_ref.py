"""TEST INFRASTRUCTURE / CPU BASELINE ONLY -- the whole SSOD step (trainer/ssod_trainer.py:587-680, 458-488) restated on
the CPU from the oracle pieces: TrunkRef (torch fp32) for teacher + student, port.nms_ssod / pseudo_label_rows /
select_targets / build_targets / det_loss, SGD-Nesterov (torch.optim) and the two EMA updates.
Used by bench.py (`cpu_baseline`, `--impl reference`) and by the step-level parity test."""
import math

import numpy as np
import torch

from . import port
from .trunk_ref import TrunkRef

ANCHORS_GRID = np.array([[[1.25, 1.625], [2.0, 3.75], [4.125, 2.875]], [[1.875, 3.8125], [3.875, 2.8125], [3.6875, 7.4375]],
                         [[3.625, 2.8125], [4.875, 6.1875], [11.65625, 10.1875]]], dtype=np.float32)
STRIDES = (8, 16, 32)


def domain_focal(feature, label):
    logits = torch.cat([f.permute(0, 2, 3, 1).reshape(-1, 2) for f in feature], 0)
    logp = torch.log_softmax(logits, 1)[:, label]
    return 0.5 * (-(1 - logp.exp()) ** 2 * logp).mean()


class CpuSSODStep:
    def __init__(self, state_dict, depth, neck_depth, lr=0.01, momentum=0.937, weight_decay=0.0005, batch_size=32,
                 ema_updates=0, semi_decay=0.999, teacher_loss_weight=3.0, bn_momentum=0.0, warmup=None, fixed_accumulate=True,
                 nc=80, anchor_t=4.0, da_loss_weight=0.0):
        """nc / anchor_t: the dataset's class count and Loss.anchor_t; the class-loss weight is derived from nc as
        ComputeLoss / ComputeStudentMatchLoss do (cls * nc / 80 * 3 / nl, models/loss/loss.py:124), and the per-class
        pseudo-label thresholds are sized by it.  da_loss_weight: SSOD.da_loss_weights when SSOD.with_da_loss is on (the
        domain losses of the labeled and unlabeled halves join the supervised loss, trainer/ssod_trainer.py:633-636), else 0.
        bn_momentum > 0: the student's running statistics are updated like nn.BatchNorm2d(momentum) does (needed for
        multi-step trajectories; the single-step parity tests leave it 0).  warmup = (nw, warmup_bias_lr, warmup_momentum):
        apply the reference's per-iteration warm-up (trainer/trainer.py:388-395: group index 2 gets warmup_bias_lr)."""
        self.bn_momentum, self.warmup, self.lr0, self.momentum0, self.ni = bn_momentum, warmup, lr, momentum, 0
        self.fixed_accumulate, self.batch_size, self.last_opt_step = fixed_accumulate, batch_size, -1
        self.student = {k: v.detach().clone().float() for k, v in state_dict.items()}
        self.teacher = {k: v.detach().clone() for k, v in self.student.items()}
        self.semi = {k: v.detach().clone() for k, v in self.student.items()}
        self.depth, self.neck_depth = depth, neck_depth
        g_b, g_w, g_bn = [], [], []
        for k, v in self.student.items():
            if not v.dtype.is_floating_point or "running_" in k or k.endswith("anchors"):
                continue
            v.requires_grad_(True)
            if k.endswith(".bn.weight"):
                g_bn.append(v)
            elif k.endswith(".bias"):
                g_b.append(v)
            else:
                g_w.append(v)
        wd = weight_decay * batch_size * max(round(64 / batch_size), 1) / 64
        self.opt = torch.optim.SGD(g_b, lr=lr, momentum=momentum, nesterov=True)
        self.opt.add_param_group({'params': g_w, 'weight_decay': wd})
        self.opt.add_param_group({'params': g_bn})
        self.ema_updates, self.semi_decay, self.tlw = ema_updates, semi_decay, teacher_loss_weight
        self.nc, self.anchor_t, self.da_w = nc, anchor_t, da_loss_weight
        self.cls_w = 0.3 * nc / 80. * 3. / len(STRIDES)

    def step(self, imgs, targets, u_strong, u_weak, Ms, conf_thres=0.1, iou_thres=0.65):
        H, W = u_weak.shape[2:]
        shapes = [(H // s, W // s) for s in STRIDES]
        with torch.no_grad():
            raw, _ = TrunkRef(self.teacher, self.depth, self.neck_depth).forward(u_weak, train=False)
            pred = port.detect_decode(raw, ANCHORS_GRID, STRIDES).numpy()
        dets = port.nms_ssod(pred, conf_thres, iou_thres)
        rows = port.pseudo_label_rows(dets, Ms, H, W)
        n_img = imgs.shape[0]
        raw, feat = TrunkRef(self.student, self.depth, self.neck_depth, bn_momentum=self.bn_momentum).forward(torch.cat([imgs, u_strong], 0), train=True)
        sup_p, un_p = [r[:n_img] for r in raw], [r[n_img:] for r in raw]
        sup_sets = [port.build_targets(np.asarray(targets), ANCHORS_GRID, shapes, self.anchor_t)]
        sup_loss, _ = port.det_loss(sup_p, sup_sets, [4.0, 1.0, 0.4], 0.05, 0.7, self.cls_w)
        sup_loss = sup_loss + domain_focal([f[:n_img] for f in feat], 0) * self.da_w + \
            domain_focal([f[n_img:] for f in feat], 1) * self.da_w
        if len(rows):
            sel = port.select_targets(rows, [0.6] * self.nc, [0.1] * self.nc, True)
            sets = [port.build_targets(sel[0][:, :6], ANCHORS_GRID, shapes, self.anchor_t)]
            sets += [port.build_targets(s, ANCHORS_GRID, shapes, self.anchor_t, with_score=True) for s in sel[1:]]
            un_loss, _ = port.det_loss(un_p, sets, [4.0, 1.0, 0.4], 0.05, 0.7, self.cls_w, with_bbox=True)
        else:
            un_loss = torch.zeros(1)
        loss = sup_loss + un_loss * self.tlw
        # ssod_trainer.py:458-488: backward (gradients accumulate), accumulate / warm-up, optimizer + EMA when due
        loss.backward()
        accumulate = 1 if self.fixed_accumulate else max(round(64 / self.batch_size), 1)
        if self.warmup is not None and self.ni <= self.warmup[0]:
            xi = [0, self.warmup[0]]
            accumulate = max(1, np.interp(self.ni, xi, [1, 1 if self.fixed_accumulate else 64 / self.batch_size]).round())
            for j, pg in enumerate(self.opt.param_groups):
                pg['lr'] = float(np.interp(self.ni, xi, [self.warmup[1] if j == 2 else 0.0, self.lr0]))
                pg['momentum'] = float(np.interp(self.ni, xi, [self.warmup[2], self.momentum0]))
        ni, self.ni = self.ni, self.ni + 1
        if ni - self.last_opt_step < accumulate:
            return float(loss.detach()), len(rows)
        self.last_opt_step = ni
        self.opt.step()
        self.opt.zero_grad()
        self.ema_updates += 1
        d = 0.9999 * (1 - math.exp(-self.ema_updates / 2000))
        with torch.no_grad():
            for k, v in self.teacher.items():
                if v.dtype.is_floating_point:
                    v.mul_(d).add_((1.0 - d) * self.student[k].detach())
                    s = self.semi[k]
                    s.mul_(self.semi_decay).add_((1.0 - self.semi_decay) * v)
        return float(loss.detach()), len(rows)
