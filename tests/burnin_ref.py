"""TEST INFRASTRUCTURE / CPU BASELINE ONLY -- the SSOD burn-in step and the hand-over to the semi-supervised phase
(trainer/ssod_trainer.py:295-317, 421-456 train_without_unlabeled, 490-533 train_without_unlabeled_da, 458-488
update_optimizer) restated on the CPU from the oracle pieces: TrunkRef (torch fp32), port.build_targets / det_loss,
domain_focal, torch.optim.SGD and one EMA.  The `0 *` terms of the reference are kept, so torch's own SGD sees zero
(not None) gradients for netD and applies weight decay + momentum to its weights."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import port
from oracle.step_ref import ANCHORS_GRID, STRIDES, CpuSSODStep, domain_focal
from oracle.trunk_ref import TrunkRef


class _GradReverse(torch.autograd.Function):     # models/detector/yolo_ssod.py:158-172
    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return -g


class _NeckTap(TrunkRef):
    """TrunkRef that also hands out the three neck outputs (the Detect / netD inputs)"""

    def c3(self, p, x, n, shortcut, train):
        y = super().c3(p, x, n, shortcut, train)
        if p in ("neck.C2", "neck.C3", "neck.C4"):
            self.taps.append(y)
        return y


class CpuBurnInStep(CpuSSODStep):
    """`teacher` is the burn-in ModelEMA, `semi` stays None until begin_epoch(burn_epochs) copies the teacher into it;
    after that, step() is the semi-supervised step of CpuSSODStep with both EMAs."""

    def __init__(self, state_dict, depth, neck_depth, burn_epochs, da_loss_weights=0.01, **kw):
        super().__init__(state_dict, depth, neck_depth, **kw)
        self.semi = None
        self.burn_epochs, self.da_w, self.epoch = burn_epochs, da_loss_weights, 0

    def begin_epoch(self, epoch):
        self.epoch = epoch
        if self.burn_epochs > 0 and epoch == self.burn_epochs:
            self.semi = {k: v.detach().clone() for k, v in self.teacher.items()}

    def _forward(self, x):
        trunk = _NeckTap(self.student, self.depth, self.neck_depth, bn_momentum=self.bn_momentum)
        trunk.taps = []
        raw, _ = trunk.forward(x, train=True, with_features=False)
        sd = self.student
        feat = [F.conv2d(F.relu(F.conv2d(_GradReverse.apply(f), sd[d + ".conv1.weight"])), sd[d + ".conv2.weight"])
                for d, f in zip(("det_8", "det_16", "det_32"), trunk.taps)]
        return raw, feat

    def burn_in_step(self, imgs, targets, u_weak=None):
        """u_weak None: train_without_unlabeled, else train_without_unlabeled_da.  Returns the loss."""
        loss = self.burn_in_loss(imgs, targets, u_weak)
        loss.backward()
        self.optimizer_ema()
        return float(loss.detach())

    def burn_in_loss(self, imgs, targets, u_weak=None):
        assert self.semi is None, "burn-in step after the hand-over"
        n = imgs.shape[0]
        H, W = imgs.shape[2:]
        shapes = [(H // s, W // s) for s in STRIDES]
        raw, feat = self._forward(imgs if u_weak is None else torch.cat([imgs, u_weak], 0))
        sets = [port.build_targets(np.asarray(targets, dtype=np.float32).reshape(-1, 6), ANCHORS_GRID, shapes)]
        loss, _ = port.det_loss([r[:n] for r in raw], sets, [4.0, 1.0, 0.4], 0.05, 0.7, 0.3)
        if u_weak is None:
            loss = loss + 0 * (feat[0].mean() + feat[1].mean() + feat[2].mean())
        else:
            loss = loss + domain_focal([f[:n] for f in feat], 0) * self.da_w + domain_focal([f[n:] for f in feat], 1) * self.da_w \
                + 0 * raw[0][n:].mean() + 0 * raw[1][n:].mean() + 0 * raw[2][n:].mean()
        return loss

    def optimizer_ema(self):
        """update_optimizer after backward: accumulate / warm-up, SGD-Nesterov + ema.update when due (no semi_ema)"""
        accumulate = 1 if self.fixed_accumulate else max(round(64 / self.batch_size), 1)
        if self.warmup is not None and self.ni <= self.warmup[0]:
            xi = [0, self.warmup[0]]
            accumulate = max(1, np.interp(self.ni, xi, [1, 1 if self.fixed_accumulate else 64 / self.batch_size]).round())
            for j, pg in enumerate(self.opt.param_groups):
                pg['lr'] = float(np.interp(self.ni, xi, [self.warmup[1] if j == 2 else 0.0, self.lr0]))
                pg['momentum'] = float(np.interp(self.ni, xi, [self.warmup[2], self.momentum0]))
        ni, self.ni = self.ni, self.ni + 1
        if ni - self.last_opt_step < accumulate:
            return
        self.last_opt_step = ni
        self.opt.step()
        self.opt.zero_grad()
        self.ema_updates += 1
        d = 0.9999 * (1 - math.exp(-self.ema_updates / 2000))
        with torch.no_grad():
            for k, v in self.teacher.items():
                if v.dtype.is_floating_point:
                    v.mul_(d).add_((1.0 - d) * self.student[k].detach())

    def grads(self):
        """{state_dict key: .grad} of every trained tensor (None where torch never materialised one)"""
        return {k: v.grad for k, v in self.student.items() if v.requires_grad}
