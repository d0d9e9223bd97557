"""CPU: the burn-in restatement (burnin_ref.CpuBurnInStep) that the GPU burn-in tests compare against -- netD receives
zero gradients (tensors, not None) and is still stepped by weight decay + momentum; the semi-supervised EMA appears only at
epoch == burn_epochs, as a copy of the burn-in EMA; the EMA update counter carries across the switch."""
import numpy as np
import pytest
import torch

import synth
from burnin_ref import CpuBurnInStep

NETD = ["det_%d.conv%d.weight" % (s, c) for s in (8, 16, 32) for c in (1, 2)]


def _setup(img=64):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(0)
    sd = {k: v.detach().clone() for k, v in Model(yolov5_ssod_cfg('s', batch_size=4, img_size=img)).state_dict().items()}
    r = np.random.RandomState(1)
    imgs = torch.from_numpy(r.rand(2, 3, img, img).astype(np.float32))
    uw = torch.from_numpy(r.rand(2, 3, img, img).astype(np.float32))
    return sd, imgs, uw


@pytest.mark.parametrize("da", [False, True])
def test_burn_in_oracle_netd_grads_and_hand_over(da):
    sd, imgs, uw = _setup()
    step = CpuBurnInStep(sd, (1, 2, 3, 1), 1, burn_epochs=2, batch_size=4, bn_momentum=0.03)
    lr, m, wd = 0.01, 0.937, step.opt.param_groups[1]["weight_decay"]
    for epoch, nt in ((0, 6), (1, 0)):
        step.begin_epoch(epoch)
        assert step.semi is None
        w0 = {k: step.student[k].detach().clone() for k in NETD}
        buf0 = {k: step.opt.state[step.student[k]].get("momentum_buffer") for k in NETD}
        buf0 = {k: None if b is None else b.clone() for k, b in buf0.items()}
        loss = step.burn_in_loss(imgs, synth.make_targets(epoch + 1, nt, 2), uw if da else None)
        assert torch.isfinite(loss).all()
        loss.backward()
        g = step.grads()
        for k in NETD:
            assert g[k] is not None, k                          # a zero tensor, never None: SGD steps the parameter
            assert (torch.count_nonzero(g[k]) > 0) == da, k      # DA variant: the domain losses train netD
        step.optimizer_ema()
        if not da:   # zero gradient: torch SGD-Nesterov == pure decay + momentum
            for k in NETD:
                d = wd * w0[k]
                buf = d + (0 if buf0[k] is None else m * buf0[k])
                want = w0[k] - lr * (d + m * buf)
                torch.testing.assert_close(step.student[k].detach(), want, rtol=1e-6, atol=1e-9)
                assert not torch.equal(step.student[k].detach(), w0[k])
    assert step.ema_updates == 2
    student = {k: v.detach().clone() for k, v in step.student.items()}
    step.begin_epoch(2)                                     # hand-over
    assert step.semi is not None and step.ema_updates == 2
    for k, v in step.teacher.items():
        assert torch.equal(step.semi[k], v)
        assert torch.equal(step.student[k].detach(), student[k])      # the student is not reset to the EMA
    with pytest.raises(AssertionError):
        step.burn_in_loss(imgs, synth.make_targets(3, 4, 2))
    step.step(imgs, synth.make_targets(3, 4, 2), uw.flip(3).contiguous(), uw, synth.make_Ms(2, 2, 64))
    assert step.ema_updates == 3
    assert any(not torch.equal(step.semi[k], v) for k, v in step.teacher.items() if v.dtype.is_floating_point)


def test_burn_in_oracle_semi_only_at_the_switch():
    sd, _, _ = _setup()
    step = CpuBurnInStep(sd, (1, 2, 3, 1), 1, burn_epochs=3, batch_size=4)
    for e in (0, 1, 2, 4):
        step.begin_epoch(e)
        assert step.semi is None, e          # resuming past burn_epochs never creates it, as in the reference
    step.begin_epoch(3)
    assert step.semi is not None
