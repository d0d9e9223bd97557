"""GPU (H100): the SSOD burn-in phase -- train_without_unlabeled[_da] (eager and captured), the label count kept on the
device by ComputeLoss(n_dev=...), and the hand-over to the semi-supervised step at epoch == burn_epochs -- against the
CPU restatement in burnin_ref.py."""
import numpy as np
import pytest
import torch

import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NETD = ["det_%d.conv%d.weight" % (s, c) for s in (8, 16, 32) for c in (1, 2)]


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _step(img, batch, da=False, burn=2, **hyp):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep
    torch.manual_seed(0)
    cfg = yolov5_ssod_cfg('l_shallow', batch_size=batch, img_size=img)
    cfg.hyp.burn_epochs = burn
    cfg.SSOD.with_da_loss = da
    for k, v in hyp.items():
        if k == "fixed_accumulate":
            cfg.SSOD.fixed_accumulate = v
        else:
            setattr(cfg.hyp, k, v)
    return SSODTrainerStep(cfg, torch.device(DEV), epochs=300)


def _images(seed, n, img):
    return torch.from_numpy(np.random.RandomState(seed).rand(n, 3, img, img).astype(np.float32))


def _cpu(st, **kw):
    from burnin_ref import CpuBurnInStep
    return CpuBurnInStep({k: v.detach().cpu().clone() for k, v in st.model.state_dict().items()}, (1, 2, 3, 1), 1,
                         st.cfg.hyp.burn_epochs, da_loss_weights=st.cfg.SSOD.da_loss_weights, batch_size=st.batch_size, **kw)


@pytest.mark.parametrize("img,da", [(256, False), (640, False), (256, True), (640, True)])
def test_burn_in_step_matches_cpu_step(img, da):
    from efficientteacher_b200.autograd_conv import SplitBatchFn
    bl, bu = 2, 2 if da else 0
    st = _step(img, bl + bu, da=da)
    cpu = _cpu(st, warmup=(st.nw, st.warmup_bias_lr, st.warmup_momentum), fixed_accumulate=False)
    imgs, uw = _images(3, bl, img), _images(4, bu, img) if da else None
    tg = synth.make_targets(7, 8 * bl, bl)
    before_w = st.model.backbone.stage1.conv.weight.detach().clone()
    before_g = st.model.backbone.stage1.bn.weight.detach().clone()
    copied = SplitBatchFn.stats["copied"]
    if da:
        loss = st.train_without_unlabeled_da(imgs.to(DEV), torch.from_numpy(tg).to(DEV), uw.to(DEV), 0)
    else:
        loss = st.train_without_unlabeled(imgs.to(DEV), torch.from_numpy(tg).to(DEV), 0)
    ref = cpu.burn_in_step(imgs, tg, uw)
    assert abs(loss.item() - ref) <= 0.03 * abs(ref), (loss.item(), ref)
    assert st.ema.updates == 1 and st.semi_ema is None and st.in_burn_in
    # ni = 0 of the warm-up: conv-weight lr is 0, the BatchNorm weights step with warmup_bias_lr
    assert torch.equal(before_w, st.model.backbone.stage1.conv.weight.detach())
    assert not torch.equal(before_g, st.model.backbone.stage1.bn.weight.detach())
    # the unlabeled half of the Detect / netD gradients went through SplitBatchFn's zero-copy backward
    assert SplitBatchFn.stats["copied"] == copied


def test_netd_zero_gradients_and_exact_decay():
    """3 burn-in steps without warm-up (lr 0.01 from the first step): netD's gradient-arena slices are exactly zero before
    every optimizer step, and its weights equal torch.optim.SGD's on the CPU -- pure fp32 decay + Nesterov momentum."""
    img, B = 256, 2
    st = _step(img, B, warmup_epochs=0, fixed_accumulate=True)
    cpu = _cpu(st, warmup=None, fixed_accumulate=True)
    params = dict(st.model.named_parameters())
    w0 = {k: params[k].detach().cpu().clone() for k in NETD}
    seen = []
    inner = st._optimizer_ema

    def checked(ni):
        for k in NETD:
            seen.append(int(torch.count_nonzero(params[k].grad)))
        return inner(ni)
    st._optimizer_ema = checked
    imgs = _images(3, B, img)
    for i in range(3):
        tg = synth.make_targets(10 + i, 6 + 4 * i, B)
        st.train_without_unlabeled(imgs.to(DEV), torch.from_numpy(tg).to(DEV), i)
        cpu.burn_in_step(imgs, tg)
    assert len(seen) == 3 * len(NETD) and not any(seen), seen
    assert st.ema.updates == cpu.ema_updates == 3
    for k in NETD:
        got, want = params[k].detach().cpu(), cpu.student[k].detach()
        assert not torch.equal(want, w0[k])
        assert ((got - want).abs().max() / want.abs().max()).item() <= 1e-6, k


@pytest.mark.parametrize("nt", [0, 5, 37])
def test_padded_labels_match_unpadded(nt):
    from efficientteacher_b200.loss import ComputeLoss
    from tiny_cfg import ssod_cfg, HeadOnlyModel
    B, cap = 2, 64
    crit = ComputeLoss(HeadOnlyModel().to(DEV), ssod_cfg())
    logits = synth.make_head_logits(21, B, img=256)
    tg = torch.from_numpy(synth.make_targets(22, nt, B)).to(DEV)
    buf = torch.from_numpy(synth.make_targets(23, cap, B)).to(DEV)    # stale rows past nt must be ignored
    buf[:nt] = tg
    out = []
    for args in ((tg,), (buf, torch.tensor([nt], dtype=torch.int32, device=DEV))):
        p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in logits]
        loss, items = crit(p, *args)
        loss.backward()
        out.append((loss.detach(), {k: v.detach() for k, v in items.items()}, [pi.grad for pi in p]))
    (la, ia, ga), (lb, ib, gb) = out
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()  # noqa: E731
    assert rel(lb, la) <= 1e-6
    for k in ia:
        assert rel(ib[k], ia[k]) <= 1e-6, k
    for a, b in zip(ga, gb):
        assert rel(b, a) <= 1e-6
    if nt == 0:
        assert float(ia["box"]) == 0.0 and float(ia["cls"]) == 0.0 and float(ia["obj"]) > 0.0


@pytest.mark.parametrize("da", [False, True])
def test_graphed_burn_in_matches_eager(da):
    """(eager, eager, graph) x 4 burn-in steps whose batches carry 16 / 0 / 9 / 24 labels: one capture serves them all;
    a batch above the label capacity re-captures once."""
    img, bl, bu = 256, 2, 2 if da else 0
    imgs = _images(3, bl, img).to(DEV)
    uw = _images(4, bu, img).to(DEV) if da else None
    tgs = [torch.from_numpy(synth.make_targets(30 + i, n, bl)).to(DEV) for i, n in enumerate((16, 0, 9, 24))]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        st = _step(img, bl + bu, da=da)
        losses = []
        for i, tg in enumerate(tgs):
            if da:
                f = st.train_without_unlabeled_da_graphed if mode == "graph" else st.train_without_unlabeled_da
                loss = f(imgs, tg, uw, i)
            else:
                f = st.train_without_unlabeled_graphed if mode == "graph" else st.train_without_unlabeled
                loss = f(imgs, tg, i)
            losses.append(float(loss.item()))
        out[mode] = (losses, {k: v.clone() for k, v in st.ema.ema.state_dict().items()}, st.ema.updates)
    assert st.burn_in_captures == 1
    assert out["eager"][2] == out["eager2"][2] == out["graph"][2] == 4
    for i, (a, b, c) in enumerate(zip(out["eager"][0], out["graph"][0], out["eager2"][0])):
        assert abs(a - b) <= 3.0 * abs(a - c) + (0.01 + 0.02 * i) * abs(a), out
    ke = [k for k, v in out["eager"][1].items() if v.dtype.is_floating_point and "running" not in k]
    a, b, c = (torch.cat([out[m][1][k].flatten() for k in ke]) for m in ("eager", "graph", "eager2"))
    rel, rel_eager = ((a - b).norm() / a.norm()).item(), ((a - c).norm() / a.norm()).item()
    assert rel <= 3.0 * rel_eager + 2e-3, (rel, rel_eager)
    # more labels than the capacity: exactly one more capture, which then serves smaller batches again
    cap = st._burn_graph["cap"]
    for i, n in enumerate((cap + 1, 3)):
        tg = torch.from_numpy(synth.make_targets(40 + i, n, bl))          # CPU labels are accepted as well
        loss = st.train_without_unlabeled_da_graphed(imgs, tg, uw, 4 + i) if da else st.train_without_unlabeled_graphed(imgs, tg, 4 + i)
        assert torch.isfinite(loss).all()
    assert st.burn_in_captures == 2 and st._burn_graph["cap"] == 2 * cap and st.ema.updates == 6


def test_hand_over_to_semi_supervised_step():
    from efficientteacher_b200.ema import CosineEMA
    img, bl, bu = 256, 2, 2
    st = _step(img, bl + bu, burn=2)
    with torch.no_grad():
        for mm in (st.model, st.ema.ema):
            for h in mm.head.m:
                h.bias.view(3, -1)[:, 4] += 6.5
                h.bias.view(3, -1)[:, 5:] += 5.0
    tg = synth.make_targets(7, 8 * bl, bl)
    imgs = torch.from_numpy(synth.make_images(3, bl, img, tg)).to(DEV)          # uint8, as the loaders deliver
    uw = torch.from_numpy(synth.make_images(4, bu, img)).to(DEV)
    us = uw.flip(3).contiguous()
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    tgd = torch.from_numpy(tg).to(DEV)
    st.begin_epoch(0)
    st.train_without_unlabeled(imgs, tgd, 0)
    st.begin_epoch(1)
    st.train_without_unlabeled_graphed(imgs, tgd, 1)
    assert st.in_burn_in and st.semi_ema is None and st.ema.updates == 2
    with pytest.raises(RuntimeError, match="burn-in"):
        st.train_instance(imgs, tgd, us, uw, None, Ms, 2)
    with pytest.raises(RuntimeError, match="burn-in"):
        st.train_instance_graphed(imgs, tgd, us, uw, None, Ms, 2)
    student = {k: v.clone() for k, v in st.model.state_dict().items()}
    st.begin_epoch(2)
    assert not st.in_burn_in and st._burn_graph is None
    assert isinstance(st.semi_ema, CosineEMA) and st.semi_ema.total_epoch == 300 - 2
    for k, v in st.ema.ema.state_dict().items():
        assert torch.equal(st.semi_ema.ema.state_dict()[k], v), k
    for k, v in st.model.state_dict().items():
        assert torch.equal(student[k], v), k                   # the student is not reset to the EMA
    assert st.ema.updates == 2
    with pytest.raises(RuntimeError):
        st.train_without_unlabeled_graphed(imgs, tgd, 2)
    loss = st.train_instance_graphed(imgs, tgd, us, uw, None, Ms, 2)
    assert torch.isfinite(loss).all() and st.ema.updates == 3
    sema = st.semi_ema.ema.state_dict()
    assert any(not torch.equal(sema[k], v) for k, v in st.ema.ema.state_dict().items() if v.dtype.is_floating_point)
