"""GPU (H100): the capture-and-replay path the SSOD, burn-in and supervised steps share -- the supervised step's graph B
(SGD + ModelEMA replayed on the iterations the cadence steps), a capture that leaves no trace of its warm-up steps, and
the device-memory EMA decay that graph B reads."""
import numpy as np
import pytest
import torch

import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _images(seed, n, img):
    return torch.from_numpy(np.random.RandomState(seed).rand(n, 3, img, img).astype(np.float32)).to(DEV)


def _flat(tensors):
    return torch.cat([t.detach().flatten().float() for t in tensors])


def _within_spread(out, what, floor=2e-3):
    """graph vs eager no further apart than 3x two eager runs of the same seed (fp32-atomic summation order)"""
    a, b, c = out["eager"][what], out["graph"][what], out["eager2"][what]
    n = a.norm().clamp_min(1e-30)
    rel, rel_eager = ((a - b).norm() / n).item(), ((a - c).norm() / n).item()
    assert rel <= 3.0 * rel_eager + floor, (what, rel, rel_eager)


def _float_state(module):
    return [v for k, v in module.state_dict().items() if v.dtype.is_floating_point and "running" not in k]


def test_supervised_graphed_step_matches_eager():
    """(eager, eager, graph) x 5 supervised steps with 16 / 0 / 9 / 24 / 9 labels.  Nominal batch 32: accumulate is 1 in the
    warm-up (ni = 0, 1: the optimizer steps every iteration) and 2 after it (ni = 1500, 1502 step, 1501 does not)."""
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.trainer import SupTrainerStep
    img, B = 256, 2
    imgs = _images(3, B, img)
    nis = (0, 1, 1500, 1501, 1502)
    tgs = [torch.from_numpy(synth.make_targets(30 + i, n, B)).to(DEV) for i, n in enumerate((16, 0, 9, 24, 9))]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        torch.manual_seed(0)
        st = SupTrainerStep(yolov5_sup_cfg('l_shallow', batch_size=B, img_size=img), torch.device(DEV), batch_size=32)
        f = st.train_step_graphed if mode == "graph" else st.train_step
        losses = [float(f(imgs, tg, ni).item()) for ni, tg in zip(nis, tgs)]
        assert st.ema.updates == 4 and st.last_opt_step == 1502 and st.accumulate == 2, mode
        out[mode] = dict(losses=losses, ema=_flat(_float_state(st.ema.ema)),
                         running_var=_flat(v for k, v in st.ema.ema.state_dict().items() if "running_var" in k))
    for i, (a, b, c) in enumerate(zip(out["eager"]["losses"], out["graph"]["losses"], out["eager2"]["losses"])):
        assert abs(a - b) <= 3.0 * abs(a - c) + (0.01 + 0.02 * i) * abs(a), out
    _within_spread(out, "ema")
    _within_spread(out, "running_var", 5e-3)


def _make(kind, img, bl, bu):
    """A step whose optimizer steps every 2nd iteration from ni = 0 (no warm-up, nominal batch 32: accumulate = 2)"""
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    torch.manual_seed(0)
    if kind == "sup":
        cfg = yolov5_sup_cfg('l_shallow', batch_size=bl, img_size=img)
        cfg.hyp.warmup_epochs = 0
        return SupTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    cfg = yolov5_ssod_cfg('l_shallow', batch_size=bl + bu, img_size=img)
    cfg.hyp.warmup_epochs = 0
    cfg.hyp.burn_epochs = 2 if kind == "burn_in" else 0
    st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    if kind == "ssod":
        with torch.no_grad():
            for mm in (st.model, st.ema.ema, st.semi_ema.ema):
                for h in mm.head.m:
                    h.bias.view(3, -1)[:, 4] += 6.5
                    h.bias.view(3, -1)[:, 5:] += 5.0
    return st


@pytest.mark.parametrize("kind", ["ssod", "burn_in", "sup"])
def test_capture_leaves_no_trace(kind):
    """The first graphed call (which captures: two warm-up steps that really train, then the restore) leaves the state an
    eager call leaves: at ni = 0 the optimizer is not due, at ni = 1 it is."""
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    us = uw.flip(3).contiguous()
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    out = [{}, {}]
    for mode in ("eager", "eager2", "graph"):
        st = _make(kind, img, bl, bu)
        g = mode == "graph"
        if kind == "ssod":
            f = lambda ni: (st.train_instance_graphed if g else st.train_instance)(imgs, tg, us, uw, None, Ms, ni)  # noqa: E731
        elif kind == "burn_in":
            f = lambda ni: (st.train_without_unlabeled_graphed if g else st.train_without_unlabeled)(imgs, tg, ni)  # noqa: E731
        else:
            f = lambda ni: (st.train_step_graphed if g else st.train_step)(imgs, tg, ni)  # noqa: E731
        emas = [e for e in (st.ema, st.semi_ema) if e is not None]
        for ni in (0, 1):
            f(ni)
            bufs = [st.optimizer.state[p].get("momentum_buffer") for grp in st.optimizer.param_groups for p in grp["params"]]
            if ni == 0:          # not due: the eager step has no momentum yet, the warm-up's buffers are zero again
                if g:
                    assert all(b is not None for b in bufs) and not any(bool(b.any()) for b in bufs)
                else:
                    assert all(b is None for b in bufs)
            out[ni][mode] = dict(
                counters=(st.last_opt_step, [e.updates for e in emas], st.accumulate,
                          [(x["lr"], x["momentum"]) for x in st.optimizer.param_groups]),
                weights=_flat(st.model.state_dict().values()),
                ema=_flat(t for e in emas for t in e.ema.state_dict().values()),
                grads=st._arena.flat.clone(),
                momentum=_flat(b for b in bufs if b is not None) if ni == 1 else None)
    for ni, o in enumerate(out):
        assert o["eager"]["counters"] == o["eager2"]["counters"] == o["graph"]["counters"], (ni, o["graph"]["counters"])
        assert o["graph"]["counters"][0] == (-1 if ni == 0 else 1)
        for what in ("weights", "ema", "grads") + (("momentum",) if ni == 1 else ()):
            _within_spread(o, what)


def test_no_garbage_collection_while_capturing():
    """The cyclic garbage collector stays off while a stream captures (a collected step would destroy its CUDA graphs in
    the middle of the capture) and is on again afterwards."""
    import gc
    img, B = 128, 2
    st = _make("sup", img, B, 0)
    seen, loss = [], st._loss

    def recording_loss(*a):
        seen.append((torch.cuda.is_current_stream_capturing(), gc.isenabled()))
        return loss(*a)
    st._loss = recording_loss
    assert gc.isenabled()
    st.train_step_graphed(_images(3, B, img), torch.from_numpy(synth.make_targets(7, 8, B)).to(DEV), 0)
    assert (True, False) in seen and (True, True) not in seen, seen
    assert gc.isenabled()


@pytest.mark.parametrize("updates", [0, 41, 100000])
def test_device_decay_matches_host_decay(updates):
    """ModelEMA._update_with(..., scalars_dev=...) (graph B of the burn-in and supervised steps) is bit-equal to
    ModelEMA.update on the same tensors."""
    from efficientteacher_b200.ema import ModelEMA, ema_scalars
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Conv2d(3, 16, 3), torch.nn.BatchNorm2d(16), torch.nn.Conv2d(16, 40, 1)).to(DEV)
    host, dev = ModelEMA(model, updates=updates), ModelEMA(model, updates=updates)
    with torch.no_grad():
        for t in model.state_dict().values():
            if t.dtype.is_floating_point:
                t.add_(torch.randn_like(t))
    before = [t.clone() for t in host.ema.state_dict().values()]
    host.update(model)
    dev.updates += 1
    dev._update_with(model, 0.0, scalars_dev=torch.tensor(ema_scalars(dev.decay(dev.updates)), dtype=torch.float32, device=DEV))
    assert host.updates == dev.updates == updates + 1
    for (k, a), b in zip(host.ema.state_dict().items(), dev.ema.state_dict().values()):
        assert torch.equal(a, b), k
    assert not all(torch.equal(a, b) for a, b in zip(before, host.ema.state_dict().values()))
