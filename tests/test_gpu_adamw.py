"""GPU (H100): FusedAdamW (csrc/adamw.cu), the optimizer of `adam: True`.  The kernel is bit-equal to torch.optim.AdamW's
default CUDA implementation on the same gradients, step after step, with the learning rate changing per group; state
dicts load both ways; a captured step replayed with refresh_hyper() advances the bias corrections like eager steps; and
the SSOD, burn-in and supervised steps build it from the config and capture and replay it like FusedSGD."""
import copy

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


# three groups in the reference's order [bias, conv weight, BN weight]: numel % 4 != 0, numel > ETB_CHUNK (4096), and
# a 1x1 1024 -> 1024 conv weight; groups 0 and 2 keep AdamW's default weight decay
SHAPES = [[(4099,), (13,)], [(1024, 1024, 1, 1), (3, 4133)], [(77,), (513,)]]
WD1 = 0.0005 * 32 * 2 / 64


def _params(seed):
    g = torch.Generator().manual_seed(seed)
    return [[(torch.randn(s, generator=g) * 0.1).to(DEV).requires_grad_() for s in grp] for grp in SHAPES]


def _groups(params):
    return [{"params": params[0]}, {"params": params[1], "weight_decay": WD1}, {"params": params[2]}]


def _grads(step):
    """gradients of very different magnitudes per element, some exactly zero"""
    g = torch.Generator().manual_seed(100 + step)
    out = []
    for grp in SHAPES:
        for s in grp:
            x = torch.randn(s, generator=g) * torch.pow(10.0, torch.empty(s).uniform_(-6, 1, generator=g))
            x[torch.rand(s, generator=g) < 0.01] = 0
            out.append(x.to(DEV))
    return out


def _lrs(step):
    """warm-up like: groups 0 / 1 rise from 0, group 2 falls from warmup_bias_lr; group 1 jumps once mid-run"""
    x = step / 6.0
    return [0.01 * x, (0.01 * x) if step != 3 else 0.02, 0.1 + (0.01 - 0.1) * x]


def _flat_params(opt):
    return [p for g in opt.param_groups for p in g["params"]]


def _set_lrs(opt, lrs):
    for g, lr in zip(opt.param_groups, lrs):
        g["lr"] = lr


def _assert_equal_state(ref, fused, what):
    for i, (a, b) in enumerate(zip(_flat_params(ref), _flat_params(fused))):
        assert torch.equal(a, b), (what, "param", i, (a - b).abs().max().item())
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(ref.state[a][k], fused.state[b][k]), (what, k, i)


def _step_both(ref, fused, step):
    _set_lrs(ref, _lrs(step))
    _set_lrs(fused, _lrs(step))
    for p, q, g in zip(_flat_params(ref), _flat_params(fused), _grads(step)):
        p.grad = g.clone()
        if q.grad is None:
            q.grad = torch.zeros_like(q)
        q.grad.copy_(g)
    ref.step()
    fused.step()


def test_kernel_matches_torch_adamw_bitwise():
    from efficientteacher_b200.optim import FusedAdamW
    pr, pf = _params(0), _params(0)
    ref = torch.optim.AdamW(_groups(pr), lr=0.01, betas=(0.937, 0.999))
    fused = FusedAdamW(_groups(pf), lr=0.01, betas=(0.937, 0.999))
    assert ref.param_groups[0]["weight_decay"] == fused.param_groups[0]["weight_decay"] == 0.01
    for step in range(7):
        _step_both(ref, fused, step)
        _assert_equal_state(ref, fused, step)
        assert all(not bool(q.grad.any()) for q in _flat_params(fused)), step      # zeroed in the same pass
        assert fused.step_count == step + 1
        for p in _flat_params(ref):
            assert float(ref.state[p]["step"]) == step + 1


def test_state_dict_round_trips():
    """torch -> fused (loaded before and after the chunk table exists) and fused -> torch: after 3 steps the state moves
    over and the next step is bit-equal; the saved step values are torch's"""
    from efficientteacher_b200.optim import FusedAdamW
    mk_ref = lambda ps: torch.optim.AdamW(_groups(ps), lr=0.01, betas=(0.937, 0.999))       # noqa: E731
    mk_fused = lambda ps: FusedAdamW(_groups(ps), lr=0.01, betas=(0.937, 0.999))            # noqa: E731
    # torch -> fused
    for built_first in (False, True):
        pr = _params(1)
        ref = mk_ref(pr)
        for step in range(3):
            _set_lrs(ref, _lrs(step))
            for p, g in zip(_flat_params(ref), _grads(step)):
                p.grad = g.clone()
            ref.step()
        pf = _params(2)
        fused = mk_fused(pf)
        if built_first:             # the flat buffers exist already: the loaded moments are copied into them
            for q in _flat_params(fused):
                q.grad = torch.randn_like(q)
            fused.step()
        fused.load_state_dict(copy.deepcopy(ref.state_dict()))
        assert fused.step_count == 3
        with torch.no_grad():
            for p, q in zip(_flat_params(ref), _flat_params(fused)):
                q.copy_(p)
        _step_both(ref, fused, 3)
        _assert_equal_state(ref, fused, ("torch->fused", built_first))
        sr, sf = ref.state_dict(), fused.state_dict()
        for i in sr["state"]:
            assert float(sf["state"][i]["step"]) == float(sr["state"][i]["step"]) == 4.0
            assert sf["state"][i]["step"].dtype == sr["state"][i]["step"].dtype
    # fused -> torch
    pf = _params(3)
    fused = mk_fused(pf)
    for step in range(3):
        _set_lrs(fused, _lrs(step))
        for q, g in zip(_flat_params(fused), _grads(step)):
            if q.grad is None:
                q.grad = torch.zeros_like(q)
            q.grad.copy_(g)
        fused.step()
    sd = copy.deepcopy(fused.state_dict())
    assert all(float(s["step"]) == 3.0 for s in sd["state"].values())
    pr = [[p.detach().clone().requires_grad_() for p in grp] for grp in pf]
    ref = mk_ref(pr)
    ref.load_state_dict(sd)
    _step_both(ref, fused, 3)
    _assert_equal_state(ref, fused, "fused->torch")
    # per-parameter steps that differ cannot become one step count
    sd = copy.deepcopy(fused.state_dict())
    sd["state"][0]["step"] = torch.tensor(2.0)
    with pytest.raises(ValueError):
        mk_fused(_params(3)).load_state_dict(sd)


def test_captured_step_replays_like_eager_steps():
    """one eager step, then step() captured once and replayed 5 times with the lr changed between replays through
    refresh_hyper(): bit-equal to 6 eager steps, so the bias corrections advance; the capture itself changes nothing"""
    from efficientteacher_b200.optim import FusedAdamW
    pe, pg = _params(4), _params(4)
    eager = FusedAdamW(_groups(pe), lr=0.01, betas=(0.937, 0.999))
    graphed = FusedAdamW(_groups(pg), lr=0.01, betas=(0.937, 0.999))
    for q in _flat_params(eager) + _flat_params(graphed):
        q.grad = torch.zeros_like(q)

    def feed(opt, step):
        _set_lrs(opt, _lrs(step))
        for q, g in zip(_flat_params(opt), _grads(step)):
            q.grad.copy_(g)

    feed(eager, 0)
    eager.step()
    feed(graphed, 0)
    graphed.step()
    torch.cuda.synchronize()
    before = [q.clone() for q in _flat_params(graphed)]
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph):
            graphed.step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert graphed.step_count == 1
    assert all(torch.equal(a, b) for a, b in zip(before, _flat_params(graphed)))
    for step in range(1, 6):
        feed(eager, step)
        eager.step()
        feed(graphed, step)
        graphed.refresh_hyper()
        graph.replay()
        torch.cuda.synchronize()
        assert graphed.step_count == eager.step_count == step + 1
        for a, b in zip(_flat_params(eager), _flat_params(graphed)):
            assert torch.equal(a, b), step
            for k in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(eager.state[a][k], graphed.state[b][k]), (step, k)
            assert not bool(b.grad.any())


# ---- the trainer steps ------------------------------------------------------------------------------------------------
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


def _make(kind, img, bl, bu, adam=True, warmup=False):
    """nominal batch 32: accumulate = 2 after the warm-up (warmup=False: no warm-up, the optimizer steps every 2nd ni)"""
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    torch.manual_seed(0)
    if kind == "sup":
        cfg = yolov5_sup_cfg('l_shallow', batch_size=bl, img_size=img)
    else:
        cfg = yolov5_ssod_cfg('l_shallow', batch_size=bl + bu, img_size=img)
        cfg.hyp.burn_epochs = 2 if kind == "burn_in" else 0
    cfg.adam = adam
    if not warmup:
        cfg.hyp.warmup_epochs = 0
    if kind == "sup":
        return SupTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    if kind == "ssod":
        with torch.no_grad():
            for mm in (st.model, st.ema.ema, st.semi_ema.ema):
                for h in mm.head.m:
                    h.bias.view(3, -1)[:, 4] += 6.5
                    h.bias.view(3, -1)[:, 5:] += 5.0
    return st


def _caller(st, kind, graphed, imgs, uw, tg, Ms):
    us = uw.flip(3).contiguous()
    if kind == "ssod":
        return lambda ni, t=tg: (st.train_instance_graphed if graphed else st.train_instance)(imgs, t, us, uw, None, Ms, ni)
    if kind == "burn_in":
        return lambda ni, t=tg: (st.train_without_unlabeled_graphed if graphed else st.train_without_unlabeled)(imgs, t, ni)
    return lambda ni, t=tg: (st.train_step_graphed if graphed else st.train_step)(imgs, t, ni)


def _moments(st, k):
    return [st.optimizer.state[p].get(k) for grp in st.optimizer.param_groups for p in grp["params"]]


@pytest.mark.parametrize("kind", ["ssod", "burn_in", "sup"])
def test_trainer_builds_fused_adamw(kind):
    from efficientteacher_b200.optim import FusedAdamW, FusedSGD
    st = _make(kind, 128, 2, 2, adam=True)
    opt = st.optimizer
    assert type(opt) is FusedAdamW
    wd1 = st.cfg.hyp.weight_decay * st.batch_size * st.accumulate / 64
    for gi, grp in enumerate(opt.param_groups):
        assert grp["lr"] == grp["initial_lr"] == st.cfg.hyp.lr0
        assert grp["betas"] == (st.cfg.hyp.momentum, 0.999) and grp["eps"] == 1e-8 and "momentum" not in grp
        assert grp["weight_decay"] == (wd1 if gi == 1 else 0.01), gi
    assert type(_make(kind, 128, 2, 2, adam=False).optimizer) is FusedSGD


@pytest.mark.parametrize("kind", ["ssod", "burn_in", "sup"])
def test_adamw_capture_leaves_no_trace(kind):
    """The first graphed call (which captures: two warm-up steps that really train, then the restore) leaves the state an
    eager call leaves, AdamW's moments and step count included: at ni = 0 the optimizer is not due, at ni = 1 it is."""
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    out = [{}, {}]
    for mode in ("eager", "eager2", "graph"):
        st = _make(kind, img, bl, bu)
        g = mode == "graph"
        f = _caller(st, kind, g, imgs, uw, tg, Ms)
        emas = [e for e in (st.ema, st.semi_ema) if e is not None]
        for ni in (0, 1):
            f(ni)
            ms, vs = _moments(st, "exp_avg"), _moments(st, "exp_avg_sq")
            if ni == 0:          # not due: the eager step has no moments yet, the warm-up's moments are zero again
                if g:
                    assert all(b is not None and not bool(b.any()) for b in ms + vs)
                else:
                    assert all(b is None for b in ms + vs)
            out[ni][mode] = dict(
                counters=(st.last_opt_step, [e.updates for e in emas], st.accumulate, st.optimizer.step_count,
                          [x["lr"] for x in st.optimizer.param_groups]),
                weights=_flat(st.model.state_dict().values()),
                ema=_flat(t for e in emas for t in e.ema.state_dict().values()),
                grads=st._arena.flat.clone(),
                exp_avg=_flat(ms) if ni == 1 else None,
                exp_avg_sq=_flat(vs) if ni == 1 else None)
    for ni, o in enumerate(out):
        assert o["eager"]["counters"] == o["eager2"]["counters"] == o["graph"]["counters"], (ni, o["graph"]["counters"])
        assert o["graph"]["counters"][0] == (-1 if ni == 0 else 1) and o["graph"]["counters"][3] == ni
        for what in ("weights", "ema", "grads") + (("exp_avg", "exp_avg_sq") if ni == 1 else ()):
            _within_spread(o, what)


@pytest.mark.parametrize("kind", ["ssod", "burn_in", "sup"])
def test_adamw_graphed_steps_match_eager(kind):
    """(eager, eager2, graph) x 5 steps with 16 / 0 / 9 / 24 / 9 labels.  Nominal batch 32: accumulate is 1 in the
    warm-up (ni = 0, 1: the optimizer steps every iteration) and 2 after it (ni = 1500, 1502 step, 1501 does not), so
    the step count ends at 4."""
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    nis = (0, 1, 1500, 1501, 1502)
    tgs = [torch.from_numpy(synth.make_targets(30 + i, n, bl)).to(DEV) for i, n in enumerate((16, 0, 9, 24, 9))]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        st = _make(kind, img, bl, bu, warmup=True)
        f = _caller(st, kind, mode == "graph", imgs, uw, tgs[0], Ms)
        losses = [float(f(ni, tg).item()) for ni, tg in zip(nis, tgs)]
        emas = [e for e in (st.ema, st.semi_ema) if e is not None]
        assert st.optimizer.step_count == 4 and st.ema.updates == 4, mode
        assert st.last_opt_step == 1502 and st.accumulate == 2, mode
        out[mode] = dict(losses=losses, weights=_flat(p for p in st.model.parameters()),
                         ema=_flat(v for e in emas for k, v in e.ema.state_dict().items()
                                   if v.dtype.is_floating_point and "running" not in k),
                         exp_avg=_flat(_moments(st, "exp_avg")), exp_avg_sq=_flat(_moments(st, "exp_avg_sq")))
    for i, (a, b, c) in enumerate(zip(out["eager"]["losses"], out["graph"]["losses"], out["eager2"]["losses"])):
        assert abs(a - b) <= 3.0 * abs(a - c) + (0.01 + 0.02 * i) * abs(a), out
    for what in ("weights", "ema", "exp_avg", "exp_avg_sq"):
        _within_spread(out, what)
