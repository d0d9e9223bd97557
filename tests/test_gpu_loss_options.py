"""GPU (H100): the loss options of the fused loss kernels -- BCE positive weights, focal loss and autobalance -- through
the native ComputeLoss / ComputeStudentMatchLoss against the live reference's values and gradients
(tests/golden/loss_opts_*.npz), the device-resident autobalance state (its trajectory, and a backward that uses the
balance from before the update), the single-target switches, and captured steps against eager ones with the options on."""
import numpy as np
import pytest
import torch

import synth
from loss_opts_cases import LOSS_CASES, check_grads, inputs, opts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOSS_RTOL = 1e-4


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)


def _cfg(o):
    from tiny_cfg import ssod_cfg
    cfg = ssod_cfg(o["nc"])
    cfg.single_cls = o["nc"] == 1
    cfg.Loss.fl_gamma, cfg.Loss.cls_pw, cfg.Loss.obj_pw = o["fl_gamma"], o["cls_pw"], o["obj_pw"]
    cfg.Loss.label_smoothing, cfg.Loss.autobalance = o["label_smoothing"], o["autobalance"]
    cfg.SSOD.ignore_obj, cfg.SSOD.pseudo_label_with_bbox, cfg.SSOD.pseudo_label_with_cls = o["ignore_obj"], o["with_bbox"], o["with_cls"]
    return cfg


def _crit(o, cfg=None):
    from efficientteacher_b200.loss import ComputeLoss
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import HeadOnlyModel
    cls = ComputeStudentMatchLoss if o["ssod"] else ComputeLoss
    return cls(HeadOnlyModel(o["nc"]).to(DEV), cfg or _cfg(o))


def _call(crit, o, k):
    logits, tg = inputs(o["nc"], o["ssod"], k)
    p = [torch.from_numpy(x).to(DEV).requires_grad_(True) for x in logits]
    loss, items = crit(p, torch.from_numpy(tg).to(DEV))
    keys = ("ss_box", "ss_obj", "ss_cls") if o["ssod"] else ("box", "obj", "cls")
    got = np.array([float(items[x]) for x in keys] + [float(loss.detach())], np.float32)
    return p, loss, got


@pytest.mark.parametrize("name", LOSS_CASES)
def test_loss_options_vs_reference(golden, name):
    """values and gradients of every case against the reference; autobalance: 6 calls, the balance after each"""
    g = golden("loss_opts_" + name)
    o = opts(g)
    crit = _crit(o)
    for k in range(o["ncalls"]):
        p, loss, got = _call(crit, o, k)
        np.testing.assert_allclose(got, g[f"c{k}_items"], rtol=LOSS_RTOL, atol=1e-8)
        loss.backward()
        check_grads(g, f"c{k}_", [pi.grad.cpu().numpy() for pi in p], LOSS_RTOL)
        if o["autobalance"] and not o["ssod"]:
            np.testing.assert_allclose(crit.balance, g[f"c{k}_balance"], rtol=1e-6)


def _close(a, b, what):
    """equal up to the fp32 atomic summation order of the loss kernels (a balance off by one update is ~1e-4 away)"""
    np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=1e-6, atol=1e-10, err_msg=what)


def test_autobalance_backward_uses_the_balance_before_the_update(golden):
    """Each autobalance call equals a fixed-balance call at the balance the state held before it, values and gradients,
    although the state has moved on by the time the backward runs"""
    o = opts(golden("loss_opts_autobal"))
    auto = _crit(o)
    fixed = _crit(dict(o, autobalance=False))
    for k in range(3):
        before = auto.balance
        assert auto.balance_state.dtype == torch.float64 and auto.balance_state.is_cuda
        fixed.balance = before
        pa, la, ga = _call(auto, o, k)
        pf, lf, gf = _call(fixed, o, k)
        assert auto.balance != before
        la.backward()
        lf.backward()
        _close(ga, gf, f"call {k} values")
        for a, b in zip(pa, pf):
            _close(a.grad.cpu().numpy(), b.grad.cpu().numpy(), f"call {k} gradients")
    ptr = auto.balance_state.data_ptr()
    auto.balance = [4.0, 1.0, 0.4]                              # the setter uploads in place
    assert auto.balance_state.data_ptr() == ptr and auto.balance == [4.0, 1.0, 0.4]


def test_autobalance_call_captures_and_advances_on_replay(golden):
    """the balance update lives in the captured loss call (capturing it also shows no host read): each replay advances
    it as an eager call does"""
    o = opts(golden("loss_opts_autobal"))
    eager, graphed = _crit(o), _crit(o)
    logits, tg = inputs(o["nc"], False, 0)
    p = [torch.from_numpy(x).to(DEV) for x in logits]
    t = torch.from_numpy(tg).to(DEV)
    nt = torch.full((1,), t.shape[0], dtype=torch.int32, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graphed(p, t, nt)                                        # warm-up (lazily built assigner state)
    torch.cuda.current_stream().wait_stream(side)
    graphed.balance = [4.0, 1.0, 0.4]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, _ = graphed(p, t, nt)
    assert graphed.balance == [4.0, 1.0, 0.4]                  # capturing runs nothing
    for k in range(3):
        g.replay()
        ref, _ = eager(p, t, nt)
        _close(out.cpu().numpy(), ref.cpu().numpy(), f"replay {k}")
        np.testing.assert_allclose(graphed.balance, eager.balance, rtol=1e-9, err_msg=f"replay {k}")
        assert graphed.balance != [4.0, 1.0, 0.4]


def test_single_targets_assign_bit_identical_to_default(golden):
    """Loss.single_targets=True and SSOD.uncertain_aug=False assign exactly as the defaults (and as the reference)"""
    from efficientteacher_b200.assigner import YOLOAnchorAssigner
    g = golden("loss_opts_single_targets")
    n, B = int(g["n"]), int(g["B"])
    t = synth.make_targets(int(g["seed"]), n, B)
    sc = np.random.RandomState(int(g["score_seed"])).uniform(0.1, 1, (n, 1)).astype(np.float32)
    p = [torch.empty(B, 3, ny, nx, 85, device=DEV) for ny, nx in synth.level_shapes()]
    t7 = np.concatenate([t, sc], 1)
    bufs = {}
    for st in (False, True):
        a = YOLOAnchorAssigner(3, 3, torch.from_numpy(synth.ANCHORS_GRID), 4.0, torch.tensor([8., 16., 32.]), single_targets=st)
        bt, uc = a.assign(p, torch.from_numpy(t).to(DEV)), a.assign(p, torch.from_numpy(t7).to(DEV), with_pseudo_score=True)
        bufs[st] = [(o.cnt, o.idx, o.tbox, o.anch, o.tcls, o.tscore) for o in (bt, uc)]
        res = a(p, torch.from_numpy(t).to(DEV)), a(p, torch.from_numpy(t7).to(DEV), with_pseudo_score=True)
        for l in range(3):
            for pref, r, owner in (("bt", res[0], "sup"), ("uc", res[1], "ssod")):
                assert np.array_equal(torch.stack(r[2][l], 1).cpu().numpy(), g[f"{owner}_{pref}_idx{l}"]), (st, pref, l)
            assert np.array_equal(res[0][1][l].cpu().numpy(), g[f"sup_bt_tbox{l}"])
            assert np.array_equal(res[1][4][l].cpu().numpy(), g[f"ssod_uc_tscore{l}"])
    for s0, s1 in zip(bufs[False], bufs[True]):
        cnt = s0[0][:3].cpu().tolist()
        assert torch.equal(s0[0], s1[0])
        for l, n_l in enumerate(cnt):
            for x, y in zip(s0[1:], s1[1:]):
                assert torch.equal(x[l, :n_l], y[l, :n_l]), l
    # the losses built on them equal the defaults'  (up to the fp32 atomic summation order)
    from tiny_cfg import ssod_cfg
    for ssod in (False, True):
        o = dict(nc=80, ssod=ssod)
        outs = []
        for flag in (False, True):
            cfg = ssod_cfg()
            cfg.Loss.single_targets = flag and not ssod
            cfg.SSOD.uncertain_aug = not (flag and ssod)
            crit = _crit(o, cfg)
            assert crit.assigner.single_targets == flag
            p, loss, got = _call(crit, o, 0)
            loss.backward()
            outs.append((got, [pi.grad for pi in p]))
        _close(outs[0][0], outs[1][0], "values")
        for a, b in zip(outs[0][1], outs[1][1]):
            _close(a.cpu().numpy(), b.cpu().numpy(), "gradients")


# ------------------------------------------------------------------------------------------------ captured steps
def _images(seed, n, img):
    return torch.from_numpy(np.random.RandomState(seed).rand(n, 3, img, img).astype(np.float32)).to(DEV)


def _flat(tensors):
    return torch.cat([t.detach().flatten().float() for t in tensors])


def _make(kind, img, bl, bu):
    """fl_gamma=1.5, obj_pw=1.3, autobalance on; AdamW for the supervised step.  No warm-up, nominal batch 32: the
    optimizer steps every 2nd iteration from ni = 0."""
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    torch.manual_seed(0)
    cfg = yolov5_sup_cfg('l_shallow', batch_size=bl, img_size=img) if kind == "sup" else \
        yolov5_ssod_cfg('l_shallow', batch_size=bl + bu, img_size=img)
    cfg.hyp.warmup_epochs = 0
    cfg.Loss.fl_gamma, cfg.Loss.obj_pw, cfg.Loss.autobalance = 1.5, 1.3, True
    if kind == "sup":
        cfg.adam = True
        return SupTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    cfg.hyp.burn_epochs = 0
    st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
    with torch.no_grad():
        for mm in (st.model, st.ema.ema, st.semi_ema.ema):
            for h in mm.head.m:
                h.bias.view(3, -1)[:, 4] += 6.5
                h.bias.view(3, -1)[:, 5:] += 5.0
    return st


def _within_spread(out, what, floor):
    """graph vs eager no further apart than 3x two eager runs of the same seed (fp32-atomic summation order)"""
    a, b, c = out["eager"][what], out["graph"][what], out["eager2"][what]
    n = a.norm().clamp_min(1e-30)
    rel, rel_eager = ((a - b).norm() / n).item(), ((a - c).norm() / n).item()
    assert rel <= 3.0 * rel_eager + floor, (what, rel, rel_eager)


@pytest.mark.parametrize("kind", ["sup", "ssod"])
def test_captured_step_with_loss_options_matches_eager(kind):
    """(eager, eager, graph) x 4 steps.  After each step the balance of the graphed run equals the eager run's: bit for bit
    when the two eager runs agree bit for bit, else within their spread.  The first graphed call captures (two warm-up
    steps, then the restore) and replays once, so equality after it shows the warm-up left the balance untouched."""
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    us = uw.flip(3).contiguous()
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    tgs = [torch.from_numpy(synth.make_targets(30 + i, n, bl)).to(DEV) for i, n in enumerate((16, 5, 9, 12))]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        st = _make(kind, img, bl, bu)
        assert st.compute_loss.autobalance and st.compute_loss.balance == [4.0, 1.0, 0.4]
        g = mode == "graph"
        if kind == "ssod":
            f = lambda tg, ni: (st.train_instance_graphed if g else st.train_instance)(imgs, tg, us, uw, None, Ms, ni)  # noqa: E731
        else:
            f = lambda tg, ni: (st.train_step_graphed if g else st.train_step)(imgs, tg, ni)  # noqa: E731
        losses, bals = [], []
        for ni, tg in enumerate(tgs):
            losses.append(float(f(tg, ni).item()))
            bals.append(st.compute_loss.balance_state.clone())
        if g:
            assert st.captures == 1
        emas = [e for e in (st.ema, st.semi_ema) if e is not None]
        out[mode] = dict(losses=losses, bals=bals, weights=_flat(st.model.state_dict().values()),
                         ema=_flat(t for e in emas for t in e.ema.state_dict().values()))
    for i, (a, b, c) in enumerate(zip(out["eager"]["losses"], out["graph"]["losses"], out["eager2"]["losses"])):
        assert abs(a - b) <= 3.0 * abs(a - c) + (0.01 + 0.02 * i) * abs(a), out
    _within_spread(out, "weights", 2e-3)
    _within_spread(out, "ema", 2e-3)
    for k, (a, b, c) in enumerate(zip(out["eager"]["bals"], out["graph"]["bals"], out["eager2"]["bals"])):
        assert not torch.equal(a, torch.tensor([4.0, 1.0, 0.4], dtype=torch.float64, device=DEV))
        if torch.equal(a, c):
            assert torch.equal(a, b), (k, a.tolist(), b.tolist())
        else:
            spread = (a - c).abs().max().item()
            assert (a - b).abs().max().item() <= 3.0 * spread + 1e-12, (k, a.tolist(), b.tolist(), c.tolist())
