"""GPU (H100): SyncBatchNorm (`sync_bn`) on the fused training BatchNorm.

a. Kernels in one process: a batch's rows split into unequal chunks (empty ones included) stand for the ranks.  Per
   chunk etb_bn_stats_sums, the [2C+1] fp64 vectors added on the host, etb_bn_finalize_global; per chunk the backward
   reduce / finalize, the [2C] sums added, etb_bn_act_bwd_apply_global over the chunk's rows with the global count.
   Against float64 torch over the whole batch and against etb_bn_finalize on it, at C = 64, 96, 160, 256, 1280, each
   activation, on a channel slice with a shortcut.
b. The synced path at world 1 through the loopback reducer against the per-rank path; sync_bn at world 1 changes nothing.
c. World 2 on one GPU: two processes (torch.multiprocessing, gloo, both on cuda:0) run
   (1) one Conv layer with unequal batches against torch's SyncBatchNorm and float64 BN on the concatenated batch,
   (2) a YOLOv5n at 128, fused synced path against torch's SyncBatchNorm between the same native convs
       (Conv.FUSED_BN = False), with the fused path on per-rank statistics as the yardstick of what a miss looks like,
   (3) the eager SSOD and supervised steps with sync_bn: statistics of the global batch, replicas bit-identical,
   (4) the reference's order Model(cfg) -> convert_sync_batchnorm -> step,
   (5) a captured step with sync_bn at world 2, which must raise.
   Both processes are joined with a timeout and killed if they outlive it."""
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_gpu_geometry import NAN, _bf, _check_bf16, _nchw64, _nhwc, _untouched

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F64 = {"relu": F.relu, "hard_swish": F.hardswish, "silu": F.silu}
ACT = {"silu": 1, "relu": 2, "hard_swish": 4}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------------ a. the kernels
@pytest.mark.parametrize("C_", [64, 96, 160, 256, 1280])
@pytest.mark.parametrize("act", ["silu", "relu", "hard_swish"])
def test_stats_sums_and_global_finalize_over_chunks(C_, act):
    from efficientteacher_b200 import _lib
    from efficientteacher_b200 import convops as co
    lib, sp = _lib.lib(), _lib.stream_ptr()
    P = _lib.ptr
    eps, mom = 1e-3, 0.03
    N, H, W = 3, 23, 17
    M = N * H * W
    chunks = [0, 400, 0, 77, M - 477]                      # unequal row counts, empty ones included
    assert M - 477 > 400
    y = (_bf((N, C_, H, W), 11, 2.0) + 0.5).to(torch.bfloat16).float()
    r, da = _bf((N, C_, H, W), 12), _bf((N, C_, H, W), 13)
    gamma = (torch.rand(C_, generator=torch.Generator().manual_seed(14)) * 2 + 0.5).to(DEV)
    beta = (torch.randn(C_, generator=torch.Generator().manual_seed(15)) * 0.5).to(DEV)
    rm0 = torch.randn(C_, generator=torch.Generator().manual_seed(16)) * 0.1
    rv0 = torch.rand(C_, generator=torch.Generator().manual_seed(17)) + 0.5
    yo, ro, dao = 8, 16, 24                                # channel slices of wider NaN-filled buffers
    ybuf, rbuf, dabuf = _nhwc(y, yo + C_ + 8, yo), _nhwc(r, ro + C_ + 16, ro), _nhwc(da, dao + C_ + 8, dao)
    yw, rw, daw = ybuf.shape[3], rbuf.shape[3], dabuf.shape[3]
    yrows, rrows, darows = ybuf.view(M, yw), rbuf.view(M, rw), dabuf.view(M, daw)

    # forward: per-chunk fp64 sums, added on the host, one global finalize
    total = torch.zeros(2 * C_ + 1, dtype=torch.float64, device=DEV)
    a0 = 0
    for n in chunks:
        rows = int(lib.etb_bn_partial_rows(n, C_, 0))
        part = torch.empty((rows, 2, C_), dtype=torch.float32, device=DEV)
        s = torch.full((2 * C_ + 1,), NAN, dtype=torch.float64, device=DEV)
        _lib.check(lib.etb_bn_stats_sums(P(yrows[a0:a0 + n, yo:]), n, C_, yw, P(part), rows, P(s), sp), "etb_bn_stats_sums")
        s2 = torch.full_like(s, NAN)
        _lib.check(lib.etb_bn_stats_sums(P(yrows[a0:a0 + n, yo:]), n, C_, yw, P(part), rows, P(s2), sp), "etb_bn_stats_sums")
        assert torch.equal(s.view(torch.int64), s2.view(torch.int64)), "run to run"
        assert s[2 * C_].item() == n and (n > 0 or not s[:2 * C_].any())
        total += s
        a0 += n
    stats = torch.full((4, C_), NAN, dtype=torch.float32, device=DEV)
    rm, rv = rm0.to(DEV), rv0.to(DEV)
    _lib.check(lib.etb_bn_finalize_global(P(total), C_, P(gamma), P(beta), eps, mom, P(rm), P(rv), P(stats[0]), P(stats[1]),
                                          P(stats[2]), P(stats[3]), sp), "etb_bn_finalize_global")
    # the whole batch through etb_bn_finalize
    rm_w, rv_w = rm0.to(DEV), rv0.to(DEV)
    _, stats_w = co.bn_forward(ybuf[..., yo:yo + C_], C_, gamma, beta, rm_w, rv_w, eps, mom, act, y_cstride=yw)
    torch.testing.assert_close(stats, stats_w, rtol=2e-5, atol=2e-6)
    torch.testing.assert_close(rm, rm_w, rtol=2e-5, atol=1e-6)
    torch.testing.assert_close(rv, rv_w, rtol=2e-5, atol=1e-6)
    # float64 torch over the whole batch
    y64 = y.double().requires_grad_(True)
    g64, b64 = gamma.double().cpu().requires_grad_(True), beta.double().cpu().requires_grad_(True)
    rm64, rv64 = rm0.double(), rv0.double()
    z = F64[act](F.batch_norm(y64, rm64, rv64, g64, b64, True, mom, eps))
    z.backward(da.double())
    mean64 = y.double().mean((0, 2, 3))
    invstd64 = (y.double().var((0, 2, 3), unbiased=False) + eps).rsqrt()
    torch.testing.assert_close(stats[2].double().cpu(), mean64, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(stats[3].double().cpu(), invstd64, rtol=1e-5, atol=0)
    torch.testing.assert_close(rm.double().cpu(), rm64, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(rv.double().cpu(), rv64, rtol=1e-5, atol=1e-7)

    # apply per chunk (shortcut added), then the backward: local reduce / finalize, sums added, apply over the chunk's rows
    # dividing by the global count (total[2C])
    obuf = torch.full((N, H, W, C_ + 16), NAN, dtype=torch.bfloat16, device=DEV)
    orows = obuf.view(M, C_ + 16)
    dybuf = torch.full((N, H, W, C_ + 8), NAN, dtype=torch.bfloat16, device=DEV)
    dyrows = dybuf.view(M, C_ + 8)
    sums = torch.zeros(2 * C_, dtype=torch.float32, device=DEV)
    dgb = torch.zeros((2, C_), dtype=torch.float32, device=DEV)
    a0 = 0
    for n in chunks:
        if n:
            _lib.check(lib.etb_bn_act_apply_res(P(yrows[a0:, yo:]), P(stats[0]), P(stats[1]), P(rrows[a0:, ro:]), P(orows[a0:, 8:]), n,
                                                C_, yw, rw, C_ + 16, ACT[act], sp), "etb_bn_act_apply_res")
            rows = int(lib.etb_bn_partial_rows(n, C_, 1))
            part = torch.empty((rows, 2, C_), dtype=torch.float32, device=DEV)
            s = torch.empty(2 * C_, dtype=torch.float32, device=DEV)
            _lib.check(lib.etb_bn_act_bwd_reduce(P(darows[a0:, dao:]), P(yrows[a0:, yo:]), P(stats[0]), P(stats[1]), P(stats[2]),
                                                 P(stats[3]), n, C_, daw, yw, ACT[act], P(part), rows, sp), "etb_bn_act_bwd_reduce")
            _lib.check(lib.etb_bn_act_bwd_finalize(P(part), rows, C_, P(s), P(dgb[0]), P(dgb[1]), 1, sp), "etb_bn_act_bwd_finalize")
            sums += s
        a0 += n
    a0 = 0
    for n in chunks:
        if n:
            _lib.check(lib.etb_bn_act_bwd_apply_global(P(darows[a0:, dao:]), P(yrows[a0:, yo:]), P(stats[0]), P(stats[1]),
                                                       P(stats[2]), P(stats[3]), P(sums), P(total), n, C_, daw, yw, C_ + 8, ACT[act],
                                                       P(dyrows[a0:]), sp), "etb_bn_act_bwd_apply_global")
        a0 += n
    _check_bf16(_nchw64(obuf, 8, C_), z.detach() + r.double(), "synced forward")
    _untouched(obuf, 8, C_, "synced forward")
    _check_bf16(_nchw64(dybuf, 0, C_), y64.grad, "synced backward")
    _untouched(dybuf, 0, C_, "synced backward")
    for got, want, what in ((dgb[0], g64.grad, "dgamma"), (dgb[1], b64.grad, "dbeta")):
        d = got.double().cpu()
        assert ((d - want).abs() <= 1e-3 * want.abs().max() + 1e-3 * want.abs()).all(), (what, (d - want).abs().max().item())


@pytest.mark.parametrize("C_", [96, 256])
def test_finalize_global_without_running_stats_and_empty_batch(C_):
    """running_mean / running_var may be NULL (the statistics only); a global count of 0 leaves them untouched"""
    from efficientteacher_b200 import _lib
    lib, P, sp = _lib.lib(), _lib.ptr, _lib.stream_ptr()
    gamma, beta = torch.ones(C_, device=DEV), torch.zeros(C_, device=DEV)
    stats = torch.empty((4, C_), device=DEV)
    total = torch.zeros(2 * C_ + 1, dtype=torch.float64, device=DEV)
    _lib.check(lib.etb_bn_stats_sums(None, 0, C_, C_, None, 0, P(total), sp), "etb_bn_stats_sums")
    rm, rv = torch.full((C_,), 0.5, device=DEV), torch.full((C_,), 2.0, device=DEV)
    _lib.check(lib.etb_bn_finalize_global(P(total), C_, P(gamma), P(beta), 1e-3, 0.03, P(rm), P(rv), P(stats[0]), P(stats[1]),
                                          P(stats[2]), P(stats[3]), sp), "etb_bn_finalize_global")
    assert (rm == 0.5).all() and (rv == 2.0).all() and (stats[2] == 0).all()
    total[:C_], total[C_:2 * C_], total[2 * C_] = 10.0, 30.0, 5.0       # mean 2, var 6 - 4 = 2
    _lib.check(lib.etb_bn_finalize_global(P(total), C_, P(gamma), P(beta), 1e-3, 0.03, None, None, P(stats[0]), P(stats[1]),
                                          P(stats[2]), P(stats[3]), sp), "etb_bn_finalize_global")
    torch.testing.assert_close(stats[2], torch.full((C_,), 2.0, device=DEV))
    torch.testing.assert_close(stats[3], torch.full((C_,), (2.0 + 1e-3) ** -0.5, device=DEV))


# ------------------------------------------------------------------------------------ b. world 1: loopback and no-op
def test_loopback_sync_layer_matches_per_rank_path():
    """A Conv layer with the synced kernels forced through the identity reducer computes what the per-rank path does
    (statistics through fp64 instead of fp32: equal to a few ulps)"""
    from efficientteacher_b200.model import Conv
    from efficientteacher_b200.parallel import BnSync
    out = {}
    for mode in ("local", "loopback"):
        torch.manual_seed(0)
        conv = Conv(32, 160, 3, 1, act=True).to(DEV).train()
        if mode == "loopback":
            conv.bn_sync = BnSync(loopback=True)
        x = _bf((3, 32, 20, 12), 5).to(DEV, torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        g = _bf((3, 160, 20, 12), 6).to(DEV)
        a = conv(x)
        (a.float() * g).sum().backward()
        out[mode] = dict(a=a.float(), dx=x.grad.float(), dw=conv.conv.weight.grad, dg=conv.bn.weight.grad, db=conv.bn.bias.grad,
                         rm=conv.bn.running_mean, rv=conv.bn.running_var)
    for k in ("a", "dx"):
        assert _rel(out["loopback"][k], out["local"][k]) < 1e-2, k
    for k in ("dw", "dg", "db"):
        assert _rel(out["loopback"][k], out["local"][k]) < 1e-3, k
    torch.testing.assert_close(out["loopback"]["rm"], out["local"]["rm"], rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(out["loopback"]["rv"], out["local"]["rv"], rtol=1e-5, atol=1e-7)


def _step_state(st):
    teacher = st.semi_ema.ema if getattr(st, "semi_ema", None) is not None else st.ema.ema
    return (torch.cat([p.detach().flatten().float() for p in st.model.parameters()]),
            torch.cat([v.detach().flatten().float() for v in teacher.state_dict().values() if v.dtype.is_floating_point]),
            torch.cat([v.detach().flatten() for k, v in st.model.state_dict().items() if "running" in k]))


def _ssod_batch(seed, bl, bu, img):
    import synth
    r = np.random.RandomState(seed)
    imgs = torch.from_numpy(r.rand(bl, 3, img, img).astype(np.float32)).to(DEV)
    uw = torch.from_numpy(r.rand(bu, 3, img, img).astype(np.float32)).to(DEV)
    return imgs, uw, uw.flip(3).contiguous(), torch.from_numpy(synth.make_targets(seed + 1, 6 * bl, bl)).to(DEV), \
        torch.from_numpy(synth.make_Ms(seed + 2, bu, img)).to(DEV)


def _make_step(kind, sync_bn, img, world_size=1, rank=-1, model=None, device=DEV):
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    torch.manual_seed(0)
    if kind == "sup":
        cfg = yolov5_sup_cfg('n', batch_size=2 * max(world_size, 1), img_size=img)
        cfg.sync_bn = sync_bn
        return SupTrainerStep(cfg, torch.device(device), rank=rank, world_size=world_size, epochs=300, model=model)
    cfg = yolov5_ssod_cfg('n', batch_size=4 * max(world_size, 1), img_size=img)
    cfg.sync_bn = sync_bn
    return SSODTrainerStep(cfg, torch.device(device), rank=rank, world_size=world_size, epochs=300, model=model)


def _run_steps(st, kind, mode, seed, img, steps=2):
    imgs, uw, us, tg, Ms = _ssod_batch(seed, 2, 2, img)
    losses = []
    for i in range(steps):
        if kind == "sup":
            f = st.train_step_graphed if mode == "graph" else st.train_step
            losses.append(f(imgs, tg, i).detach().clone())
        else:
            f = st.train_instance_graphed if mode == "graph" else st.train_instance
            losses.append(f(imgs, tg, us, uw, None, Ms, i).detach().clone())
    torch.cuda.synchronize()
    return torch.cat([l.flatten() for l in losses])


@pytest.mark.parametrize("kind", ["sup", "ssod"])
@pytest.mark.parametrize("mode", ["eager", "graph"])
def test_sync_bn_is_ignored_at_world_1(kind, mode):
    """The reference converts only when RANK != -1: a single process runs exactly the sync_bn: False step.  Its result is
    compared with sync_bn: False against the spread of two sync_bn: False runs (equal bits when the step is bit-stable)."""
    out = {}
    for name, sync in (("off", False), ("off2", False), ("on", True)):
        st = _make_step(kind, sync, 128)
        assert not st.sync_bn and not any(isinstance(m, nn.SyncBatchNorm) for m in st.model.modules())
        loss = _run_steps(st, kind, mode, 3, 128)
        out[name] = (loss,) + _step_state(st)
        del st
    for i, what in enumerate(("loss", "student", "teacher", "running")):
        on, off, off2 = out["on"][i], out["off"][i], out["off2"][i]
        spread = (off - off2).abs().max().item()
        assert (on - off).abs().max().item() <= 3.0 * spread + 1e-6 * off.abs().max().item(), (kind, mode, what, spread)


# ---------------------------------------------------------------------------------- c. world 2: two processes, one GPU
def _np(obj):
    if torch.is_tensor(obj):
        return obj.detach().cpu().numpy().copy()
    if isinstance(obj, dict):
        return {k: _np(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_np(v) for v in obj)
    return obj


def _part_layer(rank, world):
    """one Conv(32 -> 96, 3x3) + SyncBatchNorm + SiLU layer, rank r holding 2 + r images"""
    from efficientteacher_b200.autograd_conv import ConvFn
    from efficientteacher_b200.model import Conv
    torch.manual_seed(0)
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(Conv(32, 96, 3, 1, act=True)).to(DEV).train()
    with torch.no_grad():
        conv.bn.weight.uniform_(0.5, 1.5)
        conv.bn.bias.uniform_(-0.5, 0.5)
    assert isinstance(conv.bn, nn.SyncBatchNorm) and conv._sync() is not None
    gamma0, beta0 = conv.bn.weight.detach().clone(), conv.bn.bias.detach().clone()
    n = 2 + rank
    x = _bf((n, 32, 12, 12), 100 + rank).to(DEV, torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    g = _bf((n, 96, 12, 12), 200 + rank).to(DEV)
    a = conv(x)
    (a.float() * g).sum().backward()
    with torch.no_grad():
        y = ConvFn.apply(x.detach(), conv.conv.weight, 1, 1, False).float()
    tbn = nn.SyncBatchNorm(96, eps=1e-3, momentum=0.03).to(DEV).train()
    with torch.no_grad():
        tbn.weight.copy_(gamma0)
        tbn.bias.copy_(beta0)
    yt = y.clone().requires_grad_(True)
    at = F.silu(tbn(yt))
    (at * g).sum().backward()
    return dict(x=x.detach().float(), y=y, g=g, w=conv.conv.weight.detach(), gamma0=gamma0, beta0=beta0, a=a.float(),
                dx=x.grad.float(), dgamma=conv.bn.weight.grad, dbeta=conv.bn.bias.grad, rm=conv.bn.running_mean,
                rv=conv.bn.running_var, at=at.detach(), tdgamma=tbn.weight.grad, tdbeta=tbn.bias.grad, trm=tbn.running_mean,
                trv=tbn.running_var)


def _part_model(rank, world):
    """YOLOv5n (SupModel) after convert_sync_batchnorm: the fused synced path, torch's SyncBatchNorm between the same
    native convs (Conv.FUSED_BN = False), and the fused path with per-rank statistics (set_bn_sync of a group of one
    rank is not available, so a model that was never converted)"""
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.model import Conv, SupModel
    cfg = yolov5_sup_cfg('n', batch_size=4, img_size=128)
    r = np.random.RandomState(300 + rank)
    imgs = torch.from_numpy(r.rand(2 + rank, 3, 128, 128).astype(np.float32)).to(DEV)
    res = {}
    for kind in ("fused", "torch", "local"):
        torch.manual_seed(0)
        m = SupModel(cfg)
        if kind != "local":
            m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
        m = m.to(DEV).train()
        Conv.FUSED_BN = kind != "torch"
        try:
            out = m(imgs)
            gen = torch.Generator(device=DEV).manual_seed(400 + rank)
            loss = sum((o.float() * torch.randn(o.shape, generator=gen, device=DEV)).sum() for o in out)
            loss.backward()
        finally:
            Conv.FUSED_BN = True
        torch.cuda.synchronize()
        bns = [(n, b) for n, b in m.named_modules() if isinstance(b, nn.modules.batchnorm._BatchNorm)]
        res[kind] = dict(rm={n: b.running_mean.clone() for n, b in bns}, rv={n: b.running_var.clone() for n, b in bns},
                         grad={n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None},
                         nbt={n: int(b.num_batches_tracked) for n, b in bns})
        del m
    return res


def _part_steps(rank, world):
    """eager SSOD and supervised steps with sync_bn at world 2; the first forward's running statistics, then 3 steps"""
    res = {}
    for kind in ("ssod", "sup"):
        st = _make_step(kind, True, 128, world_size=world, rank=rank)
        assert st.sync_bn and all(isinstance(mod.bn, nn.SyncBatchNorm) for mod in st.model.modules() if hasattr(mod, "bn"))
        imgs, uw, us, tg, Ms = _ssod_batch(500 + rank, 2, 2, 128)
        # the first forward alone: running statistics of the global batch, from the initial ones
        init = {k: v.clone() for k, v in st.model.state_dict().items() if "running" in k}
        st._bn_broadcast()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            st.model([imgs, us] if kind == "ssod" else imgs)
        first = {k: v.clone() for k, v in st.model.state_dict().items() if "running" in k}
        with torch.no_grad():
            for k, v in st.model.state_dict().items():
                if "running" in k:
                    v.copy_(init[k])
        for i in range(3):
            if kind == "sup":
                st.train_step(imgs, tg, i)
            else:
                st.train_instance(imgs, tg, us, uw, None, Ms, i)
        torch.cuda.synchronize()
        student, teacher, running = _step_state(st)      # no broadcast first: equal running statistics come from the sync
        res[kind] = dict(imgs=imgs, us=us, first=first, student=student, teacher=teacher, running=running,
                         loss=st.last["loss"].float())
        # (5) a captured step refuses sync_bn at world 2
        try:
            if kind == "sup":
                st.train_step_graphed(imgs, tg, 3)
            else:
                st.train_instance_graphed(imgs, tg, us, uw, None, Ms, 3)
            res[kind]["graph_error"] = None
        except NotImplementedError as e:
            res[kind]["graph_error"] = str(e)
        del st
    return res


def _part_reference_order(rank, world):
    """Model(cfg), then torch's convert_sync_batchnorm, then the step built around that model (sync_bn: False: the
    conversion alone decides)"""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    from efficientteacher_b200.trainer import SSODTrainerStep
    cfg = yolov5_ssod_cfg('n', batch_size=8, img_size=128)
    torch.manual_seed(0)
    model = nn.SyncBatchNorm.convert_sync_batchnorm(Model(cfg))
    st = SSODTrainerStep(cfg, torch.device(DEV), rank=rank, world_size=world, epochs=300, model=model)
    bns = [m for m in st.model.modules() if isinstance(m, nn.SyncBatchNorm)]
    ids = lambda ps: {id(p) for p in ps}  # noqa: E731
    groups = st.optimizer.param_groups
    imgs, uw, us, tg, Ms = _ssod_batch(700 + rank, 2, 2, 128)
    st.train_instance(imgs, tg, us, uw, None, Ms, 0)
    torch.cuda.synchronize()
    return dict(n_bn=len(bns), bn_group=ids(groups[2]["params"]) == ids(b.weight for b in bns),
                bn_in_decay=bool(ids(groups[1]["params"]) & ids(b.weight for b in bns)),
                nbt=[int(b.num_batches_tracked) for b in bns], running=_step_state(st)[2], student=_step_state(st)[0],
                mirror=st._bn_sync is not None and len(st._bn_sync.modules) == len(bns))


_PARTS = (("layer", _part_layer), ("model", _part_model), ("steps", _part_steps), ("reference_order", _part_reference_order))


def _worker(rank, world, port, q):
    import datetime
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=180))
    res = {}
    for name, fn in _PARTS:
        try:
            res[name] = _np(fn(rank, world))
        except Exception:
            res[name] = {"error": traceback.format_exc()}
    q.put((rank, res))
    try:
        dist.barrier()
        dist.destroy_process_group()
    except Exception:
        pass


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.fixture(scope="module")
def world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = {}
    try:
        for _ in range(2):
            rank, res = q.get(timeout=900)
            out[rank] = res
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    return out


def _part(world2, name):
    for r in (0, 1):
        assert "error" not in world2[r][name], "rank %d: %s" % (r, world2[r][name].get("error"))
    return world2[0][name], world2[1][name]


def _t(a):
    return torch.from_numpy(np.asarray(a)).double()


def test_world2_layer_against_torch_syncbn_and_float64(world2):
    r0, r1 = _part(world2, "layer")
    eps, mom = 1e-3, 0.03
    y = torch.cat([_t(r0["y"]), _t(r1["y"])]).requires_grad_(True)
    gamma, beta = _t(r0["gamma0"]).requires_grad_(True), _t(r0["beta0"]).requires_grad_(True)
    rm, rv = torch.zeros(96, dtype=torch.float64), torch.ones(96, dtype=torch.float64)
    z = F.silu(F.batch_norm(y, rm, rv, gamma, beta, True, mom, eps))
    z.backward(torch.cat([_t(r0["g"]), _t(r1["g"])]))
    n0 = r0["y"].shape[0]
    w = _t(r0["w"]).to(torch.bfloat16).double()
    for r, res, sl in ((0, r0, slice(0, n0)), (1, r1, slice(n0, None))):
        _check_bf16(_t(res["a"]), z.detach()[sl], "rank %d activation vs float64" % r)
        _check_bf16(_t(res["a"]), _t(res["at"]), "rank %d activation vs torch SyncBatchNorm" % r)
        torch.testing.assert_close(_t(res["rm"]), rm, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(_t(res["rv"]), rv, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(_t(res["rm"]), _t(res["trm"]), rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(_t(res["rv"]), _t(res["trv"]), rtol=1e-4, atol=1e-6)
        dx = torch.nn.grad.conv2d_input(tuple(res["x"].shape), w, y.grad[sl], padding=1)
        assert _rel(_t(res["dx"]), dx) < 1e-2, ("dx", r, _rel(_t(res["dx"]), dx))
    assert np.array_equal(r0["rm"], r1["rm"]) and np.array_equal(r0["rv"], r1["rv"])
    for ours, theirs, want in (("dgamma", "tdgamma", gamma.grad), ("dbeta", "tdbeta", beta.grad)):
        d = _t(r0[ours]) + _t(r1[ours])
        assert ((d - want).abs() <= 1e-3 * want.abs().max() + 1e-3 * want.abs()).all(), (ours, (d - want).abs().max().item())
        assert _rel(d, _t(r0[theirs]) + _t(r1[theirs])) < 1e-3, ours


def test_world2_yolov5n_fused_against_torch_syncbn(world2):
    """every layer's running statistics and every gradient of the fused synced path follow torch's SyncBatchNorm between the
    same convs; per-rank statistics (the model never converted) are much further off"""
    for res in _part(world2, "model"):
        fused, tor, local = res["fused"], res["torch"], res["local"]
        assert set(fused["rm"]) == set(tor["rm"]) and len(fused["rm"]) > 50
        e_sync, e_local = [], []
        for n in fused["rm"]:
            for key, base in (("rm", 0.0), ("rv", 0.97)):          # the batch statistic, out of momentum's 3 %
                f, t, l = ((_t(d[key][n]) - base) / 0.03 for d in (fused, tor, local))
                e_sync.append(_rel(f, t))
                e_local.append(_rel(l, t))
        # the two paths round their activations differently (bf16 once after BN+act, or after BN and after the act) and a
        # random-init trunk amplifies that with depth: bounded by the median and relative to what per-rank statistics give
        e_sync, e_local = np.array(e_sync), np.array(e_local)
        assert np.median(e_sync) < 3e-2 and np.median(e_sync) < 0.1 * np.median(e_local), (np.median(e_sync), np.median(e_local))
        assert e_sync.max() < 0.25 * e_local.max(), (e_sync.max(), e_local.max())
        assert set(fused["grad"]) == set(tor["grad"])
        g_sync = np.array([_rel(fused["grad"][n], tor["grad"][n]) for n in tor["grad"]])
        g_local = np.array([_rel(local["grad"][n], tor["grad"][n]) for n in tor["grad"]])
        # gradients pass through every later layer of a random-init trunk, and the two paths round differently at each of
        # them: measured on the H100, the median relative difference is ~0.34 with global statistics and ~1.5 with per-rank
        # ones.  The layer test above pins the synced kernels themselves to torch's SyncBatchNorm and to float64.
        assert np.median(g_sync) < 0.5 * np.median(g_local), (np.median(g_sync), np.median(g_local), np.percentile(g_sync, [10, 90]))
        assert set(fused["nbt"].values()) == {1} and set(tor["nbt"].values()) == {1}


def test_world2_eager_steps_use_global_statistics_and_stay_identical(world2):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model, SupModel
    steps = _part(world2, "steps")
    for kind in ("ssod", "sup"):
        r0, r1 = steps[0][kind], steps[1][kind]
        # the first forward at world 2 == a world-1 forward on the concatenated batch
        cfg = yolov5_ssod_cfg('n', batch_size=8, img_size=128)
        torch.manual_seed(0)
        m = (Model(cfg) if kind == "ssod" else SupModel(cfg)).to(DEV).train()
        parts = [torch.from_numpy(r["imgs"]).to(DEV) for r in (r0, r1)]
        if kind == "ssod":
            parts += [torch.from_numpy(r["us"]).to(DEV) for r in (r0, r1)]
        init = {k: v.clone() for k, v in m.state_dict().items() if "running" in k}
        with torch.autocast("cuda", dtype=torch.bfloat16):
            m(parts)
        want = {k: v.detach().cpu() for k, v in m.state_dict().items() if "running" in k}
        # per-rank statistics for comparison: rank 0's batch alone
        with torch.no_grad():
            for k, v in m.state_dict().items():
                if "running" in k:
                    v.copy_(init[k])
        with torch.autocast("cuda", dtype=torch.bfloat16):
            m(parts[0::2])
        alone = {k: v.detach().cpu() for k, v in m.state_dict().items() if "running" in k}
        assert set(want) == set(r0["first"])
        e_sync, e_local = [], []
        for k, v in want.items():
            assert np.array_equal(r0["first"][k], r1["first"][k]), (kind, k)
            base = 0.0 if "mean" in k else 0.97
            ref = (v.double() - base) / 0.03
            e_sync.append(_rel((_t(r0["first"][k]) - base) / 0.03, ref))
            e_local.append(_rel((alone[k].double() - base) / 0.03, ref))
        # the same kernels on the same images: only the summation order of the statistics differs (per-rank fp32 rows summed
        # in fp64, or all rows in fp32), and a random-init trunk amplifies the bf16 rounding flips that causes with depth
        e_sync, e_local = np.array(e_sync), np.array(e_local)
        assert np.median(e_sync) < 5e-3 and e_sync.max() < 0.1, (kind, np.median(e_sync), e_sync.max())
        assert e_sync.max() < 0.25 * e_local.max(), (kind, e_sync.max(), e_local.max())
        for what in ("student", "teacher", "running", "loss"):
            if what != "loss":
                assert np.array_equal(r0[what], r1[what]), (kind, what)
        assert np.isfinite(r0["loss"]).all()


def test_world2_captured_step_refuses_sync_bn(world2):
    steps = _part(world2, "steps")
    for r in (0, 1):
        for kind in ("ssod", "sup"):
            msg = steps[r][kind]["graph_error"]
            assert msg is not None and "eager" in msg and "DESIGN" in msg, (r, kind, msg)


def test_world2_reference_order_convert_then_step(world2):
    r0, r1 = _part(world2, "reference_order")
    for res in (r0, r1):
        assert res["n_bn"] > 50 and res["bn_group"] and not res["bn_in_decay"] and res["mirror"]
        assert set(res["nbt"]) == {1}
    assert np.array_equal(r0["running"], r1["running"]) and np.array_equal(r0["student"], r1["student"])
