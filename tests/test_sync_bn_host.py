"""CPU: the host side of SyncBatchNorm (`sync_bn`) -- converting a native model keeps its parameters and buffers, every
BatchNorm walker of the package finds the SyncBatchNorm modules, copies drop the reducer, per-rank statistics stay the
default without a process group, and a captured step refuses SyncBatchNorm at world > 1.  No kernels run."""
import copy
from types import SimpleNamespace as NS

import pytest
import torch
import torch.nn as nn


def _model():
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    torch.manual_seed(0)
    return Model(yolov5_ssod_cfg('n', batch_size=4, img_size=128))


def test_sync_batchnorm_converts_in_place_and_keeps_state():
    from efficientteacher_b200.model import Conv
    m = _model()
    before = [(n, b) for n, b in m.named_modules() if isinstance(b, nn.BatchNorm2d)]
    params = {n: p for n, p in m.named_parameters()}
    bufs = {n: b for n, b in m.named_buffers()}
    assert m.sync_batchnorm() is m
    after = [(n, b) for n, b in m.named_modules() if isinstance(b, nn.modules.batchnorm._BatchNorm)]
    assert [n for n, _ in after] == [n for n, _ in before] and len(after) > 50
    assert all(isinstance(b, nn.SyncBatchNorm) for _, b in after)
    assert all(p is params[n] for n, p in m.named_parameters())              # the optimizer's tensors stay valid
    assert all(b is bufs[n] for n, b in m.named_buffers())
    convs = [c for c in m.modules() if isinstance(c, Conv)]
    assert all(c._sync() is None for c in convs)          # no process group: per-rank statistics, like torch's module


def test_bn_walkers_find_syncbatchnorm():
    from efficientteacher_b200.parallel import BnBufferSync
    m = nn.SyncBatchNorm.convert_sync_batchnorm(_model())       # the reference's call
    bns = [b for b in m.modules() if isinstance(b, nn.SyncBatchNorm)]
    sync = BnBufferSync(m)
    assert sync.modules == bns
    assert sync.flat.numel() == sum(2 * b.num_features for b in bns)
    assert bns[3].running_var.data_ptr() == sync.flat.data_ptr() + 4 * sum(2 * b.num_features for b in bns[:3]) + 4 * bns[3].num_features
    # the mirror survives a conversion made after it: the new modules take over the same buffer views
    m2 = _model()
    sync2 = BnBufferSync(m2)
    m2.sync_batchnorm()
    assert all(b.running_mean.data_ptr() == a.running_mean.data_ptr()
               for a, b in zip(sync2.modules, (b for b in m2.modules() if isinstance(b, nn.SyncBatchNorm))))


def test_copies_drop_the_forced_reducer():
    from efficientteacher_b200.model import Conv
    from efficientteacher_b200.parallel import BnSync
    m = _model().sync_batchnorm()
    lb = BnSync(loopback=True)
    m.set_bn_sync(lb)
    convs = [c for c in m.modules() if isinstance(c, Conv)]
    assert all(c._sync() is lb for c in convs)
    c2 = copy.deepcopy(m)                        # the EMA's copy
    assert all(c.bn_sync is None for c in c2.modules() if isinstance(c, Conv))
    assert all(isinstance(b, nn.SyncBatchNorm) for b in c2.modules() if isinstance(b, nn.modules.batchnorm._BatchNorm))
    assert all("bn_sync" not in c.__getstate__() for c in convs)
    m.set_bn_sync(None)
    assert all(c._sync() is None for c in convs)
    t = torch.arange(5.0)
    assert lb.all_reduce(t) is t and torch.equal(t, torch.arange(5.0)) and lb.world_size == 1


def test_captured_step_refuses_syncbatchnorm_at_world_2():
    from efficientteacher_b200.trainer import TrainerStep
    m = _model()
    for world, convert, raises in ((2, False, False), (1, True, False), (2, True, True)):
        if convert:
            m.sync_batchnorm()
        st = NS(WORLD_SIZE=world, model=m)
        if raises:
            with pytest.raises(NotImplementedError, match="eager"):
                TrainerStep._check_capturable(st)
        else:
            TrainerStep._check_capturable(st)
