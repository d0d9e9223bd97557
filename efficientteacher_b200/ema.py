"""ModelEMA / SemiSupModelEMA / CosineEMA with the reference's surface (utils/torch_utils.py:308-424),
backed by ONE fused multi-tensor kernel (etb_ema_update) instead of 2 x 518 tiny launches per update.

`.ema` is a real nn.Module in eval mode with requires_grad=False (it is the teacher, it is validated and
pickled by the trainer: trainer/ssod_trainer.py:599, 358, 398).  Integer buffers (num_batches_tracked) are
not updated, exactly like the reference.
"""
import math
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn

from . import _lib


def is_parallel(model):
    return type(model) in (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel)


def de_parallel(model):
    return model.module if is_parallel(model) else model


def copy_attr(a, b, include=(), exclude=()):
    # reference utils/torch_utils.py:279-285
    for k, v in b.__dict__.items():
        if (len(include) and k not in include) or k.startswith('_') or k in exclude:
            continue
        setattr(a, k, v)


def _float_pairs(ema_module, model):
    msd = de_parallel(model).state_dict()
    v_list, m_list = [], []
    for k, v in ema_module.state_dict().items():
        if v.dtype.is_floating_point:
            m = msd[k].detach()
            if v.dtype != torch.float32 or m.dtype != torch.float32:
                raise RuntimeError("EMA kernel expects fp32 state (key %s: %s / %s)" % (k, v.dtype, m.dtype))
            if not (v.is_contiguous() and m.is_contiguous()):
                raise RuntimeError("EMA kernel expects contiguous state tensors (key %s)" % k)
            _lib.require_cuda(v, m)
            v_list.append(v)
            m_list.append(m)
    return v_list, m_list


def ema_scalars(d, d2=0.0):
    """{d, 1-d, d2, 1-d2} rounded to fp32 the way python scalars are when they meet an fp32 tensor (SURVEY.md D9)."""
    return [float(np.float32(d)), float(np.float32(1.0 - d)), float(np.float32(d2)), float(np.float32(1.0 - d2))]


def _launch(owner, attr, streams, hyper_dev):
    """etb_ema_update over `streams` ({v, m[, s]} per tensor) with {d, 1-d, d2, 1-d2} read from hyper_dev; the chunk table
    is kept in owner.<attr> and rebuilt when a tensor moved"""
    tab = getattr(owner, attr, None)
    if tab is None or tab[2] != _lib.chunk_key(streams):
        tab = _lib.chunk_table(streams)
        setattr(owner, attr, tab)
    _lib.check(_lib.lib().etb_ema_update(_lib.ptr(tab[0]), tab[1], _lib.ptr(hyper_dev), _lib.stream_ptr()), "etb_ema_update")


class _EMABase:
    def __init__(self, model):
        self.ema = deepcopy(de_parallel(model)).eval()
        for p in self.ema.parameters():
            p.requires_grad_(False)

    def _scalars_dev(self, d, d2, device):
        """ema_scalars(d, d2) in a 4-float device tensor of this EMA, for an eager update.  A stream-ordered copy from
        pageable memory: the runtime stages the 16 bytes before returning, so the host does not wait for the device and a
        later update cannot overwrite them before this one has read them."""
        if getattr(self, "_hyper_dev", None) is None:
            self._hyper_dev = torch.empty(4, dtype=torch.float32, device=device)
        self._hyper_dev.copy_(torch.tensor(ema_scalars(d, d2), dtype=torch.float32), non_blocking=True)
        return self._hyper_dev

    def _update_with(self, model, d, scalars_dev=None):
        """scalars_dev: ema_scalars(d) in device memory (graph capture: the decay is refreshed before each replay)"""
        with torch.no_grad():
            v_list, m_list = _float_pairs(self.ema, model)
            if scalars_dev is None:
                scalars_dev = self._scalars_dev(d, 0.0, v_list[0].device)
            _launch(self, "_table", list(zip(v_list, m_list)), scalars_dev)

    def update_attr(self, model, include=(), exclude=('process_group', 'reducer')):
        copy_attr(self.ema, model, include, exclude)

    def __getstate__(self):  # the chunk tables hold raw pointers: never pickle / deepcopy them
        s = dict(self.__dict__)
        for k in ("_table", "_pair_table", "_hyper_dev"):
            s.pop(k, None)
        return s


class ModelEMA(_EMABase):
    """reference utils/torch_utils.py:308-342; decay ramp d = decay*(1-exp(-updates/2000))."""

    def __init__(self, model, decay=0.9999, updates=0):
        super().__init__(model)
        self.updates = updates
        self._decay0 = decay

    def decay(self, x):
        return self._decay0 * (1 - math.exp(-x / 2000))

    def update(self, model):
        self.updates += 1
        self._update_with(model, self.decay(self.updates))


class SemiSupModelEMA(_EMABase):
    """reference utils/torch_utils.py:344-379; constant decay."""

    def __init__(self, model, decay=0.99, updates=0):
        super().__init__(model)
        self.updates = updates
        self.decay = decay

    def update(self, model):
        self.updates += 1
        self._update_with(model, self.decay)


class CosineEMA(_EMABase):
    """reference utils/torch_utils.py:381-424; decay fixed within an epoch, cosine-scheduled by update_decay."""

    def __init__(self, model, decay_start=0.99, decay_end=0.9999, total_epoch=0):
        super().__init__(model)
        self.total_epoch = total_epoch
        self.decay_start = decay_start
        self.decay_end = decay_end
        self.decay = decay_start
        self.updates = 0

    def update(self, model):
        self._update_with(model, self.decay)

    def update_decay(self, cur_epoch):
        self.decay = self.decay_end - (self.decay_end - self.decay_start) * \
            (np.cos(np.pi * cur_epoch / self.total_epoch) + 1) / 2


def next_pair_decays(ema, semi_ema):
    """(d1, d2) of the next `ema.update(model); semi_ema.update(ema.ema)`; advances the update counters like .update()."""
    def one(e):
        if isinstance(e, ModelEMA):
            e.updates += 1
            return e.decay(e.updates)
        if isinstance(e, SemiSupModelEMA):
            e.updates += 1
        return e.decay
    return one(ema), one(semi_ema)


def update_ema_pair(ema, semi_ema, model, scalars_dev=None):
    """`ema.update(model); semi_ema.update(ema.ema)` (trainer/ssod_trainer.py:485-487) in ONE pass over HBM:
    5 streams (read v,m,s ; write v,s) instead of 6, one launch instead of two.  Bit-identical results.  The pair's chunk
    table lives on semi_ema."""
    with torch.no_grad():
        v_list, m_list = _float_pairs(ema.ema, model)
        s_list, v2_list = _float_pairs(semi_ema.ema, ema.ema)
        assert len(s_list) == len(v_list) and all(a.data_ptr() == b.data_ptr() for a, b in zip(v2_list, v_list))
        if scalars_dev is None:
            scalars_dev = semi_ema._scalars_dev(*next_pair_decays(ema, semi_ema), v_list[0].device)
        _launch(semi_ema, "_pair_table", list(zip(v_list, m_list, s_list)), scalars_dev)
