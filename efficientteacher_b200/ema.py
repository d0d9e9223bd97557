"""ModelEMA / SemiSupModelEMA / CosineEMA with the reference's surface (utils/torch_utils.py:308-424),
backed by ONE fused multi-tensor kernel (etb_ema_update) instead of 2 x 518 tiny launches per update.

`.ema` is a real nn.Module in eval mode with requires_grad=False (it is the teacher, it is validated and
pickled by the trainer: trainer/ssod_trainer.py:599, 358, 398).  Integer buffers (num_batches_tracked) are
not updated, exactly like the reference.
"""
import ctypes as C
import math
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import EtbEmaChunk


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


class _ChunkTable:
    """Device-resident chunk table for (ema tensors, model tensors[, second-ema tensors])."""

    def __init__(self, v_list, m_list, s_list=None):
        lib = _lib.lib()
        n = len(v_list)
        assert n == len(m_list) and (s_list is None or len(s_list) == n)
        self.key = tuple(t.data_ptr() for t in v_list) + tuple(t.data_ptr() for t in m_list) + \
            (tuple(t.data_ptr() for t in s_list) if s_list else ())
        numel = (C.c_int64 * n)(*[t.numel() for t in v_list])
        vp = (C.c_void_p * n)(*[t.data_ptr() for t in v_list])
        mp = (C.c_void_p * n)(*[t.data_ptr() for t in m_list])
        sp = (C.c_void_p * n)(*[t.data_ptr() for t in s_list]) if s_list else None
        self.n_chunks = int(lib.etb_ema_table_count(numel, n))
        host = (EtbEmaChunk * max(self.n_chunks, 1))()
        _lib.check(lib.etb_ema_table_fill(vp, mp, sp, numel, n, host, self.n_chunks), "etb_ema_table_fill")
        raw = np.frombuffer(host, dtype=np.uint8, count=C.sizeof(EtbEmaChunk) * self.n_chunks).copy()
        self.dev = torch.from_numpy(raw).to(v_list[0].device)
        self.elements = int(sum(t.numel() for t in v_list))
        self.streams = 5 if s_list else 3


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


def _launch(table, d, d2=0.0, scalars_dev=None):
    if scalars_dev is not None:      # graph-capture mode: the decays live in device memory, refreshed before each replay
        _lib.check(_lib.lib().etb_ema_update_dev(_lib.ptr(table.dev), table.n_chunks, _lib.ptr(scalars_dev), _lib.stream_ptr()),
                   "etb_ema_update_dev")
        return
    sc = ema_scalars(d, d2)
    _lib.check(_lib.lib().etb_ema_update(_lib.ptr(table.dev), table.n_chunks, sc[0], sc[1], sc[2], sc[3], _lib.stream_ptr()),
               "etb_ema_update")


class _EMABase:
    def _update_with(self, model, d, scalars_dev=None):
        """scalars_dev: ema_scalars(d) in device memory (graph capture: the decay is refreshed before each replay)"""
        with torch.no_grad():
            v_list, m_list = _float_pairs(self.ema, model)
            key = tuple(t.data_ptr() for t in v_list) + tuple(t.data_ptr() for t in m_list)
            tab = getattr(self, "_table", None)
            if tab is None or tab.key != key:
                tab = self._table = _ChunkTable(v_list, m_list)
            _launch(tab, d, scalars_dev=scalars_dev)

    def update_attr(self, model, include=(), exclude=('process_group', 'reducer')):
        copy_attr(self.ema, model, include, exclude)

    def __getstate__(self):  # the chunk table holds raw pointers: never pickle / deepcopy it
        s = dict(self.__dict__)
        s.pop("_table", None)
        return s


class ModelEMA(_EMABase):
    """reference utils/torch_utils.py:308-342; decay ramp d = decay*(1-exp(-updates/2000))."""

    def __init__(self, model, decay=0.9999, updates=0):
        self.ema = deepcopy(de_parallel(model)).eval()
        self.updates = updates
        self._decay0 = decay
        for p in self.ema.parameters():
            p.requires_grad_(False)

    def decay(self, x):
        return self._decay0 * (1 - math.exp(-x / 2000))

    def update(self, model):
        self.updates += 1
        self._update_with(model, self.decay(self.updates))


class SemiSupModelEMA(_EMABase):
    """reference utils/torch_utils.py:344-379; constant decay."""

    def __init__(self, model, decay=0.99, updates=0):
        self.ema = deepcopy(de_parallel(model)).eval()
        self.updates = updates
        self.decay = decay
        for p in self.ema.parameters():
            p.requires_grad_(False)

    def update(self, model):
        self.updates += 1
        self._update_with(model, self.decay)


class CosineEMA(_EMABase):
    """reference utils/torch_utils.py:381-424; decay fixed within an epoch, cosine-scheduled by update_decay."""

    def __init__(self, model, decay_start=0.99, decay_end=0.9999, total_epoch=0):
        self.ema = deepcopy(de_parallel(model)).eval()
        self.total_epoch = total_epoch
        self.decay_start = decay_start
        self.decay_end = decay_end
        self.decay = decay_start
        for p in self.ema.parameters():
            p.requires_grad_(False)
        self.updates = 0

    def update(self, model):
        self._update_with(model, self.decay)

    def update_decay(self, cur_epoch):
        self.decay = self.decay_end - (self.decay_end - self.decay_start) * \
            (np.cos(np.pi * cur_epoch / self.total_epoch) + 1) / 2


_pair_tables = {}


def next_pair_decays(ema, semi_ema, advance=True):
    """(d1, d2) of the next `ema.update(model); semi_ema.update(ema.ema)`; advances the update counters like .update()."""
    def one(e):
        if isinstance(e, ModelEMA):
            if advance:
                e.updates += 1
            return e.decay(e.updates if advance else e.updates + 1)
        if isinstance(e, SemiSupModelEMA) and advance:
            e.updates += 1
        return e.decay
    return one(ema), one(semi_ema)


def update_ema_pair(ema, semi_ema, model, scalars_dev=None):
    """`ema.update(model); semi_ema.update(ema.ema)` (trainer/ssod_trainer.py:485-487) in ONE pass over HBM:
    5 streams (read v,m,s ; write v,s) instead of 6, one launch instead of two.  Bit-identical results."""
    with torch.no_grad():
        d1, d2 = (0.0, 0.0) if scalars_dev is not None else next_pair_decays(ema, semi_ema)
        v_list, m_list = _float_pairs(ema.ema, model)
        s_list, v2_list = _float_pairs(semi_ema.ema, ema.ema)
        assert len(s_list) == len(v_list) and all(a.data_ptr() == b.data_ptr() for a, b in zip(v2_list, v_list))
        key = (id(ema), id(semi_ema))
        tab = _pair_tables.get(key)
        want = tuple(t.data_ptr() for t in v_list) + tuple(t.data_ptr() for t in m_list) + tuple(t.data_ptr() for t in s_list)
        if tab is None or tab.key != want:
            tab = _pair_tables[key] = _ChunkTable(v_list, m_list, s_list)
        _launch(tab, d1, d2, scalars_dev)
        return tab
