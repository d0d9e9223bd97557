"""FusedSGD: torch.optim.SGD(momentum, nesterov=True, weight_decay per group) as ONE launch over all parameters
(csrc/sgd.cu), a drop-in for the optimizer the reference builds in trainer/trainer.py:215-217.  It is a real
torch.optim.Optimizer (param_groups / state_dict / LambdaLR work unchanged); momentum buffers are views of one flat
buffer exposed per parameter as state[p]['momentum_buffer'] like torch's SGD.  The gradients are zeroed in the same pass
(optimizer.zero_grad() becomes a no-op for the arena).

FusedAdamW: the same for torch.optim.AdamW, the optimizer the reference builds when the config sets `adam: True`
(trainer/trainer.py:211-213), on csrc/adamw.cu."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import EtbAdamChunk, EtbSgdChunk, ETB_EMA_CHUNK


class FusedSGD(torch.optim.Optimizer):
    def __init__(self, params, lr=0.01, momentum=0.0, weight_decay=0.0, nesterov=True):
        if not nesterov or momentum <= 0:
            raise NotImplementedError("FusedSGD implements the reference's configuration: Nesterov momentum > 0")
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, nesterov=nesterov, dampening=0))
        self._table = None
        self._hyper = None

    def _build(self):
        ps = [(gi, p) for gi, g in enumerate(self.param_groups) for p in g["params"] if p.requires_grad]
        for _, p in ps:
            _lib.require_cuda(p)
            if p.grad is None:
                raise RuntimeError("FusedSGD needs materialised gradients (use parallel.GradArena or run a backward first)")
            if p.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous():
                raise RuntimeError("FusedSGD expects contiguous fp32 parameters and gradients")
        dev = ps[0][1].device
        total = sum(p.numel() for _, p in ps)
        old = [self.state[p].get("momentum_buffer") for _, p in ps]
        self._flat = torch.zeros(total, dtype=torch.float32, device=dev)
        chunks, o = [], 0
        for (gi, p), ob in zip(ps, old):
            buf = self._flat[o:o + p.numel()].view_as(p)
            if ob is not None:
                buf.copy_(ob)
            self.state[p]["momentum_buffer"] = buf
            for s in range(0, p.numel(), ETB_EMA_CHUNK):
                c = EtbSgdChunk()
                n = min(ETB_EMA_CHUNK, p.numel() - s)
                c.p, c.g, c.buf, c.n, c.group = p.data_ptr() + 4 * s, p.grad.data_ptr() + 4 * s, buf.data_ptr() + 4 * s, n, gi
                chunks.append(c)
            o += p.numel()
        arr = (EtbSgdChunk * len(chunks))(*chunks)
        self._table = torch.from_numpy(np.frombuffer(arr, dtype=np.uint8).copy()).to(dev)
        self._n = len(chunks)
        self._key = tuple((p.data_ptr(), p.grad.data_ptr()) for _, p in ps)
        self._ps = ps
        self._hyper = torch.zeros(4 * len(self.param_groups), dtype=torch.float32, device=dev)
        self._hyper_host = None

    def _sync_hyper(self):
        vals = []
        for g in self.param_groups:
            vals += [float(g["lr"]), float(g["momentum"]), float(g["weight_decay"]), 0.0]
        if vals != self._hyper_host:       # H2D only when the schedule / warm-up changed something
            self._hyper.copy_(torch.tensor(vals, dtype=torch.float32))
            self._hyper_host = vals

    @torch.no_grad()
    def step(self, closure=None, zero_grad=True):
        if closure is not None:
            raise NotImplementedError
        if self._table is None or self._key != tuple((p.data_ptr(), p.grad.data_ptr() if p.grad is not None else 0) for _, p in self._ps):
            self._build()
        if not torch.cuda.is_current_stream_capturing():
            self._sync_hyper()
        _lib.check(_lib.lib().etb_sgd_step(_lib.ptr(self._table), self._n, _lib.ptr(self._hyper), int(zero_grad), _lib.stream_ptr()),
                   "etb_sgd_step")

    def load_state_dict(self, state_dict):
        """torch's load_state_dict replaces state[p]['momentum_buffer'] by fresh tensors; copy them into the flat buffer the
        kernel reads (and keep the per-parameter views), so a resumed run really continues with the restored momentum
        (trainer/trainer.py:251: `self.optimizer.load_state_dict(ckpt['optimizer'])`)."""
        super().load_state_dict(state_dict)
        if self._table is not None:
            with torch.no_grad():
                o = 0
                for _, p in self._ps:
                    view = self._flat[o:o + p.numel()].view_as(p)
                    loaded = self.state[p].get("momentum_buffer")
                    if loaded is not None and loaded.data_ptr() != view.data_ptr():
                        view.copy_(loaded)
                    self.state[p]["momentum_buffer"] = view
                    o += p.numel()
        self._hyper_host = None      # force the next step to push lr / momentum / weight_decay again

    def refresh_hyper(self):
        """Push the current lr / momentum / weight_decay of the param groups to device memory (call before replaying a
        captured graph that contains step())."""
        if self._hyper is not None:
            self._sync_hyper()


class FusedAdamW(torch.optim.Optimizer):
    """torch.optim.AdamW (decoupled weight decay, no amsgrad) as ONE launch over all parameters (csrc/adamw.cu), bit-equal to
    torch's default CUDA implementation (foreach) on the same gradients.  exp_avg / exp_avg_sq are views of two flat
    buffers, exposed per parameter as state[p]['exp_avg'] / state[p]['exp_avg_sq'] like torch's; the gradients are zeroed in
    the same pass.  The param groups carry AdamW's keys and no 'momentum', so the warm-up leaves the betas alone as the
    reference's does (trainer/ssod_trainer.py:477), and state dicts load both ways between this and torch's AdamW.

    The step count t is one host integer (`step_count`) shared by all parameters: the bias corrections 1 - beta**t are
    computed in float64 on the host exactly as torch's Python does and rounded once to fp32 with the other per-group
    scalars.  It advances once per eager step(), and once per refresh_hyper(), which is called before each replay of a
    captured step(); capturing step() does not advance it.  state_dict() writes it into every state[p]['step']."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False):
        if amsgrad:
            raise NotImplementedError("FusedAdamW implements AdamW without amsgrad (the reference's configuration)")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False,
                                      maximize=False, foreach=None, capturable=False, differentiable=False, fused=None,
                                      decoupled_weight_decay=True))
        self.step_count = 0
        self._table = None
        self._hyper = None
        self._hyper_host = None

    def _build(self):
        ps = [(gi, p) for gi, g in enumerate(self.param_groups) for p in g["params"] if p.requires_grad]
        for _, p in ps:
            _lib.require_cuda(p)
            if p.grad is None:
                raise RuntimeError("FusedAdamW needs materialised gradients (use parallel.GradArena or run a backward first)")
            if p.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous():
                raise RuntimeError("FusedAdamW expects contiguous fp32 parameters and gradients")
        dev = ps[0][1].device
        total = sum(p.numel() for _, p in ps)
        old = [(self.state[p].get("exp_avg"), self.state[p].get("exp_avg_sq")) for _, p in ps]
        self._flat_m = torch.zeros(total, dtype=torch.float32, device=dev)
        self._flat_v = torch.zeros(total, dtype=torch.float32, device=dev)
        chunks, o = [], 0
        for (gi, p), (om, ov) in zip(ps, old):
            m = self._flat_m[o:o + p.numel()].view_as(p)
            v = self._flat_v[o:o + p.numel()].view_as(p)
            if om is not None:
                m.copy_(om)
            if ov is not None:
                v.copy_(ov)
            self.state[p]["exp_avg"], self.state[p]["exp_avg_sq"] = m, v
            for s in range(0, p.numel(), ETB_EMA_CHUNK):
                c = EtbAdamChunk()
                c.p, c.g = p.data_ptr() + 4 * s, p.grad.data_ptr() + 4 * s
                c.m, c.v = m.data_ptr() + 4 * s, v.data_ptr() + 4 * s
                c.n, c.group = min(ETB_EMA_CHUNK, p.numel() - s), gi
                chunks.append(c)
            o += p.numel()
        arr = (EtbAdamChunk * len(chunks))(*chunks)
        self._table = torch.from_numpy(np.frombuffer(arr, dtype=np.uint8).copy()).to(dev)
        self._n = len(chunks)
        self._key = tuple((p.data_ptr(), p.grad.data_ptr()) for _, p in ps)
        self._ps = ps
        self._hyper = torch.zeros(8 * len(self.param_groups), dtype=torch.float32, device=dev)
        self._hyper_host = None

    def _scalars(self):
        """Per group, the fp32 scalars of step t = step_count, each computed in float64 as torch's _multi_tensor_adam
        computes it (torch/optim/adam.py, non-capturable branch) and rounded once"""
        t = float(self.step_count)
        vals = []
        for g in self.param_groups:
            lr, wd, eps = float(g["lr"]), float(g["weight_decay"]), float(g["eps"])
            beta1, beta2 = (float(b) for b in g["betas"])
            bc1, bc2 = 1 - beta1 ** t, 1 - beta2 ** t
            vals += [1 - lr * wd, 1 - beta1, beta2, 1 - beta2, (lr / bc1) * -1, bc2 ** 0.5, eps, 0.0]
        return vals

    def _sync_hyper(self):
        vals = self._scalars()
        if vals != self._hyper_host:       # H2D only when the step or the schedule changed something
            self._hyper.copy_(torch.tensor(vals, dtype=torch.float32))
            self._hyper_host = vals

    @torch.no_grad()
    def step(self, closure=None, zero_grad=True):
        if closure is not None:
            raise NotImplementedError
        if self._table is None or self._key != tuple((p.data_ptr(), p.grad.data_ptr() if p.grad is not None else 0) for _, p in self._ps):
            self._build()
        if not torch.cuda.is_current_stream_capturing():
            self.step_count += 1
            self._sync_hyper()
        _lib.check(_lib.lib().etb_adamw_step(_lib.ptr(self._table), self._n, _lib.ptr(self._hyper), int(zero_grad),
                                             _lib.stream_ptr()), "etb_adamw_step")

    def refresh_hyper(self):
        """Before a replay of a captured graph that contains step(): advance the step count and push this step's lr /
        weight decay / bias corrections to the device memory the captured kernel reads.  Call it once per replay."""
        if self._hyper is not None:
            self.step_count += 1
            self._sync_hyper()

    def _params(self):
        return [p for g in self.param_groups for p in g["params"]]

    def state_dict(self):
        for p in self._params():
            if "exp_avg" in self.state.get(p, {}):
                self.state[p]["step"] = torch.tensor(float(self.step_count), dtype=torch.float32)
        return super().state_dict()

    def load_state_dict(self, state_dict):
        """Loads torch.optim.AdamW's state dicts as well as its own (trainer/trainer.py:249-251).  The moments go into the
        flat buffers the kernel reads (per-parameter views are kept); the per-parameter steps become step_count, so they
        have to agree."""
        super().load_state_dict(state_dict)
        ps = self._params()
        steps = [float(self.state[p].pop("step")) if "step" in self.state[p] else None for p in ps]
        if len(set(steps)) > 1:
            raise ValueError("FusedAdamW keeps one step count for all parameters; the loaded state has steps %s"
                             % sorted(set(steps), key=lambda s: -1 if s is None else s))
        self.step_count = int(steps[0]) if steps and steps[0] is not None else 0
        if self._table is not None:
            with torch.no_grad():
                o = 0
                for _, p in self._ps:
                    for k, flat in (("exp_avg", self._flat_m), ("exp_avg_sq", self._flat_v)):
                        view = flat[o:o + p.numel()].view_as(p)
                        loaded = self.state[p].get(k)
                        if loaded is None:
                            view.zero_()
                        elif loaded.data_ptr() != view.data_ptr():
                            view.copy_(loaded)
                        self.state[p][k] = view
                    o += p.numel()
        self._hyper_host = None
