"""FusedSGD: torch.optim.SGD(momentum, nesterov=True, weight_decay per group) as ONE launch over all parameters
(csrc/sgd.cu), a drop-in for the optimizer the reference builds in trainer/trainer.py:215-217.  It is a real
torch.optim.Optimizer (param_groups / state_dict / LambdaLR work unchanged); momentum buffers are views of one flat
buffer exposed per parameter as state[p]['momentum_buffer'] like torch's SGD.  The gradients are zeroed in the same pass
(optimizer.zero_grad() becomes a no-op for the arena).

FusedAdamW: the same for torch.optim.AdamW, the optimizer the reference builds when the config sets `adam: True`
(trainer/trainer.py:211-213), on csrc/adamw.cu."""
import torch

from . import _lib


class _FusedOptimizer(torch.optim.Optimizer):
    """What FusedSGD and FusedAdamW share.  Each per-parameter moment named in STATE_KEYS is a view of one flat buffer per
    key (flat_state()), exposed as state[p][key] like torch's; the kernel KERNEL runs over the chunk table of the streams
    {p, grad, *moments}, with the fp32 scalars of _scalars() (HYPER_W per param group) in device memory.  They are
    uploaded only when they change, and a captured step() reads whatever refresh_hyper() wrote last."""
    STATE_KEYS = ()
    KERNEL = ""
    HYPER_W = 4

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._table = None
        self._hyper = None
        self._hyper_host = None

    def _scalars(self):
        raise NotImplementedError

    def _next_step(self):
        """called once per eager step() and once per refresh_hyper(), before the scalars are pushed"""

    def _streams(self):
        return [(p, p.grad) + views for (_, p), views in zip(self._ps, self._views)]

    def _build(self):
        name = type(self).__name__
        ps = [(gi, p) for gi, g in enumerate(self.param_groups) for p in g["params"] if p.requires_grad]
        for _, p in ps:
            _lib.require_cuda(p)
            if p.grad is None:
                raise RuntimeError("%s needs materialised gradients (use parallel.GradArena or run a backward first)" % name)
            if p.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous():
                raise RuntimeError("%s expects contiguous fp32 parameters and gradients" % name)
        dev = ps[0][1].device
        total = sum(p.numel() for _, p in ps)
        self._flat = [torch.zeros(total, dtype=torch.float32, device=dev) for _ in self.STATE_KEYS]
        self._ps = ps
        self._rehome()
        self._table, self._n, self._key = _lib.chunk_table(self._streams(), [gi for gi, _ in ps])
        self._hyper = torch.zeros(self.HYPER_W * len(self.param_groups), dtype=torch.float32, device=dev)
        self._hyper_host = None

    @torch.no_grad()
    def _rehome(self):
        """Point state[p][key] at the flat buffers the kernel reads: a moment the state holds elsewhere (a new build, a
        loaded state dict) is copied in, and a missing one is zeroed, which both torch optimizers treat as a fresh moment
        (SGD: buf = grad on its first use; AdamW: zero moments)."""
        self._views, missing, o = [], [], 0
        for _, p in self._ps:
            views = tuple(f[o:o + p.numel()].view_as(p) for f in self._flat)
            for k, view in zip(self.STATE_KEYS, views):
                loaded = self.state[p].get(k)
                if loaded is None:
                    missing.append(view)
                elif loaded.data_ptr() != view.data_ptr():
                    view.copy_(loaded)
                self.state[p][k] = view
            self._views.append(views)
            o += p.numel()
        if missing:
            torch._foreach_zero_(missing)

    def _ensure_table(self):
        if self._table is None or self._key != _lib.chunk_key(self._streams()):
            self._build()

    def _sync_hyper(self):
        vals = self._scalars()
        if vals != self._hyper_host:       # H2D only when the step, the schedule or the warm-up changed something
            self._hyper.copy_(torch.tensor(vals, dtype=torch.float32))
            self._hyper_host = vals

    def flat_state(self):
        """The optimizer state as the flat buffers the kernel reads, one per STATE_KEYS entry (built from the current
        parameters and gradients if no step has built them yet): restoring these restores every state[p][key]."""
        self._ensure_table()
        return list(self._flat)

    @torch.no_grad()
    def step(self, closure=None, zero_grad=True):
        if closure is not None:
            raise NotImplementedError
        self._ensure_table()
        if not torch.cuda.is_current_stream_capturing():
            self._next_step()
            self._sync_hyper()
        _lib.check(getattr(_lib.lib(), self.KERNEL)(_lib.ptr(self._table), self._n, _lib.ptr(self._hyper), int(zero_grad),
                                                    _lib.stream_ptr()), self.KERNEL)

    def refresh_hyper(self):
        """Before a replay of a captured graph that contains step(): push this step's scalars to the device memory the
        captured kernel reads.  Call it once per replay."""
        if self._hyper is not None:
            self._next_step()
            self._sync_hyper()

    def load_state_dict(self, state_dict):
        """torch's load_state_dict puts fresh tensors into the state; they are copied into the flat buffers the kernel reads
        (the per-parameter views are kept), so a resumed run really continues with the restored moments
        (trainer/trainer.py:251: `self.optimizer.load_state_dict(ckpt['optimizer'])`)."""
        super().load_state_dict(state_dict)
        if self._table is not None:
            self._rehome()
        self._hyper_host = None      # force the next step to push the scalars again


class FusedSGD(_FusedOptimizer):
    STATE_KEYS = ("momentum_buffer",)
    KERNEL = "etb_sgd_step"

    def __init__(self, params, lr=0.01, momentum=0.0, weight_decay=0.0, nesterov=True):
        if not nesterov or momentum <= 0:
            raise NotImplementedError("FusedSGD implements the reference's configuration: Nesterov momentum > 0")
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, nesterov=nesterov, dampening=0))

    def _scalars(self):
        return [v for g in self.param_groups for v in (float(g["lr"]), float(g["momentum"]), float(g["weight_decay"]), 0.0)]


class FusedAdamW(_FusedOptimizer):
    """torch.optim.AdamW (decoupled weight decay, no amsgrad) as ONE launch over all parameters (csrc/adamw.cu), bit-equal to
    torch's default CUDA implementation (foreach) on the same gradients.  exp_avg / exp_avg_sq are views of two flat
    buffers, exposed per parameter as state[p]['exp_avg'] / state[p]['exp_avg_sq'] like torch's; the gradients are zeroed in
    the same pass.  The param groups carry AdamW's keys and no 'momentum', so the warm-up leaves the betas alone as the
    reference's does (trainer/ssod_trainer.py:477), and state dicts load both ways between this and torch's AdamW.

    The step count t is one host integer (`step_count`) shared by all parameters: the bias corrections 1 - beta**t are
    computed in float64 on the host exactly as torch's Python does and rounded once to fp32 with the other per-group
    scalars.  It advances once per eager step(), and once per refresh_hyper(), which is called before each replay of a
    captured step(); capturing step() does not advance it.  state_dict() writes it into every state[p]['step']."""
    STATE_KEYS = ("exp_avg", "exp_avg_sq")
    KERNEL = "etb_adamw_step"
    HYPER_W = 8

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False):
        if amsgrad:
            raise NotImplementedError("FusedAdamW implements AdamW without amsgrad (the reference's configuration)")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False,
                                      maximize=False, foreach=None, capturable=False, differentiable=False, fused=None,
                                      decoupled_weight_decay=True))
        self.step_count = 0

    def _next_step(self):
        self.step_count += 1

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

    def _params(self):
        return [p for g in self.param_groups for p in g["params"]]

    def state_dict(self):
        for p in self._params():
            if "exp_avg" in self.state.get(p, {}):
                self.state[p]["step"] = torch.tensor(float(self.step_count), dtype=torch.float32)
        return super().state_dict()

    def load_state_dict(self, state_dict):
        """Loads torch.optim.AdamW's state dicts as well as its own (trainer/trainer.py:249-251).  The per-parameter steps
        become step_count, so they have to agree."""
        super().load_state_dict(state_dict)
        ps = self._params()
        steps = [float(self.state[p].pop("step")) if "step" in self.state[p] else None for p in ps]
        if len(set(steps)) > 1:
            raise ValueError("FusedAdamW keeps one step count for all parameters; the loaded state has steps %s"
                             % sorted(set(steps), key=lambda s: -1 if s is None else s))
        self.step_count = int(steps[0]) if steps and steps[0] is not None else 0
