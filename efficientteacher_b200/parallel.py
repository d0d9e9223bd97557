"""Data parallelism of the SSOD step (SURVEY.md 8e): one process per GPU, NCCL over NVLink, and two collectives per step --
a SUM all-reduce of the flat fp32 gradient arena (191.8 MB for YOLOv5l-SSOD) after backward, and a broadcast of the
student's BatchNorm running statistics before its forward.

The reference wraps the student in DDP (trainer/trainer.py:313), multiplies both losses by WORLD_SIZE
(trainer/ssod_trainer.py:638-639,647-648) and lets DDP average the bucketed gradients: mean(W*g_r) == sum(g_r).  Here the
losses are left unscaled and the arena (GradArena) is summed once, after backward.  BatchNorm statistics stay per rank by
default (SyncBN is off in every shipped config), and the teacher EMA is updated locally from the identical post-all-reduce
weights.

SyncBatchNorm (`sync_bn: True` with WORLD_SIZE > 1, trainer/ssod_trainer.py:217-220): the student's BatchNorm layers
normalise with the statistics of the global batch.  BnSync is the object the fused BatchNorm kernels take for it: two SUM
all-reduces per layer, of the forward statistics ([2C+1] fp64: sum y, sum y^2, count) and of the backward sums ([2C]
fp32), on the current stream, over any backend (NCCL, or gloo with CUDA tensors).

BatchNorm buffers (SURVEY.md 8e caveat 2): the reference's DDP runs with broadcast_buffers=True, i.e. at the start of every
forward rank 0's running_mean / running_var overwrite every rank's.  BnBufferSync keeps all running statistics of the
student in ONE flat buffer and broadcasts it from rank 0 before the student forward (60,151 floats: one small NCCL
broadcast), reproducing that.  (The reference's per-rank teachers are therefore NOT identical across ranks either: each
rank's EMA sees 0.97 * rank0's statistics + 0.03 * its own batch's; only rank 0's teacher is validated / saved.)"""
import torch


class GradArena:
    """All gradients of `params` as views of one contiguous fp32 buffer.  Every view starts on a 16-byte boundary (the
    wgrad / BN-backward kernels accumulate into the views with float4 accesses); the pad floats stay zero."""

    ALIGN = 4   # floats

    @classmethod
    def _offsets(cls, params):
        offs, o = [], 0
        for p in params:
            offs.append(o)
            o += (p.numel() + cls.ALIGN - 1) // cls.ALIGN * cls.ALIGN
        return offs, o

    def __init__(self, params, device=None, reverse=False):
        """reverse: lay the arena out in reverse parameter order (= the order in which backward completes the gradients)."""
        self.params = [p for p in params if p.requires_grad]
        if reverse:
            self.params = self.params[::-1]
        self.offsets, n = self._offsets(self.params)
        dev = device if device is not None else self.params[0].device
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        for p, o in zip(self.params, self.offsets):
            p.grad = self.flat[o:o + p.numel()].view_as(p)
        self.average = False    # True: ncclAvg instead of ncclSum (same collective, same cost); see SSODTrainerStep.GRAD_REDUCE

    def _op(self):
        import torch.distributed as dist
        return dist.ReduceOp.AVG if self.average else dist.ReduceOp.SUM

    def zero(self):
        self.flat.zero_()

    def check_views(self):
        """True while every p.grad still aliases the arena (optimizer.zero_grad(set_to_none=True) would break it)."""
        for p, o in zip(self.params, self.offsets):
            if p.grad is None or p.grad.data_ptr() != self.flat.data_ptr() + 4 * o:
                return False
        return True

    def all_reduce_sum(self, world_size, group=None):
        if world_size > 1:
            import torch.distributed as dist
            dist.all_reduce(self.flat, op=self._op(), group=group)
        return self.flat


class BnBufferSync:
    """All BatchNorm running statistics of `model` re-homed into one flat fp32 buffer (the modules' registered buffers become
    views of it), so DDP's per-forward `broadcast_buffers` is one collective: broadcast(src=0)."""

    def __init__(self, model):
        bns = [m for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]    # SyncBatchNorm too
        n = sum(m.running_mean.numel() + m.running_var.numel() for m in bns)
        dev = bns[0].running_mean.device
        self.flat = torch.empty(n, dtype=torch.float32, device=dev)
        o = 0
        with torch.no_grad():
            for m in bns:
                for name in ("running_mean", "running_var"):
                    t = getattr(m, name)
                    v = self.flat[o:o + t.numel()]
                    v.copy_(t)
                    setattr(m, name, v)            # registered buffer name: lands in m._buffers
                    o += t.numel()
        self.modules = bns

    def broadcast(self, world_size, group=None):
        if world_size > 1:
            import torch.distributed as dist
            dist.broadcast(self.flat, src=0, group=group)


class BnSync:
    """The collective of the synced BatchNorm kernels (convops.bn_forward / bn_backward `sync=`): a SUM all-reduce over
    `group` (None: the default group).  loopback=True reduces over nothing (world 1): the synced kernels and the count
    hand-over run exactly as with several ranks, which isolates their cost from the communication."""

    def __init__(self, group=None, loopback=False):
        self.group, self.loopback = group, bool(loopback)
        if self.loopback:
            self.world_size = 1
        else:
            import torch.distributed as dist
            self.world_size = dist.get_world_size(group)

    def all_reduce(self, t):
        if not self.loopback:
            import torch.distributed as dist
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t

    @classmethod
    def of_module(cls, bn):
        """The BnSync of a torch.nn.SyncBatchNorm module's process group, or None where torch's SyncBatchNorm would not
        synchronise either (no initialised process group, or a group of one rank)."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            return None
        s = cls(bn.process_group)
        return s if s.world_size > 1 else None
