"""The SSOD training step with the reference's flow (trainer/ssod_trainer.py:587-680 train_instance,
:458-488 update_optimizer, trainer/trainer.py:193-251 build_optimizer) for `model_type == 'yolov5'`:

  teacher-EMA forward (native wgmma engine) -> NMS + pseudo labels (native, device resident) ->
  student forward on cat(labeled, strong-aug unlabeled) -> ComputeLoss + ComputeStudentMatchLoss (native fused
  fwd/bwd) -> backward -> [NCCL all-reduce of the student gradients] -> SGD-Nesterov -> ema / semi-ema update
  (native fused 5-stream kernel).

Data parallelism (SURVEY.md 8e): one process per GPU, per-rank batch and, by default, per-rank BN statistics exactly like
the reference's DDP without SyncBN; the only collective is one SUM all-reduce of the flattened gradient arena per step
(loss*WORLD_SIZE followed by DDP's mean == sum of per-rank gradients); teachers stay bit-identical on all ranks
because the reduced gradients are.  `sync_bn: True` with WORLD_SIZE > 1 converts the student to SyncBatchNorm like the
reference (trainer/ssod_trainer.py:217-220, trainer/trainer.py:84-87): the eager steps then normalise with the statistics
of the global batch (parallel.BnSync: two small all-reduces per BatchNorm layer); the captured steps refuse it.
"""
import gc
import math

import os
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .domain_loss import DomainLoss, TargetLoss
from .ema import ModelEMA, CosineEMA, SemiSupModelEMA, update_ema_pair, next_pair_decays, ema_scalars
from .loss import ComputeLoss
from .model import Model, SupModel
from .optim import FusedAdamW, FusedSGD
from .parallel import GradArena
from .pl_quality import HIT_KEYS, DeviceMetricMeter, PLQuality
from .pseudo_label import FairPseudoLabel
from .ssod_loss import ComputeStudentMatchLoss


def one_cycle(y1=0.0, y2=1.0, steps=100):  # reference utils/general.py:480-482
    return lambda x: ((1 - math.cos(x * math.pi / steps)) / 2) * (y2 - y1) + y1


# What a captured step is; TrainerStep._graphed / _capture own everything else.  Plain functions of the step:
#   static(step, key, *inputs) -> dict of static input buffers, filled from the inputs of the capturing call
#   stage(step, g, *inputs): copy one call's inputs into those buffers (stream-ordered, no host sync)
#   body(step, g) -> the detached loss: forward + loss + _backward on the static buffers (graph A)
#   ema_update(step, scalars_dev): the EMA update of graph B, decays read from device memory
#   ema_decays(step) -> the decays of this optimizer step for ema_scalars(); advances the update counters like .update()
GraphHooks = namedtuple("GraphHooks", "static stage body ema_update ema_decays")


class TrainerStep:
    """What the SSOD and the supervised step share: optimizer, warm-up / accumulate cadence, gradient arena, all-reduce,
    the eager optimizer + EMA update, and the capture / replay of a step as two CUDA graphs."""

    fixed_accumulate = False     # trainer/trainer.py has no such switch; the SSOD step reads cfg.SSOD.fixed_accumulate

    def __init__(self, cfg, model, device, rank, world_size, epochs, batch_size, amp_dtype, nb, start_epoch):
        self.cfg, self.device = cfg, device
        self.RANK, self.WORLD_SIZE = rank, world_size
        self.epochs = epochs if epochs is not None else cfg.epochs
        self.epoch = 0
        self.batch_size = batch_size if batch_size is not None else cfg.Dataset.batch_size
        self.amp_dtype = amp_dtype
        # the reference converts only when RANK != -1 (a single process ignores sync_bn); before the EMA is made, as there
        self.sync_bn = bool(getattr(cfg, "sync_bn", False)) and world_size > 1
        if self.sync_bn:
            model.sync_batchnorm()
        self.model = model.to(device)
        self.ema = ModelEMA(self.model)          # the reference keeps it on rank 0/-1 only (trainer.py:157); harmless elsewhere
        self.semi_ema = None
        self.build_optimizer(cfg)
        self.compute_loss = ComputeLoss(self.model, cfg)
        self.last_opt_step = -1
        # trainer/trainer.py:372-376: number of warm-up iterations = max(warmup_epochs * nb, 1000), capped at half the run
        self.nb = nb
        if cfg.hyp.warmup_epochs > 0:
            self.nw = max(round(cfg.hyp.warmup_epochs * (nb or 0)), 1000)
            if nb:
                self.nw = min(self.nw, (self.epochs - start_epoch) / 2 * nb)
        else:
            self.nw = -1
        self._arena = None
        self._bn_sync = None
        self.last = {}
        self.meter = DeviceMetricMeter(device)     # trainer/trainer.py:370 (rank 0's MetricMeter; here every rank keeps one)
        self.profile = False     # record CUDA events at the phase boundaries of the eager step
        self.phase_events = []
        self._graph = None       # the step captured as CUDA graphs (see _graphed)
        self.captures = 0        # how many times _graph has been captured (train_instance_graphed / train_step_graphed)

    # trainer/trainer.py:193-247: FusedAdamW for `adam: True`, else FusedSGD, with the LambdaLR schedule
    def build_optimizer(self, cfg):
        nbs = 64
        self.accumulate = max(round(nbs / self.batch_size), 1)
        weight_decay = cfg.hyp.weight_decay * self.batch_size * self.accumulate / nbs
        g_bnw, g_w, g_b = [], [], []
        for v in self.model.modules():
            if hasattr(v, 'bias') and isinstance(v.bias, nn.Parameter):
                g_b.append(v.bias)
            if isinstance(v, nn.modules.batchnorm._BatchNorm):      # nn.SyncBatchNorm too
                g_bnw.append(v.weight)
            elif hasattr(v, 'weight') and isinstance(v.weight, nn.Parameter):
                g_w.append(v.weight)
        if cfg.adam:
            # groups 0 and 2 keep AdamW's default weight_decay (0.01), as torch fills it in for the reference
            self.optimizer = FusedAdamW(g_b, lr=cfg.hyp.lr0, betas=(cfg.hyp.momentum, 0.999))      # one launch, zeroes the grads
        else:
            self.optimizer = FusedSGD(g_b, lr=cfg.hyp.lr0, momentum=cfg.hyp.momentum, nesterov=True)   # one launch, zeroes the grads
        self.optimizer.add_param_group({'params': g_w, 'weight_decay': weight_decay})
        self.optimizer.add_param_group({'params': g_bnw})
        if cfg.linear_lr:
            self.lf = lambda x: (1 - x / (self.epochs - 1)) * (1.0 - cfg.hyp.lrf) + cfg.hyp.lrf
        else:
            self.lf = one_cycle(1, cfg.hyp.lrf, self.epochs)
        self.scheduler = torch.optim.lr_scheduler.LambdaLR(self.optimizer, lr_lambda=self.lf)
        self.scheduler.last_epoch = self.epoch - 1     # trainer.py:247: the first scheduler.step() at an epoch's end gives lf(epoch)
        self.warmup_bias_lr, self.warmup_momentum, self.momentum = cfg.hyp.warmup_bias_lr, cfg.hyp.warmup_momentum, cfg.hyp.momentum

    # ---- gradient arena: all student gradients live in one flat fp32 buffer -> ONE all-reduce per step ----
    def _ensure_arena(self):
        if self._arena is None:
            self._arena = GradArena(self.model.parameters(), self.device, reverse=True)   # backward-completion order
        return self._arena

    # GRAD_REDUCE and WGRAD_SIDE_STREAM are read from SSODTrainerStep by both steps: callers set them there
    # (SSODTrainerStep.GRAD_REDUCE = "avg"), and one assignment has to govern the supervised step as well.
    def _allreduce_grads(self):
        """WORLD_SIZE > 1: one all-reduce of the whole gradient arena"""
        if self.WORLD_SIZE <= 1:
            return
        self._arena.average = (SSODTrainerStep.GRAD_REDUCE == "avg")
        self._arena.all_reduce_sum(self.WORLD_SIZE)

    def _bn_broadcast(self):
        """DDP broadcast_buffers=True: rank 0's BN running statistics overwrite every rank's before each forward"""
        if self.WORLD_SIZE > 1:
            if self._bn_sync is None:
                from .parallel import BnBufferSync
                self._bn_sync = BnBufferSync(self.model)
            self._bn_sync.broadcast(self.WORLD_SIZE)

    # trainer/ssod_trainer.py:458-488 (bf16 autocast needs no GradScaler; loss scale == 1), in parts so that the gradient
    # all-reduce can sit between two captured CUDA graphs when WORLD_SIZE > 1
    def _backward(self, loss):
        self._ensure_arena()
        from . import autograd_conv as ac
        ac.backward(loss, side=SSODTrainerStep.WGRAD_SIDE_STREAM)   # weight-gradient branch on a side stream, joined before returning
        self._mark("backward")

    def _warmup(self, ni):
        """ssod_trainer.py:462-478: accumulate + per-iteration warm-up of lr / momentum (host scalars only; the fused SGD
        kernel reads them from device memory, so this also serves the captured step).  Group 2 -- the BatchNorm weights in
        the reference's group order (trainer.py:215-217) -- is the one that falls from warmup_bias_lr."""
        self.accumulate = 1 if self.fixed_accumulate else max(round(64 / self.batch_size), 1)
        if ni <= self.nw:
            xi = [0, self.nw]
            self.accumulate = max(1, np.interp(ni, xi, [1, 1 if self.fixed_accumulate else 64 / self.batch_size]).round())
            for j, x in enumerate(self.optimizer.param_groups):
                x['lr'] = float(np.interp(ni, xi, [self.warmup_bias_lr if j == 2 else 0.0, x['initial_lr'] * self.lf(self.epoch)]))
                if 'momentum' in x:
                    x['momentum'] = float(np.interp(ni, xi, [self.warmup_momentum, self.momentum]))
        return ni - self.last_opt_step >= self.accumulate

    def _step_and_ema(self):
        self.optimizer.step(zero_grad=True)      # fused SGD-Nesterov; also performs optimizer.zero_grad() on the arena
        if self.semi_ema:
            update_ema_pair(self.ema, self.semi_ema, self.model)   # == ema.update(model); semi_ema.update(ema.ema)
        else:
            self.ema.update(self.model)

    def _optimizer_ema(self, ni):
        # the gradients are reduced only on the iterations that step, like graph B: a SUM all-reduce of an arena that already
        # holds reduced gradients (accumulate > 1) would count them WORLD_SIZE times
        if self._warmup(ni):
            self._allreduce_grads()
            self._mark("allreduce")
            self._step_and_ema()
            self.last_opt_step = ni

    def update_optimizer(self, loss, ni):
        self._backward(loss)
        self._optimizer_ema(ni)

    def _mark(self, name):
        if self.profile:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.phase_events.append((name, ev))

    def phase_times_ms(self):
        """After a synchronize: {phase: total ms} accumulated over the recorded steps."""
        out = {}
        for (n0, e0), (n1, e1) in zip(self.phase_events[:-1], self.phase_events[1:]):
            if n1 != "start":
                out[n1] = out.get(n1, 0.0) + e0.elapsed_time(e1)
        return out

    # ---- end-of-epoch validation (val.run, native: val.py) ----
    def _validate_model(self, model, dataloader, conf_thres, iou_thres, single_cls, names, half, confusion_matrix=None):
        from . import val
        return val.run({'nc': model.nc}, model=model, dataloader=dataloader, conf_thres=conf_thres, iou_thres=iou_thres,
                       single_cls=single_cls, half=half, plots=False, val_ssod=hasattr(model, "det_8"), names=names or {},
                       confusion_matrix=confusion_matrix)

    def validate(self, dataloader, conf_thres=0.001, iou_thres=0.6, single_cls=False, names=None, confusion_matrix=None):
        """trainer/trainer.py:451-464: validates ema.ema -> (results, maps, t).  As the reference's val.run leaves it, the
        EMA's floating state ends up rounded to fp16, here in place: no storage moves, so a captured step replayed afterwards
        still reads and writes the EMA it was captured with.  confusion_matrix: a metrics.ConfusionMatrix the validation adds
        into (val.run)."""
        return self._validate_model(self.ema.ema, dataloader, conf_thres, iou_thres, single_cls, names, half=True,
                                    confusion_matrix=confusion_matrix)

    # the single ModelEMA of the supervised and the burn-in step, as graph B runs it
    def _ema_update_dev(self, scalars_dev):
        self.ema._update_with(self.model, 0.0, scalars_dev=scalars_dev)

    def _ema_decays(self):
        self.ema.updates += 1
        return (self.ema.decay(self.ema.updates),)

    # ---- the labels of a captured step: a static buffer of capacity C and the count in a device int32 -----------------
    LABEL_CAPACITY = 64      # initial label capacity of a captured SSOD / supervised step; doubles when a batch has more labels

    # The same scheme holds the SSOD step's unlabeled ground truth: buffer "ugt", count "nug", capacity "gcap".
    def _label_capacity(self, slot, targets, initial, cap="cap"):
        """The label capacity of the graph in `slot` (`initial` before the first capture), doubled until the batch's
        labels fit.  It goes into the capture key, so only a batch with more labels than the capacity re-captures."""
        c = initial if getattr(self, slot) is None else getattr(self, slot).get(cap, initial)
        while c < targets.shape[0]:
            c *= 2
        return c

    def _static_labels(self, g, cap, targets, buf="targets", count="nt", cap_key="cap"):
        """g["targets"] [cap, 6] fp32 and g["nt"] int32[1], filled from the capturing call.  The loss (ComputeLoss(...,
        n_dev)) and LabelMatch's histogram read only the first nt rows, so one graph serves every label count <= cap."""
        nt = int(targets.shape[0])
        g.update({cap_key: cap, buf: torch.zeros((cap, 6), dtype=torch.float32, device=self.device),
                  count: torch.full((1,), nt, dtype=torch.int32, device=self.device)})
        g[buf][:nt].copy_(targets)

    def _stage_labels(self, g, targets, buf="targets", count="nt"):
        """one call's labels (CPU or CUDA) into the static buffers, stream-ordered, without a host sync"""
        nt = int(targets.shape[0])
        g[buf][:nt].copy_(targets, non_blocking=True)
        # pageable source: the runtime stages these few bytes before returning, so the next step cannot overwrite them early
        g[count].copy_(torch.tensor([nt], dtype=torch.int32))

    def _log(self, loss, items):
        """trainer.py:434 / ssod_trainer.py:447,524: the meter takes ComputeLoss's box obj cls loss; self.last the detached
        loss and items"""
        self.meter.update(items)
        self.last = dict(loss=loss.detach(), sup={k: v.detach() for k, v in items.items()})

    def reset_meter(self):
        """trainer/trainer.py:370 (before_epoch: a new MetricMeter): the meter's sums and counts start again from zero, in
        place, so the captured steps keep updating it without a re-capture"""
        self.meter.reset()

    # ---- the whole step as CUDA graphs ------------------------------------------------------------------------------
    def _graphed(self, slot, key, hooks, inputs, ni):
        """The step described by `hooks` (GraphHooks), captured once per `key` and replayed as two graphs: A = forward ...
        backward (gradients accumulate in the arena), B = SGD-Nesterov + the EMA update(s).  B is replayed on the
        iterations the reference's cadence steps the optimizer (ssod_trainer.py:462-488: `accumulate`, warm-up); for
        WORLD_SIZE > 1 the NCCL all-reduce sits between A and B.  The ~1.5k kernel launches + the autograd traversal
        collapse into two cudaGraphLaunch calls.  Inputs are copied into static buffers; learning rate / momentum (warm-up,
        scheduler) and the EMA decays of the step are host scalars written to device memory before the replay, so the
        schedule needs no re-capture.  The graphs and their buffers live in the attribute `slot`; a new key re-captures."""
        if getattr(self, slot) is None or getattr(self, slot)["key"] != key:
            self._check_capturable()
            setattr(self, slot, None)            # release the old graphs and their memory pool before capturing new ones
            setattr(self, slot, self._capture(key, hooks, inputs, ni))
        g = getattr(self, slot)
        hooks.stage(self, g, *inputs)
        # everything the host contributes to this iteration is enqueued BEFORE graph A, so that A, the all-reduce and B follow
        # each other on the stream without a host gap: accumulate / lr / momentum of iteration ni (host scalars), and -- when
        # the optimizer is due -- the EMA decays and the SGD hyper-parameters (stream-ordered copies: the previous replay of B
        # has consumed the old values by the time they land)
        due = self._warmup(ni)
        if due:
            # pageable source: the runtime stages the 16 bytes before returning, so the next step cannot overwrite them early
            g["ema_dev"].copy_(torch.tensor(ema_scalars(*hooks.ema_decays(self)), dtype=torch.float32))
            # lr / momentum of this step -> device memory read by the captured SGD kernel (AdamW: the step count advances
            # here, and this step's bias corrections go with the lr)
            self.optimizer.refresh_hyper()
        self._bn_broadcast()
        g["graph"].replay()
        self.last = g["last"]                # this iteration's loss items: the graph's static outputs, valid until the next replay
        if due:
            self._allreduce_grads()          # one all-reduce per optimizer step, between the two graphs (enqueued, no host sync)
            g["graph_b"].replay()
            self.last_opt_step = ni
        return g["loss"]

    def _check_capturable(self):
        if self.WORLD_SIZE > 1 and any(isinstance(m, nn.SyncBatchNorm) for m in self.model.modules()):
            raise NotImplementedError(
                "SyncBatchNorm (sync_bn) with WORLD_SIZE > 1 runs in the eager steps only (train_instance, "
                "train_without_unlabeled[_da], train_step): its per-layer all-reduces would have to be captured inside graph A, "
                "and collectives inside a CUDA graph risk the NCCL teardown hazard documented in DESIGN.md section 8")

    def _capture(self, key, hooks, inputs, ni):
        dev = self.device
        g = hooks.static(self, key, *inputs)
        g.update(key=key, ema_dev=torch.zeros(4, dtype=torch.float32, device=dev))
        was_profile, self.profile = self.profile, False
        self.last = {}
        restore = self._snapshot_training_state()
        # warm-up on a side stream (allocator + lazily-created state: momentum buffers, chunk tables, workspaces, TMA/func attrs)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
                hooks.body(self, g)
                self._allreduce_grads()
                self._warmup(ni)
                self._step_and_ema()          # the optimizer + EMA branch is exercised (and later captured) unconditionally
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        # No cyclic garbage collection while the stream captures: a step that only the collector frees (an SSOD step is in
        # a reference cycle through its `lf` closure) would destroy its CUDA graphs in the middle of this capture, and
        # destroying a graph is not permitted while a stream captures: it invalidates the capture.  Dead steps go now.
        gc.collect()
        gc_enabled = gc.isenabled()
        gc.disable()
        try:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                g["loss"] = hooks.body(self, g)
            g["graph"], g["last"] = graph, self.last
            gb = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gb, pool=graph.pool()):
                self.optimizer.step(zero_grad=True)
                hooks.ema_update(self, g["ema_dev"])
            g["graph_b"] = gb
        finally:
            if gc_enabled:
                gc.enable()
        restore()
        self.profile = was_profile
        return g

    def _snapshot_training_state(self):
        """The warm-up steps before a capture really train: snapshot every piece of state they touch (weights, BN
        statistics, the EMA model(s), the optimizer state -- SGD momentum, or AdamW's moments and step count --, the
        gradients accumulated towards the next optimizer step, the training meter, the autobalance state of the supervised
        loss, the counters, lr / momentum) and return
        the function that puts it back."""
        self._ensure_arena()
        emas = [e for e in (self.ema, self.semi_ema) if e is not None]
        tensors = [t for m in [self.model] + [e.ema for e in emas] for t in m.state_dict().values()]
        # the optimizer's moments (built here if no step has run yet: zero then, which both optimizers treat as fresh)
        tensors += self.optimizer.flat_state()
        tensors.append(self._arena.flat)     # gradients already accumulated towards the next optimizer step (accumulate > 1)
        tensors.append(self.meter.state)
        if self.compute_loss.balance_state is not None:
            tensors.append(self.compute_loss.balance_state)     # autobalance: every loss call advances it
        snap = [t.clone() for t in tensors]
        saved = (self.last_opt_step, [e.updates for e in emas], self.accumulate,
                 [(x['lr'], x.get('momentum')) for x in self.optimizer.param_groups])
        step_count = getattr(self.optimizer, "step_count", None)     # FusedAdamW's t of the bias corrections

        def restore():
            with torch.no_grad():
                for t, c in zip(tensors, snap):
                    t.copy_(c)
            if step_count is not None:
                self.optimizer.step_count = step_count
            self.last_opt_step, updates, self.accumulate, hyp = saved
            for e, u in zip(emas, updates):
                e.updates = u
            for x, (lr, mom) in zip(self.optimizer.param_groups, hyp):
                x['lr'] = lr
                if mom is not None:
                    x['momentum'] = mom
        return restore


class SSODTrainerStep(TrainerStep):
    def __init__(self, cfg, device, rank=-1, world_size=1, epochs=None, batch_size=None, amp_dtype=torch.bfloat16,
                 pseudo_label_stats=None, nb=None, start_epoch=0, model=None):
        """pseudo_label_stats (LabelMatch only): dict(target_data_len, label_num_per_image, cls_ratio_gt) that the reference
        derives from its datasets (ssod_trainer.py:71).  nb = batches per epoch (len(train_loader)); it only sizes the
        warm-up window exactly like trainer/trainer.py:372-376 (nb=None: the 1000-iteration floor).  model: a Model(cfg)
        built by the caller (e.g. already through convert_sync_batchnorm, the reference's order); None builds one."""
        super().__init__(cfg, Model(cfg) if model is None else model, device, rank, world_size, epochs, batch_size, amp_dtype, nb,
                         start_epoch)
        self.model_type = self.model.model_type
        if cfg.hyp.burn_epochs > 0:
            self.semi_ema = None
        elif cfg.SSOD.cosine_ema:
            self.semi_ema = CosineEMA(self.ema.ema, decay_start=cfg.SSOD.ema_rate, total_epoch=self.epochs)
        else:
            self.semi_ema = SemiSupModelEMA(self.ema.ema, cfg.SSOD.ema_rate)
        self.fixed_accumulate = cfg.SSOD.fixed_accumulate
        self.compute_un_sup_loss = ComputeStudentMatchLoss(self.model, cfg)
        self.domain_loss, self.target_loss = DomainLoss(), TargetLoss()       # ssod_trainer.py:262-263
        if getattr(cfg.SSOD, "pseudo_label_type", "FairPseudoLabel") == "LabelMatch":      # ssod_trainer.py:69-71
            from .labelmatch import LabelMatch
            ps = pseudo_label_stats or {}
            nc = cfg.Dataset.nc
            self.pseudo_label_creator = LabelMatch(cfg, int(ps.get("target_data_len", 0) / max(world_size, 1)), ps.get("label_num_per_image", 7.0),
                                                   ps.get("cls_ratio_gt", np.full(nc, 1.0 / nc)))
        else:
            self.pseudo_label_creator = FairPseudoLabel(cfg)
        self.da_loss_weights = cfg.SSOD.da_loss_weights
        self._teacher_stream = None
        self._teacher_keep = None
        self._burn_graph = None     # captured burn-in step (train_without_unlabeled[_da]_graphed)
        self.burn_in_captures = 0   # how many times a burn-in step has been captured
        self._plq = PLQuality(device)   # the pseudo-label statistics of the step (iouv = [0.5], ssod_trainer.py:662)

    # trainer/ssod_trainer.py:86-94: SSOD.multi_step_lr replaces the LambdaLR by MultiStepLR(milestones, gamma=0.1) on top
    # of it (the warm-up still interpolates towards initial_lr * lf(epoch)); the supervised step has no such switch
    def build_optimizer(self, cfg):
        super().build_optimizer(cfg)
        if cfg.SSOD.multi_step_lr:
            self.scheduler = torch.optim.lr_scheduler.MultiStepLR(self.optimizer, milestones=cfg.SSOD.milestones, gamma=0.1)
            self.scheduler.last_epoch = self.epoch - 1

    # "sum" = the reference (loss * WORLD_SIZE, then DDP's mean: trainer/ssod_trainer.py:638-648).  "avg" (ncclAvg: the same
    # collective at the same cost) is for synthetic benchmarks only: with SUM the effective learning rate grows with the world
    # size, and a random-init model's BatchNorm scales then drift WORLD_SIZE x faster (bench.py's self-check explains why that
    # matters); set before the first step.  Governs the supervised step too.
    GRAD_REDUCE = os.environ.get("ETB_GRAD_REDUCE", "sum")
    WGRAD_SIDE_STREAM = os.environ.get("ETB_WGRAD_SIDE", "1") == "1"   # ETB_WGRAD_SIDE=0 disables; governs the supervised step too
    TEACHER_SIDE_STREAM = os.environ.get("ETB_TEACHER_SIDE", "1") == "1"   # teacher forward + NMS concurrent with the student forward

    def split_predict_and_feature(self, total_pred, total_feature, n_img):
        """ssod_trainer.py:568-585.  split_batch == t[:n], t[n:] whose backward is a no-op (the loss kernels write both
        gradients into one buffer) instead of autograd's zeros + copy + add per slice."""
        from .autograd_conv import split_batch
        fs = [split_batch(f, n_img) for f in total_feature]
        ps = [split_batch(p, n_img) for p in total_pred]
        return [a for a, _ in ps], [a for a, _ in fs], [b for _, b in ps], [b for _, b in fs]

    @property
    def with_gt(self):
        """SSOD.ssod_hyp.with_gt (configs/defaults.py:303, default False): score the pseudo labels against the unlabeled
        images' ground truth (check_pseudo_label_with_gt) rather than by their reliable / uncertain split (check_pseudo_label)"""
        return bool(getattr(getattr(self.cfg.SSOD, 'ssod_hyp', None), 'with_gt', False))

    def _hit_rate(self, rows, n_dev, gt, m_dev):
        """ssod_trainer.py:661-671: tp fp_cls fp_loc pse_num gt_num of this step's pseudo labels as device scalars (views of
        the etb_pl_quality output), with the thresholds the unsupervised loss selects by, and batch_size // WORLD_SIZE"""
        hi, lo = self.compute_un_sup_loss._thresholds(self.device)
        vals = self._plq.run(rows.contiguous(), n_dev, hi, lo, gt if self.with_gt else None, m_dev,
                             self.batch_size // self.WORLD_SIZE, self.with_gt)
        return {k: vals[i, 0] for i, k in enumerate(HIT_KEYS)}

    # trainer/ssod_trainer.py:587-680; the meter update of :653-672 on the device
    def train_instance(self, imgs, targets, unlabeled_imgs, unlabeled_imgs_ori, unlabeled_gt, unlabeled_M, ni,
                       host_pseudo_labels=False, _stop_after_backward=False, _n_dev=None, _m_dev=None):
        """unlabeled_gt [M,6] (img, cls, x, y, w, h normalised; None: no boxes) feeds the pseudo-label statistics when
        with_gt.  _stop_after_backward: the body of the captured graph A (TrainerStep._graphed), which ends after the backward
        and leaves LabelMatch's image counters to the replay wrapper.  _n_dev (int32[1] CUDA): targets is a padded label
        buffer whose first _n_dev rows are the labels (ComputeLoss(..., n_dev), LabelMatch.update_device(..., n_dev));
        _m_dev likewise for unlabeled_gt."""
        self._require_semi_ema()
        n_img = imgs.shape[0]
        self._mark("start")
        if self.WORLD_SIZE > 1 and not torch.cuda.is_current_stream_capturing():
            self._bn_broadcast()         # (captured steps: _graphed issues it before the replay)
        # The teacher forward + NMS + pseudo-label transform feed nothing but the unsupervised loss, and the student forward
        # does not depend on them: with the device-resident pseudo labels they run on a side stream, concurrently with the
        # student forward (the teacher's batch-16 kernels leave SMs idle on the deep, small maps; the student's fill them),
        # and are joined right before ComputeStudentMatchLoss.  Inside a captured graph the fork/join become parallel branches.
        overlap = self.TEACHER_SIDE_STREAM and not host_pseudo_labels and not self.profile
        main = torch.cuda.current_stream(self.device)
        if overlap:
            if self._teacher_stream is None:
                self._teacher_stream = torch.cuda.Stream(self.device)
            fork = torch.cuda.Event()
            fork.record(main)
            self._teacher_stream.wait_event(fork)
        with torch.cuda.stream(self._teacher_stream if overlap else main):
            with torch.no_grad():
                (teacher_pred, train_out), teacher_feature = self.ema.ema(unlabeled_imgs_ori, augment=False)
            self._mark("teacher_forward")
            if hasattr(self.pseudo_label_creator, "update_device"):      # LabelMatch: ssod_trainer.py:616-617 (labeled-target histogram)
                self.pseudo_label_creator.update_device(targets, _n_dev)
                if not _stop_after_backward:
                    self._count_labelmatch_images(imgs, unlabeled_imgs)
            if host_pseudo_labels:   # the reference's return contract: CPU float64 rows + flag (one D2H sync)
                unlabeled_targets, invalid_target_shape = self.pseudo_label_creator.create_pseudo_label_online_with_gt(
                    teacher_pred, unlabeled_imgs, unlabeled_M, unlabeled_imgs_ori, unlabeled_gt, self.RANK)
                n_dev = None
                if not invalid_target_shape:
                    unlabeled_targets = unlabeled_targets.to(self.device)
            else:                    # device-resident twin: no host sync between teacher and student
                h, w = unlabeled_imgs.shape[2:]
                unlabeled_targets, n_dev = self.pseudo_label_creator.create_pseudo_label_device(teacher_pred, unlabeled_M, h, w)
                invalid_target_shape = False
            self._mark("nms_pseudo_label")
            if overlap:
                join = torch.cuda.Event()
                join.record(self._teacher_stream)
                self._teacher_keep = (teacher_pred, train_out, teacher_feature)    # alive until the join below
        with torch.autocast("cuda", dtype=self.amp_dtype):
            # == self.model(torch.cat([imgs, unlabeled_imgs], 0)) (ssod_trainer.py:620-622): the native stem reads both
            # batches in place (uint8 from the loaders or fp32), so the concatenated fp32 image never exists
            total_pred, total_feature = self.model([imgs, unlabeled_imgs])
        self._mark("student_forward")
        sup_pred, sup_feature, un_sup_pred, un_sup_feature = self.split_predict_and_feature(total_pred, total_feature, n_img)
        sup_loss, sup_loss_items = self.compute_loss(sup_pred, targets, _n_dev)
        d_loss = self.domain_loss(sup_feature)
        t_loss = self.target_loss(un_sup_feature)
        if self.cfg.SSOD.with_da_loss:
            sup_loss = sup_loss + d_loss * self.da_loss_weights + t_loss * self.da_loss_weights
        else:
            sup_loss = sup_loss + d_loss * 0 + t_loss * 0
        if overlap:
            main.wait_event(join)        # pseudo labels ready
            self._teacher_keep = None
        if invalid_target_shape:
            un_sup_loss = torch.zeros(1, device=self.device)
            un_sup_loss_items = dict(ss_box=0, ss_obj=0, ss_cls=0)
            hit_rate = dict(tp=0, fp_cls=0, fp_loc=0, pse_num=0, gt_num=0)     # no pseudo label created (:658-660)
        else:
            un_sup_loss, un_sup_loss_items = self.compute_un_sup_loss(un_sup_pred, unlabeled_targets, n_dev)
            if self.with_gt and unlabeled_gt is not None and _m_dev is None:
                unlabeled_gt = unlabeled_gt.to(self.device, torch.float32).reshape(-1, 6).contiguous()
            hit_rate = self._hit_rate(unlabeled_targets, n_dev, unlabeled_gt, _m_dev)
        # DDP: loss*WORLD_SIZE then gradient mean == plain SUM all-reduce of per-rank gradients (no scaling here)
        loss = sup_loss + un_sup_loss * self.cfg.SSOD.teacher_loss_weight
        self._mark("losses")
        # box obj cls loss ss_box ss_obj ss_cls tp fp_cls fp_loc pse_num gt_num, the reference's key order (:653-672)
        self.meter.update({**sup_loss_items, **un_sup_loss_items, **hit_rate})
        # logging values only -- detached, so that no reference to this step's autograd graph (and to the AccumulateGrad
        # nodes of the parameters, which are tied to the stream they were created on) survives the step
        det = lambda d: {k: (v.detach() if torch.is_tensor(v) else v) for k, v in d.items()}  # noqa: E731
        self.last = dict(loss=loss.detach(), sup=det(sup_loss_items), unsup=det(un_sup_loss_items), hits=hit_rate)
        if _stop_after_backward:         # captured graph A ends here
            self._backward(loss)
            return loss.detach()
        self.update_optimizer(loss, ni)
        self._mark("optimizer_ema")
        return loss.detach()

    # ---- the whole step as CUDA graphs ------------------------------------------------------------------------------
    def _ssod_static(self, key, imgs, targets, us, uw, Ms, ugt):
        g = dict(imgs=imgs.clone(), us=us.clone(), uw=uw.clone(), Ms=Ms.to(self.device, torch.float64).clone(), ugt=None, nug=None)
        self._static_labels(g, key[-2], targets)
        if ugt is not None:          # with_gt: the unlabeled ground truth, capacity key[-1]
            self._static_labels(g, key[-1], ugt, "ugt", "nug", "gcap")
        self.captures += 1
        return g

    def _ssod_stage(self, g, imgs, targets, us, uw, Ms, ugt):
        g["imgs"].copy_(imgs, non_blocking=True)
        self._stage_labels(g, targets)
        if ugt is not None:
            self._stage_labels(g, ugt, "ugt", "nug")
        g["us"].copy_(us, non_blocking=True)
        g["uw"].copy_(uw, non_blocking=True)
        g["Ms"].copy_(Ms, non_blocking=True)

    def _ssod_body(self, g):
        return self.train_instance(g["imgs"], g["targets"], g["us"], g["uw"], g["ugt"], g["Ms"], None, _stop_after_backward=True,
                                   _n_dev=g["nt"], _m_dev=g["nug"])

    _SSOD_GRAPH = GraphHooks(_ssod_static, _ssod_stage, _ssod_body,
                             lambda self, scalars_dev: update_ema_pair(self.ema, self.semi_ema, self.model, scalars_dev=scalars_dev),
                             lambda self: next_pair_decays(self.ema, self.semi_ema))

    def train_instance_graphed(self, imgs, targets, unlabeled_imgs, unlabeled_imgs_ori, unlabeled_gt, unlabeled_M, ni):
        """train_instance captured once per image shape (device-resident pseudo labels, no host sync anywhere in the step)
        and replayed as two graphs (TrainerStep._graphed): A = teacher forward ... backward, B = SGD-Nesterov + both EMA
        updates.  The labels go into a static buffer of capacity C with their count on the device (_static_labels), so
        any label count up to C replays the same graph; a batch with more re-captures once, with C doubled until it fits.
        With with_gt, unlabeled_gt (None: no boxes) goes into a static buffer the same way, with its own capacity."""
        self._require_semi_ema()
        cap = self._label_capacity("_graph", targets, self.LABEL_CAPACITY)
        ugt = None
        if self.with_gt:
            ugt = torch.zeros((0, 6)) if unlabeled_gt is None else unlabeled_gt.reshape(-1, 6)
        gcap = 0 if ugt is None else self._label_capacity("_graph", ugt, self.LABEL_CAPACITY, "gcap")
        key = (tuple(imgs.shape), tuple(unlabeled_imgs.shape), tuple(unlabeled_M.shape),
               imgs.dtype, unlabeled_imgs.dtype, unlabeled_imgs_ori.dtype, cap, gcap)   # uint8 loader batches vs fp32: different static buffers
        loss = self._graphed("_graph", key, self._SSOD_GRAPH, (imgs, targets, unlabeled_imgs, unlabeled_imgs_ori, unlabeled_M, ugt), ni)
        if hasattr(self.pseudo_label_creator, "stage_detections"):   # LabelMatch: the captured body neither stages nor counts
            self.pseudo_label_creator.stage_detections()
            self._count_labelmatch_images(imgs, unlabeled_imgs)
        return loss

    def _count_labelmatch_images(self, imgs, unlabeled_imgs):
        """LabelMatch.update's image counters (labelmatch.py:126-129): host integers, advanced once per step"""
        self.pseudo_label_creator.count += imgs.shape[0]
        self.pseudo_label_creator.pse_count += unlabeled_imgs.shape[0]

    def _snapshot_training_state(self):
        """+ LabelMatch's state that the SSOD warm-up steps before a capture touch: the device class histogram, the staged
        detections and the image counters"""
        restore = super()._snapshot_training_state()
        c = self.pseudo_label_creator
        if not hasattr(c, "class_hist"):
            return restore
        saved = (c.count, c.pse_count, list(c._pending))
        hist = c.class_hist(self.device)
        hist_snap = hist.clone()

        def restore_labelmatch():
            restore()
            c.count, c.pse_count, c._pending = saved
            hist.copy_(hist_snap)
        return restore_labelmatch

    def after_epoch(self, epoch, start_epoch=0):
        """ssod_trainer.py:319-323: LabelMatch re-estimates the per-class thresholds once per epoch; the unsupervised loss
        picks them up (and a captured step has to be re-captured because the thresholds are device constants of the graph)."""
        c = self.pseudo_label_creator
        if hasattr(c, "update_epoch_cls_thr") and epoch >= getattr(self.cfg.SSOD, "dynamic_thres_epoch", 0):
            c.update_epoch_cls_thr(epoch - start_epoch)
            self.compute_un_sup_loss.ignore_thres_high = list(c.cls_thr_high)
            self.compute_un_sup_loss.ignore_thres_low = list(c.cls_thr_low)
            self.reset_graph()

    def reset_graph(self):
        self._graph = None

    def validate(self, dataloader, conf_thres=0.001, iou_thres=0.6, single_cls=False, names=None, confusion_matrix=None):
        """ssod_trainer.py:335-383: the student, then the teacher of the current phase (semi_ema.ema after the hand-over,
        ema.ema during burn-in) -> (results, maps, t, cls_thr) of the teacher and the student's results.  The reference
        validates a deepcopy of the student only to spare it the fp16 rounding; here the student is validated in place
        without rounding (same numbers) and put back in training mode.  The teacher is rounded in place (TrainerStep.validate).
        confusion_matrix: a metrics.ConfusionMatrix the teacher's validation adds into."""
        training = self.model.training
        try:
            student = self._validate_model(self.model, dataloader, conf_thres, iou_thres, single_cls, names, half=False)
        finally:
            self.model.train(training)
        teacher = self.semi_ema.ema if self.semi_ema is not None else self.ema.ema
        results, maps, t, cls_thr = self._validate_model(teacher, dataloader, conf_thres, iou_thres, single_cls, names, half=True,
                                                         confusion_matrix=confusion_matrix)
        return results, maps, t, cls_thr, student[0]

    # ---- burn-in: trainer/ssod_trainer.py:295-317 (train_in_epoch), :421-456 / :490-533 -----------------------------
    @property
    def in_burn_in(self):
        """True while epoch < hyp.burn_epochs: the step is train_without_unlabeled[_da] (labeled data only, or + the weak
        unlabeled images with the domain losses), with ONE ModelEMA and no semi_ema."""
        return self.epoch < self.cfg.hyp.burn_epochs

    def _require_semi_ema(self):
        if self.semi_ema is None:
            raise RuntimeError("the semi-supervised step needs semi_ema, which begin_epoch(epoch) creates at epoch == "
                               "hyp.burn_epochs (%d); current epoch %d%s" % (
                                   self.cfg.hyp.burn_epochs, self.epoch,
                                   ": still in burn-in, use train_without_unlabeled[_da]" if self.in_burn_in else
                                   " is past it (a run resumed after burn-in never gets a semi_ema, as in the reference)"))

    def begin_epoch(self, epoch):
        """The trainer's side of ssod_trainer.py:295-317: sets the epoch; at epoch == burn_epochs (> 0) the semi-supervised
        EMA is created from the burn-in EMA and the burn-in graphs are dropped, so train_instance[_graphed] runs from here on.
        The reference's loop that 'copies the EMA into the student' (:306-309) only assigns into a temporary state_dict()
        dict, so it changes nothing: the student is deliberately NOT reset to the EMA here either."""
        self.epoch = epoch
        burn = self.cfg.hyp.burn_epochs
        if burn > 0 and epoch == burn:
            if self.cfg.SSOD.cosine_ema:
                self.semi_ema = CosineEMA(self.ema.ema, decay_start=self.cfg.SSOD.ema_rate, total_epoch=self.epochs - burn)
            else:
                self.semi_ema = SemiSupModelEMA(self.ema.ema, self.cfg.SSOD.ema_rate)
            self._burn_graph = None

    def _burn_in_loss(self, imgs, targets, unlabeled_imgs_ori=None, n_dev=None):
        """Forward + loss of the burn-in step (the reference computes it under autocast; the fused loss kernels read fp32).
        unlabeled_imgs_ori=None: train_without_unlabeled (:427-443), else train_without_unlabeled_da (:498-520)."""
        if self.WORLD_SIZE > 1 and not torch.cuda.is_current_stream_capturing():
            self._bn_broadcast()         # (captured steps: _graphed issues it before the replay)
        with torch.autocast("cuda", dtype=self.amp_dtype):
            # the native stem reads uint8 or fp32 batches in place; with two batches the cat is never materialised
            pred, feats = self.model(imgs if unlabeled_imgs_ori is None else [imgs, unlabeled_imgs_ori])
        if unlabeled_imgs_ori is None:
            loss, items = self.compute_loss(pred, targets, n_dev)
            # netD stays in the graph with zero gradients, so SGD still applies weight decay + momentum to its weights
            loss = loss + 0 * (feats[0].mean() + feats[1].mean() + feats[2].mean())
        else:
            sup_pred, sup_feature, un_sup_pred, un_sup_feature = self.split_predict_and_feature(pred, feats, imgs.shape[0])
            loss, items = self.compute_loss(sup_pred, targets, n_dev)
            w = self.da_loss_weights
            from .autograd_conv import ZeroTermFn
            # + 0 * un_sup_pred[i].mean(): the unlabeled half of the Detect gradient is zero-filled in place
            loss = loss + self.domain_loss(sup_feature) * w + self.target_loss(un_sup_feature) * w + ZeroTermFn.apply(*un_sup_pred)
        return loss, items

    def _burn_in_step(self, imgs, targets, unlabeled_imgs_ori, ni):
        loss, items = self._burn_in_loss(imgs, targets, unlabeled_imgs_ori)
        self._log(loss, items)
        self.update_optimizer(loss, ni)
        return loss.detach()

    def train_without_unlabeled(self, imgs, targets, ni):
        """ssod_trainer.py:421-456, one iteration: labeled images only; backward, warm-up / accumulate, SGD, ema.update"""
        return self._burn_in_step(imgs, targets, None, ni)

    def train_without_unlabeled_da(self, imgs, targets, unlabeled_imgs_ori, ni):
        """ssod_trainer.py:490-533, one iteration: labeled + weak unlabeled images, detection loss on the labeled half plus
        the domain losses (SSOD.da_loss_weights) of both halves"""
        return self._burn_in_step(imgs, targets, unlabeled_imgs_ori, ni)

    def train_without_unlabeled_graphed(self, imgs, targets, ni):
        """train_without_unlabeled replayed from captured CUDA graphs; see _burn_in_graphed"""
        return self._burn_in_graphed(imgs, targets, None, ni)

    def train_without_unlabeled_da_graphed(self, imgs, targets, unlabeled_imgs_ori, ni):
        """train_without_unlabeled_da replayed from captured CUDA graphs; see _burn_in_graphed"""
        return self._burn_in_graphed(imgs, targets, unlabeled_imgs_ori, ni)

    BURN_IN_LABEL_CAPACITY = 64       # initial label capacity of a burn-in graph; doubles when a batch has more labels

    def _burn_in_graphed(self, imgs, targets, uw, ni):
        """The burn-in step as two graphs (TrainerStep._graphed): A = forward + loss + backward, [all-reduce], B =
        SGD-Nesterov + the single EMA update with its decay read from device memory.  The labels are copied into a static
        buffer of capacity C and their count into a device int32 (stream-ordered, no host sync) that the assigner reads,
        so one capture serves every batch of a given image shape and dtype whatever its label count; a batch with more
        than C labels re-captures with C doubled until it fits."""
        if self.semi_ema is not None:
            raise RuntimeError("burn-in step requested after the hand-over to the semi-supervised phase (semi_ema exists)")
        cap = self._label_capacity("_burn_graph", targets, self.BURN_IN_LABEL_CAPACITY)
        key = (tuple(imgs.shape), imgs.dtype, None if uw is None else (tuple(uw.shape), uw.dtype), cap)
        return self._graphed("_burn_graph", key, self._BURN_IN_GRAPH, (imgs, targets, uw), ni)

    def _burn_in_static(self, key, imgs, targets, uw):
        g = dict(imgs=imgs.clone(), uw=None if uw is None else uw.clone())
        self._static_labels(g, key[-1], targets)
        self.burn_in_captures += 1
        return g

    def _burn_in_stage(self, g, imgs, targets, uw):
        g["imgs"].copy_(imgs, non_blocking=True)
        if uw is not None:
            g["uw"].copy_(uw, non_blocking=True)
        self._stage_labels(g, targets)

    def _burn_in_forward_backward(self, g):
        # returns the loss detached: nothing may keep this step's autograd graph alive, because the AccumulateGrad nodes of
        # the parameters it holds are tied to the stream they were created on (the warm-up's side stream, the capture's)
        loss, items = self._burn_in_loss(g["imgs"], g["targets"], g["uw"], g["nt"])
        self._log(loss, items)
        self._backward(loss)
        return loss.detach()

    _BURN_IN_GRAPH = GraphHooks(_burn_in_static, _burn_in_stage, _burn_in_forward_backward,
                                TrainerStep._ema_update_dev, TrainerStep._ema_decays)


class SupTrainerStep(TrainerStep):
    """The supervised step (trainer/trainer.py:406-443 train_in_epoch body + :381-404 update_optimizer), BASELINE configs
    #1/#2: student forward -> ComputeLoss -> backward -> [all-reduce] -> SGD-Nesterov -> ModelEMA.update, same native
    kernels as the SSOD step minus the teacher / pseudo-label path.  The optimizer cadence is the reference's:
    accumulate = max(round(64 / batch_size), 1) iterations per optimizer step (gradients add up in the arena in between)
    and the per-iteration warm-up of lr / momentum / accumulate while ni <= nw (trainer.py:372-376, 385-395)."""

    def __init__(self, cfg, device, rank=-1, world_size=1, epochs=None, batch_size=None, amp_dtype=torch.bfloat16, nb=None,
                 start_epoch=0, model=None):
        """model: a SupModel(cfg) built by the caller (see SSODTrainerStep); None builds one."""
        super().__init__(cfg, SupModel(cfg) if model is None else model, device, rank, world_size, epochs, batch_size, amp_dtype,
                         nb, start_epoch)

    def _loss(self, imgs, targets, n_dev=None):
        if self.WORLD_SIZE > 1 and not torch.cuda.is_current_stream_capturing():
            self._bn_broadcast()      # DDP broadcast_buffers=True (captured steps: _graphed issues it before the replay)
        with torch.autocast("cuda", dtype=self.amp_dtype):
            pred = self.model(imgs)
        loss, items = self.compute_loss(pred, targets, n_dev)
        self._log(loss, items)
        return loss

    def train_step(self, imgs, targets, ni):
        loss = self._loss(imgs, targets)
        self.update_optimizer(loss, ni)
        return loss.detach()

    def _static(self, key, imgs, targets):
        g = dict(imgs=imgs.clone())
        self._static_labels(g, key[-1], targets)
        self.captures += 1
        return g

    def _stage(self, g, imgs, targets):
        g["imgs"].copy_(imgs, non_blocking=True)
        self._stage_labels(g, targets)

    def _forward_backward(self, g):
        loss = self._loss(g["imgs"], g["targets"], g["nt"])
        self._backward(loss)
        return loss.detach()

    _GRAPH = GraphHooks(_static, _stage, _forward_backward, TrainerStep._ema_update_dev, TrainerStep._ema_decays)

    def train_step_graphed(self, imgs, targets, ni):
        """train_step replayed from two captured CUDA graphs (TrainerStep._graphed), captured once per image shape and
        dtype: A = forward + loss + backward, B = SGD-Nesterov + the ModelEMA update with its decay read from device
        memory.  The labels go into a static buffer of capacity C with their count on the device (_static_labels); a
        batch with more than C labels re-captures once, with C doubled until it fits."""
        cap = self._label_capacity("_graph", targets, self.LABEL_CAPACITY)
        key = (tuple(imgs.shape), imgs.dtype, cap)
        return self._graphed("_graph", key, self._GRAPH, (imgs, targets), ni)


class DevicePrefetcher:
    """Double-buffered host -> device staging of a batch on a side stream, so the H2D copy of step i+1 overlaps the kernels
    of step i (the reference's loop copies on the compute stream: `imgs.to(device, non_blocking=True)`,
    trainer/ssod_trainer.py:694-696).  put(batch of pinned host tensors) enqueues the copies into the next slot;
    get() makes the current stream wait for the oldest slot and returns its device tensors.  A slot is reused two put()s
    later, i.e. after the step that consumed it has been enqueued on the compute stream -- put() makes the copy stream wait
    for that point before overwriting.  A tensor whose first dimension changes between batches (the labels: a different
    count almost every batch) gets a slot buffer that grows by doubling, and get() returns a view of the batch's length."""

    def __init__(self, device, slots=2):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(self.device)
        self.slots = [dict(buf={}, view={}, ready=torch.cuda.Event(), free=None) for _ in range(slots)]
        self.head = self.tail = 0          # next slot to fill / next slot to hand out
        self.pending = 0

    def put(self, batch):
        assert self.pending < len(self.slots), "prefetcher full: call get() first"
        sl = self.slots[self.head]
        if sl["free"] is not None:
            self.stream.wait_event(sl["free"])          # the consumer of this slot's previous contents has been enqueued and finished
        with torch.cuda.stream(self.stream):
            for k, v in batch.items():
                buf = sl["buf"].get(k)
                if buf is None or buf.dtype != v.dtype or buf.shape[1:] != v.shape[1:] or buf.shape[0] < v.shape[0]:
                    n = v.shape[0]
                    if buf is not None and buf.dtype == v.dtype and buf.shape[1:] == v.shape[1:]:
                        n = max(buf.shape[0], 1)
                        while n < v.shape[0]:
                            n *= 2
                    # allocated on the copy stream after its wait on `free`: the old buffer goes back to this stream's pool
                    # only once the compute stream has finished reading it
                    buf = sl["buf"][k] = torch.empty((n,) + tuple(v.shape[1:]), dtype=v.dtype, device=self.device)
                view = sl["view"][k] = buf[:v.shape[0]]
                view.copy_(v, non_blocking=True)
            sl["ready"].record(self.stream)
        self.head = (self.head + 1) % len(self.slots)
        self.pending += 1

    def get(self):
        assert self.pending > 0, "prefetcher empty: call put() first"
        sl = self.slots[self.tail]
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(sl["ready"])
        self._last = sl
        self.tail = (self.tail + 1) % len(self.slots)
        self.pending -= 1
        return dict(sl["view"])

    def release(self):
        """call after the kernels that read the last get()'s tensors have been enqueued on the current stream"""
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._last["free"] = ev
