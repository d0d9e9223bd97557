#!/usr/bin/env python
"""bench.py -- images/sec of the YOLOv5l semi-supervised (SSOD) training step @640, 16 labeled + 16 unlabeled per GPU.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl native|reference] [--dump-outputs DIR]
  (N>1: python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 ... bench.py --gpus N ...)

One "step" = SSODTrainerStep.train_instance: teacher-EMA forward on the unlabeled batch (native wgmma engine) ->
NMS + pseudo labels (native) -> student forward/backward on cat(labeled, strong-aug) -> ComputeLoss +
ComputeStudentMatchLoss (native fused) -> gradient all-reduce (N>1) -> SGD-Nesterov -> both EMA updates (native fused).
Nothing is skipped inside the timed region.  Prints ONE JSON line (rank 0).

  value : images/s (B_l+B_u summed over ranks / max-over-ranks device time), inputs resident in HBM as fp32 [0,1]
  e2e   : same metric through the public step API from PINNED HOST uint8 batches: H2D copies + .float()/255 inside
          the timed region and a D2H read of the loss every step
  roofline : dominant native kernel class = conv_fwd_kernel (wgmma implicit GEMM): algorithmic conv FLOPs / CUDA-event
          time, vs the bf16 peak (MEASURED_PEAKS.json when present, else the H100 SXM data sheet)
  cpu_baseline : the oracle's CPU restatement of the same step (oracle/step_ref.py), bounded sample, rank 0, N=1 only
--dump-outputs DIR writes what the last timed step computed (its loss, and a fixed seeded sample of the student's and the
EMA teachers' weights after its optimizer / EMA updates) as DIR/<name>.npy, so two builds can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

B_L, B_U, IMG = 16, 16, 640
METRIC = "images/sec YOLOv5l SSOD step @640 bs32 (16 labeled + 16 unlabeled per GPU)"
NB = 369     # batches per epoch of the reference's COCO 10 % recipe (11,829 labeled images / 32): sizes the warm-up window (nw = 1107)
# --config: the headline (default) and the two other single-GPU configurations of BASELINE.json
CONFIGS = {
    "ssod640": dict(kind="ssod", bl=16, bu=16, img=640, metric=METRIC,
                    workload="YOLOv5l SSOD 640: 16 labeled + 16 unlabeled per GPU (BASELINE configs[2] per-GPU batch), optimizer+2xEMA every step"),
    "ssod1280": dict(kind="ssod", bl=8, bu=8, img=1280, metric="images/sec YOLOv5l SSOD step @1280 bs16 (8 labeled + 8 unlabeled per GPU)",
                     workload="YOLOv5l SSOD 1280: 8 labeled + 8 unlabeled per GPU (BASELINE configs[4]), optimizer+2xEMA every step"),
    "sup32": dict(kind="sup", bl=32, bu=0, img=640, metric="images/sec YOLOv5l supervised step @640 bs32",
                  workload="YOLOv5l supervised 640, batch 32 on one GPU (BASELINE configs[1]); optimizer cadence of the reference (accumulate=2 past warm-up, 1 inside it)"),
}


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))), "measured"
    except Exception:
        # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 TFLOP/s dense bf16 -- not measured, an upper bound
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0}, "h100_sxm_datasheet"


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""

    def __init__(self, index=0):
        super().__init__(daemon=True)
        self.index, self.rows, self._halt = index, [], threading.Event()

    def run(self):
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        while not self._halt.is_set():
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.split(",")])
            except Exception:
                pass
            self._halt.wait(0.2)

    def summary(self):
        self._halt.set()
        self.join(timeout=6)
        sm = [float(r[0]) for r in self.rows if r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if r[1].replace(".", "").isdigit()]
        reasons = set()
        for r in self.rows:
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(self.rows)}


def synth_batch(rank, device=None, pinned=False, bl=B_L, bu=B_U, img=IMG):
    """Per-rank seeded synthetic batch (SURVEY.md 8d, config #3): uint8 images like the loaders produce, 8 targets/img."""
    import synth
    tg = synth.make_targets(100 + rank, 8 * bl, bl)
    # structured images (smooth colour field + textured rectangles, on the labeled batch at the ground-truth boxes): i.i.d.
    # noise images make a random-init trunk ~7x more sensitive to parameter perturbations (tools/debug_teacher_sens.py)
    imgs = torch.from_numpy(synth.make_images(1 + rank, bl, img, tg))
    u_weak = torch.from_numpy(synth.make_images(1001 + rank, max(bu, 1), img))
    u_strong = u_weak.flip(3).contiguous()
    targets = torch.from_numpy(tg)
    Ms = torch.from_numpy(synth.make_Ms(200 + rank, max(bu, 1), img))
    out = dict(imgs=imgs, u_weak=u_weak, u_strong=u_strong, targets=targets, Ms=Ms)
    if pinned:
        out = {k: v.pin_memory() for k, v in out.items()}
    return out


def conv_flops_teacher(engine_model, n_img, img):
    """Algorithmic conv FLOPs (2*MACs, real Cin -- the stem counts K=108) of one eval forward of trunk + Detect."""
    flops = 0   # the spatial size of every conv's OUTPUT follows from its module path
    for name, mod in engine_model.named_modules():
        conv = getattr(mod, "conv", None) if hasattr(mod, "bn") else (mod if isinstance(mod, torch.nn.Conv2d) and name.startswith("head.m") else None)
        if conv is None:
            continue
        if name.startswith("backbone.stage1"): hw = img // 2
        elif name.startswith("backbone.stage2"): hw = img // 4
        elif name.startswith("backbone.stage3"): hw = img // 8
        elif name.startswith("backbone.stage4"): hw = img // 16
        elif name.startswith("backbone.stage5") or name.startswith("backbone.sppf"): hw = img // 32
        elif name.startswith("neck.conv1") or name.startswith("neck.conv4") or name.startswith("neck.C4"): hw = img // 32
        elif name.startswith("neck.C1") or name.startswith("neck.conv2") or name.startswith("neck.conv3") or name.startswith("neck.C3"): hw = img // 16
        elif name.startswith("neck.C2"): hw = img // 8
        elif name.startswith("head.m.0"): hw = img // 8
        elif name.startswith("head.m.1"): hw = img // 16
        elif name.startswith("head.m.2"): hw = img // 32
        else: continue
        co, ci, kh, kw = conv.weight.shape
        flops += 2 * n_img * hw * hw * co * ci * kh * kw
    return flops


def dominant_kernel_roofline(dev, peak_tflops, peak_kind):
    """The conv kernel with the raw bf16 epilogue (conv_fwd_kernel<128,0>: the wgmma implicit GEMM that runs the student's
    training forward AND, with transposed taps, its dgrad) on the shape family that carries 57% of the trunk FLOPs (3x3 s1
    C->C Bottleneck conv; here 256->256 on 40x40 maps, batch 32 = the student's batch).  30 launches timed with CUDA events
    on the launching stream, rotating over 6 input/output buffer sets (315 MB > the 50 MB L2) so no launch finds its input
    in L2.  Algorithmic FLOPs = 2*N*H*W*Cout*Cin*9; algorithmic bytes = input + weights + output, each moved once."""
    from efficientteacher_b200 import convops as co
    N, H, C_ = 32, 40, 256
    nbuf = 6
    xs = [torch.randn(N, H, H, C_, device=dev).to(torch.bfloat16) for _ in range(nbuf)]
    ys = [torch.empty(N, H, H, C_, dtype=torch.bfloat16, device=dev) for _ in range(nbuf)]
    w = co.pack_weight(torch.randn(C_, C_, 3, 3, device=dev) * (C_ * 9) ** -0.5)
    f = lambda i: co.conv_fwd(xs[i % nbuf], w, C_, C_, 3, 1, 1, None, None, None, out=ys[i % nbuf])  # noqa: E731
    for i in range(nbuf):
        f(i)
    torch.cuda.synchronize()
    n = 30
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(n):
        f(i)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / n
    flops = 2.0 * N * H * H * C_ * C_ * 9
    ach = flops / ms / 1e9
    traffic = 2.0 * (2 * N * H * H * C_ + C_ * C_ * 9)
    return {"bound": "tensor", "kernel": "conv_fwd_kernel<128,0> (wgmma implicit GEMM, TMA-fed, raw bf16 epilogue: student forward + dgrad), 3x3 s1 256->256 @40x40, batch 32",
            "achieved": ach, "peak": peak_tflops, "unit": "TFLOP/s", "frac": ach / peak_tflops,
            "traffic": traffic, "traffic_note": "algorithmic bytes per launch (bf16 input + weights + output, no re-reads)",
            "peak_kind": peak_kind, "flops_per_launch": flops, "us_per_launch": ms * 1e3, "launches_timed": n,
            "l2": "rotating 6 buffer sets (315 MB) > L2"}


DUMP_SAMPLE = 1 << 21      # weights sampled per model by --dump-outputs (8 MB of fp32 each)


def dump_outputs(path, loss, models):
    """--dump-outputs: the loss of the last timed step (float64) and, per model, the same fixed seeded sample of its floating
    state (parameters + BN statistics, flattened in state_dict order) as it stands after that step (float32)."""
    os.makedirs(path, exist_ok=True)
    arrays = {"loss": loss.double().cpu().numpy().reshape(-1)}
    idx = None
    for name, m in models.items():
        flat = torch.cat([v.detach().float().flatten() for v in m.state_dict().values() if v.is_floating_point()])
        if idx is None:
            idx = torch.randint(0, flat.numel(), (DUMP_SAMPLE,), generator=torch.Generator().manual_seed(1234)).sort().values
        arrays[name + "_state_sample"] = flat[idx.to(flat.device)].cpu().numpy()
    for k, v in arrays.items():
        np.save(os.path.join(path, k + ".npy"), v)


def kernel_table(step, ni, path, graph_ms):
    """Per-kernel GPU time of 2 eager steps from CUPTI activity records (torch.profiler): low overhead, kernels not
    serialised -- the shares are what the step really spends (unlike an ncu launch list)."""
    from torch.profiler import ProfilerActivity, profile
    nsteps = 2
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(nsteps):
            step(ni + i)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type is not None and "cuda" in str(ev.device_type).lower():
            r = rows.setdefault(ev.name, [0, 0.0])
            r[0] += 1
            r[1] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    tot = sum(v[1] for v in rows.values())
    with open(path, "w") as f:
        f.write("# per-kernel device time, eager step (CUPTI via torch.profiler), mean of %d steps; graph replay of the step: %.2f ms\n" % (nsteps, graph_ms))
        f.write("# kernels/step %d, sum of kernel time/step %.2f ms\n" % (sum(v[0] for v in rows.values()) / nsteps, tot / nsteps / 1e3))
        f.write("| kernel | launches/step | us/step | share |\n|---|---:|---:|---:|\n")
        for name, (cnt, us) in sorted(rows.items(), key=lambda kv: -kv[1][1])[:60]:
            f.write("| `%s` | %.1f | %.1f | %.1f%% |\n" % (name[:110], cnt / nsteps, us / nsteps, 100.0 * us / tot))


def _cpu_step_sample(threads, bl, bu, steps, img=IMG):
    """`steps` full SSOD steps of the oracle's CPU restatement (oracle/step_ref.py: torch fp32 trunk + port) on bl+bu images
    with `threads` host threads; returns the per-step seconds (the first step is a warm-up and is not returned)."""
    from oracle.step_ref import CpuSSODStep
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    import synth
    torch.set_num_threads(threads)
    torch.manual_seed(0)
    model = Model(yolov5_ssod_cfg('l'))
    step = CpuSSODStep(model.state_dict(), (3, 6, 9, 3), 3, batch_size=B_L + B_U, ema_updates=100000, bn_momentum=0.03,
                       warmup=(max(round(3 * NB), 1000), 0.1, 0.8))
    r = np.random.RandomState(1)
    imgs = torch.from_numpy(r.rand(bl, 3, img, img).astype(np.float32))
    uw = torch.from_numpy(r.rand(bu, 3, img, img).astype(np.float32))
    tg = synth.make_targets(100, 8 * bl, bl)
    Ms = synth.make_Ms(200, bu, img)
    ts = []
    for i in range(steps + 1):
        t0 = time.perf_counter()
        step.step(imgs, tg, uw.flip(3), uw, Ms)
        if i > 0:
            ts.append(time.perf_counter() - t0)
    return ts


def _best_threads(bl, bu):
    """torch's CPU convolutions stop scaling (and collapse when oversubscribed) well before 100+ threads.  Probe {all cores, 64,
    32, 16} on a SMALL proxy -- the fp32 YOLOv5l trunk forward+backward on one 320x320 image, a few hundred ms per try -- and
    keep the fastest setting for the real sample: the baseline gets the thread count it is fastest with, and the probe
    stays a few seconds even on a 128-core host (a full 2+2 step at 128 threads takes minutes there)."""
    from oracle.trunk_ref import TrunkRef
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    ncpu = os.cpu_count() or 1
    cands = sorted({c for c in (ncpu, 64, 32, 16) if c <= ncpu}, reverse=True)
    torch.manual_seed(0)
    sd = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and "running" not in k and "anchor" not in k)
          for k, v in Model(yolov5_ssod_cfg('l')).state_dict().items()}
    x = torch.rand(1, 3, 320, 320)
    best, seen = None, {}
    for c in cands:
        torch.set_num_threads(c)
        ts = []
        for _ in range(2):
            t0 = time.perf_counter()
            raw, _f = TrunkRef(sd, (3, 6, 9, 3), 3).forward(x, train=True, with_features=False)
            sum(r.square().mean() for r in raw).backward()
            ts.append(time.perf_counter() - t0)
            if ts[-1] > 20.0:
                break
        seen[c] = min(ts)
        if best is None or seen[c] < best[1]:
            best = (c, seen[c])
    return best[0], seen


def run_reference(args, rank, world):
    """--impl reference: the reference's CPU path of the step (the oracle's restatement of the original
    project's step, which needs none of its sources).  Rank 0 only.  Each step = one full SSOD step on a bounded sample (2 labeled + 2 unlabeled images), fp32, with
    the host thread count torch is fastest at (probed: all cores / 64 / 32 / 16)."""
    if rank != 0:
        return
    bl = bu = 2
    threads, _ = _best_threads(bl, bu)
    ts = _cpu_step_sample(threads, bl, bu, args.warmup + args.steps)[args.warmup:]
    sec = float(np.mean(ts))
    val = (bl + bu) / sec
    sample = ("full SSOD step (teacher fwd, NMS+pseudo-label, student fwd/bwd, both losses, SGD, 2x EMA) on 2 labeled + 2 unlabeled 640x640 images, "
              "fp32 torch CPU, %d threads (fastest of all-cores/64/32/16 on this host, probed on a small proxy; %d cores present)" % (threads, os.cpu_count()))
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": val, "unit": "images/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic", "config": {"workload": "YOLOv5l SSOD 640, CPU bounded sample 2+2 images/step"},
        "cpu_baseline": {"value": val, "unit": "images/s", "cores": threads, "kind": "port", "sample": sample},
        "e2e": {"value": val, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}), flush=True)


def cpu_baseline_quick():
    bl = bu = 2
    t_all = time.perf_counter()
    threads, _ = _best_threads(bl, bu)
    ts = _cpu_step_sample(threads, bl, bu, 2)
    sec = float(np.mean(ts))
    return {"value": (bl + bu) / sec, "unit": "images/s", "cores": threads, "kind": "port",
            "sample": "2 full SSOD steps (after 1 warm-up) on 2 labeled + 2 unlabeled 640x640 images (oracle/step_ref.py, torch fp32 CPU) with %d threads "
                      "= the fastest of all-cores/64/32/16 on this %d-core host (probed on a small proxy); mean step %.2f s; baseline leg %.0f s in total" % (
                          threads, os.cpu_count(), sec, time.perf_counter() - t_all)}


def nms_pseudo_label_full_load(creator, dev):
    """The metric's second half: NMS + pseudo-label transform, ms/batch at FULL candidate load, on synthetic decoded teacher
    predictions (SURVEY.md 8d recipe: 2 % of the rows are candidates): 16 x 25,200 (640) and 8 x 100,800 (1280).  CUDA events
    around 20 calls of FairPseudoLabel.create_pseudo_label_device (candidate filter -> rank -> batched greedy NMS -> affine
    pseudo-label transform; no host sync), after 3 warm-up calls."""
    import synth
    out = {}
    g = torch.Generator(device=dev).manual_seed(0)
    for name, B, P, img in (("16x25200_img640", 16, 25200, 640), ("8x100800_img1280", 8, 100800, 1280)):
        x = torch.empty((B, P, 85), dtype=torch.float32, device=dev)
        x[..., 0:2] = torch.rand((B, P, 2), generator=g, device=dev) * img
        x[..., 2:4] = torch.rand((B, P, 2), generator=g, device=dev) * 192 + 4
        hot = torch.rand((B, P), generator=g, device=dev) < 0.02
        x[..., 4] = torch.where(hot, torch.rand((B, P), generator=g, device=dev) * 0.9 + 0.1, torch.rand((B, P), generator=g, device=dev) * 0.05)
        x[..., 5:] = torch.rand((B, P, 80), generator=g, device=dev) ** 4
        Ms = torch.from_numpy(synth.make_Ms(200, B, img)).to(dev)
        for _ in range(3):
            creator.create_pseudo_label_device(x, Ms, img, img)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        s.record()
        for _ in range(n):
            rows, cnt = creator.create_pseudo_label_device(x, Ms, img, img)
        e.record()
        torch.cuda.synchronize()
        out[name] = {"ms_per_batch": s.elapsed_time(e) / n, "candidates_per_img": float((x[..., 4] > 0.1).sum(1).float().mean()),
                     "detections_per_img": float(creator.last_det[1].float().mean()), "pseudo_label_rows": int(cnt.item())}
        del x
    return out


def gpu_eager_baseline(st, host, cfg_b, dev, steps=5, warmup=3):
    """The same step with stock PyTorch on this GPU (oracle/eager_ref.py: ATen / cuDNN / torchvision eager under bf16 autocast,
    channels_last, cudnn.benchmark, torch.optim.SGD, per-tensor EMA loops, per-image torchvision NMS, host-side pseudo-label
    transform -- the way the reference executes it), started from the native step's CURRENT state (same weights, same batch).
    SURVEY.md 2.1 / 8(d): "the kernel-level bar to beat on the same box"."""
    from oracle.eager_ref import EagerSSODStep
    import synth
    torch.backends.cudnn.benchmark = True        # the reference: init_seeds(1 + RANK) -> cudnn.benchmark = True (utils/general.py)
    depth = tuple(len(getattr(st.model.backbone, n).m) for n in ("stage2_2", "stage3_2", "stage4_2", "stage5_2"))
    sd = {k: v.detach().clone() for k, v in st.model.state_dict().items()}
    eg = EagerSSODStep(sd, depth, len(st.model.neck.C1.m), dev, synth.ANCHORS_GRID, amp_dtype=torch.bfloat16, batch_size=cfg_b["bl"] + cfg_b["bu"],
                       ema_updates=st.ema.updates, warmup=(st.nw, st.warmup_bias_lr, st.warmup_momentum))
    eg.teacher = {k: v.detach().clone() for k, v in st.ema.ema.state_dict().items()}
    eg.ni = 30
    f01 = lambda t: t.to(dev).float() / 255.0  # noqa: E731
    imgs, uw, us = f01(host["imgs"]), f01(host["u_weak"]), f01(host["u_strong"])
    tg, Ms = host["targets"].to(dev), host["Ms"].to(dev)
    for _ in range(warmup):
        eg.step(imgs, tg, us, uw, Ms)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        loss = eg.step(imgs, tg, us, uw, Ms)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / steps
    out = {"value": (cfg_b["bl"] + cfg_b["bu"]) / (ms / 1e3), "unit": "images/s", "ms_per_step": ms, "steps": steps, "warmup": warmup,
           "pseudo_label_rows_last_step": int(eg.n_pseudo), "loss_last_step": float(loss),
           "what": "oracle/eager_ref.EagerSSODStep: PyTorch %s eager (cuDNN/ATen/torchvision), bf16 autocast, channels_last, cudnn.benchmark, same weights/batch as the native step, "
                   "inputs resident in HBM" % torch.__version__}
    del eg
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="native", choices=["native", "reference"])
    ap.add_argument("--config", default="ssod640", choices=sorted(CONFIGS), help="ssod640 = the headline (BASELINE.json metric); ssod1280 / sup32 = configs[4] / configs[1]")
    ap.add_argument("--scaling", default="weak", choices=["weak", "strong"],
                    help="weak (default): the config's per-GPU batch at every N; strong: the config's batch is the "
                         "GLOBAL batch, split evenly over the ranks (SURVEY.md 8d: 16+16 -> 8+8 -> 4+4 -> 2+2 per GPU at 1/2/4/8 GPUs)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-eager-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true", help="profiling runs only: skip the end-to-end leg")
    ap.add_argument("--no-graph", action="store_true", help="eager launches instead of replaying the captured CUDA graphs of the step")
    ap.add_argument("--allow-invalid", action="store_true", help="dev: print the line (marked invalid) even when the self-check fails")
    ap.add_argument("--nvtx-step", action="store_true", help="dev: wrap ONE extra eager step in the NVTX range 'etb_step' (ncu --nvtx --nvtx-include etb_step)")
    ap.add_argument("--kernel-table", default="", help="dev: write a per-kernel time table (torch.profiler/CUPTI, 2 eager steps) to this file")
    ap.add_argument("--dump-outputs", default="", metavar="DIR", help="write the last timed step's outputs as DIR/<name>.npy (see the module docstring)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        run_reference(args, rank, world)
        return
    assert world == args.gpus, "launch with torch.distributed.run --nproc-per-node %d" % args.gpus
    assert args.warmup >= 3, "timing rules: at least 3 warm-up steps"
    cb = CONFIGS[args.config]
    bl, bu, img, ssod = cb["bl"], cb["bu"], cb["img"], cb["kind"] == "ssod"
    if args.scaling == "strong":
        assert bl % world == 0 and bu % world == 0, "strong scaling: the global batch must divide by the world size"
        bl, bu = bl // world, bu // world
    import __graft_entry__ as g
    if rank == 0:
        g.build()
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
        dist.barrier()
    from efficientteacher_b200 import _lib
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep
    lib = _lib.lib()

    torch.manual_seed(0)                       # identical initial student on every rank (DDP broadcasts rank 0's)
    host = synth_batch(rank, pinned=True, bl=bl, bu=bu, img=img)
    f01 = lambda t: t.to(dev).float() / 255.0  # noqa: E731  trainer/ssod_trainer.py:694-696
    d_imgs, d_uw, d_us = f01(host["imgs"]), f01(host["u_weak"]), f01(host["u_strong"])
    d_tg, d_Ms = host["targets"].to(dev), host["Ms"].to(dev)
    if world > 1:
        # Gradients are AVERAGED across ranks in the benchmark (ncclAvg: the same single collective over the same 191.8 MB arena
        # as the reference's sum; every kernel is identical).  With the reference's SUM the effective learning rate grows with
        # the world size, the random-init student's BatchNorm scales drift world_size x faster and the EMA teacher's candidate
        # count leaves the self-check's [0.5, 2] x window within the 20 timed steps at N >= 4 (N = 2 with SUM: 0.61 x, N = 1:
        # 0.79 x).  Averaging keeps the synthetic state at every N as close to the single-GPU one as its data allows.
        SSODTrainerStep.GRAD_REDUCE = "avg"
    if ssod:
        cfg = yolov5_ssod_cfg('l', batch_size=(bl + bu) * world, img_size=img)
        cfg.SSOD.fixed_accumulate = True       # SURVEY.md 8(d): optimizer step + both EMA updates EVERY iteration
        st = SSODTrainerStep(cfg, dev, rank=rank if world > 1 else -1, world_size=world, epochs=300, nb=NB)
        # Synthetic steady state.  lr / momentum follow the reference's schedule from ni = 0 (warm-up, trainer.py:372-395:
        # conv-weight lr ramps up from 0 over nw = 1107 iterations) -- the state a from-scratch run is in, and the one in
        # which a random-init model is well conditioned (at full lr a random init blows its BN statistics up in ~10 steps
        # under ANY bf16 implementation: tools/debug_teacher_drift.py --nw 0, DESIGN.md section 7).  The EMA decay is the
        # steady-state 0.9999 (ema.updates = 100000) so the calibrated teacher stays put over the run.
        st.ema.updates = 100000
    else:
        cfg = yolov5_sup_cfg('l', batch_size=bl * world, img_size=img)
        st = SupTrainerStep(cfg, dev, rank=rank if world > 1 else -1, world_size=world, epochs=300, nb=NB)

    # Synthetic steady state (SURVEY.md 8d): random-init weights make an eval-mode teacher degenerate (default running
    # statistics -> constant outputs) and give no confident boxes.  (1) set every BN's running statistics to the batch
    # statistics of the synthetic data (one train-mode pass with momentum 1) and start teacher = student; (2) rescale / shift
    # the Detect head's objectness rows and biases so ~2% of the predictions/img have obj > 0.3 (robustly above the 0.1
    # NMS threshold) and class scores are ~0.96.  Everything else stays random-init.
    with torch.no_grad():
        bns = [m for m in st.model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
        for m in bns:
            m.momentum = 1.0
        with torch.autocast("cuda", dtype=torch.bfloat16):
            st.model((torch.cat([d_imgs, d_us], 0) if ssod else d_imgs).contiguous(memory_format=torch.channels_last))
        for m in bns:
            m.momentum = 0.03
        st.ema.ema.load_state_dict(st.model.state_dict())
        if ssod:
            st.semi_ema.ema.load_state_dict(st.model.state_dict())

    def calibrate_teacher_head(first):
        """(2): objectness of the TEACHER's Detect head so that ~2 % of its predictions are NMS candidates on this batch.
        A random-init trunk amplifies parameter perturbations by 10^2-10^3 (tools/debug_teacher_sens.py), so the few 1e-4
        EMA steps of a run move the teacher's logits visibly; the calibration is therefore repeated (bias only) right before
        every timed window -- outside the timed regions -- and the self-check below verifies the load over the window."""
        with torch.no_grad():
            (pred, raw), _ = st.ema.ema(d_uw)
            for l, m in enumerate(st.ema.ema.head.m):
                # A random-init head gives objectness logits with std ~0.15: (2a) widen them to std 3 by scaling the three
                # objectness rows of the 1x1 head conv, (2b) set the bias so the 98th percentile is obj = 0.3, (2c) class bias
                # +8 (it starts at log(0.6/(nc-0.99)) ~ -4.9) so class scores are ~0.96 and conf = obj*cls ~ obj.
                b = m.bias.view(3, -1)
                w = m.weight.view(3, -1, m.weight.shape[1])
                lin = (raw[l][..., 4].float() - b[:, 4].float().view(1, 3, 1, 1)).flatten()
                sc = 3.0 / max(float(lin.std()), 1e-6) if first else 1.0
                q98 = torch.quantile(sc * lin[:2_000_000], 0.98).item()
                if first:
                    w[:, 4] *= sc
                    b[:, 5:] += 8.0
                b[:, 4] = float(np.log(0.3 / 0.7)) - q98
                if first:
                    for other in (st.model, st.semi_ema.ema):
                        other.head.m[l].bias.data.copy_(m.bias.data)
                        other.head.m[l].weight.data.copy_(m.weight.data)
            (pred, raw), _ = st.ema.ema(d_uw)
            return float((pred[..., 4] > cfg.SSOD.nms_conf_thres).sum(1).float().mean().item())

    cand_per_img = calibrate_teacher_head(True) if ssod else None

    use_graph = not args.no_graph

    def step_resident(i):
        if ssod:
            f = st.train_instance_graphed if use_graph else st.train_instance
            return f(d_imgs, d_tg, d_us, d_uw, None, d_Ms, i)
        return (st.train_step_graphed if use_graph else st.train_step)(d_imgs, d_tg, i)

    def step_eager(i):
        if ssod:
            return st.train_instance(d_imgs, d_tg, d_us, d_uw, None, d_Ms, i)
        return st.train_step(d_imgs, d_tg, i)

    from efficientteacher_b200.trainer import DevicePrefetcher
    pf = DevicePrefetcher(dev)
    keys = ("imgs", "u_strong", "u_weak", "targets", "Ms") if ssod else ("imgs", "targets")
    host_batch = {k: host[k] for k in keys}

    def step_e2e(i):
        # every step: H2D of this step's uint8 batch from pinned memory (staged on a side stream, so the copy of step i+1
        # overlaps the kernels of step i), the step, D2H read of the loss
        if pf.pending == 0:
            pf.put(host_batch)
        b = pf.get()
        # the uint8 batches go straight into the step: the native stem (student) and the teacher engine read uint8 and divide by
        # 255 inside their im2col kernels (== `.float() / 255`, trainer/ssod_trainer.py:694-696), no fp32 image is materialised
        if ssod:
            loss = (st.train_instance_graphed if use_graph else st.train_instance)(b["imgs"], b["targets"], b["u_strong"], b["u_weak"], None, b["Ms"], i)
        else:
            loss = (st.train_step_graphed if use_graph else st.train_step)(b["imgs"], b["targets"], i)
        pf.release()
        pf.put(host_batch)                   # next step's inputs start moving now
        return float(loss.item())            # D2H read of the step's result

    def barrier():
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps, first):
        barrier()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for i in range(steps):
            fn(first + i)
        e.record()
        barrier()
        ms = torch.tensor([s.elapsed_time(e)], device=dev)
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    def pl_state():
        c = st.pseudo_label_creator
        return int(c.last_count_dev.item()), float(c.last_det[1].float().mean().item())

    ni = 0
    for _ in range(args.warmup):
        step_resident(ni); ni += 1
    torch.cuda.synchronize()
    cand_start = calibrate_teacher_head(False) if ssod else None     # synthetic-state maintenance, outside the timed region
    sampler = ClockSampler(local_rank) if rank == 0 else None
    if sampler:
        sampler.start()
    pl_probe = []

    last_loss = []

    def step_resident_probed(i):          # device-side copies of the pseudo-label counters of the first / last timed step (no sync)
        out = step_resident(i)
        if i == probe_last:
            last_loss.append(out.clone())
        if ssod and (i == probe_first or i == probe_last):
            c = st.pseudo_label_creator
            pl_probe.append((c.last_count_dev.clone(), c.last_det[1].float().mean()))
        return out
    probe_first, probe_last = ni, ni + args.steps - 1
    ms = timed(step_resident_probed, args.steps, ni); ni += args.steps
    if args.dump_outputs and rank == 0:      # before any further step moves the weights
        dump_outputs(args.dump_outputs, last_loss[0], dict(student=st.model, teacher_ema=st.ema.ema, **({"semi_ema": st.semi_ema.ema} if ssod else {})))
    if ssod:
        probes = [(int(a.item()), float(b.item())) for a, b in pl_probe]
        (n_pl0, det_per_img0), (n_pl_timed, det_timed) = probes[0], probes[-1]        # --steps 1: first == last
        with torch.no_grad():
            (pred_t, _r), _f = st.ema.ema(d_uw)
            cand_timed_end = float((pred_t[..., 4] > cfg.SSOD.nms_conf_thres).sum(1).float().mean())
            del pred_t, _r, _f
    # kernel-launch count and per-phase CUDA-event times come from an eager (un-graphed) pass of the same step
    step_eager(ni); ni += 1     # one eager step first: lazy one-time work
    torch.cuda.synchronize()
    if ssod:
        st.profile, st.phase_events = True, []
    l0 = lib.etb_launch_count()
    nprof = 3
    for _ in range(nprof):
        step_eager(ni); ni += 1
    torch.cuda.synchronize()
    launches = (lib.etb_launch_count() - l0) / nprof
    phases = {k: v / nprof for k, v in st.phase_times_ms().items()} if ssod else {}
    st.profile = False
    n_pl_e2e = None
    if args.no_e2e:
        ms_e2e = float("nan")
    else:
        for _ in range(3):
            step_e2e(ni); ni += 1
        if ssod:
            calibrate_teacher_head(False)
        ms_e2e = timed(step_e2e, args.steps, ni); ni += args.steps
        if ssod:
            n_pl_e2e = pl_state()[0]
    clocks = sampler.summary() if sampler else None
    if args.nvtx_step and rank == 0:
        torch.cuda.synchronize()
        rid = torch.cuda.nvtx.range_start("etb_step")     # start/end range: process-wide (backward runs on autograd's thread)
        step_eager(ni); ni += 1
        torch.cuda.synchronize()
        torch.cuda.nvtx.range_end(rid)
    if args.kernel_table and rank == 0:
        kernel_table(step_eager, ni, args.kernel_table, ms / args.steps)
        ni += 2

    # ---- self-check: the run is only a measurement if the whole step really ran at load --------------------------------
    health = {}
    if ssod:
        def _bnmax(mod):
            bb = [q for q in mod.modules() if isinstance(q, torch.nn.BatchNorm2d)]
            return [max(float(q.running_var.detach().max()) for q in bb), max(float(q.running_mean.detach().abs().max()) for q in bb),
                    max(float(q.weight.detach().abs().max()) for q in bb), max(float(q.bias.detach().abs().max()) for q in bb)]
        health = {"nms_candidates_per_img_after_first_calibration": cand_per_img,
                  "nms_candidates_per_img_at_start_of_timed_window": cand_start, "nms_candidates_per_img_at_end_of_timed_window": cand_timed_end,
                  "nms_detections_per_img_first_timed_step": det_per_img0, "nms_detections_per_img_last_timed_step": det_timed,
                  "pseudo_label_rows_first_timed_step": n_pl0, "pseudo_label_rows_last_timed_step": n_pl_timed,
                  "pseudo_label_rows_last_e2e_step": n_pl_e2e,
                  "student_bn_max[running_var,|running_mean|,|gamma|,|beta|]": _bnmax(st.model),
                  "teacher_bn_max[running_var,|running_mean|,|gamma|,|beta|]": _bnmax(st.ema.ema), "steps_total": ni,
                  "rule": "valid iff over the timed window: pseudo-label rows > 0 at both ends, last/first within [0.5, 2], NMS candidates/img at the end within [0.5, 2] x start, BN state finite"}
        ok = (n_pl0 > 0 and n_pl_timed > 0 and 0.5 * n_pl0 <= n_pl_timed <= 2.0 * n_pl0 and cand_start > 0
              and 0.5 * cand_start <= cand_timed_end <= 2.0 * cand_start and (n_pl_e2e is None or n_pl_e2e > 0)
              and all(np.isfinite(health["student_bn_max[running_var,|running_mean|,|gamma|,|beta|]"])))
        flags = torch.tensor([0 if ok else 1], device=dev)
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(flags, op=dist.ReduceOp.MAX)
        if int(flags.item()):
            print("[bench] INVALID RUN (rank %d): the pseudo-label branch did not stay loaded / the state diverged: %s" % (rank, json.dumps(health)),
                  file=sys.stderr, flush=True)
            if not args.allow_invalid:
                sys.exit(3)
            health["INVALID"] = True

    if rank == 0:
        pk, pk_kind = peaks()
        imgs_per_step = (bl + bu) * world
        value = imgs_per_step * args.steps / (ms / 1e3)
        e2e_val = imgs_per_step * args.steps / (ms_e2e / 1e3)
        f_img = conv_flops_teacher(st.ema.ema, 1, img)
        t_ms = phases.get("teacher_forward", float("nan"))
        peak = pk["bf16_tflops_sustained"]
        # conv FLOPs of the whole step: teacher fwd (B_U) + student fwd/dgrad/wgrad (B_L+B_U; the stem has no dgrad)
        step_flops = f_img * (bu + 3 * (bl + bu))
        roof = dominant_kernel_roofline(dev, peak, pk_kind + " bf16_tflops_sustained")
        roof["step_level"] = {"conv_flops_per_step": step_flops, "achieved_tflops": step_flops / (ms / args.steps / 1e3) / 1e12,
                              "frac_of_peak": step_flops / (ms / args.steps / 1e3) / 1e12 / peak,
                              "teacher_forward_phase_tflops": f_img * bu / (t_ms / 1e3) / 1e12 if ssod else None}
        h2d = sum(host[k].numel() * host[k].element_size() for k in keys)
        out = {
            "metric": cb["metric"], "value": value, "unit": "images/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": args.scaling, "vs_baseline": None,
            "dtype": "bf16", "data": "synthetic (seeded uint8 images, 8 gt boxes/img, random-init YOLOv5l with BN statistics calibrated on the batch; teacher objectness calibrated to ~2% NMS candidates)",
            "config": {"workload": cb["workload"], "config_name": args.config,
                       "global_batch": imgs_per_step, "per_gpu_batch": [bl, bu], "img_size": img, "parallelism": "dp%d" % world, "grad_reduce": ("ncclAvg of the flat arena (reference: sum; see bench.py)" if world > 1 else "none (1 GPU)"), "cuda_graph": use_graph,
                       "schedule": "reference warm-up from ni=0 (nw=%s, nb=%d): lr/momentum change every step (device-resident hyper-parameters)" % (st.nw, NB),
                       "l2": "inputs+activations per step (>1 GB) exceed the 50 MB L2; no explicit flush",
                       "native": "teacher trunk+head, student conv fwd/dgrad/wgrad (wgmma) + BatchNorm(train)+SiLU fwd/bwd, weight packing, NMS/pseudo-label, assigners, losses fwd/bwd, SGD, EMA",
                       "self_check": health},
            "e2e": {"value": e2e_val, "unit": "images/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4, "ms_per_step": ms_e2e / args.steps},
            "gpu_launches": launches,
            "phases_ms": phases,
            "roofline": roof,
            "clocks": clocks,
        }
        if ssod:
            out["nms_pseudo_label_ms_per_batch"] = nms_pseudo_label_full_load(st.pseudo_label_creator, dev)
        if world == 1 and ssod and not args.no_eager_baseline:
            try:
                out["gpu_eager_baseline"] = gpu_eager_baseline(st, host, cb, dev)
                out["gpu_eager_baseline"]["native_over_eager"] = value / out["gpu_eager_baseline"]["value"]
            except Exception as exc:      # a baseline must never take the bench line down; say why it is missing
                out["gpu_eager_baseline"] = {"unavailable": repr(exc)[:300]}
        if world == 1 and not args.no_cpu_baseline:
            out["cpu_baseline"] = cpu_baseline_quick()
        print(json.dumps(out), flush=True)
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
