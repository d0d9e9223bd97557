"""The inputs of the loss-option fixtures (tests/golden/loss_opts_*.npz, made by tests/golden/make_golden_loss_opts.py)
and the helpers the CPU oracle test and the GPU test share to read them."""
import numpy as np

import synth

IMG, B = 320, 4
OPT_KEYS = ("nc", "fl_gamma", "cls_pw", "obj_pw", "label_smoothing", "autobalance", "ignore_obj", "with_bbox", "with_cls",
            "ssod", "ncalls")
LOSS_CASES = ("fl1", "fl15", "fl2", "pw", "mix", "nc1", "ssod_ign", "ssod_cls", "autobal")


def inputs(nc, ssod, k):
    """(logits of call k, targets [n,6] or pseudo-label rows [n,9]) of a case"""
    logits = synth.make_head_logits(200 + k, B, img=IMG, no=nc + 5)
    if ssod:
        return logits, synth.make_pseudo_rows(43, 200, B, nc=nc)
    return logits, synth.make_targets(42, 16 * B, B, nc=nc)


def opts(g):
    """the case's options as a dict (ints for the counts, bools for the switches)"""
    o = dict(zip(OPT_KEYS, (float(v) for v in g["opts"])))
    for k in ("nc", "ncalls"):
        o[k] = int(o[k])
    for k in ("autobalance", "ignore_obj", "with_bbox", "with_cls", "ssod"):
        o[k] = bool(o[k])
    return o


def check_grads(g, prefix, grads, rtol):
    """grads: per-level numpy gradients of one call"""
    for l, gr in enumerate(grads):
        flat = gr.reshape(-1)
        np.testing.assert_allclose(flat[synth.grad_sample_idx(len(flat), l)], g[f"{prefix}g{l}_sv"], rtol=rtol, atol=1e-7)
        np.testing.assert_allclose(flat[g[f"{prefix}g{l}_ti"]], g[f"{prefix}g{l}_tv"], rtol=rtol, atol=1e-7)
        np.testing.assert_allclose(np.abs(flat).sum(dtype=np.float64), float(g[f"{prefix}g{l}_l1"]), rtol=rtol)
        np.testing.assert_allclose(gr[..., 4].reshape(-1)[::7], g[f"{prefix}g{l}_obj"], rtol=rtol, atol=1e-8)
