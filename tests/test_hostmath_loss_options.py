"""CPU: the loss-option criterion the loss kernels run on the device (etb_det_bce / etb_det_bce_grad in
csrc/loss_math.h), compiled for the host, against torch autograd of the reference's
FocalLoss(BCEWithLogitsLoss(pos_weight)) (models/loss/loss.py:37-64), and bit-identity with the plain BCE at the
default options."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
fp = C.POINTER(C.c_float)


@pytest.fixture(scope="module")
def hm(tmp_path_factory):
    d = tmp_path_factory.mktemp("hm")
    libs = []
    for name in ("hostmath", "loss_options"):
        so = str(d / f"lib{name}.so")
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                               os.path.join(HERE, "hostmath", name + ".cpp")])
        libs.append(C.CDLL(so))
    libs[0].hm_bce.restype = C.c_float
    libs[0].hm_bce.argtypes = [C.c_float, C.c_float]
    libs[1].hm_det_bce.argtypes = [fp, fp, C.c_int, C.c_float, C.c_float, fp, fp]
    return libs


def _run(lib, x, z, pw, gamma):
    val, grad = np.zeros_like(x), np.zeros_like(x)
    lib.hm_det_bce(x.ctypes.data_as(fp), z.ctypes.data_as(fp), len(x), pw, gamma, val.ctypes.data_as(fp),
                   grad.ctypes.data_as(fp))
    return val, grad


def _reference(x, z, pw, gamma):
    """per-element FocalLoss(BCEWithLogitsLoss(pos_weight=pw), gamma, alpha=0.25) as loss.py:37-64 computes it"""
    xt = torch.from_numpy(x).double().requires_grad_(True)
    zt = torch.from_numpy(z).double()
    loss = torch.nn.functional.binary_cross_entropy_with_logits(xt, zt, pos_weight=torch.tensor([pw], dtype=torch.float64),
                                                                reduction="none")
    if gamma > 0:
        s = xt.sigmoid()
        p_t = zt * s + (1 - zt) * (1 - s)
        alpha_factor = zt * 0.25 + (1 - zt) * (1 - 0.25)
        loss = loss * (alpha_factor * (1.0 - p_t) ** gamma)
    loss.sum().backward()
    return loss.detach().numpy(), xt.grad.numpy()


@pytest.mark.parametrize("gamma", [0.0, 1.0, 1.5, 2.0])
@pytest.mark.parametrize("pw", [1.0, 0.5, 2.0])
def test_det_bce_vs_autograd(hm, pw, gamma):
    r = np.random.RandomState(int(pw * 10 + gamma * 100))
    n = 8192
    x = (r.standard_normal(n) * 4).astype(np.float32)
    z = r.uniform(0, 1, n).astype(np.float32)
    z[: n // 8] = 0.0                      # the hard targets of the class term and the empty objectness cells
    z[n // 8: n // 4] = 1.0
    val, grad = _run(hm[1], x, z, pw, gamma)
    want_v, want_g = _reference(x, z, pw, gamma)
    np.testing.assert_allclose(val, want_v, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(grad, want_g, rtol=2e-4, atol=2e-6)


def test_defaults_are_the_plain_bce_bit_for_bit(hm):
    r = np.random.RandomState(7)
    x = np.concatenate([(r.standard_normal(4096) * 6), [-120.0, -30.0, 0.0, 30.0, 120.0]]).astype(np.float32)
    z = np.concatenate([r.uniform(0, 1, 4096), [0.0, 1.0, 0.5, 0.0, 1.0]]).astype(np.float32)
    val, grad = _run(hm[1], x, z, 1.0, 0.0)
    plain = np.array([hm[0].hm_bce(float(a), float(b)) for a, b in zip(x, z)], np.float32)
    assert np.array_equal(val.view(np.int32), plain.view(np.int32))
    with np.errstate(over="ignore"):
        s = (np.float32(1.0) / (np.float32(1.0) + np.exp(-x, dtype=np.float32))).astype(np.float32)
    np.testing.assert_allclose(grad, s - z, rtol=1e-6, atol=1e-7)
