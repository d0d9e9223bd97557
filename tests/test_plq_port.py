"""CPU: tests/plq_port.py (the restatement of check_pseudo_label_with_gt / check_pseudo_label that the native etb_pl_quality
follows) reproduces the live reference's outputs in tests/golden/plq_*.npz exactly -- float64 equality and the reference's
return types; the bootstrap rebinds both functions where the reference's trainer binds them by name."""
import glob
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import plq_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ETB_REFERENCE_ROOT", "/root/reference")
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "plq_*.npz")))
GT_KEYS = ("tp", "fp_cls", "fp_loc", "pse_num", "gt_num")
NOGT_KEYS = ("precision", "recall", "pse_num", "reliable_num")


def load(path):
    z = np.load(path)
    thr = (list(z["thr_low"]), list(z["thr_high"])) if bool(z["has_thr"]) else (None, None)
    return z, thr, int(z["bs"])


def assert_same(got, z, prefix, keys):
    assert len(got) == len(keys)
    for v, k in zip(got, keys):
        want = z[prefix + k]
        if bool(z[prefix + k + "_is_int"]):
            assert isinstance(v, int) and v == int(want), (k, v, want)
        elif want.ndim:
            assert isinstance(v, np.ndarray) and v.dtype == np.float64 and np.array_equal(v, want), (k, v, want)
        else:
            assert isinstance(v, float) and v == float(want), (k, v, want)


def test_golden_cases_present():
    names = {os.path.basename(p)[4:-4] for p in GOLDEN}
    assert {"random_nc80", "nc1", "nc20", "ties", "boundary", "zero_uncertain", "zero_gt", "zero_rows", "thr_none",
            "iouv10"} <= names


@pytest.mark.parametrize("path", GOLDEN, ids=lambda p: os.path.basename(p)[:-4])
def test_port_reproduces_reference(path):
    z, (lo, hi), bs = load(path)
    labels = z["gt"].copy()
    got = plq_port.check_pseudo_label_with_gt(z["rows"], labels, z["iouv"], lo, hi, bs)
    assert_same(got, z, "gt_", GT_KEYS)
    assert np.array_equal(labels, z["gt"])                 # the restatement leaves the labels as they were
    if lo is not None:
        assert_same(plq_port.check_pseudo_label(z["rows"], lo, hi, bs), z, "nogt_", NOGT_KEYS)


def test_config_reads_with_gt_off():
    from efficientteacher_b200.config import yolov5_ssod_cfg
    assert yolov5_ssod_cfg('n').SSOD.ssod_hyp.with_gt is False      # configs/defaults.py:303


SCRIPT = textwrap.dedent('''
    import sys
    sys.path.insert(0, %r)
    from oracle import ref_harness
    ref_harness.load_reference()
    import efficientteacher_b200.bootstrap as bs
    from efficientteacher_b200 import pl_quality
    import trainer.ssod_trainer as S
    import utils.self_supervised_utils as U
    for mod in (S, U):
        assert mod.check_pseudo_label_with_gt is pl_quality.check_pseudo_label_with_gt, mod.__name__
        assert mod.check_pseudo_label is pl_quality.check_pseudo_label, mod.__name__
    assert "trainer.ssod_trainer.check_pseudo_label_with_gt" in bs.rebound and "trainer.ssod_trainer.check_pseudo_label" in bs.rebound
    print("PLQ_BOOTSTRAP_OK")
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "trainer")), reason="reference checkout not present")
def test_bootstrap_rebinds_pseudo_label_checks():
    env = dict(os.environ, WANDB_MODE="disabled", PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, "-c", SCRIPT % ROOT], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PLQ_BOOTSTRAP_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
