"""CPU: with the live reference on sys.path, `import efficientteacher_b200.bootstrap` rebinds utils.metrics.ConfusionMatrix
and val.py's by-name binding to a subclass of the native efficientteacher_b200.metrics.ConfusionMatrix: CPU tensors run the
reference's own process_batch and give its matrix, plot is the reference's, and apply() stays idempotent.  Runs in a
subprocess: the patch is process-wide.  Needs the reference checkout (skipped where it is absent)."""
import os
import subprocess
import sys
import textwrap

import pytest

from oracle.ref_harness import REF_ROOT as REF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import sys
    sys.path.insert(0, %r)
    sys.path.insert(0, %r)
    from oracle import ref_harness
    ref_harness.load_reference()
    import numpy as np, torch
    import utils.metrics as MT
    import efficientteacher_b200.bootstrap as bs
    assert not bs.apply.skipped, bs.apply.skipped
    import val as V
    from efficientteacher_b200 import metrics as etb_metrics
    import confusion_port as cp
    original = MT.ConfusionMatrix.__wrapped__
    assert original.__module__ == "utils.metrics" and MT.ConfusionMatrix.__module__ == "efficientteacher_b200.bootstrap"
    assert issubclass(MT.ConfusionMatrix, etb_metrics.ConfusionMatrix)
    assert V.ConfusionMatrix is MT.ConfusionMatrix         # val.py's `from utils.metrics import ... ConfusionMatrix`
    assert "utils.metrics.ConfusionMatrix" in bs.rebound and "val.ConfusionMatrix" in bs.rebound
    for name, (nc, images) in cp.golden_cases().items():
        cm, ref = MT.ConfusionMatrix(nc=nc), original(nc=nc)
        for det, lab in images:
            cm.process_batch(torch.from_numpy(det), torch.from_numpy(lab))
            ref.process_batch(torch.from_numpy(det), torch.from_numpy(lab))
        assert np.array_equal(cm.matrix, ref.matrix), name
        assert np.array_equal(cm.matrix, np.load(%r %% name)["matrix"]), name
    assert cm.host_plot.__func__ is original.plot
    cm.reset()
    assert not cm.matrix.any()
    assert bs.apply() == []
    assert MT.ConfusionMatrix.__wrapped__ is original
    print("BOOTSTRAP_CONFUSION_OK")
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "trainer")), reason="reference checkout not present")
def test_bootstrap_rebinds_confusion_matrix():
    env = dict(os.environ, WANDB_MODE="disabled", PYTHONDONTWRITEBYTECODE="1")
    gold = os.path.join(ROOT, "tests", "golden", "confusion_%s.npz")
    r = subprocess.run([sys.executable, "-c", SCRIPT % (ROOT, os.path.join(ROOT, "tests"), gold)], capture_output=True, text=True,
                       timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "BOOTSTRAP_CONFUSION_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_native_class_surface_without_a_device():
    """what the native class does before any batch: a zero float64 matrix, print(), reset(), and plot()'s warning line"""
    import numpy as np
    from efficientteacher_b200 import metrics
    cm = metrics.ConfusionMatrix(3)
    assert cm.matrix.dtype == np.float64 and cm.matrix.shape == (4, 4) and not cm.matrix.any()
    assert (cm.conf, cm.iou_thres) == (0.25, 0.45)
    cm.reset()
    cm.print()
    cm.plot(save_dir=".", names=["a", "b", "c"])
    with pytest.raises(ValueError):
        metrics.ConfusionMatrix(0)
