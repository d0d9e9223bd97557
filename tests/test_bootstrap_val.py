"""CPU: with the live reference on sys.path, `import efficientteacher_b200.bootstrap` rebinds val.run and
utils.metrics.ap_per_class (also val.py's by-name binding) to wrappers; supported calls reach the native functions, every
other call the reference's own function (`__wrapped__`).  Runs in a subprocess: the patch is process-wide.  Needs the
reference checkout (skipped where it is absent)."""
import os
import subprocess
import sys
import textwrap

import pytest

from oracle.ref_harness import REF_ROOT as REF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import sys, types
    sys.path.insert(0, %r)
    from oracle import ref_harness
    ref_harness.load_reference()
    import torch
    import efficientteacher_b200.bootstrap as bs
    assert not bs.apply.skipped, bs.apply.skipped
    import val as V, utils.metrics as MT
    from efficientteacher_b200 import metrics as etb_metrics, val as etb_val
    assert V.run.__module__ == "efficientteacher_b200.bootstrap" and V.run.__wrapped__.__module__ == "val"
    assert MT.ap_per_class.__module__ == "efficientteacher_b200.bootstrap" and MT.ap_per_class.__wrapped__.__module__ == "utils.metrics"
    assert V.ap_per_class is MT.ap_per_class            # val.py's `from utils.metrics import ap_per_class`
    calls = []
    V.run.__wrapped__ = lambda *a, **k: calls.append(("reference", k)) or "ref"
    etb_val.run = lambda *a, **k: calls.append(("native", k)) or "native"

    class FakeParam:
        device = torch.device("cuda", 0)

    class FakeModel:
        def parameters(self):
            return iter([FakeParam()])

    m = FakeModel()
    # trainer/ssod_trainer.py:339-352: the training-time call
    assert V.run({}, batch_size=32, imgsz=640, model=m, conf_thres=0.001, single_cls=False, dataloader=[], save_dir=".",
                 plots=False, callbacks=None, compute_loss=None, num_points=0, val_ssod=True, val_kp=False) == "native"
    assert V.run({}, None, 32, 640, model=m, dataloader=[], plots=False) == "native"     # positional arguments bind the same
    # every other call: plots, txt / json output, keypoints, a CPU model, the standalone call, model_post, augment
    for kw in (dict(plots=True), dict(plots=False, save_txt=True), dict(plots=False, save_json=True), dict(plots=False, save_hybrid=True),
               dict(plots=False, num_points=4), dict(plots=False, model_post=object()), dict(plots=False, augment=True)):
        assert V.run({}, model=m, dataloader=[], **kw) == "ref", kw
    assert V.run({}, model=torch.nn.Linear(2, 2), dataloader=[], plots=False) == "ref"
    assert V.run({}, weights="x.pt") == "ref"
    assert V.run({}, no_such_argument=1) == "ref"
    assert [c[0] for c in calls] == ["native", "native"] + ["reference"] * 10, calls
    calls.clear()
    MT.ap_per_class.__wrapped__ = lambda *a, **k: calls.append("reference") or "ref"
    etb_metrics.ap_per_class = lambda *a, **k: calls.append("native") or "native"
    assert MT.ap_per_class(1, 2, 3, 4) == "native" and MT.ap_per_class(1, 2, 3, 4, plot=True, save_dir=".", names={}) == "ref"
    assert calls == ["native", "reference"], calls
    assert bs.apply() == []
    print("BOOTSTRAP_VAL_OK")
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "trainer")), reason="reference checkout not present")
def test_bootstrap_routes_val_run_and_ap_per_class():
    env = dict(os.environ, WANDB_MODE="disabled", PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, "-c", SCRIPT % ROOT], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "BOOTSTRAP_VAL_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_run_unsupported_rules():
    import torch
    from efficientteacher_b200 import val

    class P:
        device = torch.device("cuda", 0)

    class M:
        def parameters(self):
            return iter([P()])

    assert val.run_unsupported(model=M(), dataloader=[], plots=False) is None
    assert val.run_unsupported(model=M(), dataloader=[]) == "plots=True"        # the reference's default
    assert val.run_unsupported(model=None, dataloader=[], plots=False)
    assert val.run_unsupported(model=M(), dataloader=None, plots=False)
    assert val.run_unsupported(model=torch.nn.Linear(2, 2), dataloader=[], plots=False) == "model is not on a CUDA device"
    assert val.run_unsupported(model=M(), dataloader=[], plots=False, num_points=4)
