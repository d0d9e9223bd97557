"""CPU: the native loss mirrors construct from the live reference's own config tree carrying every loss option they
accept (Loss.fl_gamma / cls_pw / obj_pw / autobalance / label_smoothing / single_targets, SSOD.uncertain_aug=False) and
take the same derived settings as the reference's ComputeLoss / ComputeStudentMatchLoss (ssi, balance, smoothed targets,
the assigner's single_targets flag); SSOD.focal_loss > 0 is refused by both (the reference with NameError: FocalLoss is
not imported in ssod_loss.py), as are SimOTA and SSOD.use_ota.  Runs in a subprocess (loading the reference patches
torch process-wide); needs the reference checkout (skipped where it is absent)."""
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
    ns = ref_harness.load_reference()
    import torch
    from efficientteacher_b200.loss import ComputeLoss
    from efficientteacher_b200.ssod_loss import ComputeStudentMatchLoss
    from tiny_cfg import HeadOnlyModel

    YAML = "configs/ssod/coco-standard/yolov5l_coco_ssod_10_percent.yaml"
    SMALL = ["Model.depth_multiple", 0.33, "Model.width_multiple", 0.50]
    ALL = ["Loss.fl_gamma", 1.5, "Loss.cls_pw", 2.0, "Loss.obj_pw", 0.5, "Loss.autobalance", True,
           "Loss.label_smoothing", 0.1, "Loss.single_targets", True, "SSOD.uncertain_aug", False]
    torch.manual_seed(0)
    cfg = ref_harness.make_cfg(YAML, SMALL + ALL)
    rmodel = ns.SSODModel(cfg)
    model = HeadOnlyModel()
    for mine, ref in ((ComputeLoss(model, cfg), ns.ComputeLoss(rmodel, cfg)),
                      (ComputeStudentMatchLoss(model, cfg), ns.ComputeStudentMatchLoss(rmodel, cfg))):
        assert mine.ssi == ref.ssi == 1, (mine.ssi, ref.ssi)
        assert (mine.cp, mine.cn) == (ref.cp, ref.cn)
        assert list(mine.balance) == list(ref.balance)
        assert mine.assigner.single_targets == ref.assigner.single_targets == True
        assert float(ref.BCEcls.pos_weight if hasattr(ref.BCEcls, "pos_weight") else ref.BCEcls.loss_fcn.pos_weight) == mine.cls_pw
        assert (mine.box_w, mine.obj_w) == (ref.box_w, ref.obj_w) and abs(mine.cls_w - ref.cls_w) < 1e-12
    sup = ComputeLoss(model, cfg)
    assert sup.autobalance and sup.fl_gamma == 1.5 and (sup.cls_pw, sup.obj_pw) == (2.0, 0.5)
    assert type(ns.ComputeLoss(rmodel, cfg).BCEobj).__name__ == "FocalLoss"
    sup.balance = [2.0, 1.0, 0.5]                           # the setter uploads in place
    assert sup.balance == [2.0, 1.0, 0.5] and sup.balance_state.dtype == torch.float64

    for k, v in (("SSOD.focal_loss", 1.5),):
        bad = ref_harness.make_cfg(YAML, SMALL + [k, v])
        try:
            ns.ComputeStudentMatchLoss(rmodel, bad)
            raise AssertionError("reference accepted " + k)
        except NameError:
            pass
        try:
            ComputeStudentMatchLoss(model, bad)
            raise AssertionError("mirror accepted " + k)
        except NotImplementedError as e:
            assert "NameError" in str(e)
    for k, v, cls in (("Loss.assigner_type", "SimOTA", ComputeLoss), ("SSOD.use_ota", True, ComputeStudentMatchLoss)):
        try:
            cls(model, ref_harness.make_cfg(YAML, SMALL + [k, v]))
            raise AssertionError("mirror accepted " + k)
        except NotImplementedError:
            pass
    print("LOSS_OPTIONS_OK")
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "models")), reason="reference checkout not present")
def test_mirrors_accept_the_reference_loss_options():
    env = dict(os.environ, WANDB_MODE="disabled", PYTHONDONTWRITEBYTECODE="1")
    tests = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", SCRIPT % (ROOT, tests)], capture_output=True, text=True, timeout=600, env=env,
                       cwd=ROOT)
    assert r.returncode == 0 and "LOSS_OPTIONS_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
