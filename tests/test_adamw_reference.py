"""CPU: the optimizer the native steps build equals the one the live reference builds (trainer/trainer.py:193-247
Trainer.build_optimizer, trainer/ssod_trainer.py:86-94 SSODTrainer.build_optimizer), for `adam` on and off and
`SSOD.multi_step_lr` on and off: the same parameter groups in the same order with the same hyper-parameters, and the same
learning rate per epoch over 26 epochs of scheduler steps.  Both build_optimizer methods are called unbound on stub
steps that hold one small module with conv, bias and BatchNorm parameters.  Runs in a subprocess (loading the reference
patches torch process-wide); needs the reference checkout (skipped where it is absent).  Also: the ctypes mirror of
EtbChunk, the chunk record of the AdamW (and SGD, EMA) kernel, has the C layout."""
import ctypes as C
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
    sys.modules["wandb"] = None          # the reference's loggers would otherwise try to log in to wandb
    from oracle import ref_harness
    ref_harness.load_reference()
    import torch
    import torch.nn as nn
    import trainer.trainer as RT
    import trainer.ssod_trainer as RS
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.optim import FusedAdamW, FusedSGD
    from efficientteacher_b200.trainer import SSODTrainerStep, SupTrainerStep

    HYPER = ("lr", "initial_lr", "momentum", "dampening", "nesterov", "betas", "eps", "weight_decay")

    def module():
        torch.manual_seed(0)
        return nn.Sequential(nn.Conv2d(3, 8, 3, bias=False), nn.BatchNorm2d(8), nn.Conv2d(8, 8, 1, bias=True),
                             nn.BatchNorm2d(8), nn.Conv2d(8, 4, 1, bias=True))

    def stub(cls, model, epochs, batch_size):
        s = cls.__new__(cls)
        s.model, s.epochs, s.epoch, s.batch_size, s.cuda, s.opt_scales = model, epochs, 0, batch_size, False, None
        return s

    checked = 0
    for ssod in (True, False):
        for adam in (True, False):
            for multi_step in ((True, False) if ssod else (False,)):
                for batch_size in (16, 48):
                    cfg = yolov5_ssod_cfg("n") if ssod else yolov5_sup_cfg("n")
                    cfg.adam, cfg.SSOD.multi_step_lr = adam, multi_step
                    cfg.hyp.lr0, cfg.hyp.lrf = 0.01, 0.1                 # lrf < 1: the schedule actually moves
                    cfg.Model.RepOpt = False
                    m = module()
                    ref = stub(RS.SSODTrainer if ssod else RT.Trainer, m, 30, batch_size)
                    nat = stub(SSODTrainerStep if ssod else SupTrainerStep, m, 30, batch_size)
                    (RS.SSODTrainer if ssod else RT.Trainer).build_optimizer(ref, cfg)
                    (SSODTrainerStep if ssod else SupTrainerStep).build_optimizer(nat, cfg)
                    what = "ssod=%%s adam=%%s multi_step_lr=%%s bs=%%d" %% (ssod, adam, multi_step, batch_size)
                    assert type(ref.optimizer) is (torch.optim.AdamW if adam else torch.optim.SGD), what
                    assert type(nat.optimizer) is (FusedAdamW if adam else FusedSGD), what
                    assert type(nat.scheduler) is type(ref.scheduler), (what, type(nat.scheduler), type(ref.scheduler))
                    assert nat.accumulate == ref.accumulate, what
                    assert len(nat.optimizer.param_groups) == len(ref.optimizer.param_groups) == 3, what
                    for gi, (gn, gr) in enumerate(zip(nat.optimizer.param_groups, ref.optimizer.param_groups)):
                        assert [id(p) for p in gn["params"]] == [id(p) for p in gr["params"]], (what, gi)
                        assert len(gn["params"]) > 0, (what, gi)
                        for k in HYPER:
                            assert (k in gn) == (k in gr), (what, gi, k)
                            if k in gr:
                                assert gn[k] == gr[k], (what, gi, k, gn[k], gr[k])
                        if adam:               # AdamW state dicts load both ways: the groups carry the same keys
                            assert set(gn) == set(gr), (what, gi, set(gn) ^ set(gr))
                            assert "momentum" not in gn, (what, gi)
                    if adam:
                        assert nat.optimizer.param_groups[0]["weight_decay"] == 0.01 == nat.optimizer.param_groups[2]["weight_decay"]
                    lrs_ref, lrs_nat = [], []
                    for epoch in range(26):
                        lrs_ref.append([g["lr"] for g in ref.optimizer.param_groups])
                        lrs_nat.append([g["lr"] for g in nat.optimizer.param_groups])
                        ref.scheduler.step()
                        nat.scheduler.step()
                    assert lrs_nat == lrs_ref, (what, lrs_nat, lrs_ref)
                    if multi_step:             # milestones [10, 20]: two drops by 10x over the 26 epochs
                        assert lrs_nat[25][0] < lrs_nat[15][0] < lrs_nat[5][0], what
                    checked += 1
    assert checked == 12, checked
    print("ok", checked)
''')


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "trainer")), reason="reference checkout not present")
def test_optimizer_and_schedule_match_reference_build_optimizer():
    env = dict(os.environ, WANDB_MODE="disabled")
    r = subprocess.run([sys.executable, "-c", SCRIPT % ROOT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "ok 12" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]


def test_chunk_layout_matches_c(tmp_path):
    from efficientteacher_b200 import _lib
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "etb200.h"\nint main(){printf("%zu %zu %zu %zu\\n", '
           'sizeof(EtbChunk), offsetof(EtbChunk, t[3]), offsetof(EtbChunk, n), offsetof(EtbChunk, group));'
           'return 0;}')
    c = tmp_path / "sz.c"
    c.write_text(src)
    exe = str(tmp_path / "sz")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).decode().split()]
    S = _lib.EtbChunk
    assert got == [C.sizeof(S), S.t.offset + 3 * C.sizeof(C.c_void_p), S.n.offset, S.group.offset]
