"""CPU: the ReLU and Hardswish YOLOv5 trunks against the live reference (tests/golden/trunk_act_*.npz, written by
tests/golden/make_golden_trunk_act.py): this package's Model builds the reference's activation module at every Conv, and
the activation-aware trunk reference (tests/trunk_act_ref.py) reproduces the reference's eval / train outputs and BN
running statistics."""
import numpy as np
import pytest
import torch

from golden.make_golden_trunk_act import DEPTH, MODES, NECK_DEPTH, SIZE, initial_state_dict
from golden.make_golden_trunk import trunk_inputs
from test_trunk_ref_vs_reference import _check_sampled
from trunk_act_ref import ACT_CLASS, ActTrunkRef, act_map


def _model(backbone_act, neck_act):
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    return Model(yolov5_ssod_cfg(SIZE, backbone_act=backbone_act, neck_act=neck_act))


def _conv_acts(model):
    from efficientteacher_b200.model import Conv
    return {n: m.act for n, m in model.named_modules() if isinstance(m, Conv)}


def _want(g):
    return dict(zip(g["conv_paths"].tolist(), g["conv_acts"].tolist()))


@pytest.mark.parametrize("mode", list(MODES))
def test_model_builds_reference_activation_modules(mode, golden):
    g = golden("trunk_act_" + mode)
    assert (str(g["backbone_act"]), str(g["neck_act"])) == MODES[mode]
    got = _conv_acts(_model(*MODES[mode]))
    want = _want(g)
    assert list(got) == list(want)
    assert {n: type(a).__name__ for n, a in got.items()} == want
    for n, a in got.items():              # get_activation (common.py:28-47) builds ReLU / Hardswish in place
        assert getattr(a, "inplace", True), n
    assert set(want.values()) >= {"ReLU"} and (mode == "relu") == ("Hardswish" not in want.values())


@pytest.mark.parametrize("mode", list(MODES))
def test_act_map_matches_reference(mode, golden):
    acts = act_map(*MODES[mode], DEPTH, NECK_DEPTH)
    assert {n: ACT_CLASS[a] for n, a in acts.items()} == {n: a for n, a in _want(golden("trunk_act_" + mode)).items()
                                                          if n.startswith(("backbone.", "neck."))}


@pytest.mark.parametrize("unknown", ["LeakyReLU", "Mish", "relu", ""])
def test_unknown_activation_string_selects_hardswish_like_the_reference(unknown, golden):
    """The reference's `else` branch: any string other than 'SiLU' / 'ReLU' builds the Hardswish trunk."""
    want = _want(golden("trunk_act_hswish"))
    assert {n: type(a).__name__ for n, a in _conv_acts(_model(unknown, unknown)).items()} == want


def test_default_silu_trunk_unchanged():
    """SiLU is still every Conv's activation by default, and the activation-aware reference reduces to TrunkRef."""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    from oracle.trunk_ref import TrunkRef
    assert {type(a).__name__ for a in _conv_acts(Model(yolov5_ssod_cfg(SIZE))).values()} == {"SiLU"}
    sd = initial_state_dict("relu")
    x = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        a, fa = TrunkRef(sd, DEPTH, NECK_DEPTH).forward(x)
        b, fb = ActTrunkRef(sd, DEPTH, NECK_DEPTH, acts=act_map("SiLU", "SiLU", DEPTH, NECK_DEPTH)).forward(x)
    for u, v in zip(a + fa, b + fb):
        assert torch.equal(u, v)


@pytest.mark.parametrize("mode", list(MODES))
def test_act_trunk_ref_equals_live_reference(mode, golden):
    g = golden("trunk_act_" + mode)
    acts = act_map(*MODES[mode], DEPTH, NECK_DEPTH)
    sd = initial_state_dict(mode)
    x, x2 = trunk_inputs()
    with torch.no_grad():
        raw, feat = ActTrunkRef(sd, DEPTH, NECK_DEPTH, acts=acts).forward(x, train=False)
    _check_sampled(raw, g, "eval_raw")
    _check_sampled(feat, g, "eval_feat")
    sd_t = {k: v.clone() for k, v in sd.items()}
    raw, feat = ActTrunkRef(sd_t, DEPTH, NECK_DEPTH, acts=acts, bn_momentum=0.03).forward(x2, train=True)
    _check_sampled(raw, g, "train_raw")
    _check_sampled(feat, g, "train_feat")
    _check_sampled([torch.cat([sd_t[k].reshape(-1) for k in sd_t if "running_" in k])], g, "running")


@pytest.mark.parametrize("mode", list(MODES))
def test_act_trunk_ref_for_model_resolves_the_cfg(mode):
    m = _model(*MODES[mode])
    r = ActTrunkRef.for_model(m)
    assert (r.depth, r.neck_depth) == (DEPTH, NECK_DEPTH)
    assert {n: ACT_CLASS[a] for n, a in r.acts.items()} == {n: type(a).__name__ for n, a in _conv_acts(m).items()}
    assert np.all([k in r.sd for k in m.state_dict()])
