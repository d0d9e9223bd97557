"""CPU: the YOLOv5 sizes the reference ships (n, s, m, l, x) against the live reference (tests/golden/model_keys_sizes.npz and
trunk_m.npz, written by tests/golden/make_golden_sizes.py): the config presets carry the reference's multipliers, this
package's models have the reference's state_dict keys and shapes at n, m and x, and oracle/trunk_ref.TrunkRef -- the
reference the GPU tests at these widths compare with -- reproduces the reference's outputs at YOLOv5m width."""
import pytest
import torch

from golden.make_golden_sizes import DEPTH, NECK_DEPTH, SIZES, initial_state_dict
from golden.make_golden_trunk import trunk_inputs
from test_trunk_ref_vs_reference import _check_sampled


def _want(g, name):
    keys, ndim, dims, dtypes = list(g[name + "_keys"]), g[name + "_ndim"], list(g[name + "_dims"]), list(g[name + "_dtypes"])
    shapes, o = [], 0
    for n in ndim:
        shapes.append(dims[o:o + n])
        o += n
    return keys, dict(zip(keys, zip(shapes, dtypes)))


@pytest.mark.parametrize("size", SIZES)
def test_presets_carry_the_reference_multipliers(size, golden):
    from efficientteacher_b200.config import SIZES as PRESETS
    assert PRESETS[size] == tuple(golden("model_keys_sizes")["mult_" + size].tolist())


def test_shallow_presets_keep_the_widths():
    from efficientteacher_b200.config import SIZES as PRESETS
    for s in ("l", "m", "x"):
        assert PRESETS[s + "_shallow"] == (0.33, PRESETS[s][1])
    # the presets that existed before keep their values
    assert [PRESETS[s] for s in ("l", "s", "m", "l_shallow")] == [(1.0, 1.0), (0.33, 0.50), (0.67, 0.75), (0.33, 1.0)]


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("kind", ["sup", "ssod"])
def test_model_state_dict_keys_equal_reference(size, kind, golden):
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.model import Model, SupModel
    mine = SupModel(yolov5_sup_cfg(size)) if kind == "sup" else Model(yolov5_ssod_cfg(size))
    keys, want = _want(golden("model_keys_sizes"), "%s_%s" % (kind, size))
    sd = mine.state_dict()
    assert list(sd.keys()) == keys
    for k, v in sd.items():
        assert list(v.shape) == list(want[k][0]), k
        assert str(v.dtype) == want[k][1], k


@pytest.mark.parametrize("size", ["m", "x"])
def test_sizes_have_widths_that_are_not_powers_of_two(size):
    """what the kernels must handle: BatchNorm widths with C/8 not a power of two, conv inputs not a multiple of 64"""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Conv, Model
    convs = [m for m in Model(yolov5_ssod_cfg(size + "_shallow")).modules() if isinstance(m, Conv)]
    couts = {m.conv.out_channels for m in convs}
    assert all(c % 8 == 0 and c // 8 <= 256 for c in couts)
    assert any((c // 8) & (c // 8 - 1) for c in couts)
    assert any(m.conv.in_channels % 64 and m.conv.in_channels > 64 for m in convs)


def test_trunk_ref_equals_live_reference_at_yolov5m_width(golden):
    from oracle.trunk_ref import TrunkRef
    g = golden("trunk_m")
    sd = initial_state_dict()
    assert sd["backbone.stage2_1.conv.weight"].shape[0] == 96
    x, x2 = trunk_inputs()
    with torch.no_grad():
        raw, feat = TrunkRef(sd, DEPTH, NECK_DEPTH).forward(x, train=False)
    _check_sampled(raw, g, "eval_raw")
    _check_sampled(feat, g, "eval_feat")
    sd_t = {k: v.clone() for k, v in sd.items()}
    raw, feat = TrunkRef(sd_t, DEPTH, NECK_DEPTH, bn_momentum=0.03).forward(x2, train=True)
    _check_sampled(raw, g, "train_raw")
    _check_sampled(feat, g, "train_feat")
    _check_sampled([torch.cat([sd_t[k].reshape(-1) for k in sd_t if "running_" in k])], g, "running")

    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import Model
    r = TrunkRef.from_module(Model(yolov5_ssod_cfg("m_shallow")))
    assert (r.depth, r.neck_depth) == (DEPTH, NECK_DEPTH)
