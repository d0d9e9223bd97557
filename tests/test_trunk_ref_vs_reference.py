"""CPU: oracle/trunk_ref.TrunkRef (the fp32 trunk the wgmma kernels and the CPU step are compared with) against the
unmodified reference modules (models/detector/yolo_ssod.py:105-118 + backbone/neck/head) on the same state_dict and input:
the same outputs in eval and in train mode, the same BN running statistics after the train pass, and this repo's Model has
exactly the reference's state_dict keys / shapes.  The reference's side is stored in tests/golden/trunk_ref.npz and
model_keys.npz (tests/golden/make_golden_trunk.py ran it on this package's seeded initial weights)."""
import numpy as np
import pytest
import torch

from golden.make_golden_trunk import initial_state_dict, trunk_inputs


def _check_sampled(got, g, prefix):
    for i, t in enumerate(got):
        assert list(t.shape) == list(g["%s%d_shape" % (prefix, i)]), (prefix, i)
        want = g["%s%d" % (prefix, i)]
        have = t.detach().reshape(-1).numpy()[g["%s%d_idx" % (prefix, i)]]
        # fp32 CPU convolutions may pick other kernels on another CPU: last-bit differences, compounded over the trunk
        np.testing.assert_allclose(have, want, rtol=1e-4, atol=1e-5 * max(float(np.abs(want).max()), 1e-3), err_msg="%s%d" % (prefix, i))
    assert "%s%d" % (prefix, len(got)) not in g.files, prefix


@pytest.mark.parametrize("yaml_rel,depth,nd", [("configs/ssod/coco-standard/yolov5l_coco_ssod_10_percent.yaml", (3, 6, 9, 3), 3)])
def test_trunk_ref_equals_live_reference(yaml_rel, depth, nd, golden):
    from oracle.trunk_ref import TrunkRef
    g = golden("trunk_ref")
    sd = initial_state_dict()
    x, x2 = trunk_inputs()
    # eval (teacher pass): reference returns ((pred, raw_list), features)
    with torch.no_grad():
        raw, feat = TrunkRef(sd, depth, nd).forward(x, train=False)
    _check_sampled(raw, g, "eval_raw")
    _check_sampled(feat, g, "eval_feat")
    # train (student pass): batch statistics + running-stat update with the reference's momentum 0.03
    sd_t = {k: v.clone() for k, v in sd.items()}
    raw, feat = TrunkRef(sd_t, depth, nd, bn_momentum=0.03).forward(x2, train=True)
    _check_sampled(raw, g, "train_raw")
    _check_sampled(feat, g, "train_feat")
    _check_sampled([torch.cat([sd_t[k].reshape(-1) for k in sd_t if "running_" in k])], g, "running")


def test_model_state_dict_keys_equal_reference(golden):
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.model import Model, SupModel
    g = golden("model_keys")
    for name, mine, ordered in (("ssod_l", Model(yolov5_ssod_cfg('l')), True), ("sup_s", SupModel(yolov5_sup_cfg('s')), False)):
        sd = mine.state_dict()
        keys, ndim, dims, dtypes = list(g[name + "_keys"]), g[name + "_ndim"], list(g[name + "_dims"]), list(g[name + "_dtypes"])
        shapes, o = [], 0
        for n in ndim:
            shapes.append(dims[o:o + n])
            o += n
        want = dict(zip(keys, zip(shapes, dtypes)))
        if ordered:
            assert list(sd.keys()) == keys
        else:
            assert sorted(sd.keys()) == sorted(keys)
        for k, v in sd.items():
            assert list(v.shape) == list(want[k][0]), k
            if ordered:
                assert str(v.dtype) == want[k][1], k
