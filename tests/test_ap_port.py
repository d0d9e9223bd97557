"""CPU: tests/ap_port.ap_per_class (the stable-sort restatement the native ap_per_class follows) against the golden outputs of
the live reference's utils.metrics.ap_per_class (tests/golden/ap_per_class.npz, tests/golden/make_golden_val.py)."""
import numpy as np
import pytest

import ap_port

KEYS = ("p", "r", "ap", "f1", "ap_class", "cls_thr")


@pytest.mark.parametrize("name", ["mixed", "alltp_allfp", "np1", "nc1", "big"])
def test_port_matches_reference_golden(golden, name):
    g = golden("ap_per_class")
    got = ap_port.ap_per_class(*ap_port.golden_cases()[name])
    for k, v in zip(KEYS, got):
        want = g[name + "_" + k]
        v = np.asarray(v)
        assert v.dtype == want.dtype and v.shape == want.shape, (name, k, v.dtype, want.dtype, v.shape, want.shape)
        assert np.array_equal(v, want), (name, k)


def test_golden_cases_cover_the_edges():
    cases = ap_port.golden_cases()
    tp, conf, pcls, tcls = cases["mixed"]
    assert set(np.unique(tcls)) - set(np.unique(pcls)) == {3, 11, 42}        # labels, no predictions
    assert set(np.unique(pcls)) - set(np.unique(tcls)) == {75, 76, 77, 78, 79}  # predictions, no labels
    tp, conf, pcls, tcls = cases["alltp_allfp"]
    assert tp[pcls == 0].all() and not tp[pcls == 1].any()
    tp, conf, pcls, tcls = cases["np1"]
    assert (pcls == 0).sum() == 1
    assert np.unique(cases["nc1"][3]).size == 1 and cases["big"][0].shape[0] == 300000
    for name, (tp, conf, pcls, tcls) in cases.items():
        assert np.unique(conf).size == conf.size, name
