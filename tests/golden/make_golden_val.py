"""Generates tests/golden/ap_per_class.npz from the LIVE, UNMODIFIED reference's utils.metrics.ap_per_class (imported through
oracle/ref_harness.py).  Needs the reference checkout:  python tests/golden/make_golden_val.py
The inputs are re-created from seeds by tests/ap_port.golden_cases(); only the outputs are stored.  Every case has distinct
confidences: the reference sorts with numpy's unstable argsort."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import ap_port  # noqa: E402
from oracle import ref_harness  # noqa: E402


def main():
    ref_harness.load_reference()
    from utils.metrics import ap_per_class
    out = {}
    for name, (tp, conf, pcls, tcls) in ap_port.golden_cases().items():
        assert np.unique(conf).size == conf.size, name
        # names={}: the default names=() fails at metrics.py:75 (a tuple has no .items())
        p, r, ap, f1, ap_class, cls_thr = ap_per_class(tp, conf, pcls, tcls, plot=False, save_dir='.', names={})
        out.update({name + "_p": p, name + "_r": r, name + "_ap": ap, name + "_f1": f1, name + "_ap_class": ap_class,
                    name + "_cls_thr": np.asarray(cls_thr, dtype=np.float64)})
        print(name, tp.shape, "mAP@.5 %.6f" % ap[:, 0].mean())
    np.savez_compressed(os.path.join(HERE, "ap_per_class.npz"), **out)


if __name__ == "__main__":
    main()
