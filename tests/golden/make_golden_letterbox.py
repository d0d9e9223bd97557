"""Generates tests/golden/letterbox.npz from the LIVE, UNMODIFIED reference's letterbox (utils/augmentations.py, what
detect.py's LoadImages calls; imported through oracle/ref_harness.py).  Needs the reference checkout:
    python tests/golden/make_golden_letterbox.py
For every (h0, w0, S) of tests/letterbox_port.sweep(): the padded shape, ratio and (dw, dh) letterbox(auto=True) returns."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import letterbox_port  # noqa: E402
from oracle import ref_harness  # noqa: E402


def main():
    ref_harness.load_reference()
    from utils.augmentations import letterbox
    cases = np.asarray(letterbox_port.sweep(), dtype=np.int64)
    shape, ratio, pad = [], [], []
    for h0, w0, S in cases:
        im, r, (dw, dh) = letterbox(np.zeros((h0, w0, 3), np.uint8), int(S), auto=True, stride=32)
        shape.append(im.shape)
        ratio.append(r)
        pad.append((dw, dh))
    np.savez_compressed(os.path.join(HERE, "letterbox.npz"), cases=cases, shape=np.asarray(shape, np.int64),
                        ratio=np.asarray(ratio, np.float64), pad=np.asarray(pad, np.float64))
    print(len(cases), "cases")


if __name__ == "__main__":
    main()
