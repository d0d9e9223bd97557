"""Generates tests/golden/confusion_<case>.npz from the LIVE, UNMODIFIED reference's utils.metrics.ConfusionMatrix (imported
through oracle/ref_harness.py).  Needs the reference checkout:  python tests/golden/make_golden_confusion.py
The images are re-created from seeds by tests/confusion_port.golden_cases(); only the matrices are stored.  No case has an
IoU tie that decides a match: the reference sorts with numpy's argsort, which is not stable in general."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import confusion_port  # noqa: E402
from oracle import ref_harness  # noqa: E402


def main():
    ref_harness.load_reference()
    import torch
    from utils.metrics import ConfusionMatrix
    for name, (nc, images) in confusion_port.golden_cases().items():
        cm = ConfusionMatrix(nc=nc)
        for det, lab in images:
            assert confusion_port.deciding_ties(det, lab) == 0, name
            cm.process_batch(torch.from_numpy(det), torch.from_numpy(lab))
        np.savez_compressed(os.path.join(HERE, "confusion_%s.npz" % name), matrix=cm.matrix)
        print(name, len(images), "images, %d counts, %d on the diagonal" % (cm.matrix.sum(), np.trace(cm.matrix[:nc, :nc])))


if __name__ == "__main__":
    main()
