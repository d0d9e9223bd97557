"""CPU: the letterbox of detect.py's path (efficientteacher_b200/detect.py, csrc/letterbox.cu) without a GPU.

  * the host geometry equals the live reference's letterbox(auto=True) -- padded shape, ratio and (dw, dh) -- on the sweep
    of tests/letterbox_port.py (tests/golden/letterbox.npz);
  * the numpy restatement of the kernel's integer arithmetic equals cv2.resize(INTER_LINEAR) + copyMakeBorder(114), BGR ->
    RGB, HWC -> CHW, byte for byte, on the same sweep."""
import numpy as np
import pytest

import letterbox_port


def test_geometry_matches_reference_golden(golden):
    from efficientteacher_b200.detect import letterbox_geometry
    g = golden("letterbox")
    assert [tuple(c) for c in g["cases"]] == letterbox_port.sweep()
    for (h0, w0, S), shape, ratio, pad in zip(g["cases"], g["shape"], g["ratio"], g["pad"]):
        new_h, new_w, top, left, H, W, r, dw, dh = letterbox_geometry(int(h0), int(w0), int(S))
        assert (H, W, 3) == tuple(shape) and (r, r) == tuple(ratio) and (dw, dh) == tuple(pad), (h0, w0, S)
        assert 0 <= top <= H - new_h and 0 <= left <= W - new_w and H % 32 == 0 and W % 32 == 0


def test_geometry_refuses_empty_frames():
    from efficientteacher_b200.detect import letterbox_geometry
    with pytest.raises(ValueError):
        letterbox_geometry(1, 1999, 320)


def test_restatement_matches_cv2_byte_for_byte():
    cv2 = pytest.importorskip("cv2")
    from efficientteacher_b200.detect import letterbox_geometry
    r = np.random.RandomState(1)
    for h0, w0, S in letterbox_port.sweep():
        img = np.frombuffer(bytearray(r.bytes(h0 * w0 * 3)), np.uint8).reshape(h0, w0, 3)
        geom = letterbox_geometry(h0, w0, S)
        new_h, new_w, top, left, H, W = geom[:6]
        want = img if (h0, w0) == (new_h, new_w) else cv2.resize(img, (new_w, new_h), interpolation=cv2.INTER_LINEAR)
        want = cv2.copyMakeBorder(want, top, H - new_h - top, left, W - new_w - left, cv2.BORDER_CONSTANT, value=(114, 114, 114))
        got = letterbox_port.letterbox_chw(img, geom)
        assert np.array_equal(got, want[:, :, ::-1].transpose(2, 0, 1)), (h0, w0, S)
