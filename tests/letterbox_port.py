"""numpy restatement of etb_letterbox_u8's integer arithmetic (csrc/letterbox.cu), the oracle of its tests: cv2.resize
(INTER_LINEAR, 8UC3) as OpenCV's x86 build computes it, copyMakeBorder(114), BGR -> RGB and HWC -> CHW.  Also the sweep of
frame sizes the CPU and GPU tests share."""
import numpy as np


def _coefs(dst, src, clamp):
    """source indices (s, s + 1) and 11-bit coefficients of every destination column (clamp=True) or row (clamp=False)"""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:                                   # columns: the edge taps get coefficient 0; rows keep their fraction
        m = s < 0
        f[m], s[m] = 0, 0
        m = s >= src - 1
        f[m], s[m] = 0, src - 1
    c0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int32)
    c1 = np.rint(f * np.float32(2048)).astype(np.int32)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), c0, c1


def resize_linear(img, new_h, new_w):
    """cv2.resize(img, (new_w, new_h), interpolation=cv2.INTER_LINEAR) for uint8 [h0, w0, 3]"""
    h0, w0, _ = img.shape
    x = img.astype(np.int32)
    if 2 * new_h == h0 and 2 * new_w == w0:      # OpenCV takes INTER_AREA for an exact 2x downscale
        return ((x[0::2, 0::2] + x[0::2, 1::2] + x[1::2, 0::2] + x[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    x0, x1, a0, a1 = _coefs(new_w, w0, True)
    y0, y1, b0, b1 = _coefs(new_h, h0, False)
    rows = x[:, x0] * a0[None, :, None] + x[:, x1] * a1[None, :, None]
    S0, S1 = rows[y0], rows[y1]
    out = ((((S0 >> 4) * b0[:, None, None]) >> 16) + (((S1 >> 4) * b1[:, None, None]) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def letterbox_chw(img, geom):
    """uint8 [h0, w0, 3] BGR and letterbox_geometry(...) -> uint8 [3, H, W] RGB, what etb_letterbox_u8 writes"""
    new_h, new_w, top, left, H, W = geom[:6]
    r = img if img.shape[:2] == (new_h, new_w) else resize_linear(img, new_h, new_w)
    out = np.full((H, W, 3), 114, np.uint8)
    out[top:top + new_h, left:left + new_w] = r
    return np.ascontiguousarray(out[:, :, ::-1].transpose(2, 0, 1))


def sweep(n=2000, seed=0):
    """(h0, w0, S): n seeded random sizes in 1..2000 over S in {320, 640, 1280}, plus exact 2x downscales, upscales, one-pixel
    rows and columns, and frames already at size.  Sizes whose resized side rounds to 0 pixels are left out: letterbox
    cannot take them (cv2.resize rejects an empty size)."""
    r = np.random.RandomState(seed)
    cases = [(int(h), int(w), int(s)) for h, w, s in zip(r.randint(1, 2001, n), r.randint(1, 2001, n), r.choice([320, 640, 1280], n))]
    for S in (320, 640, 1280):
        cases += [(2 * S, 2 * S, S), (2 * S, S, S), (S, 2 * S, S), (S, S, S), (S, S // 2, S), (S // 4, S // 4, S), (1, 1, S),
                  (1, S + S // 2, S), (S + S // 2, 1, S), (1, S, S), (S, 1, S), (7, 3, S), (S - 1, S + 1, S)]
    return [(h, w, s) for h, w, s in cases if min(round(h * min(s / h, s / w)), round(w * min(s / h, s / w))) >= 1]
