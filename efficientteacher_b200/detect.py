"""Batched inference on raw frames: the reference's detect.py loop (detect.py:150-240) for a list of frames at once.

One call: the frames go to the device (pinned copies, no host sync), the letterbox geometry of utils/datasets.py letterbox
(auto=True, scaleup=True, stride 32) is computed on the host, and the frames are grouped by letterboxed shape (auto=True
gives every aspect ratio its own shape; the frames of a video share one).  Each group runs etb_letterbox_u8 (cv2.resize
INTER_LINEAR + copyMakeBorder(114) + BGR -> RGB + HWC -> CHW, bit for bit), the model's engine forward, the best-class NMS
and etb_detect_rescale (scale_coords(...).round()).  The detection counts are read back once per call."""

import numpy as np
import torch

from . import _lib
from . import nms as etb_nms
from .val import _image_meta, _to_device

STRIDE = 32
_FRAME = np.dtype(_lib.EtbLetterboxFrame)


def letterbox_geometry(h0, w0, img_size=640, stride=STRIDE):
    """utils/datasets.py letterbox(auto=True, scaleup=True) for a (h0, w0) frame, with Python's round-half-even ->
    (new_h, new_w, top, left, H, W, r, dw, dh): the resized size, its offset in the padded H x W image, and the reference's
    return values ratio = (r, r) and (dw, dh)."""
    r = min(img_size / h0, img_size / w0)
    new_w, new_h = int(round(w0 * r)), int(round(h0 * r))
    dw, dh = (img_size - new_w) % stride / 2, (img_size - new_h) % stride / 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    if new_h < 1 or new_w < 1:
        raise ValueError("Predictor: a %dx%d frame letterboxes to an empty image at img_size %d" % (h0, w0, img_size))
    return new_h, new_w, top, left, new_h + top + bottom, new_w + left + right, r, dw, dh


def letterbox_batch(frames, geoms, H, W):
    """frames: uint8 [h0, w0, 3] BGR CUDA tensors; geoms: their letterbox_geometry, all of padded size H x W -> the uint8
    [B, 3, H, W] RGB batch (one etb_letterbox_u8 launch).  The frames must stay alive until the launch has run."""
    dev = frames[0].device
    tab = np.zeros(len(frames), dtype=_FRAME)
    tab["src"] = [f.data_ptr() for f in frames]
    tab["h0"] = [f.shape[0] for f in frames]
    tab["w0"] = [f.shape[1] for f in frames]
    for k, name in enumerate(("new_h", "new_w", "top", "left")):
        tab[name] = [g[k] for g in geoms]
    table = _to_device(np.frombuffer(tab.tobytes(), dtype=np.uint8), dev)
    out = torch.empty((len(frames), 3, H, W), dtype=torch.uint8, device=dev)
    _lib.check(_lib.lib().etb_letterbox_u8(_lib.ptr(table), len(frames), H, W, _lib.ptr(out), _lib.stream_ptr(dev)), "etb_letterbox_u8")
    return out, table


def rescale_rows(det, det_cnt, meta):
    """det [B, max_det, >=6] NMS rows in the letterboxed image, det_cnt [B] int32, meta [B, 5] fp32 (val._image_meta) ->
    [B, max_det, 6]: rows < det_cnt[b] as scale_coords(...).round() leaves them (etb_detect_rescale), the rest unwritten."""
    B, max_det, ld = det.shape
    out = torch.empty((B, max_det, 6), dtype=torch.float32, device=det.device)
    _lib.check(_lib.lib().etb_detect_rescale(_lib.ptr(det), _lib.ptr(det_cnt), B, max_det, ld, _lib.ptr(meta), _lib.ptr(out),
                                             _lib.stream_ptr(det.device)), "etb_detect_rescale")
    return out


def _frame_tensor(f, device):
    t = f if isinstance(f, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(f))
    if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 or t.shape[0] < 1 or t.shape[1] < 1:
        raise ValueError("Predictor: frames are uint8 [h, w, 3] BGR images, got %s %s" % (t.dtype, tuple(t.shape)))
    return _to_device(t, device)


class Predictor:
    """detect.py's inference on the native library.

    Predictor(model)(frames) -> one [n_i, 6] fp32 CUDA tensor (x1, y1, x2, y2, conf, cls) per frame, in the frame's pixel
    space with the coordinates rounded, as detect.py's `det` after scale_coords(...).round().  frames: uint8 HWC BGR images
    (numpy arrays as cv2.imread returns them, CPU or CUDA tensors) of any sizes.  model: a Model or SupModel on a CUDA
    device, fp32 or already .half() / .bfloat16(); it is put in eval() and run under no_grad on its engine (bf16 weights
    refreshed from its parameters each call)."""

    def __init__(self, model, img_size=640, conf_thres=0.25, iou_thres=0.45, agnostic=False, max_det=1000, classes=None,
                 augment=False, half=False, num_points=0):
        if classes is not None:
            raise NotImplementedError("Predictor: classes= is not supported (the native NMS has no class filter)")
        if augment:
            raise NotImplementedError("Predictor: augment=True (test-time augmentation) is not supported")
        if half:
            raise NotImplementedError("Predictor: half=True is not supported (the engine computes in bf16; a model that is "
                                      "already .half() runs as it is)")
        if num_points or getattr(getattr(model, "head", None), "num_keypoints", 0):
            raise NotImplementedError("Predictor: keypoint heads are not supported")
        if img_size % STRIDE:
            raise ValueError("Predictor: img_size must be a multiple of %d, got %d" % (STRIDE, img_size))
        self.model = model.eval()
        self.device = next(model.parameters()).device
        _lib.require_cuda(next(model.parameters()))
        self.img_size, self.conf_thres, self.iou_thres = int(img_size), float(conf_thres), float(iou_thres)
        self.agnostic, self.max_det = bool(agnostic), int(max_det)

    @torch.no_grad()
    def __call__(self, frames):
        frames = [_frame_tensor(f, self.device) for f in frames]
        if not frames:
            return []
        geoms = [letterbox_geometry(int(f.shape[0]), int(f.shape[1]), self.img_size) for f in frames]
        groups = {}
        for i, g in enumerate(geoms):
            groups.setdefault(g[4:6], []).append(i)
        engine = self.model.engine()
        outs, cnts, order, keep = [], [], [], []
        for (H, W), idx in groups.items():
            img, table = letterbox_batch([frames[i] for i in idx], [geoms[i] for i in idx], H, W)
            (pred, _), _ = engine.forward(img, with_features=False)
            det, det_cnt, _, _ = etb_nms._run(pred, self.conf_thres, self.iou_thres, self.agnostic, self.max_det,
                                              need_cls_conf=True, ws_name="nms_detect")
            shapes = []
            for i in idx:
                h0, w0 = int(frames[i].shape[0]), int(frames[i].shape[1])
                gain = min(H / h0, W / w0)                     # scale_coords without ratio_pad (detect.py:240)
                shapes.append(((h0, w0), ((gain, gain), ((W - w0 * gain) / 2, (H - h0 * gain) / 2))))
            meta = _to_device(_image_meta(shapes), self.device)
            outs.append(rescale_rows(det, det_cnt, meta))
            cnts.append(det_cnt)
            order += idx
            keep += [table, meta]
        cnt = torch.cat(cnts).tolist()                          # the one host sync of the call
        result = [None] * len(frames)
        rows = [o[j] for o in outs for j in range(o.shape[0])]
        for k, i in enumerate(order):
            result[i] = rows[k][:cnt[k]]
        return result
