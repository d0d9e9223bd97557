"""The reference's validation pass (val.py:149-465) on the device.

val_batch: one batch -- half-precision forward (the native engine computes in bf16), multi-label NMS (etb_nms_val), rescale
to the native image space, and the true-positive matching process_batch (etb_val_process_batch) for all images of the batch
in one launch -- returning the per-image tuples val.py appends to `stats`.

run: the training-time val.run (a model and a dataloader given; plots, txt / json output, keypoints, model_post and
augmented inference stay with the host application).  Every batch goes into a device-resident ValEpoch (etb_val_epoch_append:
rescale, match and append without a host sync) and ap_per_class runs natively at the end (metrics.py).  With
confusion_matrix= (a metrics.ConfusionMatrix) every batch is also added into the detection confusion matrix on the device.
The COCO json is not computed."""
import itertools
from pathlib import Path

import numpy as np
import torch

from . import _lib, _ws
from . import metrics
from . import nms as etb_nms


def box_iou(box1, box2):
    """utils/metrics.py:252-273 for callers that want the matrix itself (plain torch ops; not on the hot path)"""
    area1 = (box1[:, 2] - box1[:, 0]) * (box1[:, 3] - box1[:, 1])
    area2 = (box2[:, 2] - box2[:, 0]) * (box2[:, 3] - box2[:, 1])
    inter = (torch.min(box1[:, None, 2:], box2[:, 2:]) - torch.max(box1[:, None, :2], box2[:, :2])).clamp(0).prod(2)
    return inter / (area1[:, None] + area2 - inter)


def process_batch_batched(det, det_cnt, labels, iouv):
    """det [B,max_det,>=6] fp32 (x1,y1,x2,y2,conf,cls) and labels [nt,6] (img,cls,x1,y1,x2,y2) in the same coordinate space;
    det_cnt [B] int32 or None; iouv [T] -> correct [B,max_det,T] bool (rows >= det_cnt are False)."""
    _lib.require_cuda(det, iouv)
    det = det.float().contiguous()
    labels = labels.to(det.device).float().contiguous()
    iouv = iouv.to(det.device).float().contiguous()
    B, max_det, ld = det.shape
    T = iouv.numel()
    correct = torch.empty((B, max_det, T), dtype=torch.uint8, device=det.device)
    overflow = torch.zeros(1, dtype=torch.int32, device=det.device)
    _lib.check(_lib.lib().etb_val_process_batch(_lib.ptr(det), _lib.ptr(det_cnt), B, max_det, ld, _lib.ptr(labels), int(labels.shape[0]),
                                                _lib.ptr(iouv), T, _lib.ptr(correct), _lib.ptr(overflow), _lib.stream_ptr()),
               "etb_val_process_batch")
    return correct.bool()


def process_batch(detections, labels, iouv):
    """val.py:123-145: detections [N,6] (x1,y1,x2,y2,conf,cls), labels [M,5] (cls,x1,y1,x2,y2) -> correct [N,len(iouv)] bool"""
    n = detections.shape[0]
    if n == 0:
        return torch.zeros((0, iouv.numel()), dtype=torch.bool, device=detections.device)
    lab = torch.cat([torch.zeros((labels.shape[0], 1), device=labels.device, dtype=labels.dtype), labels], 1)
    return process_batch_batched(detections[None, :, :6], None, lab, iouv)[0]


def scale_coords_(img1_shape, coords, img0_shape, ratio_pad=None):
    """utils/general.py:702-715 (in place, xyxy in columns 0..3)"""
    if ratio_pad is None:
        gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
        pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    else:
        gain = ratio_pad[0][0]
        pad = ratio_pad[1]
    coords[:, [0, 2]] -= pad[0]
    coords[:, [1, 3]] -= pad[1]
    coords[:, :4] /= gain
    coords[:, 0].clamp_(0, img0_shape[1]); coords[:, 1].clamp_(0, img0_shape[0])
    coords[:, 2].clamp_(0, img0_shape[1]); coords[:, 3].clamp_(0, img0_shape[0])
    return coords


@torch.no_grad()
def val_batch(model, img, targets, shapes, conf_thres=0.001, iou_thres=0.6, iouv=None, single_cls=False):
    """One batch of val.run (val.py:300-372, detection branch): img [B,3,H,W] (uint8 or fp32 in [0,1]) -> forward (native
    engine) -> non_max_suppression(multi_label=True) -> native-space predictions -> process_batch.  targets [nt,6] (img, cls,
    xywh normalised); shapes[i] = (shape0, (ratio, pad)) like the reference's loader.  Returns a list of (correct [n,T] bool,
    conf [n], pcls [n], tcls list) per image -- the tuples val.py appends to `stats`."""
    if iouv is None:
        iouv = torch.linspace(0.5, 0.95, 10, device=img.device)
    B, _, H, W = img.shape
    out = model(img)
    pred = out[0] if isinstance(out, tuple) else out
    pred = pred[0] if isinstance(pred, tuple) else pred            # SSOD model: ((pred, raw), features)
    dets = etb_nms.non_max_suppression(pred, conf_thres, iou_thres, multi_label=True, agnostic=single_cls)
    tg = targets.to(img.device).float().clone()
    tg[:, 2:6] *= torch.tensor([W, H, W, H], device=img.device, dtype=torch.float32)
    max_det = max(max((d.shape[0] for d in dets), default=0), 1)
    det_pad = torch.zeros((B, max_det, 6), dtype=torch.float32, device=img.device)
    cnt = torch.zeros(B, dtype=torch.int32, device=img.device)
    labs = []
    for si, p in enumerate(dets):
        predn = p.clone()
        if single_cls:
            predn[:, 5] = 0
        scale_coords_((H, W), predn[:, :4], shapes[si][0], shapes[si][1])
        det_pad[si, :predn.shape[0]] = predn
        cnt[si] = predn.shape[0]
        l = tg[tg[:, 0] == si, 1:]
        if l.shape[0]:
            tb = torch.cat((l[:, 1:3] - l[:, 3:5] / 2, l[:, 1:3] + l[:, 3:5] / 2), 1)       # xywh2xyxy
            scale_coords_((H, W), tb, shapes[si][0], shapes[si][1])
            labs.append(torch.cat((torch.full((l.shape[0], 1), float(si), device=img.device), l[:, 0:1], tb), 1))
    lab = torch.cat(labs, 0) if labs else torch.zeros((0, 6), device=img.device)
    correct = process_batch_batched(det_pad, cnt, lab, iouv)
    stats = []
    for si, p in enumerate(dets):
        n = p.shape[0]
        tcls = tg[tg[:, 0] == si, 1].tolist()
        stats.append((correct[si, :n], det_pad[si, :n, 4], det_pad[si, :n, 5], tcls))
    return stats


def _image_meta(shapes):
    """loader shapes[i] = ((h0, w0), ((gain, _), (padw, padh))) -> [B, 5] fp32 (h0, w0, 1 / gain, padw, padh), each value
    rounded to fp32 as torch rounds it: `coords /= gain` on a CUDA tensor multiplies by 1 / gain taken in float64"""
    return np.asarray([(s[0][0], s[0][1], 1.0 / s[1][0][0], s[1][1][0], s[1][1][1]) for s in shapes],
                      dtype=np.float32).reshape(-1, 5)


def _to_device(t, device, dtype=None):
    """host -> device without a host sync (pinned staging); device tensors pass through"""
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(np.asarray(t))
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if t.device.type == "cpu":
        return t.contiguous().pin_memory().to(device, non_blocking=True)
    return t.to(device).contiguous()


class ValEpoch:
    """The epoch's statistics (val.py:376 `stats`) in device memory: conf, class and correct bits of every detection in an
    arena that doubles when the host-side bound (images * max_det) outgrows it, and the label classes in an int32 histogram.
    add() never waits for the device; finish() copies the counters back once and runs ap_per_class.
    confusion_matrix: a metrics.ConfusionMatrix that every batch is also added into (val.py:372-373), from the same rescaled
    rows and labels, in the same launch sequence plus one kernel."""

    def __init__(self, device, nc, iouv=None, single_cls=False, capacity=0, confusion_matrix=None):
        self.device, self.nc, self.single_cls = torch.device(device), int(nc), bool(single_cls)
        self.iouv = (torch.linspace(0.5, 0.95, 10) if iouv is None else torch.as_tensor(iouv)).to(self.device, torch.float32).contiguous()
        self.T = self.iouv.numel()
        if not 0 < self.T <= 16:
            raise ValueError("ValEpoch: 1..16 IoU thresholds supported, got %d" % self.T)
        self.n_dev = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.hist = torch.zeros(self.nc + 1, dtype=torch.int32, device=self.device)
        self.flags = torch.zeros(2, dtype=torch.int32, device=self.device)
        self.cap = self.bound = 0
        self.conf = self.cls = self.tp = None
        self.seen = self.n_labels = 0
        self.cm = confusion_matrix
        if self.cm is not None:
            self.cm.buffers(self.device)
        self._grow(capacity)

    def _grow(self, need):
        if need <= self.cap and self.conf is not None:
            return
        cap = max(self.cap, 4096)
        while cap < need:
            cap *= 2
        conf = torch.empty(cap, dtype=torch.float32, device=self.device)
        cls = torch.empty(cap, dtype=torch.float32, device=self.device)
        tp = torch.empty(cap, dtype=torch.uint16, device=self.device)
        if self.conf is not None and self.cap:
            conf[:self.cap].copy_(self.conf)
            cls[:self.cap].copy_(self.cls)
            tp.view(torch.int16)[:self.cap].copy_(self.tp.view(torch.int16))
        self.conf, self.cls, self.tp, self.cap = conf, cls, tp, cap

    def add(self, det, det_cnt, targets, shapes, img_hw):
        """det [B, max_det, >=6] fp32 NMS rows and det_cnt [B] int32 on the device (etb_nms_val's layout); targets [nt, 6]
        (img, cls, xywh normalised); shapes: the loader's per-image ((h0, w0), ((gain, _), (padw, padh))); img_hw: (H, W) of
        the letterboxed batch."""
        B, max_det, ld = det.shape
        self.bound += B * max_det
        self._grow(self.bound)
        meta = _to_device(_image_meta(shapes), self.device)
        tg = _to_device(targets, self.device, torch.float32).reshape(-1, 6)
        nt = tg.shape[0]
        lib = _lib.lib()
        ws = _ws.workspace("val_epoch", lib.etb_val_epoch_append_workspace_bytes(B, max_det, nt, self.T), self.device)
        args = (_lib.ptr(det), _lib.ptr(det_cnt), B, max_det, ld, _lib.ptr(meta), _lib.ptr(tg), nt, int(img_hw[0]), int(img_hw[1]),
                int(self.single_cls), _lib.ptr(self.iouv), self.T, self.nc, _lib.ptr(self.conf), _lib.ptr(self.cls), _lib.ptr(self.tp),
                self.cap, _lib.ptr(self.n_dev), _lib.ptr(self.hist), _lib.ptr(self.flags))
        tail = (_lib.ptr(ws), ws.numel(), _lib.stream_ptr(self.device))
        if self.cm is None:
            _lib.check(lib.etb_val_epoch_append(*args, *tail), "etb_val_epoch_append")
        else:
            cm = self.cm
            counts, cm_flags = cm.buffers(self.device)
            _lib.check(lib.etb_val_epoch_append_confusion(*args, cm.nc, float(cm.conf), float(cm.iou_thres), _lib.ptr(counts),
                                                          _lib.ptr(cm_flags), *tail), "etb_val_epoch_append_confusion")
        self._keep = (meta, tg)       # the pinned staging buffers stay alive until the next batch
        self.seen += B
        self.n_labels += nt

    def finish(self):
        """-> (any_tp, per-class label counts [nc] (numpy), ap_per_class tuple or None when no detection is a TP)"""
        n = int(self.n_dev.item())
        flags = self.flags.cpu().numpy()
        hist = self.hist.cpu().numpy()
        if flags[1]:
            raise RuntimeError("ValEpoch: an image carries more than 1024 labels (etb_val_process_batch's limit)")
        if hist[self.nc]:
            raise IndexError("ValEpoch: %d labels have a class outside [0, %d)" % (hist[self.nc], self.nc))
        if self.cm is not None:
            self.cm.check()
        nt = hist[:self.nc]
        if not flags[0]:
            return False, nt, None
        unique = np.flatnonzero(nt)
        res = metrics.ap_from_device(self.conf, self.cls, self.tp, n, self.T, unique.astype(np.float64), nt[unique])
        return True, nt, res


def _registered(callbacks, hook):
    if callbacks is None:
        return False
    get = getattr(callbacks, "get_registered_actions", None)
    try:
        return bool(get(hook)) if get is not None else bool(getattr(callbacks, "_callbacks", {}).get(hook))
    except Exception:
        return True


def round_fp16_(model):
    """model.half(); model.float() (val.py:190, :455) in place: every floating parameter and buffer takes its fp16-rounded
    value without moving storage, so pointers held by captured CUDA graphs, EMA tables and weight packers stay valid."""
    with torch.no_grad():
        for t in itertools.chain(model.parameters(), model.buffers()):
            if t.is_floating_point():
                t.copy_(t.half())


def run_unsupported(model=None, dataloader=None, plots=True, save_txt=False, save_hybrid=False, save_json=False, num_points=0,
                    model_post=None, augment=False, **_):
    """The reason run() cannot take this call (None if it can)."""
    if model is None or dataloader is None:
        return "model and dataloader must be given (the training-time call)"
    try:
        dev = next(model.parameters()).device
    except (StopIteration, AttributeError):
        return "model has no parameters"
    if dev.type != "cuda":
        return "model is not on a CUDA device"
    for name, v in (("plots", plots), ("save_txt", save_txt), ("save_hybrid", save_hybrid), ("save_json", save_json),
                    ("augment", augment)):
        if v:
            return name + "=True"
    if num_points:
        return "num_points > 0 (keypoint heads)"
    if model_post is not None:
        return "model_post"
    return None


def _nms(out, conf_thres, iou_thres, single_cls, max_det=300):
    """utils/general.py non_max_suppression(multi_label=True) as val.py:335 calls it, device-resident (no per-image lists);
    multi_label applies only when nc > 1, as in the reference"""
    if out.shape[2] - 5 > 1:
        return etb_nms._run_val(out, conf_thres, iou_thres, single_cls, max_det)
    det, det_cnt, _, _ = etb_nms._run(out, conf_thres, iou_thres, single_cls, max_det, need_cls_conf=True, ws_name="nms_val1")
    return det, det_cnt


def _unwrap(outputs):
    """val.py:307-312 applied to the model's output: a tuple's first element, twice for a 2-sequence"""
    out = outputs
    if type(outputs) is tuple:
        out = outputs[0]
    if len(outputs) == 2:
        out = outputs[0]
    if not isinstance(out, torch.Tensor):
        raise TypeError("val.run: the model's output unwraps to %s, not a prediction tensor (an SSOD model needs val_ssod=True)"
                        % type(out).__name__)
    return out


@torch.no_grad()
def val_step(model, img, targets, shapes, epoch, conf_thres=0.001, iou_thres=0.6, single_cls=False, val_ssod=False, events=None,
             stream=None):
    """One batch of run() (val.py:279-376) into the ValEpoch `epoch`, without a host sync: upload, forward, NMS, append.
    events: 4 CUDA timing events recorded around pre-process, inference and NMS.  -> (img on the device, det, det_cnt)"""
    device = epoch.device
    if events is not None:
        events[0].record(stream)
    img = img.to(device, non_blocking=True)
    if img.dtype != torch.uint8:             # uint8 goes to the engine as is: its stem divides by 255
        img = img.float() / 255.0
    height, width = img.shape[2:]
    if events is not None:
        events[1].record(stream)
    if val_ssod:
        outputs, _ = model(img)
    else:
        outputs = model(img)
    out = _unwrap(outputs)
    if events is not None:
        events[2].record(stream)
    det, det_cnt = _nms(out, conf_thres, iou_thres, single_cls)
    if events is not None:
        events[3].record(stream)
    epoch.add(det, det_cnt, targets, shapes, (height, width))
    return img, det, det_cnt


@torch.no_grad()
def run(data, weights=None, batch_size=32, imgsz=640, conf_thres=0.001, iou_thres=0.6, task='val', device='', single_cls=False,
        augment=False, verbose=False, save_txt=False, save_hybrid=False, save_conf=False, save_json=False, project=None, name='exp',
        exist_ok=False, half=True, model=None, dataloader=None, save_dir=Path(''), plots=True, callbacks=None, compute_loss=None,
        model_post=None, eval_num=-1, cfg=None, val_ssod=False, num_points=0, val_kp=False, val_dp1000=False, dnn=False, names={},
        confusion_matrix=None):
    """val.py:149-465, the training-time call: returns ((mp, mr, map50, map, 0, 0, 0), maps, t[, cls_thr]).  The loss terms
    are zero as in the reference (its compute_loss branch is unreachable: `outputs is not list` always holds).  t is ms per
    image for (pre-process, inference, NMS), timed with CUDA events.  With half=True the model's floating state is rounded
    to fp16 in place (what model.half(); model.float() leaves); the model is left in eval().  confusion_matrix (native only,
    a metrics.ConfusionMatrix): every image with NMS rows and labels is added into it, as val.py:372-373 does with plots=True."""
    why = run_unsupported(model=model, dataloader=dataloader, plots=plots, save_txt=save_txt, save_hybrid=save_hybrid,
                          save_json=save_json, num_points=num_points, model_post=model_post, augment=augment)
    if why:
        raise NotImplementedError("efficientteacher_b200.val.run: " + why)
    device = next(model.parameters()).device
    if half:
        round_fp16_(model)
    model.eval()
    nc = 1 if single_cls else int(data['nc'])
    iouv = torch.linspace(0.5, 0.95, 10).to(device)
    try:
        names = {k: v for k, v in enumerate(model.names if hasattr(model, 'names') else model.module.names)}
    except Exception:
        pass
    per_image = _registered(callbacks, 'on_val_image_end')
    s = ('%20s' + '%11s' * 6) % ('Class', 'Images', 'Labels', 'P', 'R', 'mAP@.5', 'mAP@.5:.95')
    print(s)
    epoch = ValEpoch(device, nc, iouv, single_cls, confusion_matrix=confusion_matrix)
    stream = torch.cuda.current_stream(device)
    events = []
    for batch_i, (img, targets, paths, shapes) in enumerate(dataloader):
        if batch_i == eval_num:
            break
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        events.append(ev)
        img, det, det_cnt = val_step(model, img, targets, shapes, epoch, conf_thres, iou_thres, single_cls, val_ssod, ev, stream)
        nb = img.shape[0]
        if per_image:                            # val.py:383, only when a hook wants the per-image rows (host sync)
            cnt = det_cnt.tolist()
            for si in range(nb):
                pred = det[si, :cnt[si], :6].clone()
                if single_cls:
                    pred[:, 5] = 0
                predn = pred.clone()
                scale_coords_(img[si].shape[1:], predn[:, :4], shapes[si][0], shapes[si][1])
                callbacks.run('on_val_image_end', pred, predn, Path(paths[si]), names, img[si])
    seen = epoch.seen
    any_tp, nt_cls, res = epoch.finish()
    dt = [0.0, 0.0, 0.0]
    for ev in events:
        for k in range(3):
            dt[k] += ev[k].elapsed_time(ev[k + 1]) / 1e3
    mp = mr = map50 = map = 0.0
    ap_class = []
    if any_tp:
        p, r, ap, f1, ap_class, cls_thr = res
        ap50, ap = ap[:, 0], ap.mean(1)
        mp, mr, map50, map = p.mean(), r.mean(), ap50.mean(), ap.mean()
        nt = nt_cls
    else:
        cls_thr = []
        nt = torch.zeros(1)
    pf = '%20s' + '%11i' * 2 + '%11.3g' * 4
    print(pf % ('all', seen, nt.sum(), mp, mr, map50, map))
    if verbose and nc > 1 and any_tp:
        for i, c in enumerate(ap_class):
            print(pf % (names[c], seen, nt[c], p[i], r[i], ap50[i], ap[i]))
    t = tuple(x / seen * 1E3 for x in dt)
    maps = np.zeros(nc) + map
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    loss = (torch.zeros(3) / len(dataloader)).tolist()
    if val_ssod:
        return (mp, mr, map50, map, *loss), maps, t, cls_thr
    return (mp, mr, map50, map, *loss), maps, t
