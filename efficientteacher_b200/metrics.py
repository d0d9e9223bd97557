"""ap_per_class and fitness with the reference's surface (utils/metrics.py:16-126).

The per-class work -- sort by confidence, cumulative TP / FP counts, precision and recall, the precision envelope and every
numpy.interp of compute_ap and of the P / R curves -- runs in one native call (etb_ap_per_class, csrc/metrics.cu).  What is
left is O(nc * 1000) and stays in numpy so that its summation order is numpy's: trapz over the 101 interpolated points, F1,
the argmax of the mean F1 and the per-class F1 thresholds.  Equal confidences within a class keep their row order (a stable
sort); numpy's argsort(-conf) leaves that order unspecified, so results agree with the reference whenever the confidences of
a class are distinct.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, _ws

NPX = 1000      # the P / R / F1 curves' confidence grid (metrics.py:45)
NXS = 101       # COCO's 101 recall points (metrics.py:120)
_trapz = getattr(np, "trapezoid", None) or np.trapz


def fitness(x):
    """metrics.py:16-19: 0.1 * mAP@0.5 + 0.9 * mAP@0.5:0.95 of rows [P, R, mAP@0.5, mAP@0.5:0.95, ...]"""
    w = [0.0, 0.0, 0.1, 0.9]
    return (x[:, :4] * w).sum(1)


def _grids(device):
    return (torch.from_numpy(np.linspace(0, 1, NPX)).to(device), torch.from_numpy(np.linspace(0, 1, NXS)).to(device))


def pack_tp_bits(tp):
    """[n, T] bool -> [n] uint16 with bit t = tp[:, t] (T <= 16)"""
    T = tp.shape[1]
    w = torch.tensor([1 << t for t in range(T)], dtype=torch.int32, device=tp.device)
    return (tp.to(torch.int32) * w).sum(1).to(torch.int16).view(torch.uint16) if T else torch.zeros(tp.shape[0], dtype=torch.uint16,
                                                                                                       device=tp.device)


def ap_from_device(conf, pred_cls, tp_bits, n, T, target_classes, n_l):
    """conf / pred_cls fp32 [>=n], tp_bits uint16 [>=n] on the device; target_classes: the sorted unique label classes (numpy
    float64), n_l their label counts.  -> (p, r, ap, f1, ap_class, cls_thr) as the reference returns them."""
    dev = conf.device
    unique = np.asarray(target_classes, dtype=np.float64)
    nu = unique.shape[0]
    if nu and (np.any(unique < 0) or np.any(unique != np.floor(unique))):
        raise ValueError("ap_per_class: class indices must be non-negative integers, got %s" % unique[:8])
    ncls = int(unique[-1]) + 1 if nu else 0
    slot = np.full(max(ncls, 1), -1, dtype=np.int32)
    slot[unique.astype(np.int64)] = np.arange(nu, dtype=np.int32)
    slot_d = torch.from_numpy(slot).to(dev)
    nl_d = torch.from_numpy(np.asarray(n_l, dtype=np.int32).reshape(-1)).to(dev)
    px, xs = _grids(dev)
    points = torch.empty((max(nu, 1), T, NXS), dtype=torch.float64, device=dev)
    pc = torch.empty((max(nu, 1), NPX), dtype=torch.float64, device=dev)
    rc = torch.empty_like(pc)
    n_p = torch.empty(max(nu, 1), dtype=torch.int32, device=dev)
    lib = _lib.lib()
    ws = _ws.workspace("ap_per_class", lib.etb_ap_per_class_workspace_bytes(int(n), nu), dev)
    _lib.check(lib.etb_ap_per_class(_lib.ptr(conf), _lib.ptr(pred_cls), _lib.ptr(tp_bits), int(n), T, _lib.ptr(slot_d), ncls, nu,
                                    _lib.ptr(nl_d), _lib.ptr(px), _lib.ptr(xs), _lib.ptr(points), _lib.ptr(pc), _lib.ptr(rc),
                                    _lib.ptr(n_p), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev)), "etb_ap_per_class")
    points, p, r, n_p = points[:nu].cpu().numpy(), pc[:nu].cpu().numpy(), rc[:nu].cpu().numpy(), n_p[:nu].cpu().numpy()
    return _host_tail(points, p, r, n_p, unique)


def _host_tail(points, p, r, n_p, unique):
    """metrics.py:68-98 after the interpolations: trapz, F1 and the thresholds, in numpy"""
    px = np.linspace(0, 1, NPX)
    ap = np.zeros(points.shape[:2])
    has = n_p > 0
    if has.any():
        ap[has] = _trapz(points[has], np.linspace(0, 1, NXS), axis=-1)
    f1 = 2 * p * r / (p + r + 1e-16)
    i = f1.mean(0).argmax()
    cls_thr = [px[f1[k, :].argmax()] for k in range(f1.shape[0])]
    return p[:, i], r[:, i], ap, f1[:, i], unique.astype('int32'), cls_thr


def _to_device(x, dev, dtype):
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
    return t.to(device=dev, dtype=dtype).contiguous()


def ap_per_class(tp, conf, pred_cls, target_cls, plot=False, save_dir='.', names=()):
    """metrics.py:22-98.  tp [n, T] bool, conf [n], pred_cls [n], target_cls [m]: numpy arrays or tensors (CUDA or CPU);
    the work runs on the CUDA device of the tensors (the current device for numpy input).  plot=True is not implemented
    (the plots stay with the host application)."""
    if plot:
        raise NotImplementedError("efficientteacher_b200.metrics.ap_per_class: plot=True (the PR / F1 plots are not native)")
    dev = next((x.device for x in (tp, conf, pred_cls) if isinstance(x, torch.Tensor) and x.is_cuda), None)
    if dev is None:
        _lib.require_cuda()
        dev = torch.device("cuda", torch.cuda.current_device())
    tp_t = _to_device(tp, dev, torch.bool)
    if tp_t.dim() == 1:
        tp_t = tp_t[:, None]
    n, T = tp_t.shape
    if not 0 < T <= 16:
        raise ValueError("ap_per_class: 1..16 IoU columns supported, got %d" % T)
    conf_t = _to_device(conf, dev, torch.float32).reshape(-1)
    cls_t = _to_device(pred_cls, dev, torch.float32).reshape(-1)
    tc = target_cls.detach().cpu().numpy() if isinstance(target_cls, torch.Tensor) else np.asarray(target_cls)
    unique, n_l = np.unique(tc.astype(np.float64).reshape(-1), return_counts=True)
    return ap_from_device(conf_t, cls_t, pack_tp_bits(tp_t), n, T, unique, n_l)


class ConfusionMatrix:
    """utils/metrics.py:129-204 with the reference's surface; process_batch runs on the device (etb_confusion_matrix,
    csrc/val.cu) and adds into an int64 count matrix there, without a host sync.  `matrix` reads it back as the reference's
    float64 [nc+1, nc+1] (rows: predicted class, columns: true class, index nc: background).  A ValEpoch given this object
    (val.run(..., confusion_matrix=cm)) adds every validation batch into it the same way.

    Matches are decided by fp32 IoU; on an exact IoU tie the later label, then the later detection wins (the order numpy's
    argsort()[::-1] gives where its sort is stable).  A class outside [0, nc) raises IndexError when the matrix is read:
    numpy's indexing in the reference would raise for most of them, and take class nc or a negative class silently."""
    host_plot = None        # the host application's ConfusionMatrix.plot, bound by efficientteacher_b200.bootstrap

    def __init__(self, nc, conf=0.25, iou_thres=0.45):
        self.nc, self.conf, self.iou_thres = int(nc), conf, iou_thres
        if self.nc < 1:
            raise ValueError("ConfusionMatrix: nc must be >= 1, got %d" % self.nc)
        self.counts = None      # int64 [(nc+1)^2] on the device of the first batch
        self.flags = None       # int32 [2]: an image with more than 1024 labels, a class outside [0, nc)
        self.host = np.zeros((self.nc + 1, self.nc + 1))    # counts added on the host (the bootstrap's route for CPU tensors)

    def buffers(self, device):
        """(counts, flags) on `device`, allocated on first use"""
        device = torch.device(device)
        if self.counts is None:
            self.counts = torch.zeros((self.nc + 1) ** 2, dtype=torch.int64, device=device)
            self.flags = torch.zeros(2, dtype=torch.int32, device=device)
        elif self.counts.device != device:
            raise RuntimeError("ConfusionMatrix: counts live on %s, got a batch on %s" % (self.counts.device, device))
        return self.counts, self.flags

    def process_batch(self, detections, labels):
        """one image: detections [N, >=6] (x1, y1, x2, y2, conf, cls) and labels [M, 5] (cls, x1, y1, x2, y2), CUDA tensors in
        the same coordinate space.  fp16 rows are widened to fp32, exactly as torch promotes them against fp32 labels."""
        _lib.require_cuda(detections, labels)
        det = detections.float().contiguous()
        if det.dim() != 2 or det.shape[1] < 6 or labels.dim() != 2 or labels.shape[1] != 5:
            raise ValueError("ConfusionMatrix.process_batch: detections [N, 6] and labels [M, 5], got %s and %s"
                             % (tuple(detections.shape), tuple(labels.shape)))
        if det.shape[0] > 1024:
            raise ValueError("ConfusionMatrix.process_batch: at most 1024 detections per image, got %d" % det.shape[0])
        if det.shape[0] == 0:       # the reference counts every label as missed: one row below any conf threshold does that
            det = torch.full((1, 6), float("-inf"), device=det.device)
        counts, flags = self.buffers(det.device)
        lab = torch.nn.functional.pad(labels.to(det.device, torch.float32), (1, 0))        # (img 0, cls, x1, y1, x2, y2)
        _lib.check(_lib.lib().etb_confusion_matrix(_lib.ptr(det), None, 1, det.shape[0], det.shape[1], _lib.ptr(lab), lab.shape[0],
                                                   self.nc, float(self.conf), float(self.iou_thres),
                                                   _lib.ptr(counts), _lib.ptr(flags), _lib.stream_ptr(det.device)),
                   "etb_confusion_matrix")

    def check(self):
        """raises if a batch overflowed or met a class outside [0, nc) (one read-back of the flags)"""
        if self.flags is None:
            return
        f = self.flags.cpu().numpy()
        if f[0]:
            raise RuntimeError("ConfusionMatrix: an image carries more than 1024 labels (etb_confusion_matrix's limit)")
        if f[1]:
            raise IndexError("ConfusionMatrix: a class outside [0, %d) was to be counted" % self.nc)

    @property
    def matrix(self):
        self.check()
        m = self.host.copy()
        if self.counts is not None:
            m += self.counts.cpu().numpy().reshape(self.nc + 1, self.nc + 1)
        return m

    def reset(self):
        self.host[:] = 0
        if self.counts is not None:
            self.counts.zero_()
            self.flags.zero_()

    def plot(self, normalize=True, save_dir='', names=()):
        """the host application's drawing (seaborn) when the bootstrap has bound it; else the reference's warning line"""
        if self.host_plot is None:
            print('WARNING: ConfusionMatrix plot failure: no host plot bound (import efficientteacher_b200.bootstrap)')
            return
        self.host_plot(normalize=normalize, save_dir=save_dir, names=names)

    def print(self):
        m = self.matrix
        for i in range(self.nc + 1):
            print(' '.join(map(str, m[i])))
