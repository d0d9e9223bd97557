"""Pseudo-label quality statistics and the training meter of the SSOD step, on the device.

check_pseudo_label_with_gt / check_pseudo_label mirror utils/self_supervised_utils.py:481-587 / :589-606 with the reference's
signatures and return types: numpy float64 arrays [T] (or the int 0 when there is no uncertain row) and Python floats.
The reference selects the rows with one `.cpu()` per row (select_targets, :456-479) and matches them with numpy; here one
etb_pl_quality call does both (csrc/plq.cu restates the algorithm): the inputs are uploaded, the kernels run, and one
buffer is read back.  One deliberate difference: the reference scales `labels[:, 2:6]` by 640 IN PLACE (`gt *= ...` on a
view, :521), so the caller's labels come back changed; the mirror leaves them as they were.

DeviceMetricMeter is MetricMeter / AverageMeter (utils/metrics.py:352-414) with its sums on the device, so that a
captured training step can update it without reading anything back.
"""
import ctypes as C
from collections import OrderedDict

import numpy as np
import torch

from . import _lib

HIT_KEYS = ("tp", "fp_cls", "fp_loc", "pse_num", "gt_num")     # trainer/ssod_trainer.py:671


class PLQuality:
    """The buffers of etb_pl_quality for one launch site: vals [5][T] float64 and the int32 counts (see
    include/etb200.h) share one float64 buffer, so that a caller on the host reads both with one copy.  Allocated once;
    run() neither allocates nor synchronises, so it can be captured in a CUDA graph."""

    def __init__(self, device, iouv=(0.5,)):
        self.device = torch.device(device)
        self.iouv = torch.as_tensor(iouv).to(self.device, torch.float64).reshape(-1).contiguous()
        self.T = T = int(self.iouv.numel())
        if not 0 < T <= 16:
            raise ValueError("etb_pl_quality takes 1 to 16 IoU thresholds, got %d" % T)
        ncnt = 5 + 3 * T
        self.buf = torch.zeros(5 * T + (ncnt + 1) // 2, dtype=torch.float64, device=self.device)
        self.vals = self.buf[:5 * T].view(5, T)
        self.cnt = self.buf[5 * T:].view(torch.int32)[:ncnt]
        self.ws = torch.empty(int(_lib.lib().etb_pl_quality_workspace_bytes()), dtype=torch.uint8, device=self.device)

    def run(self, rows, n_dev, thr_high, thr_low, gt, m_dev, batch_size, with_gt, iou64=False):
        """rows [cap,9] float64 CUDA (n_dev int32[1] or None: all cap rows); thr_high / thr_low [nc] float64 CUDA or both
        None; gt [capG,6] fp32 CUDA or None (m_dev int32[1] or None: all capG rows).  Returns self.vals."""
        _lib.require_cuda(rows, gt)
        assert rows.dtype == torch.float64 and rows.is_contiguous() and (rows.numel() == 0 or rows.shape[1] == 9)
        assert gt is None or (gt.dtype == torch.float32 and gt.is_contiguous() and (gt.numel() == 0 or gt.shape[1] == 6))
        nc = 0 if thr_high is None else int(thr_high.numel())
        _lib.check(_lib.lib().etb_pl_quality(
            _lib.ptr(rows), _lib.ptr(n_dev), int(rows.shape[0]), _lib.ptr(thr_high), _lib.ptr(thr_low), nc, _lib.ptr(gt),
            _lib.ptr(m_dev), 0 if gt is None else int(gt.shape[0]), _lib.ptr(self.iouv), self.T, int(batch_size),
            int(bool(with_gt)), int(bool(iou64)), _lib.ptr(self.vals), _lib.ptr(self.cnt), _lib.ptr(self.ws), self.ws.numel(),
            _lib.stream_ptr(self.device)), "etb_pl_quality")
        return self.vals

    def read(self):
        """-> (vals [5,T] float64, counts dict) after one device-to-host copy"""
        b = self.buf.cpu().numpy()
        T = self.T
        c = b[5 * T:].view(np.int32)
        counts = dict(n=int(c[0]), n_uc=int(c[1]), n_reliable=int(c[2]), m=int(c[3]), overflow=int(c[4]),
                      tp=c[5:5 + T].copy(), fp_cls=c[5 + T:5 + 2 * T].copy(), fp_loc=c[5 + 2 * T:5 + 3 * T].copy())
        return b[:5 * T].reshape(5, T).copy(), counts


def _device(*tensors):
    for t in tensors:
        if torch.is_tensor(t) and t.is_cuda:
            return t.device
    _lib.require_cuda()
    return torch.device("cuda", torch.cuda.current_device())


def _rows(detections, dev):
    d = torch.as_tensor(detections)
    return d.to(dev, torch.float64).reshape(-1, 9).contiguous(), d.dtype


def _thresholds(thr, dev):
    return None if thr is None else torch.as_tensor(np.asarray(thr, dtype=np.float64)).to(dev)


def _run(detections, labels, iouv, ignore_thres_low, ignore_thres_high, batch_size, with_gt):
    dev = _device(detections, labels)
    rows, dtype = _rows(detections, dev)
    select = ignore_thres_low is not None
    hi, lo = (_thresholds(ignore_thres_high, dev), _thresholds(ignore_thres_low, dev)) if select else (None, None)
    gt = None if labels is None else torch.as_tensor(labels).to(dev, torch.float32).reshape(-1, 6).contiguous()
    plq = PLQuality(dev, iouv)
    plq.run(rows, None, hi, lo, gt, None, batch_size, with_gt, iou64=not select and dtype == torch.float64)
    vals, counts = plq.read()
    if counts["overflow"]:
        raise RuntimeError("pseudo-label quality: an image with more than 1024 labels, a class index outside the thresholds "
                           "or a negative image index")
    return vals, counts


def check_pseudo_label_with_gt(detections, labels, iouv=torch.tensor([0.5]), ignore_thres_low=None, ignore_thres_high=None,
                               batch_size=1):
    """utils/self_supervised_utils.py:481-587.  detections [N,9] (img, cls, x, y, w, h, conf, obj_conf, cls_conf; float64 as
    FairPseudoLabel makes them), labels [M,6] (img, cls, x, y, w, h), both normalised xywh, CPU or CUDA.  With thresholds
    only the uncertain rows (low <= conf < high of their class) are scored.  -> (tp_rate, fp_cls_rate, fp_loc_rate,
    pse_num, gt_num): three float64 arrays [len(iouv)] (the int 0 when no row is scored) and two floats.  `labels` is not
    modified (the reference scales its box columns in place)."""
    vals, c = _run(detections, labels, iouv, ignore_thres_low, ignore_thres_high, batch_size, True)
    n_uc = c["n_uc"]
    rates = (0, 0, 0) if n_uc == 0 else tuple(vals[s].copy() for s in range(3))
    return rates + (n_uc / batch_size, c["m"] / batch_size)


def check_pseudo_label(detections, ignore_thres_low=None, ignore_thres_high=None, batch_size=1):
    """utils/self_supervised_utils.py:589-606 -> (reliable / (reliable + uncertain), (reliable + uncertain) * batch_size / N,
    reliable + uncertain, reliable) with the counts divided by batch_size; 0 (int) for the ratios whose denominator is 0."""
    if ignore_thres_low is None or ignore_thres_high is None:
        raise TypeError("check_pseudo_label needs ignore_thres_low and ignore_thres_high (select_targets indexes them)")
    _, c = _run(detections, None, (0.5,), ignore_thres_low, ignore_thres_high, batch_size, False)
    reliable_num, uncertain_num = c["n_reliable"] / batch_size, c["n_uc"] / batch_size
    denorm = reliable_num + uncertain_num
    precision_rate = 0 if denorm == 0 else reliable_num / denorm
    recall_rate = 0 if c["n"] == 0 else (reliable_num + uncertain_num) * batch_size / c["n"]
    return precision_rate, recall_rate, reliable_num + uncertain_num, reliable_num


class AverageMeterView:
    """One meter of DeviceMetricMeter.meters: AverageMeter's val / sum / count / avg, read at one point in time."""
    __slots__ = ("val", "sum", "count", "avg")

    def __init__(self, val, sum_, count):
        self.val, self.sum, self.count = val, sum_, count
        self.avg = sum_ / count


class DeviceMetricMeter:
    """MetricMeter (utils/metrics.py:369-414) whose AverageMeters live on the device: state [3][capacity] float64 holds
    sum, count and the last value of each key; update() is one etb_meter_update launch per 16 keys and reads nothing
    back, so it can be captured in a CUDA graph (CUDA tensors are read where they are when the kernel runs).  The sums are
    float64 additions in update order, as the reference's Python floats (a fp32 tensor enters as its exact float64 value,
    like .item()).  Reading (meters, get_avg, str) copies the state to the host once per call.  Keys keep their
    first-insertion order; a key is listed once it has been updated since the last reset().  reset() zeroes the state in
    place, so a captured graph keeps valid pointers across epochs."""

    CAPACITY = 32

    def __init__(self, device, delimiter='\t', capacity=CAPACITY):
        self.device = torch.device(device)
        self.delimiter = delimiter
        self.state = torch.zeros((3, capacity), dtype=torch.float64, device=self.device)
        self._slots = OrderedDict()

    def _slot(self, name):
        s = self._slots.get(name)
        if s is None:
            s = len(self._slots)
            if s >= self.state.shape[1]:
                raise RuntimeError("DeviceMetricMeter: more than %d keys" % self.state.shape[1])
            self._slots[name] = s
        return s

    def update(self, input_dict):
        if input_dict is None:
            return
        if not isinstance(input_dict, dict):
            raise TypeError('Input to MetricMeter.update() must be a dictionary')
        dev_src, host_slots, host_vals = [], [], []
        for k, v in input_dict.items():
            s = self._slot(k)
            if torch.is_tensor(v) and v.device == self.device:
                if v.numel() != 1:
                    raise ValueError("DeviceMetricMeter: %r has %d elements, expected 1" % (k, v.numel()))
                if v.dtype not in (torch.float32, torch.float64):
                    v = v.double()
                dev_src.append((s, v))
            else:
                a = np.asarray(v.detach().cpu() if torch.is_tensor(v) else v, dtype=np.float64).reshape(-1)
                if a.size != 1:
                    raise ValueError("DeviceMetricMeter: %r has %d elements, expected 1" % (k, a.size))
                host_slots.append(s)
                host_vals.append(float(a[0]))
        if host_vals:
            staged = torch.tensor(host_vals, dtype=torch.float64).to(self.device)
            dev_src += [(s, staged[i]) for i, s in enumerate(host_slots)]
        lib = _lib.lib()
        for i in range(0, len(dev_src), 16):
            chunk = dev_src[i:i + 16]
            n = len(chunk)
            src = (C.c_void_p * n)(*[t.data_ptr() for _, t in chunk])
            slot = (C.c_int32 * n)(*[s for s, _ in chunk])
            f64 = (C.c_int32 * n)(*[int(t.dtype == torch.float64) for _, t in chunk])
            _lib.check(lib.etb_meter_update(_lib.ptr(self.state), self.state.shape[1], src, slot, f64, n,
                                            _lib.stream_ptr(self.device)), "etb_meter_update")

    def reset(self):
        self.state.zero_()

    @property
    def meters(self):
        st = self.state.cpu().numpy()
        return OrderedDict((k, AverageMeterView(float(st[2, s]), float(st[0, s]), int(st[1, s])))
                           for k, s in self._slots.items() if st[1, s] > 0)

    def get_avg(self):
        return [m.avg for m in self.meters.values()]

    def __str__(self):
        return self.delimiter.join('{} {:.4f} ({:.4f})'.format(name, m.val, m.avg) for name, m in self.meters.items())
