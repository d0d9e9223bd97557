"""One-launch weight preparation for the wgmma convolutions.

Every step the student's fp32 OIHW parameters change (SGD) and so does the teacher (EMA), so the bf16 K-major GEMM operands
must be rebuilt: forward operand [Cout][kh*kw*Cin], dgrad operand per output-parity class [Cin][taps*Cout], stem operand
[Cout][128], and -- teacher only -- the folded eval-BatchNorm scale/bias.  Instead of ~3 tiny launches per conv (~440 per
step) a WeightPacker owns persistent destination buffers and a device-resident descriptor table, and rebuilds everything
with ONE etb_pack_multi launch (+ ONE etb_fold_bn_multi)."""
import torch

from . import _lib
from ._lib import EtbFoldDesc, EtbPackDesc, ETB_PACK_CHUNK


def _ceil64(c):
    return (c + 63) // 64 * 64


def dgrad_classes(k, s, pad):
    """[(kh list, kw list)] per output-parity class in the order etb_conv_dgrad visits them (ph outer, pw inner)."""
    out = []
    for ph in range(s):
        for pw in range(s):
            khs, kws = [], []
            for kh in range(k):
                if (ph + pad - kh) % s:
                    continue
                for kw in range(k):
                    if (pw + pad - kw) % s:
                        continue
                    khs.append(kh)
                    kws.append(kw)
            out.append((khs, kws))
    return out


class PackedConv:
    """Destination buffers of one conv (views into the packer's arenas)."""
    __slots__ = ("fwd", "dgrad", "scale", "bias", "Cin", "Cout", "k", "s", "p")


class WeightPacker:
    def __init__(self, device):
        self.device = device
        self.items = []          # (weight tensor, PackedConv, kind)
        self.folds = []          # (bn module, PackedConv)
        self._built = None

    def add(self, weight, stride, pad, want_dgrad, stem=False, negate_dgrad=False):
        Cout, Cin, k, _ = weight.shape
        pc = PackedConv()
        pc.Cin, pc.Cout, pc.k, pc.s, pc.p = (128 if stem else Cin), Cout, (1 if stem else k), (1 if stem else stride), (0 if stem else pad)
        # every tap is padded to a multiple of the 64-channel K block (YOLOv5s widths: 32-channel layers); pads stay zero
        pc.fwd = torch.zeros((Cout, 128 if stem else k * k * _ceil64(Cin)), dtype=torch.bfloat16, device=self.device)
        pc.dgrad = None
        if want_dgrad and not stem:
            pc.dgrad = torch.zeros(Cin * k * k * _ceil64(Cout), dtype=torch.bfloat16, device=self.device)
        pc.scale = pc.bias = None
        self.items.append((weight, pc, "stem" if stem else ("conv_neg" if negate_dgrad else "conv")))
        self._built = None
        return pc

    def add_fold(self, bn, pc):
        pc.scale = torch.empty(bn.weight.shape[0], dtype=torch.float32, device=self.device)
        pc.bias = torch.empty_like(pc.scale)
        self.folds.append((bn, pc))
        self._built = None

    def _build(self):
        descs, chunks = [], []

        def push(w, out_ptr, elems, Cout, Cin, k, mode, taps=((), ()), out_ld=0):
            d = EtbPackDesc()
            d.w, d.out, d.elems = w.data_ptr(), out_ptr, elems
            d.Cout, d.Cin, d.k, d.mode, d.ntaps, d.out_ld = Cout, Cin, k, mode, len(taps[0]), out_ld
            for t, (a, b) in enumerate(zip(*taps)):
                d.kh[t], d.kw[t] = a, b
            idx = len(descs)
            descs.append(d)
            for c in range((elems + ETB_PACK_CHUNK - 1) // ETB_PACK_CHUNK):
                chunks.append((idx, c))

        for w, pc, kind in self.items:
            Cout, Cin, k, _ = w.shape
            if kind == "stem":
                push(w, pc.fwd.data_ptr(), Cout * 128, Cout, 3, 6, 2)
                continue
            push(w, pc.fwd.data_ptr(), Cout * k * k * Cin, Cout, Cin, k, 0, out_ld=_ceil64(Cin))
            if pc.dgrad is not None:
                ld = _ceil64(Cout)
                off = 0
                for khs, kws in dgrad_classes(k, pc.s, pc.p):
                    nt = len(khs)
                    push(w, pc.dgrad.data_ptr() + 2 * off, Cin * nt * Cout, Cout, Cin, k, 3 if kind == "conv_neg" else 1, (khs, kws), ld)
                    off += Cin * nt * ld
        self._descs = _lib.upload((EtbPackDesc * len(descs))(*descs), self.device)
        self._chunks = torch.tensor(chunks, dtype=torch.int32).reshape(-1, 2).contiguous().to(self.device)
        self._nchunks = len(chunks)
        self._keep = [w for w, *_ in self.items]
        self._ptrs = tuple(w.data_ptr() for w in self._keep)
        self._fold_descs = None
        if self.folds:
            f = []
            for bn, pc in self.folds:
                d = EtbFoldDesc()
                d.gamma, d.beta = bn.weight.data_ptr(), bn.bias.data_ptr()
                d.mean, d.var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
                d.scale, d.bias, d.C, d.eps = pc.scale.data_ptr(), pc.bias.data_ptr(), bn.weight.shape[0], float(bn.eps)
                f.append(d)
            self._fold_descs = _lib.upload((EtbFoldDesc * len(f))(*f), self.device)
            self._fold_ptrs = tuple(t.data_ptr() for bn, _ in self.folds for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
        self._built = True

    def _stale(self):
        if self._built is None:
            return True
        if tuple(w.data_ptr() for w in self._keep) != self._ptrs:
            return True
        if self.folds and tuple(t.data_ptr() for bn, _ in self.folds for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var)) != self._fold_ptrs:
            return True
        return False

    def run(self):
        """Rebuild every packed operand from the current parameter values (2 launches)."""
        if self._stale():
            self._build()
        lib = _lib.lib()
        _lib.check(lib.etb_pack_multi(_lib.ptr(self._descs), _lib.ptr(self._chunks), self._nchunks, _lib.stream_ptr()), "etb_pack_multi")
        if self._fold_descs is not None:
            _lib.check(lib.etb_fold_bn_multi(_lib.ptr(self._fold_descs), len(self.folds), _lib.stream_ptr()), "etb_fold_bn_multi")
