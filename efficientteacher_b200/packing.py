"""One-launch weight preparation for the wgmma convolutions.

Every step the student's fp32 OIHW parameters change (SGD) and so does the teacher (EMA), so the bf16 K-major GEMM operands
must be rebuilt: forward operand [Cout][kh*kw*Cin], dgrad operand per output-parity class [Cin][taps*Cout], stem operand
[Cout][128], and -- teacher only -- the folded eval-BatchNorm scale/bias.  Instead of ~3 tiny launches per conv (~440 per
step) a WeightPacker owns persistent destination buffers and a device-resident descriptor table, and rebuilds everything
with ONE etb_pack_multi launch (+ ONE etb_fold_bn_multi).

The sources may be fp32, fp16 or bf16 (a model after .half() or .bfloat16(), as val.py and detect.py --half leave it): the
kernels read each one as stored and widen it to fp32, so the operands equal those of the fp32 model holding the same values.
Any other dtype, or a BatchNorm whose four tensors do not share one, raises NotImplementedError before anything runs."""
import torch

from . import _lib
from ._lib import EtbFoldDesc, EtbPackDesc, ETB_DT, ETB_PACK_CHUNK


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


class PackedBias:
    """The fp32 bias of one conv for the epilogue: `fp32` is the copy the pack launch refreshes when the bias is stored in
    fp16 / bf16, None when it is fp32 (the epilogue then reads the parameter itself)."""
    __slots__ = ("conv", "copy", "fp32")


def _dtype_code(t, name):
    code = ETB_DT.get(t.dtype)
    if code is None:
        raise NotImplementedError("%s is %s: the native weight packer reads fp32, fp16 and bf16" % (name or "a packed tensor", t.dtype))
    return code


def _bn_tensors(bn):
    return bn.weight, bn.bias, bn.running_mean, bn.running_var


class WeightPacker:
    def __init__(self, device):
        self.device = device
        self.items = []          # (weight tensor, PackedConv, kind, name)
        self.folds = []          # (bn module, PackedConv, name)
        self.biases = []         # (PackedBias, name)
        self._built = None

    def add(self, weight, stride, pad, want_dgrad, stem=False, negate_dgrad=False, name=""):
        """name: what an error about this weight calls it (e.g. its state_dict key)"""
        Cout, Cin, k, _ = weight.shape
        pc = PackedConv()
        pc.Cin, pc.Cout, pc.k, pc.s, pc.p = (128 if stem else Cin), Cout, (1 if stem else k), (1 if stem else stride), (0 if stem else pad)
        # every tap is padded to a multiple of the 64-channel K block (YOLOv5s widths: 32-channel layers); pads stay zero
        pc.fwd = torch.zeros((Cout, 128 if stem else k * k * _ceil64(Cin)), dtype=torch.bfloat16, device=self.device)
        pc.dgrad = None
        if want_dgrad and not stem:
            pc.dgrad = torch.zeros(Cin * k * k * _ceil64(Cout), dtype=torch.bfloat16, device=self.device)
        pc.scale = pc.bias = None
        self.items.append((weight, pc, "stem" if stem else ("conv_neg" if negate_dgrad else "conv"), name))
        self._built = None
        return pc

    def add_fold(self, bn, pc, name=""):
        pc.scale = torch.empty(bn.weight.shape[0], dtype=torch.float32, device=self.device)
        pc.bias = torch.empty_like(pc.scale)
        self.folds.append((bn, pc, name))
        self._built = None

    def add_bias(self, conv, name=""):
        """-> PackedBias of conv.bias (read from the module at every rebuild, so a replaced parameter is followed)"""
        pb = PackedBias()
        pb.conv, pb.fp32 = conv, None
        pb.copy = torch.empty(conv.bias.numel(), dtype=torch.float32, device=self.device)
        self.biases.append((pb, name))
        self._built = None
        return pb

    def _key(self):
        """(pointer, dtype) of every source: a moved or converted tensor (model.half(), .float(), .to()) makes it differ"""
        ts = [w for w, *_ in self.items]
        ts += [t for bn, *_ in self.folds for t in _bn_tensors(bn)]
        ts += [pb.conv.bias for pb, _ in self.biases]
        return tuple((t.data_ptr(), t.dtype) for t in ts)

    def _build(self):
        descs, chunks = [], []

        def push(w, out_ptr, elems, Cout, Cin, k, mode, dtype, taps=((), ()), out_ld=0):
            d = EtbPackDesc()
            d.w, d.out, d.elems, d.dtype = w.data_ptr(), out_ptr, elems, dtype
            d.Cout, d.Cin, d.k, d.mode, d.ntaps, d.out_ld = Cout, Cin, k, mode, len(taps[0]), out_ld
            for t, (a, b) in enumerate(zip(*taps)):
                d.kh[t], d.kw[t] = a, b
            idx = len(descs)
            descs.append(d)
            for c in range((elems + ETB_PACK_CHUNK - 1) // ETB_PACK_CHUNK):
                chunks.append((idx, c))

        # every dtype is checked before anything is uploaded or launched
        dts = [_dtype_code(w, name) for w, _, _, name in self.items]
        fold_dts = []
        for bn, _, name in self.folds:
            codes = {_dtype_code(t, name) for t in _bn_tensors(bn)}
            if len(codes) != 1:
                raise NotImplementedError("%s mixes %s: the BatchNorm fold reads its weight, bias, running_mean and running_var "
                                          "in one dtype" % (name or "a BatchNorm", sorted({str(t.dtype) for t in _bn_tensors(bn)})))
            fold_dts.append(codes.pop())
        bias_dts = [_dtype_code(pb.conv.bias, name) for pb, name in self.biases]
        for (w, pc, kind, _), dt in zip(self.items, dts):
            Cout, Cin, k, _ = w.shape
            if kind == "stem":
                push(w, pc.fwd.data_ptr(), Cout * 128, Cout, 3, 6, 2, dt)
                continue
            push(w, pc.fwd.data_ptr(), Cout * k * k * Cin, Cout, Cin, k, 0, dt, out_ld=_ceil64(Cin))
            if pc.dgrad is not None:
                ld = _ceil64(Cout)
                off = 0
                for khs, kws in dgrad_classes(k, pc.s, pc.p):
                    nt = len(khs)
                    push(w, pc.dgrad.data_ptr() + 2 * off, Cin * nt * Cout, Cout, Cin, k, 3 if kind == "conv_neg" else 1, dt, (khs, kws), ld)
                    off += Cin * nt * ld
        for (pb, _), dt in zip(self.biases, bias_dts):
            pb.fp32 = None
            if dt != ETB_DT[torch.float32]:          # an fp32 bias is read in place, as before
                b = pb.conv.bias
                push(b, pb.copy.data_ptr(), b.numel(), 0, 0, 0, 4, dt)
                pb.fp32 = pb.copy
        self._descs = _lib.upload((EtbPackDesc * len(descs))(*descs), self.device)
        self._chunks = torch.tensor(chunks, dtype=torch.int32).reshape(-1, 2).contiguous().to(self.device)
        self._nchunks = len(chunks)
        self._fold_descs = None
        if self.folds:
            f = []
            for (bn, pc, _), dt in zip(self.folds, fold_dts):
                d = EtbFoldDesc()
                d.gamma, d.beta = bn.weight.data_ptr(), bn.bias.data_ptr()
                d.mean, d.var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
                d.scale, d.bias, d.C, d.eps, d.dtype = pc.scale.data_ptr(), pc.bias.data_ptr(), bn.weight.shape[0], float(bn.eps), dt
                f.append(d)
            self._fold_descs = _lib.upload((EtbFoldDesc * len(f))(*f), self.device)
        self._built_key = self._key()
        self._built = True

    def _stale(self):
        return self._built is None or self._key() != self._built_key

    def run(self):
        """Rebuild every packed operand, fold and bias copy from the current parameter values (2 launches)."""
        if self._stale():
            self._build()
        lib = _lib.lib()
        _lib.check(lib.etb_pack_multi(_lib.ptr(self._descs), _lib.ptr(self._chunks), self._nchunks, _lib.stream_ptr()), "etb_pack_multi")
        if self._fold_descs is not None:
            _lib.check(lib.etb_fold_bn_multi(_lib.ptr(self._fold_descs), len(self.folds), _lib.stream_ptr()), "etb_fold_bn_multi")
