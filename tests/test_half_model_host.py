"""CPU: the host side of half-precision models on the native engine -- the dtype codes and descriptor fields the packing
kernels read, the weight packer's refusals (before anything is uploaded or launched) and staleness on a dtype change,
and the fp32 guard of the training forward."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    return open(os.path.join(ROOT, "include", "etb200.h")).read()


def test_dtype_codes_match_the_header():
    from efficientteacher_b200 import _lib
    h = _header()
    codes = {name: int(v) for name, v in re.findall(r"#define (ETB_DT_\w+|ETB_STEM_SRC_\w+) (\d+)", h)}
    assert _lib.ETB_DT == {torch.float32: codes["ETB_DT_F32"], torch.float16: codes["ETB_DT_F16"],
                           torch.bfloat16: codes["ETB_DT_BF16"]}
    assert _lib.ETB_STEM_SRC == {torch.float32: codes["ETB_STEM_SRC_F32"], torch.uint8: codes["ETB_STEM_SRC_U8"],
                                 torch.float16: codes["ETB_STEM_SRC_F16"]}
    # 0 and 1 keep the meaning etb_stem_im2col_into's former is_u8 flag gave them
    assert codes["ETB_STEM_SRC_F32"] == 0 and codes["ETB_STEM_SRC_U8"] == 1


def test_descriptor_offsets_match_c(tmp_path):
    from efficientteacher_b200 import _lib
    fields = [("EtbPackDesc", f) for f, _ in _lib.EtbPackDesc._fields_] + [("EtbFoldDesc", f) for f, _ in _lib.EtbFoldDesc._fields_]
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "etb200.h"\nint main(){' + "".join(
        'printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (s, f, s, f) for s, f in fields) + "return 0;}"
    c = tmp_path / "off.c"
    c.write_text(src)
    exe = str(tmp_path / "off")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe])
    out = dict(l.split() for l in subprocess.check_output([exe]).decode().splitlines())
    for s, f in fields:
        assert int(out["%s.%s" % (s, f)]) == getattr(getattr(_lib, s), f).offset, (s, f)


def _conv(dtype, cout=16, cin=8):
    return torch.nn.Conv2d(cin, cout, 3, 1, 1, bias=False).to(dtype)


def test_packer_refuses_dtypes_it_cannot_read():
    from efficientteacher_b200.packing import WeightPacker
    pk = WeightPacker(torch.device("cpu"))
    pk.add(_conv(torch.float16).weight, 1, 1, want_dgrad=True, name="a.weight")
    pk.add(_conv(torch.float64).weight, 1, 1, want_dgrad=False, name="b.weight")
    with pytest.raises(NotImplementedError, match=r"b\.weight is torch\.float64"):
        pk.run()
    assert pk._built is None
    pk = WeightPacker(torch.device("cpu"))
    pc = pk.add(_conv(torch.bfloat16).weight, 1, 1, want_dgrad=False, name="c.conv.weight")
    bn = torch.nn.BatchNorm2d(16).half()
    bn.running_var = bn.running_var.float()
    pk.add_fold(bn, pc, name="c.bn")
    with pytest.raises(NotImplementedError, match=r"c\.bn mixes \['torch\.float16', 'torch\.float32'\]"):
        pk.run()
    head = torch.nn.Conv2d(8, 24, 1).double()
    pk = WeightPacker(torch.device("cpu"))
    pk.add(head.weight.float(), 1, 0, want_dgrad=False, name="head.weight")
    pk.add_bias(head, name="head.bias")
    with pytest.raises(NotImplementedError, match=r"head\.bias is torch\.float64"):
        pk.run()


def test_packer_key_follows_dtype_and_storage():
    from efficientteacher_b200.packing import WeightPacker
    conv = torch.nn.Conv2d(8, 24, 1)
    bn = torch.nn.BatchNorm2d(24)
    pk = WeightPacker(torch.device("cpu"))
    pc = pk.add(conv.weight, 1, 0, want_dgrad=False)
    pk.add_fold(bn, pc)
    pk.add_bias(conv)
    k0 = pk._key()
    assert len(k0) == 1 + 4 + 1
    conv.half()
    k1 = pk._key()
    assert k1 != k0 and k1[0][1] == torch.float16 and k1[-1][1] == torch.float16
    bn.bfloat16()                         # new buffer objects: the packer reads them from the module
    k2 = pk._key()
    assert all(dt == torch.bfloat16 for _, dt in k2[1:5])
    # the same storage seen as another dtype is a change too
    ptr = conv.weight.data_ptr()
    conv.weight.data = conv.weight.data.view(torch.bfloat16)
    k3 = pk._key()
    assert k3[0] == (ptr, torch.bfloat16) and k3 != k2


def test_training_forward_needs_an_fp32_model():
    from efficientteacher_b200.config import yolov5_sup_cfg
    from efficientteacher_b200.model import SupModel
    m = SupModel(yolov5_sup_cfg("n", batch_size=2, img_size=64))
    m._require_fp32()
    assert m._state_fp32
    m.half()
    assert m._state_fp32 is None
    with pytest.raises(NotImplementedError, match=r"backbone\.stage1\.conv\.weight is torch\.float16"):
        m._require_fp32()
    m.float()
    m._require_fp32()
    m.bfloat16()
    with pytest.raises(NotImplementedError, match=r"is torch\.bfloat16: the native training forward needs an fp32 model"):
        m._require_fp32()
    m.head.float()                                  # a partial conversion still leaves bf16 state behind
    m.head.anchors = m.head.anchors.float()
    with pytest.raises(NotImplementedError, match=r"backbone\.stage1\.conv\.weight is torch\.bfloat16"):
        m._require_fp32()
