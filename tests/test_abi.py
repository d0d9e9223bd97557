"""CPU: the C-ABI shared library loads, exports every symbol include/etb200.h declares, and the ctypes struct
mirrors in efficientteacher_b200/_lib.py have the sizes the C compiler gives them.  No compute calls."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    syms = set()
    for fn in os.listdir(os.path.join(ROOT, "include")):
        if fn.endswith(".h"):
            src = open(os.path.join(ROOT, "include", fn)).read()
            src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
            syms |= set(re.findall(r"\b(etb_[a-z0-9_]+)\s*\(", src))
    return sorted(syms)


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    from efficientteacher_b200 import _lib
    return _lib


def test_library_exports_all_declared_symbols(built):
    lib = built.lib()
    declared = _header_symbols()
    assert len(declared) >= 12
    for s in declared:
        assert hasattr(lib, s), "libetb200.so does not export %s" % s
    assert set(built.exported_symbols()) == set(declared), "ctypes signature table out of sync with include/*.h"
    assert lib.etb_version() >= 100


def test_ctypes_struct_sizes_match_c(built, tmp_path):
    names = ["EtbChunk", "EtbNmsParams", "EtbAssignLevels", "EtbAssignOut", "EtbLossParams", "EtbFocalParams", "EtbPackDesc", "EtbFoldDesc", "EtbV8Levels"]
    if hasattr(built, "EtbConvParams") and "EtbConvParams" in open(os.path.join(ROOT, "include", "etb200.h")).read():
        names.append("EtbConvParams")
    src = '#include <stdio.h>\n#include "etb200.h"\nint main(){' + "".join(
        'printf("%s %%zu\\n", sizeof(%s));' % (n, n) for n in names) + "return 0;}"
    c = tmp_path / "sz.c"
    c.write_text(src)
    exe = str(tmp_path / "sz")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe])
    out = dict(l.split() for l in subprocess.check_output([exe]).decode().splitlines())
    for n in names:
        assert int(out[n]) == C.sizeof(getattr(built, n)), n


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    from efficientteacher_b200 import loss
    with pytest.raises(RuntimeError):
        loss.bbox_iou(torch.zeros(4, 3), torch.zeros(3, 4), x1y1x2y2=False, CIoU=True)
