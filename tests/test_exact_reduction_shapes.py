"""CPU: the layer shapes the exact-reduction GPU tests (test_gpu_exact_reductions.py) run at, taken from the models.

Every YOLOv5 size the reference ships (n, s, m, l, x) is built and run once on the CPU at a 64x64 image with forward
pre-hooks on its convolutions, BatchNorms, pools, upsamples and concats.  Every map of the trunk is image/stride, so the
recorded maps scale exactly to the 640x640 training image; the batch is 32, the student batch of both bench configs.
The stem (6x6 s2 p2 on the image) runs its weight gradient as a pointwise K=128 GEMM over the im2col buffer and is listed
apart.  netD's conv2 (C -> 2) is not a weight-gradient GEMM (etb_netd_tail_bwd) and is left out.

The tests here keep the lists honest: a change of the model builder that emptied them, or a change of the split-K plan
that moved every model shape out of a branch of the plan or of the second-stage reduce, fails here without a GPU."""
import ctypes as C
import functools

import pytest
import torch
import torch.nn as nn

SIZES = ("n", "s", "m", "l", "x")
N_BATCH = 32
IMG = 640
PROBE = 64          # the CPU forward's image side: the stride-32 level is 2x2


@functools.lru_cache(maxsize=None)
def model_layers(size):
    """dict of the layers of Model(yolov5_ssod_cfg(size)) at a PROBE x PROBE image, shapes scaled to IMG:
    conv: [(name, Cin, Cout, k, s, p, H, W)] (H, W: the input map), bn: [(name, C, H, W)], pool: [(name, C, H, W)] (SPPF's
    5x5 pools), up: [(name, C, H, W)] (the upsample's input), cat: [(name, [C of each part], H, W)]"""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.model import SPPF, Concat, Model
    torch.manual_seed(0)
    m = Model(yolov5_ssod_cfg(size)).train()     # train: the Detect head returns its maps (no decode)
    rec = {"conv": [], "bn": [], "pool": [], "up": [], "cat": []}
    scale = IMG // PROBE

    def hw(t):
        H, W = t.shape[2:]
        assert PROBE % H == 0 and PROBE % W == 0, (H, W)     # every map is image/stride: the scaling is exact
        return H * scale, W * scale

    def hook(name, mod):
        def f(_, args):
            x = args[0]
            if isinstance(mod, nn.Conv2d):
                if not (name.startswith("det_") and name.endswith(".conv2")):
                    rec["conv"].append((name, mod.in_channels, mod.out_channels, mod.kernel_size[0], mod.stride[0], mod.padding[0], *hw(x)))
            elif isinstance(mod, nn.BatchNorm2d):
                rec["bn"].append((name, x.shape[1], *hw(x)))
            elif isinstance(mod, SPPF):
                rec["pool"].append((name, mod.cv1.conv.out_channels, *hw(x)))
            elif isinstance(mod, nn.Upsample):
                rec["up"].append((name, x.shape[1], *hw(x)))
            elif isinstance(mod, Concat):
                rec["cat"].append((name, [t.shape[1] for t in x], *hw(x[0])))
        return f

    for name, mod in m.named_modules():
        if isinstance(mod, (nn.Conv2d, nn.BatchNorm2d, SPPF, nn.Upsample, Concat)):
            mod.register_forward_pre_hook(hook(name, mod))
    with torch.no_grad():
        f = m.neck(m.backbone(torch.zeros(1, 3, PROBE, PROBE)))
        m.head(f)
        for d, x in zip((m.det_8, m.det_16, m.det_32), f):
            d(x, True)
    return rec


def wgrad_cases(size):
    """(N, Cin, H, W, Cout, k, s, p) of every weight-gradient GEMM of `size` but the stem, in model order, deduplicated"""
    out = []
    for name, Cin, Cout, k, s, p, H, W in model_layers(size)["conv"]:
        case = (N_BATCH, Cin, H, W, Cout, k, s, p)
        if name != "backbone.stage1.conv" and case not in out:
            out.append(case)
    return out


def stem_case(size):
    """the stem's weight gradient as etb_conv_wgrad runs it: a flat K=128 GEMM over the [N, H/2, W/2, 128] im2col buffer"""
    (name, Cin, Cout, k, s, p, H, W), = [c for c in model_layers(size)["conv"] if c[0] == "backbone.stage1.conv"]
    assert (Cin, k, s, p) == (3, 6, 2, 2)
    return (N_BATCH, 128, H // 2, W // 2, Cout, 1, 1, 0)


def bn_cases(size):
    """(M = N*H*W, C) of every BatchNorm of `size`, deduplicated"""
    out = []
    for _, C_, H, W in model_layers(size)["bn"]:
        if (N_BATCH * H * W, C_) not in out:
            out.append((N_BATCH * H * W, C_))
    return out


def _merge(fn):
    out = []
    for size in SIZES:
        for c in fn(size):
            if c not in out:
                out.append(c)
    return out


# synthetic weight-gradient shapes for branches of the plan no model layer reaches: none today (test_plan_coverage)
SYNTHETIC_WGRAD = {}


def all_wgrad_cases():
    model = _merge(wgrad_cases)
    return model + [c for c in SYNTHETIC_WGRAD.values() if c not in model]


def all_stem_cases():
    return _merge(lambda s: [stem_case(s)])


def all_bn_cases():
    return _merge(bn_cases)


def glue_cases():
    """(pool: (N, C, H, W) of SPPF's pools, up: (N, C, H, W) of the upsample inputs, cat: (N, H, W, C of the copied part,
    its channel offset, width of the concat)) of every size, deduplicated.  The first part of every neck concat is written
    in place by its producer (upsample or stride-2 conv); the second, the lateral, is copied in by etb_copy_slice_nhwc."""
    pool = _merge(lambda s: [(N_BATCH, C_, H, W) for _, C_, H, W in model_layers(s)["pool"]])
    up = _merge(lambda s: [(N_BATCH, C_, H, W) for _, C_, H, W in model_layers(s)["up"]])
    cat = _merge(lambda s: [(N_BATCH, H, W, cs[1], cs[0], sum(cs)) for _, cs, H, W in model_layers(s)["cat"]])
    return pool, up, cat


# ------------------------------------------------------------------------------------------------------------------ tests
def test_shapes_are_listed_for_every_size():
    from test_conv_plan import REAL
    want_real = [c for c in REAL if c[0] == N_BATCH and c[2] == c[3]]      # the square batch-32 shapes of the plan test
    assert want_real
    for size in SIZES:
        rec = model_layers(size)
        assert wgrad_cases(size) and bn_cases(size), size
        assert len(rec["pool"]) == 1 and len(rec["up"]) == 2 and len(rec["cat"]) == 4, size
        assert stem_case(size)[1:4] == (128, IMG // 2, IMG // 2), size
    merged = all_wgrad_cases()
    for c in want_real:
        if c[1] <= 1024 and c[4] <= 1024:       # (32, 2048, 20, 20, 1024) is a synthetic shape of the plan test
            assert c in merged, c
    # YOLOv5l: 61 convs in the backbone, 40 in the neck, 3 Detect convs, 3 netD conv1 (+ 3 netD conv2, not listed)
    rec = model_layers("l")
    assert len(rec["conv"]) == 107 and len(rec["bn"]) == 101
    assert (N_BATCH * 320 * 320, 64) in bn_cases("l")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from efficientteacher_b200 import _lib
    return _lib


def wgrad_splits(lib, case):
    """split-K count of the plan (etb_conv_wgrad_workspace_bytes / one fp32 [Cout, k*k*Cin] slice)"""
    N, Cin, H, W, Cout, k, s, p = case
    cp = lib.EtbConvParams(N=N, H=H, W=W, Cin=Cin, Cout=Cout, kh=k, kw=k, stride=s, pad=p, x_cstride=Cin,
                           y_cstride=(Cout + 7) // 8 * 8)
    nbytes = int(lib.lib().etb_conv_wgrad_workspace_bytes(C.byref(cp)))
    slice_bytes = Cout * k * k * Cin * 4
    assert nbytes > 0 and nbytes % slice_bytes == 0, (case, nbytes)
    return nbytes // slice_bytes


def wgrad_branches(lib, case, stem=False):
    """the branches of etb_conv_wgrad's plan and second stage that `case` runs"""
    N, Cin, H, W, Cout, k, s, p = case
    sk = wgrad_splits(lib, case)
    out = {"BN = %d" % (128 if Cin >= 128 else 64)}
    out.add("flat" if (k == 1 and s == 1 and p == 0) else "tiled")
    if s == 2:
        out.add("stride 2")
    if Cout % 128:
        out.add("Cout % 128 != 0")
    if stem:
        out.add("stem")
    if k * k > 1 and not stem:
        out.add("reduce_taps")
        out.add("reduce_taps, Cin % 64 != 0" if Cin % 64 else "reduce_taps, Cin % 64 == 0")
        if sk > 4 and sk % 4:
            out.add("reduce_taps, splitk > 4, splitk % 4 != 0")
    elif sk >= 32:
        out.add("reduce<16>, splitk >= 32")
    elif sk >= 6:
        out.add("reduce<4>, splitk 6-31")
    elif sk >= 2:
        out.add("reduce<1>, splitk 2-5")
    else:
        out.add("reduce<1>, splitk 1")
    return out


REQUIRED_BRANCHES = {
    "reduce<1>, splitk 1", "reduce<1>, splitk 2-5", "reduce<4>, splitk 6-31", "reduce<16>, splitk >= 32",
    "reduce_taps, Cin % 64 != 0", "reduce_taps, Cin % 64 == 0", "reduce_taps, splitk > 4, splitk % 4 != 0",
    "stride 2", "flat", "tiled", "BN = 64", "BN = 128", "stem", "Cout % 128 != 0",
}


def test_plan_coverage(lib):
    """the model shapes plus SYNTHETIC_WGRAD reach every branch of the split-K plan and of the second-stage reduce"""
    seen = set()
    for case in all_wgrad_cases():
        seen |= wgrad_branches(lib, case)
    for case in all_stem_cases():
        seen |= wgrad_branches(lib, case, stem=True)
    assert REQUIRED_BRANCHES <= seen, sorted(REQUIRED_BRANCHES - seen)
    # each synthetic shape earns its place: it reaches a branch the model shapes alone miss
    model_only = set()
    for case in _merge(wgrad_cases):
        model_only |= wgrad_branches(lib, case)
    for case in all_stem_cases():
        model_only |= wgrad_branches(lib, case, stem=True)
    for name, case in SYNTHETIC_WGRAD.items():
        assert wgrad_branches(lib, case) - model_only, name
