"""GPU (H100): half-precision models on the native engine -- model.half() / model.bfloat16() state read as stored by the
weight packer (etb_pack_multi), the BatchNorm fold (etb_fold_bn_multi) and the Detect bias copy, and fp16 images read by
the stem im2col (etb_stem_im2col_into).

  * a .half() model gives, bit for bit, what the fp32 model holding its fp16 values (val.round_fp16_) gives: predictions,
    raw levels and netD features, for Model and SupModel at sizes n, s and l under the SiLU, ReLU and Hardswish trunks;
    a .bfloat16() model likewise against the fp32 model holding its bf16 values;
  * an fp16 image batch gives what its .float() copy gives;
  * .half() -> forward -> .float() -> forward repacks from the new storage every time, and so does load_state_dict;
  * the reference's after_train validation of best.pt (checkpoint stored .half(), loaded, .float(), eval, .half(), forward
    on img.half() / 255, NMS, process_batch) restated on the native side;
  * a Predictor on a .half() copy of the teacher between a captured SSOD step and its replay leaves the replay as eager;
  * a float64 model in eval and a .half() model in training raise NotImplementedError before any launch."""
import io
from copy import deepcopy

import numpy as np
import pytest
import torch

import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# cfg.Model.{Backbone,Neck}.activation of the three native trunks (model.trunk_acts)
TRUNKS = {"silu": ("SiLU", "SiLU"), "relu": ("ReLU", "ReLU"), "hswish": ("Hardswish", "Hardswish")}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _model(sup, size="s", trunk="silu", seed=0):
    """A model with random BatchNorm state and conv weights whose fp16 / bf16 roundings differ from fp32, and a head that
    keeps classes 0..3 (so NMS has rows to compare)"""
    from efficientteacher_b200.config import yolov5_ssod_cfg, yolov5_sup_cfg
    from efficientteacher_b200.model import Model, SupModel
    torch.manual_seed(seed)
    bb, nk = TRUNKS[trunk]
    cfg = (yolov5_sup_cfg if sup else yolov5_ssod_cfg)(size, batch_size=2, img_size=256, backbone_act=bb, neck_act=nk)
    m = (SupModel if sup else Model)(cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
                mod.weight.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.1)
        for h in m.head.m:
            b = h.bias.view(3, -1)
            b[:, 4] += 6.0
            b[:, 5:] = -12.0
            b[:, 5:9] = 1.0 + torch.rand(b[:, 5:9].shape, generator=g) * 1e-3   # not representable in fp16
    return m.to(DEV).eval()


def _round_(model, dtype):
    """model.to(dtype); model.float() in place (val.round_fp16_ for fp16)"""
    from efficientteacher_b200.val import round_fp16_
    if dtype == torch.float16:
        round_fp16_(model)
        return model
    with torch.no_grad():
        for t in list(model.parameters()) + list(model.buffers()):
            if t.is_floating_point():
                t.copy_(t.to(dtype))
    return model


def _outputs(model, x):
    """(pred, raw levels, netD features) of an eval forward under no_grad, all fp32"""
    with torch.no_grad():
        out = model(x)
    (pred, raw), feat = out if hasattr(model, "det_8") else (out, [])     # Model: ((pred, raw), features); SupModel: (pred, raw)
    return [pred] + list(raw) + list(feat)


def _equal(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == torch.float32 and a.shape == b.shape, (what, i, a.dtype, a.shape, b.shape)
        assert torch.equal(a, b), (what, i, (a - b).abs().max().item())


def _u8(seed, B, H, W):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, 256, (B, 3, H, W)).astype(np.uint8)).to(DEV)


@pytest.mark.parametrize("trunk", list(TRUNKS))
@pytest.mark.parametrize("size", ["n", "s", "l"])
@pytest.mark.parametrize("sup", [False, True], ids=["ssod", "sup"])
def test_half_and_bf16_models_equal_the_rounded_fp32_model(sup, size, trunk):
    m = _model(sup, size, trunk)
    u = _u8(1, 2, 256, 384)
    x = u.half() / 255                              # val.py:281
    for dtype in (torch.float16, torch.bfloat16):
        lowp = deepcopy(m).to(dtype)
        assert all(p.dtype == dtype for p in lowp.parameters()) and lowp.head.anchors.dtype == dtype
        ref = _round_(deepcopy(m), dtype)
        want = _outputs(ref, x.float())
        assert want[0].shape[1] == 3 * (32 * 48 + 16 * 24 + 8 * 12)
        _equal(_outputs(lowp, x), want, (dtype, "fp16 image"))
        _equal(_outputs(lowp, x.float()), want, (dtype, "fp32 image"))
        _equal(_outputs(lowp, u), _outputs(ref, u), (dtype, "uint8 image"))
    # the rounding matters here: the fp32 model itself gives different numbers
    assert not torch.equal(_outputs(m, x.float())[0], want[0])


def test_fp16_images_equal_their_float_copy():
    from efficientteacher_b200 import convops as co
    u = _u8(2, 3, 130, 198)                         # odd multiples of 2: partial 64-pixel tiles
    x = u.half() / 255
    got = co.stem_im2col_parts([x], 1.0)
    assert torch.equal(got, co.stem_im2col_parts([x.float()], 1.0))
    # several fp16 parts into one buffer: the batch concatenation
    assert torch.equal(co.stem_im2col_parts([x[:1], x[1:]], 1.0), got)
    # the model: an fp16 batch and its .float() copy give the same outputs
    m = _model(False, "s").half()
    x = _u8(3, 2, 256, 384).half() / 255
    _equal(_outputs(m, x), _outputs(m, x.float()), "model")


def test_fp16_image_rounding_against_the_uint8_path():
    """img.half() / 255 rounds to fp16 before the stem rounds to bf16.  Of the 256 pixel values, 26 (1, 2, 4, 8, 16, 17,
    ...) then land one bf16 ulp away from where uint8 / 255 rounds: the stem reproduces each route as it is."""
    from efficientteacher_b200 import convops as co
    v = torch.arange(256, dtype=torch.uint8, device=DEV)
    u = v.repeat(3)[:3 * 4 * 64].view(1, 3, 4, 64)
    # input pixel (2oh, 2ow) of channel c is K slot (c*6 + 2)*6 + 2 of output pixel (oh, ow)
    centre = lambda t: t[..., :108].reshape(1, 2, 32, 3, 6, 6)[..., 2, 2].permute(0, 3, 1, 2)   # noqa: E731
    from_u8 = (u.float() / 255).to(torch.bfloat16)
    from_f16 = (u.half() / 255).float().to(torch.bfloat16)
    assert torch.equal(centre(co.stem_im2col_parts([u], 255.0)), from_u8[:, :, ::2, ::2])
    assert torch.equal(centre(co.stem_im2col_parts([u.half() / 255], 1.0)), from_f16[:, :, ::2, ::2])
    a, b = (v.float() / 255).to(torch.bfloat16), (v.half() / 255).float().to(torch.bfloat16)
    step = (a.view(torch.int16).int() - b.view(torch.int16).int()).abs()      # positive bf16: adjacent values differ by 1
    assert int((step != 0).sum()) == 26 and int(step.max()) == 1


def test_half_float_round_trip_and_load_state_dict_repack():
    m0 = _model(False, "s")
    x = _u8(4, 2, 256, 384)
    m = deepcopy(m0).half()
    fp16 = _outputs(m, x)
    m.float()
    back = _outputs(m, x)
    want = _outputs(_round_(deepcopy(m0), torch.float16), x)
    _equal(fp16, want, "half")
    _equal(back, want, "half -> float")
    other = _model(False, "s", seed=5)
    m.load_state_dict(other.state_dict())
    new = _outputs(m, x)
    assert not torch.equal(new[0], back[0])
    _equal(new, _outputs(other, x), "load_state_dict")
    # and once more to fp16: the packer follows the new storage again
    m.half()
    _equal(_outputs(m, x), _outputs(_round_(deepcopy(other), torch.float16), x), "load_state_dict -> half")


def test_half_anchors_get_their_own_decode_cache_key():
    from efficientteacher_b200 import head
    m = _model(True, "n")
    x = _u8(5, 1, 256, 256)
    _outputs(m, x)
    a32 = m.head.anchors
    k32 = (a32.data_ptr(), a32._version, a32.dtype)
    assert k32 in head._ANCHOR_CACHE
    m.half()
    a16 = m.head.anchors
    k16 = (a16.data_ptr(), a16._version, a16.dtype)
    assert k16 != k32
    _outputs(m, x)
    assert torch.equal(head._ANCHOR_CACHE[k16], a16.float().cpu())


def _labels_from(dets, r):
    """[n,5] (cls, x1, y1, x2, y2) labels: jittered copies of a third of an image's detections plus two unmatched boxes"""
    rows = []
    for x1, y1, x2, y2, _, c in dets.cpu().numpy():
        if r.rand() < 0.3:
            j = r.uniform(0.9, 1.1, 4)
            rows.append((c, x1 * j[0], y1 * j[1], x2 * j[2], y2 * j[3]))
    rows += [(0, 10, 10, 60, 80), (2, 100, 50, 180, 120)]
    return torch.tensor(rows, dtype=torch.float32, device=DEV)


def test_after_train_validation_of_a_half_checkpoint():
    """trainer.py after_train: val.run(model=attempt_load(best).half(), ...), where the checkpoint holds
    deepcopy(ema).half() and attempt_load returns ckpt.float().eval(); val.py then forwards img.half() / 255 under no_grad,
    runs non_max_suppression(multi_label=True) and process_batch.  The result equals that of the native val.run's route --
    the fp32 model rounded in place (round_fp16_) given the uint8 batch -- bit for bit, on pixel values whose fp16 / 255 and
    fp32 / 255 round to the same bf16 (test_fp16_image_rounding_against_the_uint8_path covers the others)."""
    from efficientteacher_b200 import nms as etb_nms
    from efficientteacher_b200 import val
    ema = _model(False, "s")
    buf = io.BytesIO()
    torch.save({"ema": deepcopy(ema).half(), "model": None}, buf)            # trainer.py:477-478
    buf.seek(0)
    ckpt = torch.load(buf, map_location="cpu", weights_only=False)            # experimental.py attempt_load
    model = (ckpt.get("ema") or ckpt["model"]).to(DEV).float().eval()
    model.half()                                                               # attempt_load(best).half()
    assert next(model.parameters()).dtype == torch.float16 and model._engine is None
    v = torch.arange(256)
    same = v[(v.float() / 255).to(torch.bfloat16) == (v.half() / 255).float().to(torch.bfloat16)]
    r = np.random.RandomState(6)
    u = same[torch.from_numpy(r.randint(0, len(same), (3, 3, 256, 384)))].to(torch.uint8).to(DEV)
    with torch.no_grad():
        out, _ = model(u.half() / 255)                                         # val.py:281, :307 (val_ssod)
    got = etb_nms.non_max_suppression(out[0], 0.001, 0.65, multi_label=True)  # iou_thres=0.65 as after_train passes
    ref = deepcopy(ema)
    val.round_fp16_(ref)                                                       # the native val.run(half=True)
    with torch.no_grad():
        out_ref, _ = ref(u)
    want = etb_nms.non_max_suppression(out_ref[0], 0.001, 0.65, multi_label=True)
    iouv = torch.linspace(0.5, 0.95, 10, device=DEV)
    tp = 0
    for si, (g, w) in enumerate(zip(got, want)):
        assert g.shape[0] > 0 and g.shape == w.shape and torch.equal(g, w), (si, g.shape, w.shape)
        labels = _labels_from(w, r)
        cg, cw = val.process_batch(g, labels, iouv), val.process_batch(w, labels, iouv)
        assert torch.equal(cg, cw), si
        tp += int(cw[:, 0].sum())
    assert tp > 0


def _images(seed, n, img):
    return torch.from_numpy(np.random.RandomState(seed).rand(n, 3, img, img).astype(np.float32)).to(DEV)


def _flat(tensors):
    return torch.cat([t.detach().flatten().float() for t in tensors])


def _frame(r, h0, w0):
    return np.frombuffer(bytearray(r.bytes(h0 * w0 * 3)), np.uint8).reshape(h0, w0, 3)


def test_captured_ssod_step_replayed_after_half_predictor_matches_eager():
    """step (graph: the capture), Predictor on a .half() copy of the teacher, step (graph: a replay): the state the eager
    run leaves, within the spread of two eager runs.  The copy has its own engine and packer: the teacher's storage and
    the workspaces the graph reads stay where they are."""
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.detect import Predictor
    from efficientteacher_b200.trainer import SSODTrainerStep
    img, bl, bu = 256, 2, 2
    imgs, uw = _images(3, bl, img), _images(4, bu, img)
    us = uw.flip(3).contiguous()
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    r = np.random.RandomState(11)
    frames = [_frame(r, 720, 1280) for _ in range(3)] + [_frame(r, 1280, 720)]
    out = {}
    for mode in ("eager", "eager2", "graph"):
        torch.manual_seed(0)
        cfg = yolov5_ssod_cfg('l_shallow', batch_size=bl + bu, img_size=img)
        cfg.hyp.warmup_epochs = 0
        cfg.hyp.burn_epochs = 0
        st = SSODTrainerStep(cfg, torch.device(DEV), epochs=300, batch_size=32)
        with torch.no_grad():
            for mm in (st.model, st.ema.ema, st.semi_ema.ema):
                for h in mm.head.m:
                    h.bias.view(3, -1)[:, 4] += 6.5
                    h.bias.view(3, -1)[:, 5:] += 5.0
        g = mode == "graph"
        f = lambda ni: (st.train_instance_graphed if g else st.train_instance)(imgs, tg, us, uw, None, Ms, ni)  # noqa: E731
        emas = [st.ema, st.semi_ema]
        f(1)
        ptrs = [t.data_ptr() for e in emas for t in e.ema.state_dict().values()]
        dets = Predictor(deepcopy(st.ema.ema).half(), img_size=640, max_det=1000)(frames)
        want = Predictor(_round_(deepcopy(st.ema.ema), torch.float16), img_size=640, max_det=1000)(frames)
        assert len(dets) == 4 and sum(d.shape[0] for d in dets) > 0 and st.model.training
        assert all(torch.equal(a, b) for a, b in zip(dets, want))
        assert [t.data_ptr() for e in emas for t in e.ema.state_dict().values()] == ptrs
        assert all(t.dtype == torch.float32 for e in emas for t in e.ema.state_dict().values() if t.is_floating_point())
        f(3)
        torch.cuda.synchronize()
        out[mode] = dict(weights=_flat(st.model.state_dict().values()), ema=_flat(t for e in emas for t in e.ema.state_dict().values()))
    for what in ("weights", "ema"):
        a, b, c = out["eager"][what], out["graph"][what], out["eager2"][what]
        assert torch.isfinite(b).all(), what
        n = a.norm().clamp_min(1e-30)
        rel, rel_eager = ((a - b).norm() / n).item(), ((a - c).norm() / n).item()
        assert rel <= 3.0 * rel_eager + 2e-3, (what, rel, rel_eager)


def _launches():
    from efficientteacher_b200 import _lib
    torch.cuda.synchronize()
    return int(_lib.lib().etb_launch_count())


def test_unsupported_dtypes_raise_before_any_launch():
    m = _model(False, "n")
    x = _u8(8, 1, 256, 256)
    _outputs(m, x)                                   # library loaded, workspaces made
    d = deepcopy(m).double()
    n0 = _launches()
    for _ in range(2):                               # the packer refuses on every call, not only while it is built
        with pytest.raises(NotImplementedError, match=r"backbone\.stage1\.conv\.weight is torch\.float64"):
            with torch.no_grad():
                d(x)
    assert _launches() == n0
    # a BatchNorm whose tensors the fold cannot read in one dtype
    mix = deepcopy(m)
    mix.neck.C2.cv3.bn.running_var = mix.neck.C2.cv3.bn.running_var.half()
    with pytest.raises(NotImplementedError, match=r"neck\.C2\.cv3\.bn mixes"):
        with torch.no_grad():
            mix(x)
    assert _launches() == n0
    # training forward of a half-precision model
    h = deepcopy(m).half().train()
    nbt = [b.num_batches_tracked.clone() for b in h.modules() if isinstance(b, torch.nn.BatchNorm2d)]
    with pytest.raises(NotImplementedError, match="is torch.float16: the native training forward needs an fp32 model"):
        h(_images(9, 2, 256))
    assert _launches() == n0
    assert all(torch.equal(a, b.num_batches_tracked) for a, b in zip(nbt, (b for b in h.modules() if isinstance(b, torch.nn.BatchNorm2d))))
    # ... and after .float() it trains again
    h.float()
    out, feats = h(_images(9, 2, 256))
    assert len(out) == 3 and len(feats) == 3 and _launches() > n0
