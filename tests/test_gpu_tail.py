"""GPU (H100): the native tail of the student's step (csrc/tail.cu) against plain PyTorch references of the same ops:
Detect backward layout + bias gradient, netD tail (C -> 2) forward/backward, Domain/Target focal loss forward/backward
(also against the oracle's restatement of models/loss/loss.py:312-421), the uint8 stem loader, and the zero-copy batch split."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__ as g
    g.build()
    torch.cuda.set_device(0)


def _bf(x):
    return x.to(torch.bfloat16).float()


@pytest.mark.parametrize("N,H,W", [(2, 20, 20), (3, 9, 7), (16, 80, 80)])
def test_detect_dy_pack_and_bias_grad(N, H, W):
    from efficientteacher_b200 import convops as co
    na, no = 3, 85
    g = torch.randn((N, na, H, W, no), generator=torch.Generator().manual_seed(1)).to(DEV)
    dy, partials = co.detect_dy_pack(g, 256)
    want = g.permute(0, 2, 3, 1, 4).reshape(N, H, W, na * no)
    assert torch.equal(dy[..., :255].float(), _bf(want))
    assert float(dy[..., 255:].abs().max()) == 0.0
    db = co.column_sum(partials)
    torch.testing.assert_close(db, g.sum((0, 2, 3)).reshape(-1), rtol=1e-5, atol=1e-4)
    base = torch.randn(255, device=DEV)
    acc = base.clone()
    co.column_sum(partials, out=acc, accumulate=True)
    torch.testing.assert_close(acc, base + db, rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize("C_,N,H", [(256, 2, 20), (512, 2, 10), (1024, 3, 5), (64, 2, 16)])
def test_netd_tail_fwd_bwd_vs_torch(C_, N, H):
    from efficientteacher_b200 import convops as co
    g = torch.Generator().manual_seed(2)
    h = torch.relu(torch.randn((N, H, H, C_), generator=g)).to(DEV).to(torch.bfloat16)
    w2 = (torch.randn((2, C_, 1, 1), generator=g) * C_ ** -0.5).to(DEV)
    o = co.netd_tail_fwd(h, C_, w2)
    hr = h.double().permute(0, 3, 1, 2).requires_grad_(True)          # float64 reference (cuDNN fp32 convs default to TF32)
    w2r = w2.double().requires_grad_(True)
    orf = F.conv2d(hr, w2r)
    torch.testing.assert_close(o.permute(0, 3, 1, 2).double(), orf.detach(), rtol=1e-5, atol=1e-5)
    do = torch.randn((N, H, H, 2), generator=g).to(DEV)
    orf.backward(do.double().permute(0, 3, 1, 2))
    dh, partials = co.netd_tail_bwd(do, h, C_, w2)
    want_dh = (hr.grad.permute(0, 2, 3, 1) * (h.double() > 0)).float()
    assert float((dh.float() - _bf(want_dh)).abs().max()) <= 1e-2 * max(float(want_dh.abs().max()), 1.0)
    dw2 = co.column_sum(partials).view(2, C_)
    torch.testing.assert_close(dw2.double(), w2r.grad.view(2, C_), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("label", [0, 1])
def test_domain_focal_loss_fwd_bwd(label):
    from efficientteacher_b200.domain_loss import DomainLoss, TargetLoss
    from oracle.step_ref import domain_focal
    g = torch.Generator().manual_seed(3)
    feats = [(torch.randn((4, 2, s, s), generator=g) * 2.0).to(DEV).requires_grad_(True) for s in (40, 20, 10)]
    loss = (DomainLoss() if label == 0 else TargetLoss())(feats)
    ref_in = [f.detach().clone().requires_grad_(True) for f in feats]
    ref = domain_focal(ref_in, label)
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    (loss * 3.0).backward()
    (ref * 3.0).backward()
    for a, b in zip(feats, ref_in):
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-4, atol=1e-7)
    # the native netD layout: NCHW-shaped views of [B,H,W,2] buffers, split along the batch without copies
    from efficientteacher_b200.autograd_conv import SplitBatchFn, split_batch
    base = [(torch.randn((4, s, s, 2), generator=g) * 2.0).to(DEV).requires_grad_(True) for s in (40, 20, 10)]
    views = [b.permute(0, 3, 1, 2) for b in base]
    before = dict(SplitBatchFn.stats)
    parts = [split_batch(v, 1) for v in views]
    tot = DomainLoss()([a for a, _ in parts]) + TargetLoss()([b for _, b in parts])
    tot.backward()
    assert SplitBatchFn.stats["zero_copy"] - before["zero_copy"] == 3 and SplitBatchFn.stats["copied"] == before["copied"]
    ref_b = [b.detach().clone().requires_grad_(True) for b in base]
    rv = [b.permute(0, 3, 1, 2) for b in ref_b]
    (domain_focal([v[:1] for v in rv], 0) + domain_focal([v[1:] for v in rv], 1)).backward()
    for a, b in zip(base, ref_b):
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-4, atol=1e-7)


def test_stem_im2col_uint8_parts_equal_float_path():
    from efficientteacher_b200 import convops as co
    r = np.random.RandomState(4)
    a = torch.from_numpy(r.randint(0, 256, (2, 3, 64, 96), dtype=np.uint8)).to(DEV)
    b = torch.from_numpy(r.randint(0, 256, (3, 3, 64, 96), dtype=np.uint8)).to(DEV)
    got = co.stem_im2col_parts([a, b], 255.0)
    want = co.stem_im2col_parts([torch.cat([a, b], 0).float() / 255.0], 1.0)   # trainer/ssod_trainer.py:694-696 then torch.cat (:620)
    assert torch.equal(got, want)
    got_f = co.stem_im2col_parts([a.float() / 255.0, b.float() / 255.0], 1.0)
    assert torch.equal(got_f, want)


def test_ssod_step_from_uint8_batches_and_zero_copy_split():
    """The whole step fed with the loaders' uint8 batches gives the loss of the fp32 path bit for bit (same bf16 stem operand),
    and every batch split of the step (3 head levels + 3 netD maps) takes the zero-copy backward."""
    from efficientteacher_b200.autograd_conv import SplitBatchFn
    from efficientteacher_b200.config import yolov5_ssod_cfg
    from efficientteacher_b200.trainer import SSODTrainerStep
    import synth
    img, bl, bu = 128, 2, 2
    r = np.random.RandomState(6)
    imgs8 = torch.from_numpy(r.randint(0, 256, (bl, 3, img, img), dtype=np.uint8)).to(DEV)
    uw8 = torch.from_numpy(r.randint(0, 256, (bu, 3, img, img), dtype=np.uint8)).to(DEV)
    us8 = uw8.flip(3).contiguous()
    tg = torch.from_numpy(synth.make_targets(7, 8 * bl, bl)).to(DEV)
    Ms = torch.from_numpy(synth.make_Ms(9, bu, img)).to(DEV)
    losses = []
    for as_u8 in (True, False):
        torch.manual_seed(0)
        st = SSODTrainerStep(yolov5_ssod_cfg('l_shallow', batch_size=bl + bu, img_size=img), torch.device(DEV), epochs=300)
        with torch.no_grad():
            for mm in (st.model, st.ema.ema, st.semi_ema.ema):
                for h in mm.head.m:
                    h.bias.view(3, -1)[:, 4] += 6.5
                    h.bias.view(3, -1)[:, 5:] += 5.0
        f = (lambda t: t) if as_u8 else (lambda t: t.float() / 255.0)
        before = dict(SplitBatchFn.stats)
        losses.append(float(st.train_instance(f(imgs8), tg, f(us8), f(uw8), None, Ms, 0)))
        assert SplitBatchFn.stats["zero_copy"] - before["zero_copy"] == 6 and SplitBatchFn.stats["copied"] == before["copied"]
        assert int(st.pseudo_label_creator.last_count_dev.item()) > 0
    assert losses[0] == losses[1], losses
