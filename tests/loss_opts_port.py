"""CPU restatement of the detection losses with the cfg.Loss options (torch CPU fp32, differentiable): oracle/port.det_loss
plus BCE positive weights, focal loss and autobalance (reference models/loss/loss.py:37-64,98-124,191-197,
models/loss/ssod/ssod_loss.py:32-38).  Pinned to the live reference by tests/test_oracle_loss_options.py."""
import torch

from oracle.port import _bce, _t, ciou


def crit(x, z, pw=1.0, gamma=0.0):
    """mean of BCEWithLogitsLoss(pos_weight=pw), wrapped in FocalLoss(gamma, alpha=0.25) when gamma > 0"""
    if pw == 1.0 and gamma == 0.0:
        return _bce(x, z).mean()
    lw = 1.0 + (pw - 1.0) * z
    loss = (1.0 - z) * x + lw * (torch.log1p(torch.exp(-x.abs())) + torch.clamp(-x, min=0))
    if gamma > 0.0:
        s = x.sigmoid()
        pt = z * s + (1.0 - z) * (1.0 - s)
        at = z * 0.25 + (1.0 - z) * (1.0 - 0.25)
        loss = loss * (at * (1.0 - pt) ** gamma)
    return loss.mean()


def det_loss(p, sets, balance, box_w, obj_w, cls_w, cp=1.0, cn=0.0, ignore_obj=False, with_bbox=False, with_cls=False,
             cls_pw=1.0, obj_pw=1.0, fl_gamma=0.0, autobalance=False, ssi=1):
    """oracle/port.det_loss with the loss options; at their defaults it computes what port.det_loss computes.
    autobalance=True: `balance` is a list of Python floats advanced in place as loss.py:191-197 does it (ssi = the
    stride-16 level); the objectness term of each level uses the value from before its update."""
    lbox = torch.zeros(1); lobj = torch.zeros(1); lcls = torch.zeros(1)
    for l, pi in enumerate(p):
        nc = pi.shape[-1] - 5
        tobj = torch.zeros(pi.shape[:-1])

        def gather(s):
            idx = _t(s["idx"], torch.int64)
            return pi[idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]], idx

        def box_term(s):
            ps, idx = gather(s)
            pxy = ps[:, :2].sigmoid() * 2.0 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * _t(s["anch"])
            return ciou(torch.cat([pxy, pwh], 1), _t(s["tbox"])), ps, idx

        def cls_term(ps, s):
            z = torch.full_like(ps[:, 5:], cn)
            z[torch.arange(len(ps)), _t(s["tcls"], torch.int64)] = cp
            return crit(ps[:, 5:], z, cls_pw, fl_gamma)

        s0 = sets[0][l]
        if len(s0["idx"]):
            iou, ps, idx = box_term(s0)
            lbox = lbox + (1.0 - iou).mean()
            v = iou.detach().clamp(0)
            for r in range(len(idx)):                           # last row wins (CPU index_put_ semantics)
                tobj[idx[r, 0], idx[r, 1], idx[r, 2], idx[r, 3]] = v[r]
            if nc > 1:
                lcls = lcls + cls_term(ps, s0)
        if len(sets) > 1:
            s1 = sets[1][l]
            idx1 = _t(s1["idx"], torch.int64)
            sc = _t(s1["tscore"])
            for r in range(len(idx1)):
                tobj[idx1[r, 0], idx1[r, 1], idx1[r, 2], idx1[r, 3]] = -1.0 if ignore_obj else sc[r]
            if with_bbox and len(sets[2][l]["idx"]):
                iou2, _, _ = box_term(sets[2][l])
                lbox = lbox + (1.0 - iou2).mean()
            if with_cls and nc > 1 and len(sets[3][l]["idx"]):
                ps3, _ = gather(sets[3][l])
                lcls = lcls + cls_term(ps3, sets[3][l])
        valid = tobj >= 0
        obji = crit(pi[..., 4][valid], tobj[valid], obj_pw, fl_gamma)
        lobj = lobj + obji * balance[l]
        if autobalance:
            balance[l] = balance[l] * 0.9999 + 0.0001 / obji.detach().item()
    if autobalance:
        balance[:] = [x / balance[ssi] for x in balance]
    lbox = lbox * box_w; lobj = lobj * obj_w; lcls = lcls * cls_w
    B = p[0].shape[0]
    return (lbox + lobj + lcls) * B, (lbox, lobj, lcls)
