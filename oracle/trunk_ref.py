"""TEST INFRASTRUCTURE ONLY -- plain PyTorch fp32 functional forward of the YOLOv5 trunk + Detect + netD from a
state_dict with the reference's key names (models/backbone/yolov5_backbone.py:76-88, models/neck/yolov5_neck.py:88-109,
models/head/yolov5_head.py:47-87, models/detector/yolo_ssod.py:105-118, models/backbone/common.py Conv/Bottleneck/C3/SPPF).
It is the torch reference the wgmma trunk is compared with, and the trunk of the CPU baseline in bench.py.
Works on any device; train=True uses batch statistics and, with bn_momentum > 0, updates the running statistics in the
state_dict in place like nn.BatchNorm2d does (default 0: leaves them alone)."""
import torch
import torch.nn.functional as F


class TrunkRef:
    def __init__(self, state_dict, depth=(3, 6, 9, 3), neck_depth=3, bn_eps=1e-3, bn_momentum=0.0):
        self.sd = state_dict
        self.eps = bn_eps
        self.momentum = bn_momentum
        self.depth, self.neck_depth = depth, neck_depth

    @classmethod
    def from_module(cls, model):
        bb = model.backbone
        depth = tuple(len(getattr(bb, n).m) for n in ("stage2_2", "stage3_2", "stage4_2", "stage5_2"))
        return cls(dict(model.state_dict()), depth, len(model.neck.C1.m))

    def conv(self, p, x, k, s, train, act=True):
        sd = self.sd
        y = F.conv2d(x, sd[p + ".conv.weight"], None, s, k // 2 if k != 6 else 2)
        if train and self.momentum > 0:
            y = F.batch_norm(y, sd[p + ".bn.running_mean"], sd[p + ".bn.running_var"], sd[p + ".bn.weight"], sd[p + ".bn.bias"], True,
                             self.momentum, self.eps)
        elif train:
            y = F.batch_norm(y, None, None, sd[p + ".bn.weight"], sd[p + ".bn.bias"], True, 0.0, self.eps)
        else:
            y = F.batch_norm(y, sd[p + ".bn.running_mean"], sd[p + ".bn.running_var"], sd[p + ".bn.weight"], sd[p + ".bn.bias"],
                             False, 0.0, self.eps)
        return F.silu(y) if act else y

    def c3(self, p, x, n, shortcut, train):
        t = self.conv(p + ".cv1", x, 1, 1, train)
        for i in range(n):
            u = self.conv("%s.m.%d.cv2" % (p, i), self.conv("%s.m.%d.cv1" % (p, i), t, 1, 1, train), 3, 1, train)
            t = t + u if shortcut else u
        return self.conv(p + ".cv3", torch.cat([t, self.conv(p + ".cv2", x, 1, 1, train)], 1), 1, 1, train)

    def forward(self, x, train=False, with_features=True):
        d = self.depth
        x = self.conv("backbone.stage1", x, 6, 2, train)
        x = self.c3("backbone.stage2_2", self.conv("backbone.stage2_1", x, 3, 2, train), d[0], True, train)
        c3 = self.c3("backbone.stage3_2", self.conv("backbone.stage3_1", x, 3, 2, train), d[1], True, train)
        c4 = self.c3("backbone.stage4_2", self.conv("backbone.stage4_1", c3, 3, 2, train), d[2], True, train)
        x5 = self.c3("backbone.stage5_2", self.conv("backbone.stage5_1", c4, 3, 2, train), d[3], True, train)
        s = self.conv("backbone.sppf.cv1", x5, 1, 1, train)
        y1 = F.max_pool2d(s, 5, 1, 2); y2 = F.max_pool2d(y1, 5, 1, 2); y3 = F.max_pool2d(y2, 5, 1, 2)
        p5 = self.conv("backbone.sppf.cv2", torch.cat([s, y1, y2, y3], 1), 1, 1, train)
        nd = self.neck_depth
        xp1 = self.conv("neck.conv1", p5, 1, 1, train)
        x1 = self.c3("neck.C1", torch.cat([F.interpolate(xp1, scale_factor=2, mode="nearest"), c4], 1), nd, False, train)
        xp2 = self.conv("neck.conv2", x1, 1, 1, train)
        x2 = self.c3("neck.C2", torch.cat([F.interpolate(xp2, scale_factor=2, mode="nearest"), c3], 1), nd, False, train)
        x3 = self.c3("neck.C3", torch.cat([self.conv("neck.conv3", x2, 3, 2, train), xp2], 1), nd, False, train)
        x4 = self.c3("neck.C4", torch.cat([self.conv("neck.conv4", x3, 3, 2, train), xp1], 1), nd, False, train)
        feats = (x2, x3, x4)
        raw = []
        for i, f in enumerate(feats):
            y = F.conv2d(f, self.sd["head.m.%d.weight" % i], self.sd["head.m.%d.bias" % i])
            B, _, ny, nx = y.shape
            raw.append(y.view(B, 3, -1, ny, nx).permute(0, 1, 3, 4, 2).contiguous())
        feature = None
        if with_features and "det_8.conv1.weight" in self.sd:
            feature = [F.conv2d(F.relu(F.conv2d(f, self.sd[d_ + ".conv1.weight"])), self.sd[d_ + ".conv2.weight"])
                       for d_, f in zip(("det_8", "det_16", "det_32"), feats)]
        return raw, feature
