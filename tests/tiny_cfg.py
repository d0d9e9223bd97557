"""A minimal stand-in for the yacs cfg tree + a head-only model, so the loss mirrors can be constructed in tests
without the full trunk (values = configs/ssod/coco-standard/yolov5l_coco_ssod_10_percent.yaml)."""
from types import SimpleNamespace as NS

import torch

import synth


def ssod_cfg(nc=80):
    return NS(
        single_cls=False,
        Loss=NS(autobalance=False, cls_pw=1.0, obj_pw=1.0, label_smoothing=0.0, fl_gamma=0.0, box=0.05, obj=0.7, cls=0.3,
                anchor_t=4.0, single_targets=False, assigner_type='TAL', top_k=13),
        Dataset=NS(nc=nc, np=0, names=[str(i) for i in range(nc)], img_size=640),
        SSOD=NS(focal_loss=0.0, box_loss_weight=0.05, obj_loss_weight=0.7, cls_loss_weight=0.3, ignore_thres_high=0.6,
                ignore_thres_low=0.1, uncertain_aug=True, use_ota=False, ignore_obj=False, pseudo_label_with_obj=True,
                pseudo_label_with_bbox=True, pseudo_label_with_cls=False, nms_conf_thres=0.1, nms_iou_thres=0.65,
                debug=False, multi_label=False),
    )


class _Head(torch.nn.Module):
    def __init__(self, nc):
        super().__init__()
        self.na, self.nc, self.nl, self.num_keypoints = 3, nc, 3, 0
        self.register_buffer("anchors", torch.from_numpy(synth.ANCHORS_GRID.copy()))
        self.stride = torch.tensor([8., 16., 32.])


class HeadOnlyModel(torch.nn.Module):
    def __init__(self, nc=80):
        super().__init__()
        self.head = _Head(nc)
        self.dummy = torch.nn.Parameter(torch.zeros(1))
