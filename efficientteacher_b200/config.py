"""Standalone restatement of the slice of the reference's yacs config tree the hot path reads
(configs/defaults.py + configs/ssod/coco-standard/yolov5l_coco_ssod_10_percent.yaml + configs/sup/public/yolov5l_coco.yaml).
The real trainer passes its own frozen CfgNode; these namespaces exist so bench.py / smoke() / tests can build the
same objects on a box without the reference checkout.  Attribute names and values are the reference's."""
from types import SimpleNamespace as NS

COCO_NAMES = [str(i) for i in range(80)]
ANCHORS = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]


def _model(depth, width, backbone_act='SiLU', neck_act='SiLU'):
    return NS(depth_multiple=depth, width_multiple=width, ch=3, inplace=True, anchors=[list(a) for a in ANCHORS],
              RepOpt=False, weights='',
              Backbone=NS(name='YoloV5', activation=backbone_act),
              Neck=NS(name='YoloV5', activation=neck_act, in_channels=[256, 512, 1024], out_channels=[256, 512, 1024]),
              Head=NS(name='YoloV5', activation='SiLU', strides=[8, 16, 32]))


def _hyp():
    return NS(lr0=0.01, lrf=1.0, momentum=0.937, weight_decay=0.0005, warmup_epochs=3, warmup_momentum=0.8,
              warmup_bias_lr=0.1, burn_epochs=0)


def _loss():
    return NS(type='ComputeLoss', autobalance=False, cls_pw=1.0, obj_pw=1.0, label_smoothing=0.0, fl_gamma=0.0, box=0.05,
              obj=0.7, cls=0.3, anchor_t=4.0, single_targets=False, assigner_type='TAL', top_k=13)


def _ssod():
    return NS(train_domain=True, nms_conf_thres=0.1, nms_iou_thres=0.65, teacher_loss_weight=3.0, cls_loss_weight=0.3,
              box_loss_weight=0.05, obj_loss_weight=0.7, loss_type='ComputeStudentMatchLoss', ignore_thres_low=0.1,
              ignore_thres_high=0.6, uncertain_aug=True, use_ota=False, multi_label=False, ignore_obj=False,
              pseudo_label_with_obj=True, pseudo_label_with_bbox=True, pseudo_label_with_cls=False, with_da_loss=False,
              da_loss_weights=0.01, epoch_adaptor=True, ema_rate=0.999, cosine_ema=True, imitate_teacher=False,
              focal_loss=0.0, pseudo_label_type='FairPseudoLabel', debug=False, fixed_accumulate=False,
              extra_teachers=[], multi_step_lr=False, milestones=[10, 20], ssod_hyp=NS(with_gt=False))


# (depth_multiple, width_multiple) of the reference's five YOLOv5 sizes (configs/sup/public/yolov5{n,s,m,l,x}_coco.yaml),
# plus shallow variants (depth 0.33: one or two Bottlenecks per C3) that keep a size's widths for quick tests
SIZES = {'n': (0.33, 0.25), 's': (0.33, 0.50), 'm': (0.67, 0.75), 'l': (1.0, 1.0), 'x': (1.33, 1.25),
         'l_shallow': (0.33, 1.0), 'm_shallow': (0.33, 0.75), 'x_shallow': (0.33, 1.25)}


def yolov5_ssod_cfg(size='l', batch_size=32, img_size=640, backbone_act='SiLU', neck_act='SiLU'):
    """backbone_act / neck_act: cfg.Model.{Backbone,Neck}.activation -- 'SiLU', 'ReLU', or anything else for the Hardswish
    trunk (the reference's defaults, configs/defaults.py, are 'LeakyReLU' and 'ReLU': a Hardswish backbone, a ReLU neck)"""
    depth, width = SIZES[size]
    return NS(epochs=300, adam=False, linear_lr=True, single_cls=False, sync_bn=False,
              hyp=_hyp(), Model=_model(depth, width, backbone_act, neck_act), Loss=_loss(), SSOD=_ssod(),
              Dataset=NS(nc=80, np=0, names=list(COCO_NAMES), img_size=img_size, batch_size=batch_size))


def yolov5_sup_cfg(size='l', batch_size=32, img_size=640, backbone_act='SiLU', neck_act='SiLU'):
    cfg = yolov5_ssod_cfg(size, batch_size, img_size, backbone_act, neck_act)
    cfg.SSOD.train_domain = False
    cfg.linear_lr = False
    return cfg
