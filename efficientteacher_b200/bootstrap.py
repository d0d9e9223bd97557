"""`import efficientteacher_b200.bootstrap` (first line of the reference's train.py / val.py, before its trainers are
imported) rebinds the reference's hot-path symbols to the native mirrors -- see INTEGRATION.md section 1.  Requires the
reference checkout on sys.path (it is the host application) and libetb200.so (no CPU fallback).

The reference binds these symbols BY NAME with `from X import Y` in several places, and it loads some files twice under
two module names (`sys.path` contains both the checkout root and `models/`, so `models/loss/loss.py` exists as
`models.loss.loss` AND as `loss.loss`: models/loss/__init__.py:1, trainer/trainer.py:30).  Patching the defining module
alone would therefore leave e.g. `models.loss.build_ssod_loss` (models/loss/__init__.py:3,17-19, called from
trainer/ssod_trainer.py:261) on the original class.  apply() does three things:
  1. imports the modules that define the originals and, when importable, the ones that bind them by name
     (trainer.trainer, trainer.ssod_trainer, models.loss, val);
  2. for every patch collects ALL original objects (same __name__, defined in a module whose dotted name is a suffix of the
     defining module: `loss.loss` for `models.loss.loss`);
  3. sweeps the namespaces of every loaded module and rebinds each attribute that IS one of those objects.
Modules of the host application imported later with `from X import Y` see the patched attribute of X anyway.
"""
import importlib
import inspect
import sys
import types

from . import _lib, ema, labelmatch, loss, metrics, model, nms, pl_quality, pseudo_label, ssod_loss, assigner, tal
from . import val as etb_val

_lib.lib()  # fail loudly now if the kernels are not built


def _val_nms(original):
    """utils.general.non_max_suppression (general.py:994-1098).  The best-class variant (training path) and the val.py variant
    (`multi_label=True`, val.py:335: etb_nms_val) run on the native kernels; calls with `classes` / a-priori `labels` or CPU
    tensors keep going to the host application's own function."""
    def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False, multi_label=False,
                            labels=(), max_det=300):
        if classes is not None or (labels is not None and len(labels)) or not prediction.is_cuda:
            return original(prediction, conf_thres, iou_thres, classes, agnostic, multi_label, labels, max_det)
        return nms.non_max_suppression(prediction, conf_thres, iou_thres, classes, agnostic, multi_label, (), max_det)
    non_max_suppression.__wrapped__ = original
    return non_max_suppression


def _bbox_iou(original):
    """utils.metrics.bbox_iou (metrics.py:207-249): the branch the losses use (xywh, CIoU, CUDA tensors) -> etb_bbox_ciou;
    every other variant (GIoU/DIoU/plain IoU, xyxy, CPU) stays with the reference's function."""
    def bbox_iou(box1, box2, x1y1x2y2=True, GIoU=False, DIoU=False, CIoU=False, eps=1e-7):
        if (not x1y1x2y2) and CIoU and not GIoU and not DIoU and eps == 1e-7 and box1.is_cuda and box2.is_cuda \
                and box1.dim() == 2 and box2.dim() == 2 and box1.shape[0] == 4 and not (box1.requires_grad or box2.requires_grad):
            return loss.bbox_iou(box1, box2, x1y1x2y2, GIoU, DIoU, CIoU, eps)
        return original(box1, box2, x1y1x2y2, GIoU, DIoU, CIoU, eps)
    bbox_iou.__wrapped__ = original
    return bbox_iou


def _val_run(original):
    """val.run (val.py:149-465): the training-time call (model and dataloader given, CUDA, plots=False, no txt / json /
    hybrid output, no keypoints, no model_post, no augment) runs natively (efficientteacher_b200.val.run); every other call
    goes to the host application's own run."""
    sig = inspect.signature(etb_val.run)

    def run(*args, **kwargs):
        try:
            bound = sig.bind(*args, **kwargs)
        except TypeError:
            return run.__wrapped__(*args, **kwargs)
        if etb_val.run_unsupported(**bound.arguments) is None:
            return etb_val.run(*args, **kwargs)
        return run.__wrapped__(*args, **kwargs)
    run.__wrapped__ = original
    return run


def _ap_per_class(original):
    """utils.metrics.ap_per_class (metrics.py:22-126): native (efficientteacher_b200.metrics); plot=True (the PR / F1 plots)
    goes to the host application's own function."""
    def ap_per_class(tp, conf, pred_cls, target_cls, plot=False, save_dir='.', names=()):
        if plot:
            return ap_per_class.__wrapped__(tp, conf, pred_cls, target_cls, plot=plot, save_dir=save_dir, names=names)
        return metrics.ap_per_class(tp, conf, pred_cls, target_cls)
    ap_per_class.__wrapped__ = original
    return ap_per_class


def _confusion_matrix(original):
    """utils.metrics.ConfusionMatrix (metrics.py:129-204), also val.py's by-name binding: the native class
    (efficientteacher_b200.metrics), whose process_batch runs on the device for CUDA tensors; calls with a CPU tensor run the
    host application's own process_batch into a host-side matrix that `matrix` adds in.  plot is the original plot, which
    reads only self.matrix and self.nc."""
    class ConfusionMatrix(metrics.ConfusionMatrix):
        host_plot = original.plot

        def process_batch(self, detections, labels):
            if detections.is_cuda and labels.is_cuda:
                return super().process_batch(detections, labels)
            host = types.SimpleNamespace(matrix=self.host, nc=self.nc, conf=self.conf, iou_thres=self.iou_thres)
            return original.process_batch(host, detections, labels)
    ConfusionMatrix.__wrapped__ = original
    return ConfusionMatrix


# (defining module, attribute, replacement | factory(original) -> replacement)
_PATCHES = [
    ("utils.torch_utils", "ModelEMA", ema.ModelEMA),
    ("utils.torch_utils", "SemiSupModelEMA", ema.SemiSupModelEMA),
    ("utils.torch_utils", "CosineEMA", ema.CosineEMA),
    ("utils.general", "non_max_suppression_ssod", nms.non_max_suppression_ssod),
    ("utils.general", "non_max_suppression", _val_nms),
    ("utils.metrics", "bbox_iou", _bbox_iou),
    ("utils.metrics", "ap_per_class", _ap_per_class),
    ("utils.metrics", "ConfusionMatrix", _confusion_matrix),
    ("val", "run", _val_run),
    ("utils.self_supervised_utils", "FairPseudoLabel", pseudo_label.FairPseudoLabel),
    ("utils.self_supervised_utils", "check_pseudo_label_with_gt", pl_quality.check_pseudo_label_with_gt),   # ssod_trainer.py:46
    ("utils.self_supervised_utils", "check_pseudo_label", pl_quality.check_pseudo_label),
    ("utils.labelmatch", "LabelMatch", labelmatch.LabelMatch),
    ("models.loss.loss", "ComputeLoss", loss.ComputeLoss),
    ("models.loss.ssod.ssod_loss", "ComputeStudentMatchLoss", ssod_loss.ComputeStudentMatchLoss),
    ("models.assigner.yolo_anchor_assigner", "YOLOAnchorAssigner", assigner.YOLOAnchorAssigner),
    ("models.assigner.tal_assigner", "TaskAlignedAssigner", tal.TaskAlignedAssigner),     # the only consumer, tal_loss.py, is unimportable
    ("models.detector.yolo_ssod", "Model", model.Model),
    ("models.detector.yolo", "Model", model.SupModel),
]
_FACTORIES = (_val_nms, _bbox_iou, _ap_per_class, _confusion_matrix, _val_run)
# defining modules whose import may fail (val.py pulls in optional dependencies of the host application): their patches are
# skipped, listed in apply.skipped
_OPTIONAL = ("val",)
# modules of the host application that bind the names above with `from X import Y` (imported here when possible so that the
# sweep reaches them; a missing optional dependency of one of them only skips that module)
_BINDERS = ["models.loss", "loss.loss", "models.assigner", "models.backbone.common", "trainer.trainer", "trainer.ssod_trainer", "val"]


def _is_original(obj, attr, mod_name):
    m = getattr(obj, "__module__", None)
    return (getattr(obj, "__name__", None) == attr and isinstance(m, str)
            and (m == mod_name or mod_name.endswith("." + m)) and not m.startswith("efficientteacher_b200"))


def apply(import_binders=True):
    """Returns the sorted list of `module.attribute` names that were rebound."""
    skipped = []
    for mod_name in dict.fromkeys(m for m, _, _ in _PATCHES):
        try:
            importlib.import_module(mod_name)
        except Exception as e:  # the host application is not on sys.path
            if mod_name in _OPTIONAL:
                skipped.append((mod_name, repr(e)))
                continue
            raise RuntimeError("efficientteacher_b200.bootstrap: cannot import reference module %s (%s)" % (mod_name, e))
    if import_binders:
        for mod_name in _BINDERS:
            if mod_name in sys.modules or any(mod_name == m for m, _ in skipped):
                continue
            try:
                importlib.import_module(mod_name)
            except Exception as e:
                skipped.append((mod_name, repr(e)))
    done = []
    for mod_name, attr, repl in _PATCHES:
        defining = sys.modules.get(mod_name)
        if defining is None:     # an optional module that could not be imported
            continue
        originals = {}
        for m in list(sys.modules.values()):
            d = getattr(m, "__dict__", None)
            if not isinstance(d, dict):
                continue
            v = d.get(attr)
            if v is not None and _is_original(v, attr, mod_name):
                originals[id(v)] = v
        if not originals:       # already patched (apply() is idempotent)
            continue
        primary = defining.__dict__.get(attr)
        new = repl(primary if id(primary) in originals else next(iter(originals.values()))) if repl in _FACTORIES else repl
        for name, m in list(sys.modules.items()):
            d = getattr(m, "__dict__", None)
            if not isinstance(d, dict) or name.startswith("efficientteacher_b200"):
                continue
            for k, v in list(d.items()):
                if id(v) in originals:
                    d[k] = new
                    done.append(name + "." + k)
    apply.skipped = skipped
    return sorted(done)


rebound = apply()
