"""TEST INFRASTRUCTURE ONLY -- oracle/trunk_ref.TrunkRef and oracle/step_ref.CpuSSODStep with a per-Conv activation, for
the ReLU and Hardswish YOLOv5 trunks.  The activation of each Conv is resolved from the two config strings with the
reference's rules (models/backbone/yolov5_backbone.py:47-55, models/neck/yolov5_neck.py:48-56, C3 common.py:566-592,
SPPF :682-700), restated here independently of efficientteacher_b200.model so the two can be checked against each other
and against tests/golden/trunk_act_*.npz."""
import torch.nn.functional as F

from oracle import step_ref
from oracle.step_ref import CpuSSODStep
from oracle.trunk_ref import TrunkRef

ACT_FN = {"silu": F.silu, "relu": F.relu, "hard_swish": F.hardswish}
ACT_CLASS = {"silu": "SiLU", "relu": "ReLU", "hard_swish": "Hardswish"}


def _modes(activation):
    """(CONV_ACT, C3 inner, C3 last) of one cfg.Model.{Backbone,Neck}.activation string"""
    if activation in ("SiLU", "ReLU"):
        a = activation.lower()
        return a, a, a
    return "hard_swish", "relu", "hard_swish"


def act_map(backbone_act, neck_act, depth=(3, 6, 9, 3), neck_depth=3):
    """module path of every trunk Conv -> 'silu' / 'relu' / 'hard_swish'"""
    acts = {}

    def c3(p, n, inner, last):
        for c in ("cv1", "cv2"):
            acts["%s.%s" % (p, c)] = inner
        for i in range(n):
            acts["%s.m.%d.cv1" % (p, i)] = acts["%s.m.%d.cv2" % (p, i)] = inner
        acts[p + ".cv3"] = last

    conv, inner, last = _modes(backbone_act)
    for s in ("stage1", "stage2_1", "stage3_1", "stage4_1", "stage5_1", "sppf.cv1", "sppf.cv2"):
        acts["backbone." + s] = conv           # SPPF is built with CONV_ACT: both of its convs take it
    for s, n in zip(("stage2_2", "stage3_2", "stage4_2", "stage5_2"), depth):
        c3("backbone." + s, n, inner, last)
    conv, inner, last = _modes(neck_act)
    for s in ("conv1", "conv2", "conv3", "conv4"):
        acts["neck." + s] = conv
    for s in ("C1", "C2", "C3", "C4"):
        c3("neck." + s, neck_depth, inner, last)
    return acts


class ActTrunkRef(TrunkRef):
    """TrunkRef whose Conv at path p applies ACT_FN[acts[p]] instead of SiLU (acts=None: SiLU everywhere, as TrunkRef)"""

    def __init__(self, state_dict, depth=(3, 6, 9, 3), neck_depth=3, acts=None, **kw):
        super().__init__(state_dict, depth, neck_depth, **kw)
        self.acts = acts or {}

    @classmethod
    def for_model(cls, model, **kw):
        """the reference trunk of a Model: its weights, depths and the activations its cfg strings select"""
        r = TrunkRef.from_module(model)
        acts = act_map(model.cfg.Model.Backbone.activation, model.cfg.Model.Neck.activation, r.depth, r.neck_depth)
        return cls(r.sd, r.depth, r.neck_depth, acts=acts, **kw)

    def conv(self, p, x, k, s, train, act=True):
        y = super().conv(p, x, k, s, train, act=False)
        return ACT_FN[self.acts.get(p, "silu")](y) if act else y


class ActCpuSSODStep(CpuSSODStep):
    """CpuSSODStep whose teacher and student trunks are ActTrunkRef(acts)"""

    def __init__(self, *args, acts=None, **kw):
        super().__init__(*args, **kw)
        self.acts = acts

    def step(self, *args, **kw):
        # CpuSSODStep.step builds its trunks through the module-level name TrunkRef
        orig = step_ref.TrunkRef
        step_ref.TrunkRef = lambda *a, **k: ActTrunkRef(*a, acts=self.acts, **k)
        try:
            return super().step(*args, **kw)
        finally:
            step_ref.TrunkRef = orig
