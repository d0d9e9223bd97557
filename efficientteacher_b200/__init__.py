"""efficientteacher_b200 -- H100 (sm_90a) kernels behind EfficientTeacher's semi-supervised YOLOv5 step.

Host-side mirrors of the reference's hot-path interface (same class / function names and call contracts,
SURVEY.md section 8b) over the C ABI of libetb200.so.  Reference = AlibabaResearch/efficientteacher.
"""
from . import _lib  # noqa: F401

__all__ = ["_lib"]
__version__ = "0.1.0"
