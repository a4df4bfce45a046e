"""squeezedet_b200 — H100-native SqueezeDet inference hot path (see DESIGN.md).

Host side mirrors the reference's Python surface (config / nets / nn_skeleton /
utils); all arithmetic runs in ``lib/libsqdet_b200.so`` (hand-written sm_90a CUDA,
C ABI in ``include/sqdet_b200.h``).  No CPU fallback."""
from ._lib import SqdetError, MATH_FP32_SIMT, MATH_TF32X3_TC, DET_DTYPE  # noqa: F401
from .nn_skeleton import ModelSkeleton, Session  # noqa: F401

__all__ = ['SqdetError', 'MATH_FP32_SIMT', 'MATH_TF32X3_TC', 'DET_DTYPE',
           'ModelSkeleton', 'Session']
