"""hyperqueue_b200 — H100-native (sm_90a) task->worker assignment solver for HyperQueue's tako scheduler tick.

Only the hot path is here (SURVEY.md §8): the CUDA kernels + C ABI (csrc/hqsched.cu, include/hqsched.h)
and a thin host-side mirror of tako's scheduler seam (scheduler.py).  There is no CPU fallback: every
entry point needs the compiled library and a CUDA device and fails loudly otherwise.
"""
from ._lib import (HqsError, LibraryNotBuilt, assignment_dtype, load_library, HQS_AMOUNT_MAX, HQS_TIME_INF,
                   HQS_MAX_RESOURCES, HQS_MAX_VARIANTS, HQS_MAX_WORKERS, HQS_MAX_CLASSES, HQS_MAX_GROUPS)
from .scheduler import (FRACTIONS_PER_UNIT, GpuScheduler, RequestVariant, WorkerTaskMapping, priority_from_user)

__all__ = ["GpuScheduler", "RequestVariant", "WorkerTaskMapping", "HqsError", "LibraryNotBuilt", "load_library",
           "assignment_dtype", "priority_from_user", "FRACTIONS_PER_UNIT", "HQS_AMOUNT_MAX", "HQS_TIME_INF",
           "HQS_MAX_RESOURCES", "HQS_MAX_VARIANTS", "HQS_MAX_WORKERS", "HQS_MAX_CLASSES", "HQS_MAX_GROUPS"]
