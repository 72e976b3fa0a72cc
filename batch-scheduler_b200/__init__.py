"""batch-scheduler_b200 — H100-native gang-scheduling feasibility engine (the name is historical).

Replaces the PreFilter / Permit / Less hot path of tenstack/batch-scheduler
(pkg/scheduler/core/core.go) with hand-written sm_90a kernels behind the C ABI of
include/bsched.h.  The directory name carries a hyphen (it mirrors the reference
repository's name), so import it with
    importlib.import_module("batch-scheduler_b200")
"""
from . import snapshot, capi  # noqa: F401
from .engine import Engine  # noqa: F401

__all__ = ["snapshot", "capi", "Engine"]
