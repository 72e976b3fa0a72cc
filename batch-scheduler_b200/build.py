"""Builds the C-ABI shared library in-tree: nvcc, sm_90a (H100) only.

Translation units (compiled in parallel, then linked into libbsched.so):
  engine.cu            the C ABI, host sequencing and every kernel the units below do not hold
  plugin.cpp           the C++ host mirror of the reference plugin + snapshot packer
  priority_inst.cu x 6 the 96 priority_pod_kernel builds (csrc/priority.cuh), one slice per -DBS_PRIO_SLICE=k: lane
                       bound 5, 9, 16 by k / 2, IPA off or on by k % 2; slice 0 also the LOC and IPA pre-passes
  replay_inst.cu x 6   the 60 replay_kernel builds (csrc/replay.cuh), one slice per -DBS_REPLAY_SLICE=k: lane bound
                       5, 9, 16 by k / 2, IPF off or on by k % 2
  fit_inst.cu x 9      the gang_fit_kernel variant table, one slice per -DBS_FIT_SLICE=n (csrc/fit.cuh)

    python -m importlib ...  # not importable by dotted name (hyphen); use __graft_entry__.build()
"""
from __future__ import annotations

import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libbsched.so")
OBJ = os.path.join(HERE, "build")
HEADERS = ["devmem.hpp", "common.cuh", "kernels.cuh", "fit.cuh", "sort.cuh", "replay.cuh", "preempt.cuh", "priority.cuh", "interpod_filter.cuh",
           "plugin.hpp",
           os.path.join("..", "..", "include", "bsched.h")]
FIT_SLICES = 9
PRIO_SLICES = 6
REPLAY_SLICES = 6


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the engine is CUDA-only, there is no CPU build")


def _units():
    """(source, object, extra flags) of every translation unit."""
    u = [("engine.cu", "engine.o", []), ("plugin.cpp", "plugin.o", [])]
    for k in range(PRIO_SLICES):
        u.append(("priority_inst.cu", f"priority_inst_{k}.o", [f"-DBS_PRIO_SLICE={k}"]))
    for k in range(REPLAY_SLICES):
        u.append(("replay_inst.cu", f"replay_inst_{k}.o", [f"-DBS_REPLAY_SLICE={k}"]))
    for n in range(FIT_SLICES):
        u.append(("fit_inst.cu", f"fit_inst_{n}.o", [f"-DBS_FIT_SLICE={n}"]))
    return u


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    files = [os.path.join(CSRC, f) for f in HEADERS] + [os.path.join(CSRC, src) for src, _, _ in _units()]
    return any(os.path.exists(f) and os.path.getmtime(f) > t for f in files)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compiles every unit whose object is older than its sources (all of them with force) and links."""
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    base = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
            "-Xcompiler", "-fPIC,-Wall,-fopenmp", "-fmad=false", "-diag-suppress=186,550"]
    if verbose:
        base.insert(1, "-Xptxas=-v")
    hdr_t = max(os.path.getmtime(os.path.join(CSRC, h)) for h in HEADERS if os.path.exists(os.path.join(CSRC, h)))

    def compile_one(unit):
        src, obj, flags = unit
        srcp, objp = os.path.join(CSRC, src), os.path.join(OBJ, obj)
        if not force and os.path.exists(objp) and os.path.getmtime(objp) > max(hdr_t, os.path.getmtime(srcp)):
            return objp
        subprocess.check_call(base + flags + ["-c", srcp, "-o", objp], cwd=CSRC)
        return objp

    with ThreadPoolExecutor(max_workers=max(1, min(os.cpu_count() or 1, len(_units())))) as ex:
        objs = list(ex.map(compile_one, _units()))
    subprocess.check_call([nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB] + objs +
                          ["-lgomp"], cwd=CSRC)
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force=True, verbose="-v" in sys.argv))
