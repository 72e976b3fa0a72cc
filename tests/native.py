"""TEST INFRASTRUCTURE — the native code the tests compile: the C restatements and the C++ plugin programs.

ref_lib() compiles every C restatement (tests/*_ref.c) into one library linked against oracle/libbs_oracle.so; the
*_ref.py modules bind their own functions from it.  cpp_program(name) builds tests/cpp/<name>.cpp against
libbsched.so.  Both build once per process into a temporary directory, because the tree may be read-only.
"""
from __future__ import annotations

import ctypes as C
import functools
import importlib
import os
import subprocess
import tempfile

from oracle import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_REF_SOURCES = ("fit_reasons_ref.c", "preempt_ref.c", "priority_ref.c", "replay_priority_ref.c", "ratio_priority_ref.c")


@functools.cache
def _out_dir() -> tempfile.TemporaryDirectory:
    """The process's build directory, removed when the interpreter exits."""
    return tempfile.TemporaryDirectory(prefix="bs_tests_")


@functools.cache
def ref_lib() -> C.CDLL:
    """The C restatements as one library.  -ffp-contract=off makes every double operation round on its own (the
    priority scorers); -fopenmp runs preempt_ref.c over the preemptors in parallel."""
    so = oracle.build()
    out = os.path.join(_out_dir().name, "libbs_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-ffp-contract=off", "-fopenmp",
                           "-shared", "-o", out, *(os.path.join(_HERE, f) for f in _REF_SOURCES),
                           "-I" + os.path.join(_ROOT, "oracle"), so, "-Wl,-rpath," + os.path.dirname(so), "-lm"])
    oracle.lib()   # the oracle library first, so that its symbols resolve
    return C.CDLL(out)


@functools.cache
def cpp_program(name: str) -> str:
    """The path of tests/cpp/<name>.cpp built against libbsched.so (which is built first if it is missing)."""
    importlib.import_module("batch-scheduler_b200").capi.load()
    libdir = os.path.join(_ROOT, "batch-scheduler_b200")
    out = os.path.join(_out_dir().name, name)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", out, os.path.join(_HERE, "cpp", name + ".cpp"),
                           "-L" + libdir, "-lbsched", "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64",
                           "-Wl,-rpath,/usr/local/cuda/lib64"])
    return out
