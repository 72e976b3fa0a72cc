"""bs_replay against bs_replay_priority on cfg4 in device-sort order on one GPU; writes profiles/replay_priority_h100.jsonl.

    python profiles/tools/replay_priority_bench.py [--out PATH] [--reps 3]

  cfg4 (100k pods x 10k nodes, 5 lanes): the queue is the order the round's device sort produced.  One engine walks
  the whole queue with bs_replay (first-fit), bs_replay_priority under (1, 0, 1) and under (0, 1, 0), alternating
  `reps` times in one process (the order flips every repetition); each walk is timed with a host clock around the call,
  which ends in a device synchronise, and by the engine's own BS_K_REPLAY events (profiling on).  No after-state is
  read back.
  cfg4 widened to 10 lanes (lanes 5-9 absent on every node and pod, so every decision is the same): the same walks in
  the MAXL = 16 kernels, whose scored build spills, against the 5-lane ones.
The non-zero request columns come from snapshot.nonzero_requests.  The first line records the card's name and power
limit (nvidia-smi query only)."""
import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

pkg = importlib.import_module("batch-scheduler_b200")
S = pkg.snapshot


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                  text=True).strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power}


def walk(eng, order, mode):
    """(host seconds, BS_K_REPLAY milliseconds, placed pods) of one walk of the whole queue."""
    if mode != "first_fit":
        eng.set_score_weights(*mode)
    t0 = time.perf_counter()
    out = eng.replay(order, after_state=False, priority=mode != "first_fit")
    host = time.perf_counter() - t0
    ms, n = C.c_float(), C.c_uint32()
    eng._check(eng.lib.bs_kernel_ms(eng.h, pkg.capi.K_REPLAY, C.byref(ms), C.byref(n)))
    return host, float(ms.value), int((out["node"] >= 0).sum())


def widen(snap, lanes):
    """The snapshot with absent lanes appended up to `lanes`: every [L, n] column gets zero rows."""
    s = snap.copy()
    for t in (s.nodes, s.pods, s.groups):
        for f in t.__dataclass_fields__:
            v = getattr(t, f)
            if isinstance(v, np.ndarray) and v.ndim == 2:
                setattr(t, f, np.vstack([v, np.zeros((lanes - v.shape[0], v.shape[1]), v.dtype)]))
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "replay_priority_h100.jsonl"))
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("replay_priority_bench: no CUDA device (this measurement needs the GPU)")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    f = open(a.out, "w")

    def emit(rec):
        f.write(json.dumps(rec) + "\n")
        f.flush()
        print(json.dumps(rec), flush=True)

    emit({"kind": "card", **card(), "reps": a.reps})
    snap = S.config(4)
    node_nz, pod_nz = S.nonzero_requests(snap, 4)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, score=False)
    eng.upload(snap)
    order = eng.evaluate().order.copy()
    eng.close()
    wide = widen(snap, 10)
    legs = {"cfg4_device_order": (snap, {"first_fit": "first_fit", "priority_least_balanced": (1, 0, 1),
                                         "priority_most": (0, 1, 0)}),
            "cfg4_10_lanes_device_order": (wide, {"first_fit": "first_fit", "priority_least_balanced": (1, 0, 1)})}
    placed = {}
    for kind, (sn, modes) in legs.items():
        eng = pkg.Engine(sn.lanes, 0, fit_bitmap=False, score=False)
        eng.upload(sn)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        eng.set_profiling(True)
        walk(eng, order[:1000], "first_fit")   # module load and scratch allocation
        res = {m: [] for m in modes}
        for rep in range(a.reps):
            for m in (list(modes) if rep % 2 == 0 else list(modes)[::-1]):
                res[m].append(walk(eng, order, modes[m]))
        eng.close()
        ref = float(np.median([r[0] for r in res["first_fit"]]))
        for m, w in modes.items():
            host = [r[0] for r in res[m]]
            rec = {"kind": kind, "mode": m, "weights": None if w == "first_fit" else list(w),
                   "P": sn.pods.n, "N": sn.nodes.n, "lanes": sn.lanes, "walk_s": host,
                   "walk_s_median": float(np.median(host)), "kernel_ms": [r[1] for r in res[m]],
                   "placed": res[m][0][2], "vs_first_fit": float(np.median(host)) / ref}
            if m in placed:
                rec["placed_equals_5_lanes"] = placed[m] == rec["placed"]
            placed.setdefault(m, rec["placed"])
            emit(rec)
    f.close()


if __name__ == "__main__":
    main()
