"""Reason rows (BS_OUT_REASONS) against the same rounds without them on one GPU; writes profiles/reasons_h100.jsonl.

    python profiles/tools/reasons_bench.py [--out PATH] [--steps 30] [--warmup 5] [--reps 3]

cfg4 (100k pods x 10k nodes, 5 lanes) in three output modes: decisions-only, bitmap-only and top-K with K = 16, each
with and without the reason rows.  The two engines of a mode alternate `reps` times in one process (the order flips
every repetition).  Per engine and repetition: the round (CUDA events on the engine stream around `steps` back-to-back
rounds of the uploaded snapshot) and, in a separate pass with stage events on, the reasons stage (bs_kernel_ms,
BS_K_REASONS).  The per-class part of the rows is rebuilt only when the node table or the pods' classes change, so
back-to-back rounds of one snapshot time the per-pod sweep; the class part is timed once per engine from a fresh
upload (BS_K_NODE_LEFT with and without the flag).  The first line records the card's name and power limit
(nvidia-smi query only)."""
import argparse
import importlib
import json
import os
import subprocess
import sys

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


def timed(eng, steps, warmup):
    """ms per round over `steps` back-to-back rounds (events on the engine stream)."""
    ext = torch.cuda.ExternalStream(eng.stream())
    for _ in range(warmup):
        eng.evaluate_async()
    eng.sync()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(ext)
    for _ in range(steps):
        eng.evaluate_async()
    b.record(ext)
    eng.sync()
    b.synchronize()
    return a.elapsed_time(b) / steps


def stage_ms(eng, rounds, name):
    """median time of one stage over `rounds` rounds with stage events on."""
    eng.set_profiling(True)
    ms = []
    for _ in range(rounds):
        eng.evaluate_async()
        eng.sync()
        ms.append(eng.reasons_ms() if name == "reasons" else eng.kernel_ms()[name][0])
    eng.set_profiling(False)
    return float(np.median(ms))


def prepare_ms(eng, snap):
    """BS_K_NODE_LEFT of the first round after a fresh upload: node_left, class fit bits and, with the flag, the
    per-class half of the reason rows."""
    eng.set_profiling(True)
    eng.upload(snap)
    eng.evaluate()
    ms = eng.kernel_ms()["node_left"][0]
    eng.set_profiling(False)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "reasons_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if a.steps < 20:
        raise SystemExit("reasons_bench: at least 20 steps per measurement")
    if not torch.cuda.is_available():
        raise SystemExit("reasons_bench: no CUDA device (this measurement needs the GPU)")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    f = open(a.out, "w")

    def emit(rec):
        f.write(json.dumps(rec) + "\n")
        f.flush()
        print(json.dumps(rec), flush=True)

    emit({"kind": "card", **card(), "steps": a.steps, "warmup": a.warmup, "reps": a.reps})
    snap = S.config(4)
    modes = {"decisions": dict(fit_bitmap=False), "bitmap": dict(fit_bitmap=True),
             "topk16": dict(fit_bitmap=False, topk=16)}
    ref = None
    for m, kw in modes.items():
        engs = {}
        for r in (False, True):
            engs[r] = pkg.Engine(snap.lanes, 0, reasons=r, **kw)
            engs[r].upload(snap)
            engs[r].evaluate()
        step = {False: [], True: []}
        for rep in range(a.reps):
            for r in ((False, True) if rep % 2 == 0 else (True, False)):
                step[r].append(timed(engs[r], a.steps, a.warmup))
        reasons = stage_ms(engs[True], 20, "reasons")
        prep = {r: prepare_ms(engs[r], snap) for r in (False, True)}
        for e in engs.values():
            e.close()
        off, on = float(np.median(step[False])), float(np.median(step[True]))
        if m == "decisions":
            ref = off
        emit({"kind": "cfg4", "mode": m, "P": snap.pods.n, "N": snap.nodes.n, "lanes": snap.lanes,
              "step_ms_without": step[False], "step_ms_with": step[True],
              "step_ms_without_median": off, "step_ms_with_median": on,
              "step_spread_without": float(np.max(step[False]) - np.min(step[False])),
              "added_ms": on - off, "added_ratio_to_decisions_round": (on - off) / ref,
              "reasons_stage_ms_median": reasons,
              "node_left_stage_ms_first_round_without": prep[False], "node_left_stage_ms_first_round_with": prep[True]})
    f.close()


if __name__ == "__main__":
    main()
