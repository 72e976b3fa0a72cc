"""The TaintToleration and preferred NodeAffinity priorities on cfg4 on one GPU; writes
profiles/node_priority_h100.jsonl.

    python profiles/tools/node_priority_bench.py [--out PATH] [--steps 20] [--warmup 3] [--reps 4]

cfg4 (100k pods x 10k nodes, 5 lanes) with the priority lists at K = 16 and resource weights (1, 0, 1), under two
settings: the node priorities off (0, 0) and on (1, 1), the columns from snapshot.node_preferences.  The two engines
alternate `reps` times in one process (the order flips every repetition); per engine and repetition, CUDA events on the
engine stream around `steps` back-to-back rounds, and the device time of priority_pod_kernel per round from
torch.profiler in a separate pass.  The first line records the card's name and power limit (nvidia-smi query only)."""
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


def kernel_ms(eng, rounds):
    """Device time of priority_pod_kernel per round, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    eng.evaluate()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            eng.evaluate_async()
        eng.sync()
    total = 0.0
    for ev in prof.key_averages():
        if "priority_pod_kernel" in ev.key:
            total += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
    return total / 1000.0 / rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "node_priority_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("node_priority_bench: no CUDA device (this measurement needs the GPU)")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    f = open(a.out, "w")

    def emit(rec):
        f.write(json.dumps(rec) + "\n")
        f.flush()
        print(json.dumps(rec), flush=True)

    emit({"kind": "card", **card(), "reps": a.reps})
    snap = S.config(4)
    L = snap.lanes
    nz = S.nonzero_requests(snap, 4)
    prefs = S.node_preferences(snap, 4)
    settings = {"node_prio_off": (0, 0), "node_prio_w11": (1, 1)}
    engs = {}
    for m, pw in settings.items():
        eng = pkg.Engine(L, 0, fit_bitmap=False, score=False, priority_k=16)
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_score_weights(1, 0, 1)
        eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
        eng.set_node_priority_weights(*pw)
        eng.evaluate()
        engs[m] = eng
    res = {m: [] for m in settings}
    for rep in range(a.reps):
        for m in (list(settings) if rep % 2 == 0 else list(settings)[::-1]):
            res[m].append(timed(engs[m], a.steps, a.warmup))
    for m, pw in settings.items():
        emit({"kind": "cfg4_round_k16", "mode": m, "weights": [1, 0, 1], "node_priority_weights": list(pw),
              "pref_classes": int(prefs[1].shape[0]), "prefer_bits": 6, "P": snap.pods.n, "N": snap.nodes.n,
              "lanes": L, "round_ms": res[m], "round_ms_median": float(np.median(res[m])),
              "round_ms_spread": float(max(res[m]) - min(res[m])),
              "priority_kernel_ms_profiler": kernel_ms(engs[m], 5)})
    for eng in engs.values():
        eng.close()
    f.close()


if __name__ == "__main__":
    main()
