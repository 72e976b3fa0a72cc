"""The SelectorSpread priority on cfg4 on one GPU; writes profiles/spread_priority_h100.jsonl.

    python profiles/tools/spread_priority_bench.py [--out PATH] [--steps 20] [--warmup 3] [--reps 4]

cfg4 (100k pods x 10k nodes, 5 lanes) with the priority lists at K = 16 and resource weights (1, 0, 1), in five
modes: off; SelectorSpread 1; TaintToleration / NodeAffinity (1, 1) alone; (1, 1) plus SelectorSpread 1; and v1.17's
full default profile: resource weights (1, 0, 1), TaintToleration / NodeAffinity (1, 1), ImageLocality /
NodePreferAvoidPods (1, 10000) and SelectorSpread 1.  The columns come from snapshot.node_spread (8 zones, some
unzoned nodes, 32 classes), snapshot.node_preferences and snapshot.node_locality.  The engines alternate `reps` times
in one process (the order flips every repetition); per engine and repetition, CUDA events on the engine stream around
`steps` back-to-back rounds.  In a separate pass, torch.profiler gives the device time per round of
priority_pod_kernel.  The first line records the card's name and power limit (nvidia-smi query only, in the same
process as the measurement)."""
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
    """Device ms per round of priority_pod_kernel, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    eng.evaluate()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            eng.evaluate()
    tot = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if "priority_pod_kernel" in ev.key:
            tot += t
    return tot / 1000.0 / rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "spread_priority_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spread_priority_bench: no CUDA device (this measurement needs the GPU)")
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
    spread = S.node_spread(snap, 4, n_zones=8, n_classes=32)
    prefs = S.node_preferences(snap, 4)
    loc = S.node_locality(snap, 4)
    # mode: (node priority weights, locality weights, spread weight)
    modes = {"off": ((0, 0), (0, 0), 0), "spread_1": ((0, 0), (0, 0), 1), "pref_11": ((1, 1), (0, 0), 0),
             "pref_11_spread_1": ((1, 1), (0, 0), 1), "default_profile": ((1, 1), (1, 10000), 1)}
    engs = {}
    for m, (pw, lw, sw) in modes.items():
        eng = pkg.Engine(L, 0, fit_bitmap=False, score=False, priority_k=16)
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_score_weights(1, 0, 1)
        if any(pw):
            eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
            eng.set_node_priority_weights(*pw)
        if any(lw):
            eng.upload_locality(node=loc[0], pods=loc[1])
            eng.set_locality_weights(*lw)
        if sw:
            eng.upload_spread(node=spread[0], pods=spread[1])
            eng.set_spread_weight(sw)
        eng.evaluate()
        engs[m] = eng
    res = {m: [] for m in modes}
    for rep in range(a.reps):
        for m in (list(modes) if rep % 2 == 0 else list(modes)[::-1]):
            res[m].append(timed(engs[m], a.steps, a.warmup))
    for m, (pw, lw, sw) in modes.items():
        emit({"kind": "cfg4_round_k16", "mode": m, "weights": [1, 0, 1], "node_priority_weights": list(pw),
              "locality_weights": list(lw), "spread_weight": sw, "zones": 8, "spread_classes": 32,
              "P": snap.pods.n, "N": snap.nodes.n, "lanes": L, "round_ms": res[m],
              "round_ms_median": float(np.median(res[m])), "round_ms_spread": float(max(res[m]) - min(res[m])),
              "priority_kernel_ms_profiler": kernel_ms(engs[m], 5)})
    for eng in engs.values():
        eng.close()
    f.close()


if __name__ == "__main__":
    main()
