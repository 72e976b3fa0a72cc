"""The InterPodAffinity priority on cfg4 on one GPU; writes profiles/interpod_priority_h100.jsonl.

    python profiles/tools/interpod_priority_bench.py [--out PATH] [--steps 20] [--warmup 3] [--reps 4] [--bound 300000]

cfg4 (100k pods x 10k nodes, 5 lanes) with the priority lists at K = 16 and resource weights (1, 0, 1), in four
modes: off; InterPodAffinity 1 alone; v1.17's default profile without InterPodAffinity (TaintToleration /
NodeAffinity (1, 1), ImageLocality / NodePreferAvoidPods (1, 10000), SelectorSpread 1); and the whole default profile,
that plus InterPodAffinity 1.  The columns come from snapshot.node_interpod (a hostname, a zone and a rack key,
`bound` bound pods over the nodes), snapshot.node_preferences, snapshot.node_locality and snapshot.node_spread (8 zones,
32 classes).  The engines alternate `reps` times in one process (the order flips every repetition); per engine and
repetition, CUDA events on the engine stream around `steps` back-to-back rounds.  In a separate pass, torch.profiler
gives the device time per round of priority_pod_kernel and of the IPA pre-pass (interpod_mass_kernel +
interpod_class_kernel), which runs only after a side changes: the pass uploads the node side again before every
profiled round of a mode with IPA so that both pre-pass kernels run in each.  The first line records the card's name
and power limit (nvidia-smi query only, in the same process as the measurement)."""
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


def kernel_ms(eng, rounds, node_side):
    """Device ms per round of priority_pod_kernel and of the IPA pre-pass, from torch.profiler; the node side is
    uploaded again before every round (when the mode has one) so that the whole pre-pass runs in each."""
    from torch.profiler import ProfilerActivity, profile
    eng.evaluate()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            if node_side is not None:
                eng.upload_interpod(node=node_side)
            eng.evaluate()
    tot = {"priority": 0.0, "prepass": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if "priority_pod_kernel" in ev.key:
            tot["priority"] += t
        elif "interpod_mass_kernel" in ev.key or "interpod_class_kernel" in ev.key:
            tot["prepass"] += t
    return {k: v / 1000.0 / rounds for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "interpod_priority_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--bound", type=int, default=300_000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("interpod_priority_bench: no CUDA device (this measurement needs the GPU)")
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
    node_side, pod_side = S.node_interpod(snap, 4, n_bound=a.bound)
    spread = S.node_spread(snap, 4, n_zones=8, n_classes=32)
    prefs = S.node_preferences(snap, 4)
    loc = S.node_locality(snap, 4)
    # mode: (whether the other default-profile priorities are on, InterPodAffinity weight)
    modes = {"off": (False, 0), "ipa_1": (False, 1), "default_profile_without_ipa": (True, 0),
             "default_profile": (True, 1)}
    engs = {}
    for m, (others, w) in modes.items():
        eng = pkg.Engine(L, 0, fit_bitmap=False, score=False, priority_k=16)
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_score_weights(1, 0, 1)
        if others:
            eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
            eng.set_node_priority_weights(1, 1)
            eng.upload_locality(node=loc[0], pods=loc[1])
            eng.set_locality_weights(1, 10000)
            eng.upload_spread(node=spread[0], pods=spread[1])
            eng.set_spread_weight(1)
        if w:
            eng.upload_interpod(node=node_side, pods=pod_side)
            eng.set_interpod_weight(w)
        eng.evaluate()
        engs[m] = eng
    res = {m: [] for m in modes}
    for rep in range(a.reps):
        for m in (list(modes) if rep % 2 == 0 else list(modes)[::-1]):
            res[m].append(timed(engs[m], a.steps, a.warmup))
    for m, (others, w) in modes.items():
        k = kernel_ms(engs[m], 5, node_side if w else None)
        emit({"kind": "cfg4_round_k16", "mode": m, "weights": [1, 0, 1],
              "node_priority_weights": [1, 1] if others else [0, 0],
              "locality_weights": [1, 10000] if others else [0, 0], "spread_weight": 1 if others else 0,
              "interpod_weight": w, "hard_pod_affinity_weight": 1, "bound_pods": a.bound,
              "P": snap.pods.n, "N": snap.nodes.n, "lanes": L, "round_ms": res[m],
              "round_ms_median": float(np.median(res[m])), "round_ms_spread": float(max(res[m]) - min(res[m])),
              "priority_kernel_ms_profiler": k["priority"], "prepass_ms_profiler": k["prepass"]})
    for eng in engs.values():
        eng.close()
    f.close()


if __name__ == "__main__":
    main()
