"""The ImageLocality and NodePreferAvoidPods priorities on cfg4 on one GPU; writes
profiles/locality_priority_h100.jsonl.

    python profiles/tools/locality_priority_bench.py [--out PATH] [--steps 20] [--warmup 3] [--reps 4]

cfg4 (100k pods x 10k nodes, 5 lanes) with the priority lists at K = 16 and resource weights (1, 0, 1), under five
settings of (ImageLocality, NodePreferAvoidPods): (0, 0), (1, 0), (0, 10000), (1, 10000), and (1, 10000) with the
TaintToleration / NodeAffinity weights (1, 1); the columns from snapshot.node_locality and snapshot.node_preferences.
The engines alternate `reps` times in one process (the order flips every repetition); per engine and repetition, CUDA
events on the engine stream around `steps` back-to-back rounds.  In a separate pass, torch.profiler gives the device
time per round of priority_pod_kernel and of the pre-pass (image_spread_kernel + locality_class_kernel), which runs
only after a column or weight changes: the pass re-uploads the pod side before each profiled round to make it run.
Then bs_replay_priority walks cfg4's 100k pods in the round's device-sort order with the terms off and on at
(1, 10000), alternating `reps` times, host clock around the synchronising call.  The first line records the card's
name and power limit (nvidia-smi query only, in the same process as the measurement)."""
import argparse
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


def kernel_ms(eng, rounds, pods_side):
    """Device ms per round of priority_pod_kernel and of the pre-pass, from torch.profiler; the pod side is uploaded
    again before every round (when the setting has one) so that the pre-pass runs in each."""
    from torch.profiler import ProfilerActivity, profile
    eng.evaluate()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            if pods_side is not None:
                eng.upload_locality(pods=pods_side)
            eng.evaluate()
    tot = {"priority": 0.0, "prepass": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if "priority_pod_kernel" in ev.key:
            tot["priority"] += t
        elif "image_spread_kernel" in ev.key or "locality_class_kernel" in ev.key:
            tot["prepass"] += t
    return {k: v / 1000.0 / rounds for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "locality_priority_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("locality_priority_bench: no CUDA device (this measurement needs the GPU)")
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
    node_side, pod_side = S.node_locality(snap, 4)
    prefs = S.node_preferences(snap, 4)
    settings = {"loc_off": ((0, 0), (0, 0)), "img_1": ((1, 0), (0, 0)), "avoid_10000": ((0, 10000), (0, 0)),
                "img_1_avoid_10000": ((1, 10000), (0, 0)), "img_1_avoid_10000_pref_11": ((1, 10000), (1, 1))}
    engs = {}
    for m, (lw, pw) in settings.items():
        eng = pkg.Engine(L, 0, fit_bitmap=False, score=False, priority_k=16)
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_score_weights(1, 0, 1)
        if any(pw):
            eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
            eng.set_node_priority_weights(*pw)
        if any(lw):
            eng.upload_locality(node=node_side, pods=pod_side)
        eng.set_locality_weights(*lw)
        eng.evaluate()
        engs[m] = eng
    res = {m: [] for m in settings}
    for rep in range(a.reps):
        for m in (list(settings) if rep % 2 == 0 else list(settings)[::-1]):
            res[m].append(timed(engs[m], a.steps, a.warmup))
    for m, (lw, pw) in settings.items():
        k = kernel_ms(engs[m], 5, pod_side if any(lw) else None)
        emit({"kind": "cfg4_round_k16", "mode": m, "weights": [1, 0, 1], "locality_weights": list(lw),
              "node_priority_weights": list(pw), "images": int(len(node_side[0])),
              "image_classes": int(len(pod_side[1]) - 1), "P": snap.pods.n, "N": snap.nodes.n, "lanes": L,
              "round_ms": res[m], "round_ms_median": float(np.median(res[m])),
              "round_ms_spread": float(max(res[m]) - min(res[m])), "priority_kernel_ms_profiler": k["priority"],
              "prepass_ms_profiler": k["prepass"]})
    order = engs["loc_off"].evaluate().order.copy()
    for eng in engs.values():
        eng.close()

    eng = pkg.Engine(L, 0, fit_bitmap=False, score=False)
    eng.upload(snap)
    eng.upload_nonzero(node=nz[0], pods=nz[1])
    eng.set_score_weights(1, 0, 1)
    eng.upload_locality(node=node_side, pods=pod_side)
    walks = {"replay_loc_off": (0, 0), "replay_img_1_avoid_10000": (1, 10000)}
    for lw in walks.values():   # module load, scratch allocation and the IL table
        eng.set_locality_weights(*lw)
        eng.replay(order[:1000], after_state=False, priority=True)
    out = {m: [] for m in walks}
    for rep in range(a.reps):
        for m in (list(walks) if rep % 2 == 0 else list(walks)[::-1]):
            eng.set_locality_weights(*walks[m])
            t0 = time.perf_counter()
            r = eng.replay(order, after_state=False, priority=True)
            out[m].append((time.perf_counter() - t0, int((r["node"] >= 0).sum())))
    eng.close()
    for m, lw in walks.items():
        host = [x[0] for x in out[m]]
        emit({"kind": "cfg4_replay_priority_device_order", "mode": m, "weights": [1, 0, 1], "locality_weights": list(lw),
              "P": snap.pods.n, "N": snap.nodes.n, "lanes": L, "walk_s": host, "walk_s_median": float(np.median(host)),
              "walk_s_spread": float(max(host) - min(host)), "placed": out[m][0][1]})
    f.close()


if __name__ == "__main__":
    main()
