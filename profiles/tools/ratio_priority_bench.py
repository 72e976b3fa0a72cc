"""The RequestedToCapacityRatio priority on cfg4 on one GPU; writes profiles/ratio_priority_h100.jsonl.

    python profiles/tools/ratio_priority_bench.py [--out PATH] [--steps 20] [--warmup 3] [--reps 3]

  round   cfg4 (100k pods x 10k nodes, 5 lanes, lane 4 the GPU lane) with the priority lists at K = 16 under three
          settings: weights (1, 0, 1) with the ratio off; (0, 0, 0) with the ratio on alone, weights {cpu 1, memory 1,
          gpu 3} and the bin-pack shape; (1, 0, 1) plus that ratio.  The three engines alternate `reps` times in one
          process (the order flips every repetition); per engine and repetition, CUDA events on the engine stream
          around `steps` back-to-back rounds, and the device time of priority_pod_kernel per round from torch.profiler.
  replay  bs_replay (first-fit), bs_replay_priority under (1, 0, 1), and bs_replay_priority with the GPU bin-pack
          ratio alone (weights (0, 0, 0), ratio {gpu 1}), over the whole queue in the round's device-sort order,
          alternating `reps` times: walk time (host clock around the call, which ends in a device synchronise), pods
          placed and gangs that reached ready.
The non-zero request columns come from snapshot.nonzero_requests.  The first line records the card's name and power
limit (nvidia-smi query only)."""
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

BIN_PACK = ((0, 0), (100, 100))
GPU_LANE = 4


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


def lane_weights(L, cpu, mem, gpu):
    lw = [0] * L
    lw[0], lw[1], lw[GPU_LANE] = cpu, mem, gpu
    return lw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "ratio_priority_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ratio_priority_bench: no CUDA device (this measurement needs the GPU)")
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
    ratio = (1, BIN_PACK, lane_weights(L, 1, 1, 3), 0)
    settings = {"w101_ratio_off": ((1, 0, 1), None), "w000_ratio_binpack": ((0, 0, 0), ratio),
                "w101_plus_ratio_binpack": ((1, 0, 1), ratio)}
    engs = {}
    for m, (w, r) in settings.items():
        eng = pkg.Engine(L, 0, fit_bitmap=False, score=False, priority_k=16)
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_score_weights(*w)
        if r is not None:
            eng.set_ratio_priority(*r)
        eng.evaluate()
        engs[m] = eng
    res = {m: [] for m in settings}
    for rep in range(a.reps):
        for m in (list(settings) if rep % 2 == 0 else list(settings)[::-1]):
            res[m].append(timed(engs[m], a.steps, a.warmup))
    for m, (w, r) in settings.items():
        emit({"kind": "cfg4_round_k16", "mode": m, "weights": list(w), "ratio": None if r is None else
              {"weight": r[0], "shape": [list(p) for p in r[1]], "lane_weights": r[2]},
              "P": snap.pods.n, "N": snap.nodes.n, "lanes": L, "round_ms": res[m],
              "round_ms_median": float(np.median(res[m])), "priority_kernel_ms_profiler": kernel_ms(engs[m], 5)})
    order = engs["w101_ratio_off"].evaluate().order.copy()
    for eng in engs.values():
        eng.close()

    walks = {"first_fit": None, "priority_w101": ((1, 0, 1), None),
             "gpu_binpack_ratio_only": ((0, 0, 0), (1, BIN_PACK, lane_weights(L, 0, 0, 1), 0))}
    eng = pkg.Engine(L, 0, fit_bitmap=False, score=False)
    eng.upload(snap)
    eng.upload_nonzero(node=nz[0], pods=nz[1])
    eng.replay(order[:1000], after_state=False)   # module load and scratch allocation
    out = {m: [] for m in walks}
    gid = snap.pods.gid
    for rep in range(a.reps):
        for m in (list(walks) if rep % 2 == 0 else list(walks)[::-1]):
            setting = walks[m]
            if setting is not None:
                eng.set_score_weights(*setting[0])
                eng.set_ratio_priority(*(setting[1] or (0, BIN_PACK, [0] * L, 0)))
            t0 = time.perf_counter()
            r = eng.replay(order, after_state=False, priority=setting is not None)
            host = time.perf_counter() - t0
            g = gid[order][(r["ready"] == 1)]
            out[m].append((host, int((r["node"] >= 0).sum()), int(np.unique(g[g >= 0]).size)))
    eng.close()
    for m in walks:
        host = [x[0] for x in out[m]]
        emit({"kind": "cfg4_replay_device_order", "mode": m, "P": snap.pods.n, "N": snap.nodes.n, "lanes": L,
              "walk_s": host, "walk_s_median": float(np.median(host)), "placed": out[m][0][1],
              "gangs_ready": out[m][0][2]})
    f.close()


if __name__ == "__main__":
    main()
