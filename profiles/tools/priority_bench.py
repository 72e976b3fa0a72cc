"""Priority lists (BS_OUT_PRIORITY) against the same rounds without them on one GPU; writes profiles/priority_h100.jsonl.

    python profiles/tools/priority_bench.py [--out PATH] [--steps 30] [--warmup 5] [--reps 3] [--skip-cfg5]

  cfg4  (100k pods x 10k nodes, 5 lanes, no bitmap): decisions-only, then with the priority lists at K = 1 and K = 16
        with the default weights (1, 0, 1), and K = 16 with (0, 1, 0).  The four engines alternate `reps` times in one
        process (the order flips every repetition); per engine and repetition, CUDA events on the engine stream around
        `steps` back-to-back rounds of the uploaded snapshot.  The priority stage's kernel time comes from a separate
        torch.profiler pass (device time of priority_pod_kernel per round).
  cfg5  (1M pods x 50k nodes, 9 lanes) on one GPU with K = 16: the round time, and 50 sampled pods' lists checked
        against the CPU restatement (tests/priority_ref.c) in the same run.
The non-zero request columns come from snapshot.nonzero_requests (the synthetic tables carry no containers).  The
first line records the card's name and power limit (nvidia-smi query only)."""
import argparse
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

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


def engine(snap, nz, kw, weights):
    eng = pkg.Engine(snap.lanes, 0, **kw)
    eng.upload(snap)
    if kw.get("priority_k"):
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_score_weights(*weights)
    eng.evaluate()
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "priority_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-cfg5", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("priority_bench: no CUDA device (this measurement needs the GPU)")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    f = open(a.out, "w")

    def emit(rec):
        f.write(json.dumps(rec) + "\n")
        f.flush()
        print(json.dumps(rec), flush=True)

    emit({"kind": "card", **card(), "steps": a.steps, "warmup": a.warmup, "reps": a.reps})
    snap = S.config(4)
    nz = S.nonzero_requests(snap, 4)
    modes = {"decisions": (dict(fit_bitmap=False), None),
             "priority_k1": (dict(fit_bitmap=False, priority_k=1), (1, 0, 1)),
             "priority_k16": (dict(fit_bitmap=False, priority_k=16), (1, 0, 1)),
             "priority_k16_most": (dict(fit_bitmap=False, priority_k=16), (0, 1, 0))}
    engs = {m: engine(snap, nz, kw, w) for m, (kw, w) in modes.items()}
    step = {m: [] for m in modes}
    for rep in range(a.reps):
        for m in (list(modes) if rep % 2 == 0 else list(modes)[::-1]):
            step[m].append(timed(engs[m], a.steps, a.warmup))
    ref = float(np.median(step["decisions"]))
    for m, (kw, w) in modes.items():
        rec = {"kind": "cfg4", "mode": m, "P": snap.pods.n, "N": snap.nodes.n, "lanes": snap.lanes,
               "K": kw.get("priority_k", 0), "weights": w, "step_ms": step[m],
               "step_ms_median": float(np.median(step[m])),
               "step_spread": float(np.max(step[m]) - np.min(step[m])),
               "added_ms": float(np.median(step[m])) - ref}
        if kw.get("priority_k"):
            rec["priority_kernel_ms_profiler"] = kernel_ms(engs[m], 10)
        emit(rec)
    for e in engs.values():
        e.close()
    del engs, snap

    if not a.skip_cfg5:
        import priority_ref
        snap = S.config(5)
        nz = S.nonzero_requests(snap, 5)
        eng = engine(snap, nz, dict(fit_bitmap=False, priority_k=16), (1, 0, 1))
        st = [timed(eng, 3, 1) for _ in range(2)]
        km = kernel_ms(eng, 2)
        res = eng.evaluate()
        nodes, scores = eng.priority_rows()
        eng.close()
        idx = np.sort(np.random.default_rng(5).choice(snap.pods.n, 50, replace=False))
        wn, ws = priority_ref.priority_rows(snap, nz[0], nz[1], 16, (1, 0, 1), pods=idx)
        ok = bool(np.array_equal(nodes[idx], wn) and np.array_equal(scores[idx], ws) and
                  np.array_equal((nodes >= 0).sum(axis=1), np.minimum(16, res.feasible_count)))
        emit({"kind": "cfg5_one_gpu", "mode": "priority_k16", "P": snap.pods.n, "N": snap.nodes.n, "lanes": snap.lanes,
              "step_ms": st, "step_ms_median": float(np.median(st)), "priority_kernel_ms_profiler": km,
              "sampled_pods": len(idx), "sampled_pods_match_restatement": ok})
        if not ok:
            raise SystemExit("cfg5 priority lists differ from the restatement")
    f.close()


if __name__ == "__main__":
    main()
