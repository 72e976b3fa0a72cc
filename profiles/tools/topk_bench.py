"""Top-K rounds (BS_OUT_TOPK) against the other output modes on one GPU; writes profiles/topk_h100.jsonl.

    python profiles/tools/topk_bench.py [--out PATH] [--steps 50] [--warmup 5] [--reps 3] [--skip-cfg5]

  cfg4       (100k pods x 10k nodes, 5 lanes): decisions-only, bitmap-only, top-K with K = 1, 8, 16, 32 and score
             mode, alternated `reps` times in one process.  Per mode and repetition: the round (CUDA events on the
             engine stream around `steps` back-to-back rounds) and, in a separate pass with stage events on, the
             gang_fit kernel (bs_kernel_ms).  Ratios are to decisions-only.
  worst      cfg4's node table reordered so that every node's free cpu rises with its index: most fitting nodes
             enter the running lists (decisions-only and K = 16).
  cfg5       (1M pods x 50k nodes, 9 lanes) on one GPU with K = 16, no bitmap: its score matrix (400 GB) does not fit
             one GPU.  300 sampled pods' lists are checked against the CPU oracle in the same run.
The first line records the card's name and power limit (nvidia-smi query only)."""
import argparse
import dataclasses
import importlib
import json
import os
import subprocess
import sys
import time

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


def fit_ms(eng, rounds):
    """median gang_fit kernel time over `rounds` rounds with stage events on."""
    eng.set_profiling(True)
    ms = []
    for _ in range(rounds):
        eng.evaluate_async()
        eng.sync()
        ms.append(eng.kernel_ms()["gang_fit"][0])
    eng.set_profiling(False)
    return float(np.median(ms))


def permute_nodes(nt, perm):
    cols = {}
    for f in dataclasses.fields(nt):
        v = getattr(nt, f.name)
        cols[f.name] = None if v is None else (v[:, perm] if v.ndim == 2 else v[perm])
    return type(nt)(**cols)


def expected_topk(score, K):
    from test_gpu_topk import expected_topk as e
    return e(score, K)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "topk_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-cfg5", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("topk_bench: no CUDA device (this measurement needs the GPU)")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    f = open(a.out, "w")

    def emit(rec):
        f.write(json.dumps(rec) + "\n")
        f.flush()
        print(json.dumps(rec), flush=True)

    emit({"kind": "card", **card(), "steps": a.steps, "warmup": a.warmup, "reps": a.reps})

    snap = S.config(4)
    modes = {"decisions": dict(fit_bitmap=False), "bitmap": dict(fit_bitmap=True),
             "topk1": dict(fit_bitmap=False, topk=1), "topk8": dict(fit_bitmap=False, topk=8),
             "topk16": dict(fit_bitmap=False, topk=16), "topk32": dict(fit_bitmap=False, topk=32),
             "score": dict(fit_bitmap=True, score=True)}
    engs = {}
    for m, kw in modes.items():
        engs[m] = pkg.Engine(snap.lanes, 0, **kw)
        engs[m].upload(snap)
        engs[m].evaluate()
    step = {m: [] for m in modes}
    fit = {m: [] for m in modes}
    for rep in range(a.reps):
        for m in (list(modes) if rep % 2 == 0 else list(modes)[::-1]):
            step[m].append(timed(engs[m], a.steps, a.warmup))
            fit[m].append(fit_ms(engs[m], 20))
    ref_step, ref_fit = np.median(step["decisions"]), np.median(fit["decisions"])
    for m in modes:
        emit({"kind": "cfg4", "mode": m, "P": snap.pods.n, "N": snap.nodes.n, "lanes": snap.lanes,
              "shape": engs[m].fit_shape(), "step_ms": step[m], "gang_fit_ms": fit[m],
              "step_ms_median": float(np.median(step[m])), "gang_fit_ms_median": float(np.median(fit[m])),
              "step_ratio_to_decisions": float(np.median(step[m]) / ref_step),
              "gang_fit_ratio_to_decisions": float(np.median(fit[m]) / ref_fit)})
    for e in engs.values():
        e.close()
    del engs

    # worst-case ordering: free cpu rising with node index
    free = snap.nodes.alloc[0] - snap.nodes.requested[0]
    worst = S.Snapshot(permute_nodes(snap.nodes, np.argsort(free, kind="stable")), snap.pods, snap.groups, "cfg4-rising")
    assert getattr(snap, "aff_bits", None) is None
    for m, kw in (("decisions", dict(fit_bitmap=False)), ("topk16", dict(fit_bitmap=False, topk=16))):
        eng = pkg.Engine(worst.lanes, 0, **kw)
        eng.upload(worst)
        eng.evaluate()
        st = [timed(eng, a.steps, a.warmup) for _ in range(a.reps)]
        ft = fit_ms(eng, 20)
        emit({"kind": "cfg4_rising_free_cpu", "mode": m, "step_ms": st, "step_ms_median": float(np.median(st)),
              "gang_fit_ms_median": ft})
        eng.close()
    del worst, snap

    if not a.skip_cfg5:
        from oracle import oracle
        oracle.build()
        t0 = time.perf_counter()
        snap = S.config(5)
        t_gen = time.perf_counter() - t0
        eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, topk=16)
        eng.upload(snap)
        res = eng.evaluate()
        st = [timed(eng, a.steps, 2) for _ in range(a.reps)]
        ft = fit_ms(eng, 10)
        idx = np.sort(np.random.default_rng(5).choice(snap.pods.n, 300, replace=False))
        nodes, scores = eng.topk_rows()
        eng.close()
        sub = S.Snapshot(snap.nodes, snap.pods.take(idx), snap.groups)
        o2 = oracle.round(sub, want_bitmap=False, want_score=True, want_sort=False, threads=0)
        en, es = expected_topk(o2.score, 16)
        ok = bool(np.array_equal(nodes[idx], en) and np.array_equal(scores[idx], es) and
                  np.array_equal(nodes[:, 0], res.best_node) and np.array_equal(scores[:, 0], res.best_score))
        emit({"kind": "cfg5_one_gpu", "mode": "topk16", "P": snap.pods.n, "N": snap.nodes.n, "lanes": snap.lanes,
              "step_ms": st, "step_ms_median": float(np.median(st)), "gang_fit_ms_median": ft,
              "lists_bytes": int(nodes.nbytes + scores.nbytes), "sampled_pods_match_oracle": ok,
              "snapshot_gen_s": t_gen})
        if not ok:
            raise SystemExit("cfg5 top-K lists differ from the oracle")
    f.close()


if __name__ == "__main__":
    main()
