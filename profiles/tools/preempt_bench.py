"""bs_preempt on cfg4's node table; writes profiles/preempt_h100.jsonl, or with --violating
profiles/preempt_pdb_h100.jsonl.

    python profiles/tools/preempt_bench.py [--out PATH] [--reps 20] [--warmup 3] [--sample 2000] [--violating FRAC]

Workload: cfg4's 10k nodes (5 lanes), a bound-pod table from their pod_count (snapshot.bound_pods: about 300k pods),
and 1k and 10k preemptors whose cpu request exceeds every node's free cpu, so that each one needs victims.  Two
bound tables: "mixed" (the generator's defaults: online, missing-group and locked pods on most nodes, so most
(preemptor, node) pairs end in a RemovePod refusal) and "evictable" (every node's cpu fully requested, every bound
pod online, online preemptors asking 1-3 cpus: nothing fits without victims, nothing is refused, and the reprieve walk
runs on every node with room once its lower-priority pods are gone).  --violating FRAC flags that share of the
"evictable" table's pods BS_BOUND_PDB_VIOLATING (snapshot.bound_pods' `violating` draw), so that the reprieve walk
takes its two passes; 0, the default, gives the tables and lines without the flag.  bs_preempt is timed with a host clock around the synchronising call (median of
`reps` after `warmup`).  The CPU restatement tests/preempt_ref.c (mutating a copy of each node, OpenMP over the
preemptors on every host thread) is compiled before any timing, timed on the first `sample` preemptors, and its
outputs are compared with the GPU's for all of them; with --violating it is tests/preempt_pdb_ref.c, the same
restatement with the budgets' reprieve order and pick.  The first line records the card's name and power limit
(nvidia-smi query only)."""
import argparse
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

pkg = importlib.import_module("batch-scheduler_b200")
S = pkg.snapshot
import preempt_pdb_ref  # noqa: E402
import preempt_ref  # noqa: E402


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                  text=True).strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=2000)
    ap.add_argument("--violating", type=float, default=0.0)
    args = ap.parse_args()
    if args.out is None:
        args.out = os.path.join(ROOT, "profiles", "preempt_pdb_h100.jsonl" if args.violating > 0 else "preempt_h100.jsonl")
    ref = preempt_pdb_ref if args.violating > 0 else preempt_ref
    ref.warm()   # gcc runs here, not inside a timed region
    snap = S.config(4)
    nt, pt = snap.nodes, snap.pods
    free_cpu = nt.alloc[0] - nt.requested[0]
    rng = np.random.default_rng(4)
    n_max = 10000
    pt.req[0, :n_max] = int(free_cpu.max()) + 1 + rng.integers(0, 2000, n_max)
    pt.priority[:n_max] = rng.choice([1000, 100000, 2**30], n_max)
    mixed_gid = np.where(rng.random(n_max) < 0.5, S.GID_NONE, pt.gid[:n_max])
    lines = [dict(card(), workload="cfg4", nodes=int(nt.n), lanes=int(nt.lanes), cpu_threads=os.cpu_count())]
    for table in ("mixed", "evictable"):
        if table == "mixed":
            bound = S.bound_pods(snap, 4)
            pt.gid[:n_max] = mixed_gid
        else:
            nt.requested[0] = nt.alloc[0]
            bound = S.bound_pods(snap, 4, online=1.0, missing=0.0, locked=0.0, violating=args.violating)
            pt.gid[:n_max] = S.GID_NONE
            pt.req[0, :n_max] = 1000 + rng.integers(0, 2000, n_max)
        eng = pkg.Engine(nt.lanes, fit_bitmap=False)
        eng.upload(snap)
        t0 = time.perf_counter()
        eng.upload_bound_pods(bound)
        lines.append(dict(table=table, bound_pods=int(bound.n), stage="upload_bound_pods",
                          ms=(time.perf_counter() - t0) * 1e3))
        if table == "evictable" and args.violating > 0:
            lines[-1].update(violating=args.violating,
                             violating_pods=int(((bound.flags & S.BOUND_PDB_VIOLATING) != 0).sum()))
        run(eng, snap, bound, table, args, lines, ref)
        eng.close()
    with open(args.out, "w") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")


def run(eng, snap, bound, table, args, lines, ref):
    for n in (1000, 10000):
        pods = np.arange(n, dtype=np.uint32)
        for _ in range(args.warmup):
            r = eng.preempt(pods)
        ms = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            r = eng.preempt(pods)
            ms.append((time.perf_counter() - t0) * 1e3)
        sample = np.arange(min(args.sample, n), dtype=np.uint32)
        t0 = time.perf_counter()
        want = ref.preempt(snap, bound, sample)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        same = (np.array_equal(r.node[sample], want.node) and np.array_equal(r.n_victims[sample], want.n_victims) and
                np.array_equal(r.n_candidates[sample], want.n_candidates) and
                all(r.victims_of(int(p)) == want.victims_of(k) for k, p in enumerate(sample)))
        lines.append(dict(table=table, preemptors=n, gpu_ms_median=float(np.median(ms)), gpu_ms_min=float(np.min(ms)),
                          reps=args.reps, with_node=int((r.node >= 0).sum()), victims_total=int(len(r.victims)),
                          cpu_ref_ms=cpu_ms, cpu_ref_threads=os.cpu_count(), cpu_ref_preemptors=int(len(sample)),
                          sample_equal=bool(same)))
        print(json.dumps(lines[-1]), flush=True)


if __name__ == "__main__":
    main()
