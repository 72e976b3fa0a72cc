"""bs_preempt_walk beside bs_preempt on cfg4's node table; writes profiles/preempt_walk_h100.jsonl.

    python profiles/tools/preempt_walk_bench.py [--out PATH] [--reps 5] [--warmup 1] [--sample 200]

Workload: cfg4's 10k nodes (5 lanes) with three bound tables and their preemptors, as walk lists of 1k and 10k pods in
queue order (priority descending).  "mixed" and "evictable" are preempt_bench.py's tables.  "offline" is "evictable"
with every bound pod in an unlocked group instead of online, so that gang preemptors may evict them.  Each list is
walked three ways: without gang units, and in gangs of 8 and of 64 (consecutive pods of the list form one group with
one priority, walked with BS_PREEMPT_GANG).  On the "offline" table the last member of every fourth gang asks for more
cpu than any node has, so that unit evicts for its other members and then rolls back: the undo path runs with real
evictions.  bs_preempt answers the same lists as independent what-ifs.  Both calls are timed with a host clock around
the synchronising call (median of `reps` after `warmup`), each with a victims_cap that holds the whole answer (sized by
an untimed call first), so that a timed call is one walk.  The walk's first `sample` preemptors (a whole number of
units) are checked against the CPU restatement tests/preempt_walk_ref.c, which walks a prefix of the list the way the
engine walks the whole.  The first line records the card's name and power limit (nvidia-smi query only)."""
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
import preempt_walk_ref  # noqa: E402


def card():
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                  text=True).strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power}


def timed(fn, reps, warmup):
    for _ in range(warmup):
        r = fn()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    return r, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "preempt_walk_h100.jsonl"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=200)
    args = ap.parse_args()
    preempt_walk_ref.warm()   # gcc runs here, not inside a timed region
    snap = S.config(4)
    nt, pt = snap.nodes, snap.pods
    free_cpu = nt.alloc[0] - nt.requested[0]
    rng = np.random.default_rng(4)
    n_max = 10000
    pt.req[0, :n_max] = int(free_cpu.max()) + 1 + rng.integers(0, 2000, n_max)
    prio = rng.choice([1000, 100000, 2**30], n_max)
    mixed_gid = np.where(rng.random(n_max) < 0.5, S.GID_NONE, pt.gid[:n_max])
    lines = [dict(card(), workload="cfg4", nodes=int(nt.n), lanes=int(nt.lanes), cpu_threads=os.cpu_count())]
    cpu0 = pt.req[0, :n_max].copy()
    for table in ("mixed", "evictable", "offline"):
        if table == "mixed":
            bound = S.bound_pods(snap, 4)
            gid0 = mixed_gid
        else:
            nt.requested[0] = nt.alloc[0]
            online = 1.0 if table == "evictable" else 0.0
            bound = S.bound_pods(snap, 4, online=online, missing=0.0, locked=0.0)
            gid0 = np.full(n_max, S.GID_NONE, np.int32)
            if table == "evictable":
                cpu0 = 1000 + rng.integers(0, 2000, n_max)
        for gang in (0, 8, 64):
            for n in (1000, 10000):
                pods = np.arange(n)
                pt.req[0, :n_max] = cpu0
                if gang:   # consecutive pods form one group, one priority per group
                    pt.gid[:n] = pods // gang
                    pt.priority[:n] = np.repeat(prio[:n:gang], gang)[:n]
                    if table == "offline":   # every fourth unit's last member fits nowhere: the unit rolls back
                        pt.req[0, np.arange(4 * gang - 1, n, 4 * gang)] = 1 << 40
                else:
                    pt.gid[:n] = gid0[:n]
                    pt.priority[:n] = prio[:n]
                order = np.array(sorted(pods.tolist(), key=lambda p: (-int(pt.priority[p]), int(pt.gid[p]), p)),
                                 np.uint32)
                eng = pkg.Engine(nt.lanes, fit_bitmap=False)
                eng.upload(snap)
                eng.upload_bound_pods(bound)
                cap_walk = len(eng.preempt_walk(order, gang=gang > 0).victims)
                cap_plain = len(eng.preempt(order).victims)
                walk, walk_ms = timed(lambda: eng.preempt_walk(order, gang=gang > 0, victims_cap=cap_walk), args.reps,
                                      args.warmup)
                plain, plain_ms = timed(lambda: eng.preempt(order, victims_cap=cap_plain), args.reps, args.warmup)
                eng.close()
                k = min(n, args.sample - args.sample % max(gang, 1))
                t0 = time.perf_counter()
                want = preempt_walk_ref.walk(snap, bound, order[:k], gang > 0)
                cpu_ms = (time.perf_counter() - t0) * 1e3
                same = (np.array_equal(walk.node[:k], want.node) and np.array_equal(walk.n_victims[:k], want.n_victims)
                        and np.array_equal(walk.n_candidates[:k], want.n_candidates)
                        and np.array_equal(walk.outcome[:k], want.outcome)
                        and all(walk.victims_of(i) == want.victims_of(i) for i in range(k)))
                rolled = walk.outcome == 2
                lines.append(dict(table=table, bound_pods=int(bound.n), preemptors=n, gang=gang,
                                  walk_ms_median=float(np.median(walk_ms)), walk_ms_min=float(np.min(walk_ms)),
                                  walk_us_per_step=float(np.median(walk_ms)) * 1e3 / n,
                                  preempt_ms_median=float(np.median(plain_ms)), reps=args.reps,
                                  walk_nominated=int((walk.outcome == 1).sum()), walk_rolled_back=int(rolled.sum()),
                                  walk_rolled_back_with_candidates=int((rolled & (walk.n_candidates > 0)).sum()),
                                  walk_victims=int(len(walk.victims)), preempt_with_node=int((plain.node >= 0).sum()),
                                  preempt_victims=int(len(plain.victims)), cpu_ref_preemptors=k, cpu_ref_ms=cpu_ms,
                                  sample_equal=bool(same)))
                print(json.dumps(lines[-1]), flush=True)
    with open(args.out, "w") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
