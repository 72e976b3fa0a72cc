"""bs_preempt and bs_preempt_walk with the PodFitsHostPorts filter off and on; writes
profiles/preempt_host_ports_h100.jsonl.

    python profiles/tools/preempt_host_ports_bench.py [--out PATH] [--reps 3] [--warmup 1] [--rounds 2]

Workload: cfg4's 10k nodes (5 lanes) with preempt_walk_bench.py's "mixed" and "evictable" bound tables and
preemptors, and host_ports_bench.py's dictionary and used masks.  Each bound row holds each of its node's used entries
with probability 1/2, and each of the first 10k pods wants one entry with probability 1/2.  bs_preempt answers 10k
preemptors, bs_preempt_walk walks 1k and 10k in queue order without gang units.  Every (table, call, size) is timed
with the filter off and on, the two alternated `rounds` times on one engine, each a host clock around the synchronising
call (median of `reps` after `warmup`) with a victims_cap that holds the whole answer.  The first line records the
card's name and power limit (nvidia-smi query only)."""
import argparse
import importlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

import host_ports_bench  # noqa: E402
from preempt_walk_bench import card, timed  # noqa: E402

pkg = importlib.import_module("batch-scheduler_b200")
S = pkg.snapshot


def bound_ports(bound, used, rng):
    """[V]: each row holds each entry its node uses with probability 1/2."""
    u = used[bound.node.astype(np.int64)]
    out = np.zeros(bound.n, np.uint64)
    for k in range(64):
        bit = np.uint64(1) << np.uint64(k)
        out |= np.where(((u & bit) != 0) & (rng.random(bound.n) < 0.5), bit, np.uint64(0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "preempt_host_ports_h100.jsonl"))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    snap = S.config(4)
    nt, pt = snap.nodes, snap.pods
    free_cpu = nt.alloc[0] - nt.requested[0]
    rng = np.random.default_rng(4)
    n_max = 10000
    pt.req[0, :n_max] = int(free_cpu.max()) + 1 + rng.integers(0, 2000, n_max)
    pt.priority[:n_max] = rng.choice([1000, 100000, 2**30], n_max)
    mixed_gid = np.where(rng.random(n_max) < 0.5, S.GID_NONE, pt.gid[:n_max])
    (entries, used), want = host_ports_bench.columns(snap)
    K = len(entries)
    want[:n_max] = np.where(rng.random(n_max) < 0.5, np.uint64(1) << rng.integers(0, K, n_max).astype(np.uint64),
                            np.uint64(0))
    lines = [dict(card(), workload="cfg4", nodes=int(nt.n), lanes=int(nt.lanes), entries=K,
                  nodes_with_ports=int((used != 0).sum()), preemptors_with_ports=int((want[:n_max] != 0).sum()))]
    print(json.dumps(lines[-1]), flush=True)
    for table in ("mixed", "evictable"):
        if table == "mixed":
            bound = S.bound_pods(snap, 4)
            pt.gid[:n_max] = mixed_gid
        else:
            nt.requested[0] = nt.alloc[0]
            bound = S.bound_pods(snap, 4, online=1.0, missing=0.0, locked=0.0)
            pt.gid[:n_max] = S.GID_NONE
            pt.req[0, :n_max] = 1000 + rng.integers(0, 2000, n_max)
        ports = bound_ports(bound, used, rng)
        order = np.array(sorted(range(n_max), key=lambda p: (-int(pt.priority[p]), int(pt.gid[p]), p)), np.uint32)
        eng = pkg.Engine(nt.lanes, fit_bitmap=False)
        eng.upload(snap)
        eng.upload_bound_pods(bound)
        eng.upload_host_ports(node=(entries, used), pods=want)
        eng.upload_bound_host_ports(ports)
        calls = [("preempt", 10000, lambda o, cap: eng.preempt(o, victims_cap=cap)),
                 ("walk", 1000, lambda o, cap: eng.preempt_walk(o, victims_cap=cap)),
                 ("walk", 10000, lambda o, cap: eng.preempt_walk(o, victims_cap=cap))]
        for rnd in range(args.rounds):
            for on in (False, True):
                eng.set_host_port_filter(on)
                for call, n, fn in calls:
                    o = order[:n]
                    cap = len(fn(o, None).victims)
                    res, ms = timed(lambda: fn(o, cap), args.reps, args.warmup)
                    lines.append(dict(table=table, bound_pods=int(bound.n),
                                      bound_rows_with_ports=int((ports != 0).sum()), call=call, preemptors=n,
                                      filter=on, round=rnd, ms_median=float(np.median(ms)), ms_min=float(np.min(ms)),
                                      reps=args.reps, with_node=int((res.node >= 0).sum()),
                                      victims=int(len(res.victims)), candidates_sum=int(res.n_candidates.sum())))
                    print(json.dumps(lines[-1]), flush=True)
        eng.close()
    with open(args.out, "w") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
