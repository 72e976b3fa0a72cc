"""The PodFitsHostPorts filter on cfg4 on one GPU; writes profiles/host_ports_h100.jsonl.

    python profiles/tools/host_ports_bench.py [--out PATH] [--steps 20] [--warmup 3] [--reps 2]

cfg4 (100k pods x 10k nodes, 5 lanes) with host-port columns from a seeded generator: a dictionary of 12 entries over
the wildcard and two specific ips, TCP and UDP and five ports; about 30 % of the gangs want one or two entries (every
worker of a gang the same ones), and each node uses up to two.  Three round kinds, each with the filter on and off in
one engine: decisions only, top-K at K = 16, and the priority lists at K = 16 with reason rows.  The switch alternates
`reps` times per kind (the order flips every repetition); per setting, CUDA events on the engine stream around `steps`
back-to-back rounds.  Then bs_replay and bs_replay_priority over the whole 100k-pod queue in the round's order, filter
on and off alternated, with CUDA events around each walk, and the pods placed and gangs made ready by each.  The first
line records the card's name and power limit (nvidia-smi query only, in the same process as the measurement)."""
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


def columns(snap, seed=4, n_entries=12, grouped=0.3, node_bits=2):
    """((entries [K, 3], used [N]), want [P]) as the docstring describes."""
    rng = np.random.default_rng(seed)
    seen, entries = set(), []
    while len(entries) < n_entries:
        e = (int(rng.choice([0, 0, 1, 2])), int(rng.integers(0, 2)), int(rng.choice([22, 1234, 29500, 8080, 6379])))
        if e not in seen:
            seen.add(e)
            entries.append(e)
    K, N, G = len(entries), snap.nodes.n, snap.groups.n
    used = np.zeros(N, np.uint64)
    for _ in range(node_bits):
        on = rng.random(N) < 0.5
        used[on] |= np.uint64(1) << rng.integers(0, K, int(on.sum())).astype(np.uint64)
    gwant = np.zeros(max(G, 1), np.uint64)
    pick = rng.random(G) < grouped
    for _ in range(2):
        more = pick & (rng.random(G) < 0.5)
        gwant[:G][pick] |= np.uint64(1) << rng.integers(0, K, int(pick.sum())).astype(np.uint64)
        pick = more
    gid = snap.pods.gid
    ok = (gid >= 0) & (gid < G)
    want = np.where(ok, gwant[np.clip(gid, 0, max(G - 1, 0))], np.uint64(0)).astype(np.uint64)
    return (np.array(entries, np.int64), used), want


def timed(eng, steps, warmup):
    """ms per round over `steps` rounds (events on the engine stream)."""
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


def walk(eng, order, priority):
    """(ms, pods placed, gangs made ready) of one walk over `order`."""
    ext = torch.cuda.ExternalStream(eng.stream())
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(ext)
    out = eng.replay(order, after_state=False, priority=priority)
    b.record(ext)
    b.synchronize()
    return a.elapsed_time(b), int((out["node"] >= 0).sum()), int(out["ready"].sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "host_ports_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    snap = S.config(4)
    cols = columns(snap)
    nz = S.nonzero_requests(snap, 4)
    lines = [dict(kind="card", **card(), reps=args.reps)]
    kinds = {"decisions": dict(fit_bitmap=False), "topk16": dict(fit_bitmap=False, topk=16),
             "priority16_reasons": dict(fit_bitmap=False, priority_k=16, reasons=True)}
    order = None
    for kind, kw in kinds.items():
        eng = pkg.Engine(snap.lanes, 0, **kw)
        eng.upload(snap)
        if kw.get("priority_k"):
            eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.upload_host_ports(node=cols[0], pods=cols[1])
        ms = {"on": [], "off": []}
        for r in range(args.reps):
            for on in ((True, False) if r % 2 == 0 else (False, True)):
                eng.set_host_port_filter(on)
                ms["on" if on else "off"].append(timed(eng, args.steps, args.warmup))
        eng.set_host_port_filter(True)
        feasible = eng.evaluate().feasible_count.copy()
        eng.set_host_port_filter(False)
        res = eng.evaluate()
        feasible_off = res.feasible_count.copy()
        order = res.order.copy()
        eng.close()
        lines.append(dict(kind=kind, P=snap.pods.n, N=snap.nodes.n, lanes=snap.lanes, entries=int(len(cols[0][0])),
                          pods_wanting_ports=int((cols[1] != 0).sum()),
                          round_ms_on=ms["on"], round_ms_off=ms["off"],
                          round_ms_on_median=float(np.median(ms["on"])), round_ms_off_median=float(np.median(ms["off"])),
                          spread_on=float(np.ptp(ms["on"])), spread_off=float(np.ptp(ms["off"])),
                          pods_losing_nodes=int((feasible < feasible_off).sum()),
                          pods_fitting_nowhere_on=int((feasible == 0).sum()),
                          pods_fitting_nowhere_off=int((feasible_off == 0).sum())))
        print(json.dumps(lines[-1]), flush=True)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False)
    eng.upload(snap)
    eng.upload_nonzero(node=nz[0], pods=nz[1])
    eng.upload_host_ports(node=cols[0], pods=cols[1])
    for priority in (False, True):
        res = {"on": [], "off": []}
        for r in range(args.reps):
            for on in ((True, False) if r % 2 == 0 else (False, True)):
                eng.set_host_port_filter(on)
                res["on" if on else "off"].append(walk(eng, order, priority))
        ln = dict(kind="replay_priority" if priority else "replay", queue=int(len(order)))
        for k in ("on", "off"):
            ln[f"ms_{k}"] = [x[0] for x in res[k]]
            ln[f"ms_{k}_median"] = float(np.median(ln[f"ms_{k}"]))
            ln[f"spread_{k}"] = float(np.ptp(ln[f"ms_{k}"]))
            ln[f"placed_{k}"] = res[k][0][1]
            ln[f"ready_{k}"] = res[k][0][2]
        lines.append(ln)
        print(json.dumps(ln), flush=True)
    eng.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
