"""The MatchInterPodAffinity filter in the walks on cfg4 on one GPU; writes profiles/interpod_walk_h100.jsonl.

    python profiles/tools/interpod_walk_bench.py [--out PATH] [--reps 2]

cfg4 (100k pods x 10k nodes, 5 lanes) with snapshot.node_interpod_walk's seeded columns: node_interpod_filter's two
sides (hostname anti-affinity gangs, parameter-server and self-affine zone affinity, zone blockers, filler bound pods)
and the placed side derived from them, with pending parameter servers.  bs_replay and bs_replay_priority walk the whole
queue in the round's order with the filter on (placed side uploaded) and off, alternated `reps` times (the order flips
every repetition), with CUDA events on the engine stream around each walk; per walk the pods placed and the gangs made
ready.  The first line records the card's name and power limit (nvidia-smi query only, in the same process as the
measurement)."""
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


def walk(eng, order, priority, gid):
    """(ms, pods placed, gangs made ready) of one walk over `order`."""
    ext = torch.cuda.ExternalStream(eng.stream())
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(ext)
    out = eng.replay(order, after_state=False, priority=priority)
    b.record(ext)
    b.synchronize()
    ready = gid[order][out["ready"] != 0]
    return a.elapsed_time(b), int((out["node"] >= 0).sum()), int(len(np.unique(ready[ready >= 0])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "interpod_walk_h100.jsonl"))
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    snap = S.config(4)
    node, pods, placed = S.node_interpod_walk(snap, 4)
    nz = S.nonzero_requests(snap, 4)
    lines = [dict(kind="card", **card(), reps=args.reps, P=snap.pods.n, N=snap.nodes.n, lanes=snap.lanes,
                  terms=int(len(node[2])), bound=int(len(node[3])),
                  pods_with_filter_class=int((pods[0] != S.IPF_NONE).sum()),
                  pods_with_placed_class=int((placed[0] != S.IPF_NONE).sum()))]
    print(json.dumps(lines[-1]), flush=True)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False)
    eng.upload(snap)
    eng.upload_nonzero(node=nz[0], pods=nz[1])
    eng.upload_interpod_filter(node=node, pods=pods)
    eng.upload_interpod_placed(*placed)
    order = eng.evaluate().order.copy()
    walk(eng, order, False, snap.pods.gid)   # warm-up: module load and scratch allocation
    for priority in (False, True):
        res = {"on": [], "off": []}
        for r in range(args.reps):
            for on in ((True, False) if r % 2 == 0 else (False, True)):
                eng.set_interpod_filter(on)
                res["on" if on else "off"].append(walk(eng, order, priority, snap.pods.gid))
        ln = dict(kind="replay_priority" if priority else "replay", queue=int(len(order)))
        for k in ("on", "off"):
            ln[f"ms_{k}"] = [x[0] for x in res[k]]
            ln[f"ms_{k}_median"] = float(np.median(ln[f"ms_{k}"]))
            ln[f"spread_{k}"] = float(np.ptp(ln[f"ms_{k}"]))
            ln[f"placed_{k}"] = res[k][0][1]
            ln[f"gangs_ready_{k}"] = res[k][0][2]
        lines.append(ln)
        print(json.dumps(ln), flush=True)
    eng.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
