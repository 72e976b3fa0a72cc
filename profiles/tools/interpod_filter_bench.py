"""The MatchInterPodAffinity filter on cfg4 on one GPU; writes profiles/interpod_filter_h100.jsonl.

    python profiles/tools/interpod_filter_bench.py [--out PATH] [--steps 20] [--warmup 3] [--reps 2]

cfg4 (100k pods x 10k nodes, 5 lanes) with the filter's columns from snapshot.node_interpod_filter (hostname and zone
keys; shares of the gangs one per host with siblings bound, zone-affine to a bound "ps" pod, or zone-affine to their
own job under the first-pod exception; 16 bound pods with zone anti-affinity; two class-less bound pods per node).  Three round kinds, each with the filter on
and off in one engine: decisions only, top-K at K = 16, and the priority lists at K = 16 with reason rows.  The
switch alternates `reps` times per kind (the order flips every repetition); per setting, CUDA events on the engine
stream around `steps` back-to-back rounds; also a round after the node side is uploaded again (the pre-pass and the
class rebuild) against a steady one.  In passes of their own, torch.profiler gives each kernel's device time per
round: steady with the filter on and off (the reason stage is reason_pod_kernel) and after a node-side upload (the
pre-pass alone is ipf_presence_kernel + ipf_class_kernel).  The first
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


def timed(eng, steps, warmup, before=None):
    """ms per round over `steps` rounds (events on the engine stream); before() runs ahead of each timed round."""
    ext = torch.cuda.ExternalStream(eng.stream())
    for _ in range(warmup):
        if before:
            before()
        eng.evaluate_async()
    eng.sync()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(ext)
    for _ in range(steps):
        if before:
            before()
        eng.evaluate_async()
    b.record(ext)
    eng.sync()
    b.synchronize()
    return a.elapsed_time(b) / steps


KERNELS = ("ipf_presence_kernel", "ipf_class_kernel", "node_left_kernel", "class_fit_kernel", "reason_class_kernel",
           "reason_pod_kernel", "priority_pod_kernel", "gang_fit")


def kernel_ms(eng, rounds, node_side=None):
    """Device ms per round of each kernel of KERNELS, from torch.profiler in a pass of its own; with node_side, the
    filter's node side is uploaded again before every round, so that the pre-pass and the class rebuild run in each."""
    from torch.profiler import ProfilerActivity, profile
    eng.evaluate()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            if node_side is not None:
                eng.upload_interpod_filter(node=node_side)
            eng.evaluate()
    tot = dict.fromkeys(KERNELS, 0.0)
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        for k in KERNELS:
            if k in ev.key:
                tot[k] += t
    return {k: v / 1000.0 / rounds for k, v in tot.items() if v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "interpod_filter_h100.jsonl"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    snap = S.config(4)
    cols = S.node_interpod_filter(snap, 4)
    nz = S.nonzero_requests(snap, 4)
    lines = [dict(kind="card", **card(), reps=args.reps)]
    kinds = {"decisions": dict(fit_bitmap=False), "topk16": dict(fit_bitmap=False, topk=16),
             "priority16_reasons": dict(fit_bitmap=False, priority_k=16, reasons=True)}
    for kind, kw in kinds.items():
        eng = pkg.Engine(snap.lanes, 0, **kw)
        eng.upload(snap)
        if kw.get("priority_k"):
            eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.upload_interpod_filter(node=cols[0], pods=cols[1])
        ms = {"on": [], "off": []}
        for r in range(args.reps):
            for on in ((True, False) if r % 2 == 0 else (False, True)):
                eng.set_interpod_filter(on)
                ms["on" if on else "off"].append(timed(eng, args.steps, args.warmup))
        eng.set_interpod_filter(True)
        prepass = timed(eng, args.steps, args.warmup, before=lambda: eng.upload_interpod_filter(node=cols[0]))
        prof = {"steady_on": kernel_ms(eng, 5), "after_node_side": kernel_ms(eng, 5, cols[0])}
        eng.set_interpod_filter(False)
        prof["steady_off"] = kernel_ms(eng, 5)
        eng.set_interpod_filter(True)
        feasible = eng.evaluate().feasible_count.copy()
        eng.set_interpod_filter(False)
        feasible_off = eng.evaluate().feasible_count.copy()
        eng.close()
        lines.append(dict(kind=kind, P=snap.pods.n, N=snap.nodes.n, lanes=snap.lanes,
                          bound_pods=int(len(cols[0][3])), terms=int(len(cols[0][2])),
                          filter_classes=int(len(cols[1][1][0]) - 1),
                          round_ms_on=ms["on"], round_ms_off=ms["off"],
                          round_ms_on_median=float(np.median(ms["on"])), round_ms_off_median=float(np.median(ms["off"])),
                          spread_on=float(np.ptp(ms["on"])), spread_off=float(np.ptp(ms["off"])),
                          round_ms_after_node_side=prepass,
                          extra_ms_after_node_side=prepass - float(np.median(ms["on"])),
                          kernel_ms_profiler=prof,
                          pods_losing_nodes=int((feasible < feasible_off).sum()),
                          pods_fitting_nowhere_on=int((feasible == 0).sum()),
                          pods_fitting_nowhere_off=int((feasible_off == 0).sum())))
        print(json.dumps(lines[-1]), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for ln in lines:
            f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
