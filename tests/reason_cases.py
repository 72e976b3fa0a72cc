"""A hand-built round for the reason rows (include/bsched.h BS_REASON_*): one node per rule, with the bins each of
two pods must count there written out node by node.

Lanes (L = 6): 0 cpu, 1 memory, 2 ephemeral-storage, 3 pods, 4 and 5 scalar.  Every node starts as a node where
both pods fit (1000 on lanes 0-2, 10 pods, 5 on both scalar lanes with both keys present, label bit 0, no taint,
affinity class 0 matched) and changes one thing or a few.

  pod 0: sel 0b1, tol 0b1, affinity class 0; requests 100 / 100 / 100 / 1 pod, 2 on lane 4, 0 on lane 5 (both keys)
  pod 1: sel 0, tol 0, no affinity class; requests nothing.  Its presence mask carries the stray bits 0-3 and
         bit 10 (>= L), which compareResourceAndRequire never reads, and lane 4 holds 100 without the key.
"""
from __future__ import annotations

import numpy as np

from randsnap import S

L = 6
UNSCHED, UNAVAIL, SEL, TAINT = 0, 1, 2, 3
CPU, MEM, EPH, PODS, LANE4, LANE5 = 4, 5, 6, 7, 8, 9

# (what changes, bins of pod 0, bins of pod 1)
NODES = [
    ("fits", (), ()),
    ("nil + unschedulable", (UNAVAIL,), (UNAVAIL,)),
    ("unschedulable + taints error", (UNSCHED,), (UNSCHED,)),
    ("no node + taints error", (UNAVAIL,), (UNAVAIL,)),
    ("nil + no node", (UNAVAIL,), (UNAVAIL,)),
    ("taints error", (UNAVAIL,), (UNAVAIL,)),
    ("unschedulable", (UNSCHED,), (UNSCHED,)),
    ("selector only", (SEL,), ()),
    ("taint only", (TAINT,), (TAINT,)),
    ("selector and taint", (SEL, TAINT), (TAINT,)),
    ("affinity bit only", (SEL,), ()),
    ("cpu short by 1", (CPU,), ()),
    ("cpu exact", (), ()),
    ("memory short by 1", (MEM,), ()),
    ("ephemeral-storage short by 1", (EPH,), ()),
    ("pods short: len(Pods()) = 10", (PODS,), ()),
    ("pods exact: len(Pods()) = 9", (), ()),
    ("lane 4 short by 1", (LANE4,), ()),
    ("lane 4 exact", (), ()),
    ("lane 4 key absent from allocatable, request 2", (LANE4,), ()),
    ("lane 5 key absent from requested, request 0", (), ()),
    ("requested pods 10 overrides len(Pods()) = 0", (PODS,), ()),
    ("selector fails and cpu short: no lane bin", (SEL,), ()),
    ("unschedulable and selector fails: guard only", (UNSCHED,), (UNSCHED,)),
    ("cpu short and lane 4 absent: both lanes", (CPU, LANE4), ()),
    ("lane 4 left negative", (LANE4,), ()),
    ("taint tolerated by pod 0 only", (), (TAINT,)),
]
N = len(NODES)


def snapshot() -> S.Snapshot:
    nt = S.NodeTable.empty(N, L)
    nt.alloc[:3] = 1000
    nt.alloc[3] = 10
    nt.alloc[4:] = 5
    both = np.uint32((1 << 4) | (1 << 5))
    nt.alloc_present[:] = both
    nt.req_present[:] = both
    nt.label_mask[:] = 1
    aff = np.ones(N, bool)
    f = nt.flags
    f[1] = S.NODE_NIL | S.NODE_UNSCHEDULABLE
    f[2] = S.NODE_UNSCHEDULABLE | S.NODE_TAINTS_ERR
    f[3] = S.NODE_NO_NODE | S.NODE_TAINTS_ERR
    f[4] = S.NODE_NIL | S.NODE_NO_NODE
    f[5] = S.NODE_TAINTS_ERR
    f[6] = S.NODE_UNSCHEDULABLE
    nt.label_mask[7] = 0
    nt.taint_mask[8] = 0b10
    nt.label_mask[9], nt.taint_mask[9] = 0, 0b10
    aff[10] = False
    nt.requested[0, 11] = 901
    nt.requested[0, 12] = 900
    nt.requested[1, 13] = 901
    nt.requested[2, 14] = 901
    nt.pod_count[15] = 10
    nt.pod_count[16] = 9
    nt.requested[4, 17] = 4
    nt.requested[4, 18] = 3
    nt.alloc_present[19] = np.uint32(1 << 5)
    nt.req_present[20] = np.uint32(1 << 4)
    nt.requested[3, 21] = 10
    nt.label_mask[22], nt.requested[0, 22] = 0, 901
    f[23], nt.label_mask[23] = S.NODE_UNSCHEDULABLE, 0
    nt.requested[0, 24], nt.alloc_present[24] = 901, np.uint32(1 << 5)
    nt.requested[4, 25] = 9
    nt.taint_mask[26] = 0b01

    pt = S.PodTable.empty(2, L)
    pt.req[:, 0] = [100, 100, 100, 1, 2, 0]
    pt.req_present[0] = (1 << 4) | (1 << 5)
    pt.sel_mask[0], pt.tol_mask[0] = 1, 1
    pt.req[:, 1] = [0, 0, 0, 0, 100, 0]
    pt.req_present[1] = 0xF | (1 << 10)
    pt.aff_class = np.array([0, S.AFF_NONE], np.uint32)
    gt = S.GroupTable.empty(1, L)
    gt.min_member[:] = 1
    snap = S.Snapshot(nt, pt, gt, "reason_cases")
    W = (N + 31) // 32
    by = np.packbits(np.concatenate([aff, np.zeros(W * 32 - N, bool)]), bitorder="little")
    snap.aff_bits = by.view(np.uint32).reshape(1, W).copy()
    return snap


def expected() -> np.ndarray:
    """[2, 4 + L] rows summed from the per-node table."""
    out = np.zeros((2, 4 + L), np.uint32)
    for _, b0, b1 in NODES:
        for p, bins in ((0, b0), (1, b1)):
            for b in bins:
                out[p, b] += 1
    return out
