"""TEST INFRASTRUCTURE — hand-built walks under the MatchInterPodAffinity filter with their placements written out.

Each case: (name, nodes {name: labels} in order, existing pods, pending pods, queue (pending indices in pop order, None:
table order), expected node per queue position).  snapshot() gives the table every case runs on: one gang of all the
pending pods with MinMember = their count, and nodes so roomy that only the filter decides (first fit).
"""
import numpy as np

from pyref_interpod_filter import Pod, Term
from randsnap import random_snapshot

H = "kubernetes.io/hostname"
Z = "zone"


def _nodes(*zones):
    """n0, n1, ... with a hostname label and the given zone (None: no zone label)."""
    out = {}
    for i, z in enumerate(zones):
        lab = {H: f"n{i}"}
        if z is not None:
            lab[Z] = z
        out[f"n{i}"] = lab
    return out


def _ps():
    return Pod("ps", labels={"role": "ps", "job": "j"})


def _follower(name, one_per_host=False):
    """A worker that needs the zone of job j's parameter server (and, one_per_host, a host without a sibling)."""
    return Pod(name, labels={"job": "j", "role": "worker"}, affinity=[Term({"role": "ps", "job": "j"}, Z)],
               anti=[Term({"job": "j", "role": "worker"}, H)] if one_per_host else [])


CASES = [
    # one worker per host: eight workers, five hosts; the round admits the gang, the walk places five
    ("eight-anti-workers", _nodes(*["a"] * 5), [],
     [Pod(f"w{i}", labels={"job": "j"}, anti=[Term({"job": "j"}, H)]) for i in range(8)],
     None, [0, 1, 2, 3, 4, -1, -1, -1]),
    # the parameter server pops first: the workers follow it into zone b, one per host
    ("ps-before-workers", _nodes("b", "a", "b"), [],
     [_ps(), _follower("w0", True), _follower("w1", True)],
     None, [0, 0, 2]),
    # the workers pop before the parameter server: no node has it in its zone yet
    ("ps-after-workers", _nodes("b", "a", "b"), [],
     [_ps(), _follower("w0", True), _follower("w1", True)],
     [1, 2, 0], [-1, -1, 0]),
    # a self-affine gang, one per host: the first worker goes anywhere under the first-pod exception, the others
    # follow its zone until it has no free host
    ("self-affine-gang", _nodes("b", "a", "b"), [],
     [Pod(f"w{i}", labels={"job": "s"}, affinity=[Term({"job": "s"}, Z)], anti=[Term({"job": "s"}, H)])
      for i in range(3)],
     None, [0, 2, -1]),
    # a pod without terms of its own (filter class BS_IPF_NONE) kept off a host by an earlier pod's anti-affinity
    ("none-pod-kept-out", _nodes("a", "a"), [],
     [Pod("guard", labels={"app": "web"}, anti=[Term({"app": "db"}, H)]), Pod("db", labels={"app": "db"})],
     None, [0, 1]),
    # nodes without the key and an empty topology key: a zone anti-affinity owned on an unzoned node blocks nobody, an
    # empty key is carried by no node, and pods on unzoned nodes give an affinity term no pair
    ("no-key-and-empty-key", _nodes(None, "a"), [],
     [Pod("p0", labels={"app": "x"}, anti=[Term({"app": "x"}, Z)]),
      Pod("p1", labels={"app": "x"}, anti=[Term({"app": "x"}, "")]),
      Pod("p2", labels={"app": "x"}),
      Pod("p3", affinity=[Term({"app": "x"}, Z)])],
     None, [0, 0, 0, -1]),
    # a bound pod's anti-affinity and an assumed one's together
    ("bound-and-assumed-anti", _nodes("a", "a", "b"),
     [Pod("old", labels={"app": "y"}, anti=[Term({"app": "x"}, H)], node="n0")],
     [Pod("p0", labels={"app": "x"}, anti=[Term({"app": "x"}, Z)]), Pod("p1", labels={"app": "x"})],
     None, [1, 2]),
]


def snapshot(n_nodes: int, n_pods: int):
    """One gang of n_pods tiny pods (MinMember n_pods) on n_nodes roomy nodes without taints, labels or selectors."""
    snap = random_snapshot(31, P=n_pods, N=n_nodes, G=1, L=5, case="mixed")
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    nt.flags[:] = 0
    nt.label_mask[:] = 0
    nt.taint_mask[:] = 0
    nt.alloc[:4] = 1 << 40
    nt.requested[:] = 0
    nt.pod_count[:] = 0
    nt.alloc_present[:] = 0xF
    nt.req_present[:] = 0
    pt.req[:] = 1
    pt.req_present[:] = 0xF
    pt.gid[:] = 0
    pt.flags[:] = 0
    pt.sel_mask[:] = 0
    pt.tol_mask[:] = 0
    if pt.aff_class is not None:
        pt.aff_class[:] = 0xFFFFFFFF
    gt.min_member[:] = n_pods
    gt.scheduled[:] = 0
    gt.matched[:] = 0
    gt.flags[:] = 0
    return snap


def queue_of(case):
    return None if case[4] is None else np.asarray(case[4], np.uint32)
