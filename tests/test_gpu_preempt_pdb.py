"""GPU: bs_preempt with PodDisruptionBudget-violating bound pods (BS_BOUND_PDB_VIOLATING) bit-exact against the CPU
restatement tests/preempt_pdb_ref.c (node, n_victims, n_candidates, offsets, victims in order): the hand-built cases of
tests/pdb_cases.py, random tables at every register width of the kernels (MAXL 5, 9 and 16), several node tiles with
ties across them, a launch split over preemptors, a victims cap that is too small, and the generator's default table
with bits added."""
import ctypes as C
import importlib
import itertools

import numpy as np
import pytest

import pdb_cases
import preempt_pdb_ref
import randsnap

S = importlib.import_module("batch-scheduler_b200.snapshot")
E = importlib.import_module("batch-scheduler_b200.engine")
capi = importlib.import_module("batch-scheduler_b200.capi")

pytestmark = pytest.mark.gpu


def _engine(snap, bound):
    eng = E.Engine(snap.lanes)
    eng.upload(snap)
    eng.upload_bound_pods(bound)
    return eng


def _same(got, want):
    np.testing.assert_array_equal(got.node, want.node)
    np.testing.assert_array_equal(got.n_victims, want.n_victims)
    np.testing.assert_array_equal(got.n_candidates, want.n_candidates)
    np.testing.assert_array_equal(got.victim_offset, want.victim_offset)
    np.testing.assert_array_equal(got.victims, want.victims)


def _run(snap, bound, pods=None):
    pods = np.arange(snap.pods.n, dtype=np.uint32) if pods is None else np.asarray(pods, np.uint32)
    eng = _engine(snap, bound)
    got = eng.preempt(pods)
    eng.close()
    _same(got, preempt_pdb_ref.preempt(snap, bound, pods))
    return got


@pytest.mark.parametrize("name", sorted(pdb_cases.cases()))
def test_hand_built_case(name):
    snap, bound, pods, want, plain = pdb_cases.cases()[name]
    got = _run(snap, bound, pods)
    assert [(int(got.node[k]), got.victims_of(k)) for k in range(len(pods))] == want
    got = _run(snap, pdb_cases.without_bits(bound), pods)
    assert [(int(got.node[k]), got.victims_of(k)) for k in range(len(pods))] == plain


@pytest.mark.parametrize("seed,L,violating", list(itertools.product(range(3), (5, 9, 16), (0.1, 0.5, 1.0))))
def test_random(seed, L, violating):
    """L 5, 9 and 16 run the MAXL 5, 9 and 16 builds of the node and emit kernels; every other node is full."""
    snap = randsnap.random_snapshot(seed, P=64, N=90, G=10, L=L, aff=4 if seed % 2 else 0)
    snap.nodes.requested[:3, ::2] = snap.nodes.alloc[:3, ::2]
    snap.pods.gid[::2] = S.GID_NONE
    bound = S.bound_pods(snap, seed, max_per_node=40, priorities=(-5, 0, 1, 100, 2**31 - 1, -2**31),
                         online=0.5, locked=0.1, violating=violating)
    got = _run(snap, bound)
    assert ((got.node >= 0) & (got.n_victims > 0)).any()


def test_many_node_tiles():
    """Several 256-node tiles and a partial last one, a third of the bound pods violating."""
    snap = randsnap.random_snapshot(1, P=48, N=1300, G=8, L=5)
    snap.nodes.requested[:3] = snap.nodes.alloc[:3]   # full nodes: a pod fits only where it evicts
    snap.pods.priority[:] = 2**31 - 1
    snap.pods.gid[::2] = S.GID_NONE
    bound = S.bound_pods(snap, 1, max_per_node=12, online=0.5, locked=0.1, violating=0.3)
    got = _run(snap, bound)
    chosen = got.node[got.node >= 0]
    assert len(got.victims) > 0 and len(set((chosen // 256).tolist())) > 2


def test_ties_across_tiles():
    """Identical nodes in several tiles; the pods of nodes 700-999 violate a budget, so the winner is node 1000 in
    tile 3, its violating twins in tiles 2 and 3 lose on the first criterion, and its twins after it tie with it."""
    snap = randsnap.random_snapshot(3, P=16, N=1100, G=4, L=5)
    nt = snap.nodes
    for f in nt.__dataclass_fields__:
        a = getattr(nt, f)
        a[...] = a[..., :1]
    nt.flags[:] = 0
    nt.flags[:700] = S.NODE_UNSCHEDULABLE
    nt.label_mask[:] = ~np.uint64(0)
    nt.taint_mask[:] = 0
    nt.pod_count[:] = 3
    nt.requested[3] = 0
    nt.alloc[3] = 3
    snap.aff_bits = None
    snap.pods.aff_class = None
    snap.pods.gid[:] = S.GID_NONE
    snap.pods.priority[:] = 1000
    snap.pods.req[:] = 0
    snap.pods.req[3] = 1
    snap.pods.req_present[:] = 0
    bound = S.bound_pods(snap, 3, priorities=(5,), n_starts=1, online=1.0)
    bound.flags[bound.node < 1000] |= S.BOUND_PDB_VIOLATING
    got = _run(snap, bound)
    assert (got.node == 1000).all() and (got.n_candidates == 400).all()


def test_many_preemptors():
    """More preemptors than one launch takes (gridDim.y <= 65535)."""
    snap = randsnap.random_snapshot(7, P=70000, N=40, G=8, L=5)
    bound = S.bound_pods(snap, 7, max_per_node=20, violating=0.4)
    pods = np.arange(snap.pods.n, dtype=np.uint32)
    eng = _engine(snap, bound)
    got = eng.preempt(pods)
    eng.close()
    sample = np.concatenate([pods[:300], pods[65400:65700], pods[-300:]])
    want = preempt_pdb_ref.preempt(snap, bound, sample)
    np.testing.assert_array_equal(got.node[sample], want.node)
    np.testing.assert_array_equal(got.n_victims[sample], want.n_victims)
    np.testing.assert_array_equal(got.n_candidates[sample], want.n_candidates)
    for k, p in enumerate(sample):
        assert got.victims_of(int(p)) == want.victims_of(k)


def test_victims_cap_too_small():
    snap = randsnap.random_snapshot(5, P=30, N=30, G=4, L=5)
    bound = S.bound_pods(snap, 5, max_per_node=20, online=1.0, violating=0.5)
    snap.pods.gid[:] = S.GID_NONE
    snap.pods.priority[:] = 2**31 - 1
    eng = _engine(snap, bound)
    n = 30
    full = eng.preempt(np.arange(n, dtype=np.uint32))
    _same(full, preempt_pdb_ref.preempt(snap, bound, np.arange(n)))
    assert len(full.victims) > 0
    idx = np.arange(n, dtype=np.uint32)
    node, nv, cand, off = np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n + 1, np.uint32)
    vict = np.full(4, 7, np.uint32)
    r = capi.PreemptResultC(capi.ptr(node), capi.ptr(nv), capi.ptr(cand), capi.ptr(off), capi.ptr(vict),
                            len(full.victims) - 1, 0)
    rc = eng.lib.bs_preempt(eng.h, capi.ptr(idx), n, C.byref(r))
    eng.close()
    assert rc == capi.BS_E_INVAL and r.victims_total == len(full.victims)
    assert (vict == 7).all()


@pytest.mark.parametrize("violating", [0.3, 1.0])
def test_generator_default_table_with_bits(violating):
    """snapshot.bound_pods' defaults (online, missing-group and locked pods) with bits added, on full nodes.  With some
    pods violating, the bits change some answer against the same table without them."""
    snap = randsnap.random_snapshot(12, P=64, N=200, G=10, L=5)
    snap.nodes.requested[:3] = snap.nodes.alloc[:3]
    snap.pods.priority[:] = 2**31 - 1
    snap.pods.gid[::2] = S.GID_NONE
    bound = S.bound_pods(snap, 12, violating=violating)
    got = _run(snap, bound)
    plain = _run(snap, pdb_cases.without_bits(bound))
    assert violating == 1.0 or any((int(got.node[k]), got.victims_of(k)) != (int(plain.node[k]), plain.victims_of(k))
               for k in range(snap.pods.n))
