"""CPU: preemption with PodDisruptionBudget-violating bound pods (include/bsched.h BS_BOUND_PDB_VIOLATING) on both CPU
restatements, tests/preempt_pdb_ref.c and tests/pyref_preempt_pdb.py: the hand-built cases of tests/pdb_cases.py with
and without the bits, the two restatements against each other on random tables, both against the budget-free
restatement tests/preempt_ref.c on tables without the bit, and the generator's `violating` draw.  The GPU is compared
with the C restatement in tests/test_gpu_preempt_pdb.py."""
import importlib
import itertools

import numpy as np
import pytest

import pdb_cases
import preempt_pdb_ref
import preempt_ref
import pyref_preempt
import pyref_preempt_pdb
import randsnap

S = importlib.import_module("batch-scheduler_b200.snapshot")


def _check(snap, bound, pods, want=None):
    got = preempt_pdb_ref.preempt(snap, bound, pods)
    py = pyref_preempt_pdb.preempt(snap, bound, pods)
    for k in range(len(pods)):
        assert (int(got.node[k]), got.victims_of(k), int(got.n_candidates[k])) == py[k], k
        if want is not None:
            assert (int(got.node[k]), got.victims_of(k)) == tuple(want[k]), k
    return got


@pytest.mark.parametrize("name", sorted(pdb_cases.cases()))
def test_hand_built_case(name):
    snap, bound, pods, want, plain = pdb_cases.cases()[name]
    _check(snap, bound, pods, want)
    _check(snap, pdb_cases.without_bits(bound), pods, plain)


def _table(seed, L, violating):
    snap = randsnap.random_snapshot(seed, P=8, N=12, G=4, L=L, aff=3 if seed % 2 else 0)
    bound = S.bound_pods(snap, seed, max_per_node=5, priorities=(-5, 0, 1, 100, 2**31 - 1, -2**31), n_starts=3,
                         online=0.3 if seed % 3 else 0.0, locked=0.2 if seed % 4 else 0.0, violating=violating)
    return snap, bound


@pytest.mark.parametrize("seed,L,violating", list(itertools.product(range(12), (5, 9), (0.1, 0.5, 1.0))))
def test_c_restatement_agrees_with_pyref_random(seed, L, violating):
    snap, bound = _table(seed, L, violating)
    assert (bound.flags & S.BOUND_PDB_VIOLATING).any()
    _check(snap, bound, np.arange(snap.pods.n))


def test_random_tables_reach_the_new_rules():
    """Over the random tables above, the bits change some answer (node or victim order) against the same table
    without them."""
    changed = 0
    for seed, L, violating in itertools.product(range(12), (5, 9), (0.1, 0.5, 1.0)):
        snap, bound = _table(seed, L, violating)
        pods = np.arange(snap.pods.n)
        a = preempt_pdb_ref.preempt(snap, bound, pods)
        b = preempt_pdb_ref.preempt(snap, pdb_cases.without_bits(bound), pods)
        changed += sum((int(a.node[k]), a.victims_of(k)) != (int(b.node[k]), b.victims_of(k)) for k in range(len(pods)))
    assert changed > 0


@pytest.mark.parametrize("seed,L", list(itertools.product(range(12), (4, 5, 9, 16))))
def test_bit_free_tables_give_the_budget_free_answers(seed, L):
    """Without the bit both restatements give exactly what the budget-free ones (tests/preempt_ref.c,
    tests/pyref_preempt.py) give, victims in the same order."""
    snap, bound = _table(seed, L, 0.0)
    pods = np.arange(snap.pods.n)
    got = _check(snap, bound, pods)
    want = preempt_ref.preempt(snap, bound, pods)
    py = pyref_preempt.preempt(snap, bound, pods)
    for k in range(len(pods)):
        assert (int(got.node[k]), got.victims_of(k), int(got.n_candidates[k])) == \
            (int(want.node[k]), want.victims_of(k), int(want.n_candidates[k])) == py[k], k


def test_generator_violating_draw():
    """violating=0 gives the table of a call without the parameter; a fraction sets the bit on about that share of
    the rows and leaves every other column and bit as it was."""
    snap = randsnap.random_snapshot(3, P=4, N=40, G=6, L=7)
    base = S.bound_pods(snap, 1)
    zero = S.bound_pods(snap, 1, violating=0.0)
    half = S.bound_pods(snap, 1, violating=0.5)
    for f in base.__dataclass_fields__:
        np.testing.assert_array_equal(getattr(base, f), getattr(zero, f))
        if f != "flags":
            np.testing.assert_array_equal(getattr(base, f), getattr(half, f))
    np.testing.assert_array_equal(half.flags & ~np.uint8(S.BOUND_PDB_VIOLATING), base.flags)
    share = float(((half.flags & S.BOUND_PDB_VIOLATING) != 0).mean())
    assert 0.3 < share < 0.7
    full = S.bound_pods(snap, 1, violating=1.0)
    assert ((full.flags & S.BOUND_PDB_VIOLATING) != 0).all()
