"""bs_update_groups with affinity classes: the representative's class (rep_aff) of every changed row reaches the
engine, and each round stays bit-exact against the oracle on the mutated snapshot."""
import numpy as np
import pytest

from parity import assert_round_equal
from randsnap import random_snapshot

pytestmark = pytest.mark.gpu

GROUP_COLUMNS = ("min_member", "scheduled", "matched", "flags", "min_res", "min_res_present", "rep_sel", "rep_tol",
                 "creation_ns", "name_rank", "rep_aff")


def changed_rows(S, gt, idx, aff, rng):
    """Rows `idx` of `gt`, each with a carried-in representative (HAS_POD) whose affinity class differs from its own."""
    rows = S.GroupTable(*(getattr(gt, f)[..., idx].copy() for f in GROUP_COLUMNS))
    rows.flags |= S.GROUP_HAS_POD
    classes = np.append(np.arange(aff), S.AFF_NONE).astype(np.uint32)   # AFF_NONE is the last choice
    pos = np.where(rows.rep_aff == S.AFF_NONE, aff, rows.rep_aff)
    rows.rep_aff = classes[(pos + rng.integers(1, aff + 1, len(idx))) % (aff + 1)]
    return rows


def test_incremental_group_update_affinity(pkg, oracle, snapshot_mod):
    S = snapshot_mod
    aff = 4
    # seeds where a changed row's class decides PreFilter verdicts (one class fits no node): every round differs
    # from one in which the changed rows lost their class
    snap = random_snapshot(6172, P=260, N=300, G=40, L=6, aff=aff)
    gt = snap.groups
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=True, score=True)
    eng.upload(snap)
    eng.evaluate()
    rng = np.random.default_rng(5)
    for _ in range(3):
        idx = np.sort(rng.choice(gt.n, size=9, replace=False)).astype(np.uint32)
        rows = changed_rows(S, gt, idx, aff, rng)
        for f in GROUP_COLUMNS:
            getattr(gt, f)[..., idx] = getattr(rows, f)
        eng.update_groups(idx, rows)
        res = eng.evaluate()
        orc = oracle.round(snap, want_bitmap=True, want_score=True)
        assert_round_equal(res, eng.fit_rows(), eng.score_rows(), orc)
    eng.close()
