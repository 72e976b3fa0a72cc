"""CPU: the group decomposition of DESIGN §6, pinned on the CPU references before the GPU test relies on it.

For every case of tests/shard_cases.py, every world size of 2, 3 and 4 and every rank, each round's references on the
rank's shard (tables and side columns cut by shard_cases.shard) equal the references on the whole snapshot restricted
to the shard: every per-pod row (PreFilter, the feasible count, best node and score, the fit, score and Filter rows, the
reason and both filters' companion rows, top-K and the priority lists with every weight and both filters on),
admit and new_denied of the rank's own group range and of the groups no rank holds pods of, max_group and max_finished
on every rank, and the queue order as the whole order filtered to the shard.  The rounds in between apply the same
group row updates on every rank, and the cases are checked to do what their names say."""
import functools

import numpy as np
import pytest

import shard_cases as sc


@functools.cache
def _rounds(name):
    """[(Model, every output of its round)] for the case's rounds on the whole snapshot."""
    m = sc.case(name)
    out = [(m, m.expect(sc.EVERY_OUTPUT))]
    for upd in sc.group_updates(m):
        m = sc.updated(m, upd)
        out.append((m, m.expect(sc.EVERY_OUTPUT)))
    return out


@pytest.mark.parametrize("world", sc.WORLDS)
@pytest.mark.parametrize("name", sc.CASES)
def test_shard_equals_whole_restricted(oracle, name, world):
    for k, (m, full) in enumerate(_rounds(name)):
        idle = sc.idle_groups(m)
        for rank in range(world):
            s, idx, (g0, g1) = sc.shard(m, rank, world)
            got = s.expect(sc.EVERY_OUTPUT)
            d = sc.first_diff(full, got, idx, g0, g1, idle)
            assert d is None, f"case {name} world {world} rank {rank} round {k}: {d}"


@pytest.mark.parametrize("name", sc.CASES)
def test_rounds_move_admits_and_max_group(oracle, name):
    rounds = _rounds(name)
    admits = [full["admit"] for _, full in rounds]
    assert all(not np.array_equal(a, b) for a, b in zip(admits, admits[1:])), "a group row update left every admit"
    assert len({full["max_group"] for _, full in rounds}) > 1, "max_group never moved"


def _shards(name, world):
    m = sc.case(name)
    return [sc.shard(m, r, world) for r in range(world)], m


def test_case_shapes(oracle):
    """Each case is the regime its name claims."""
    G = {n: sc.case(n).groups.n for n in sc.CASES}
    assert 32 * 256 < G["many_groups"] <= 32 * 512 < G["many_groups3"] <= 32 * 768
    assert all(g % 32 for n, g in G.items() if n != "empty_shard")
    for world in sc.WORLDS:
        sh, m = _shards("ungrouped", world)
        for r, (_, idx, (g0, g1)) in enumerate(sh):
            gid = m.pods.gid[idx]
            assert (gid < 0).any() and (idx[gid < 0] % world == r).all()
        sh, m = _shards("empty_shard", world)
        if world > 2:   # a rank without pods; with four, one without groups too
            assert any(len(idx) == 0 for _, idx, _ in sh)
            assert world == 3 or any(len(idx) == 0 and g0 == g1 for _, idx, (g0, g1) in sh)
    m = sc.case("idle")
    idle = sc.idle_groups(m)
    assert idle[0] and idle[-1] and idle[50] and (~idle).sum() == 42
    heavy = np.bincount(sc.case("unbalanced").pods.gid.clip(0), minlength=48)[[5, 6, 30]].sum()
    assert heavy > 0.6 * sc.case("unbalanced").pods.n
