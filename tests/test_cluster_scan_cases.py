"""The designed cluster-scan tables on the CPU: the plain reference walk against the C oracle and the Python
restatement, and proof that each table's designated needs reach the engine's full prefix scan (step 3) both ways."""
import collections

import numpy as np
import pytest

import pyref
import scan_cases as sc

TABLES = {t.name: t for t in sc.tables()}


def test_tables_are_the_designed_shapes():
    L = {t.name: t.lanes for t in TABLES.values()}
    N = {t.name: t.nodes.n for t in TABLES.values()}
    assert 4 in L.values() and 16 in L.values()
    assert N["two_nodes"] == 2 and max(N.values()) > 5 * 256 and max(N.values()) >= 3 * 1024
    assert N["edges"] % 32 and N["edges"] - 4 in TABLES["edges"].targets     # a target in the partial last warp
    assert TABLES["big"].nodes.n == TABLES["big_bump"].nodes.n
    # big_bump's running sum passes 2^62 and returns; big stays far below it
    pre, _, _ = sc.ref_prefixes(TABLES["big_bump"], sc.SEL, sc.TOL, 1.0)
    assert np.abs(pre).max() > 1 << 62
    pre, _, _ = sc.ref_prefixes(TABLES["big"], sc.SEL, sc.TOL, 1.0)
    assert np.abs(pre).max() < 1 << 20


@pytest.mark.parametrize("name", sorted(TABLES))
def test_designated_needs_reach_the_full_scan(name):
    t = TABLES[name]
    pre, keys, vis = sc.ref_prefixes(t, sc.SEL, sc.TOL, t.pct)
    st = sc.stats(pre, keys, vis)
    # every lane's maximum is attained once, so the argmax tie rule cannot change which prefixes are candidates
    assert all(st.unique_max), st.unique_max
    seen = collections.Counter()
    for need, npres, expect, at in t.needs:
        kind = sc.classify(pre, keys, vis, st, need, npres)
        assert kind == "step3-" + expect, (need, hex(npres), kind)
        hit = sc.first_hit(pre, keys, vis, need, npres)
        assert hit == (at if expect == "true" else -1), (need, hit, at)
        seen[expect] += 1
    assert seen["true"] >= 1 and seen["false"] >= 1


def test_designated_positions():
    # the satisfying prefixes sit where the issue of exactness is: warp and chunk edges, the first and last
    # visited nodes, a chunk of otherwise skipped nodes, before and after an int64 wrap
    at = {n: {a for _, _, e, a in t.needs if e == "true"} for n, t in TABLES.items()}
    assert {0, 31, 32, 63, 255, 256, 257, 600, 1346} <= at["edges"]
    e = TABLES["edges"]
    assert all(e.nodes.flags[512:768][np.arange(256) != 600 - 512] & 0x07)
    assert not e.nodes.flags[1347] and all(e.nodes.flags[1348:] & 0x07)
    assert all(TABLES["leading_skip"].nodes.flags[:40] & 0x07) and 40 in at["leading_skip"]
    assert at["wrap"] == {110, 160}


def test_step_totals(capsys):
    """Per path, over the designated needs and a few hundred random ones per table: how many the bounds reject,
    how many a candidate accepts, and how many only the full scan decides (true / false)."""
    total = collections.Counter()
    for t in TABLES.values():
        pre, keys, vis = sc.ref_prefixes(t, sc.SEL, sc.TOL, t.pct)
        st = sc.stats(pre, keys, vis)
        need, npres = sc.random_needs(t, sc.SEL, sc.TOL, t.pct, 200, seed=7)
        rows = [(need[:, j], int(npres[j])) for j in range(need.shape[1])] + [(n[0], n[1]) for n in t.needs]
        c = collections.Counter(sc.classify(pre, keys, vis, st, n, p) for n, p in rows)
        assert c[sc.STEP3_TRUE] >= 1 and c[sc.STEP3_FALSE] >= 1
        total += c
        with capsys.disabled():
            print(f"\n{t.name:13s} N={t.nodes.n:5d} L={t.lanes:2d} " +
                  " ".join(f"{k}={c[k]}" for k in (sc.BOUNDS, sc.CANDIDATE, sc.STEP3_TRUE, sc.STEP3_FALSE)))
    with capsys.disabled():
        print("total " + " ".join(f"{k}={total[k]}" for k in (sc.BOUNDS, sc.CANDIDATE, sc.STEP3_TRUE, sc.STEP3_FALSE)))


def _pyref_nodes(nt):
    return [pyref.Node(nt, i) for i in range(nt.n)]


@pytest.mark.parametrize("name", sorted(TABLES) + ["one_node"])
def test_reference_agrees_with_oracle_and_pyref(oracle, name):
    t = TABLES[name] if name in TABLES else sc.one_node_table()
    nt, L = t.nodes, t.lanes
    nodes = _pyref_nodes(nt)
    for k, ((sel, tol), pct) in enumerate([(c, p) for c in sc.CLASSES for p in (1.0, 0.7)]):
        need, npres = sc.random_needs(t, sel, tol, pct, 60, seed=k)
        if (sel, tol, pct) == (sc.SEL, sc.TOL, t.pct) and t.needs:
            dn, dp = sc.need_arrays(t.needs, L)
            need, npres = np.concatenate([dn, need], axis=1), np.concatenate([dp, npres])
        ref = sc.reference_answers(t, sel, tol, pct, need, npres)
        orc = np.array([oracle.compare_cluster(nt, sel, tol, need[:, j], int(npres[j]), pct)
                        for j in range(need.shape[1])])
        np.testing.assert_array_equal(orc, ref, err_msg=f"oracle, class {(sel, tol)} at {pct}")
        # the Python restatement walks Go-like objects: the designated needs and a sample of the rest
        for j in list(range(len(t.needs) if (sel, tol, pct) == (sc.SEL, sc.TOL, t.pct) else 0)) + [0, 7, 23, 41]:
            if j >= need.shape[1]:
                continue
            r = pyref.resource_from(need[:, j], int(npres[j]), L)
            assert pyref.compare_cluster(nodes, sel, tol, r, pct) == ref[j], (j, sel, tol, pct)
    if t.needs:
        dn, dp = sc.need_arrays(t.needs, L)
        exp = [e == "true" for _, _, e, _ in t.needs]
        np.testing.assert_array_equal(sc.reference_answers(t, sc.SEL, sc.TOL, t.pct, dn, dp), exp)
