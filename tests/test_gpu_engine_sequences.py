"""GPU: one long-lived engine through seeded sequences of uploads, row updates, affinity tables, side columns, weights,
the MatchInterPodAffinity filter's switch, halves and placed side, the PodFitsHostPorts filter's switch and halves,
failing calls, rounds, walks with either filter or both, preemption with PodDisruptionBudget bits and the preemption walk (tests/engine_model.py), with every output on.  After each op the engine
answers the error code the host model predicts, and every round, walk and preemption is bit-exact against the CPU
restatements on the model's state.  A mismatch reports the seed, the step, the ops up to it, the first differing
output and whether a fresh engine loaded with the model's state agrees (stale engine state) or not (a kernel)."""
import numpy as np
import pytest

import engine_model as em

pytestmark = pytest.mark.gpu

CONFIGS = {
    "score_filter_reasons_priority": dict(score=True, fit_bitmap=True, filter=True, reasons=True, priority_k=8),
    "topk_priority_reasons": dict(fit_bitmap=False, topk=8, priority_k=8, reasons=True),
}


def _engine(pkg, L, cfg):
    return pkg.Engine(L, 0, fit_bitmap=cfg.get("fit_bitmap", False), score=cfg.get("score", False),
                      filter=cfg.get("filter", False), topk=cfg.get("topk", 0), reasons=cfg.get("reasons", False),
                      priority_k=cfg.get("priority_k", 0))


def _side(eng, op):
    name, half, cols = op["name"], op["half"], op["cols"]
    kw = {half if half == "node" else "pods": cols}
    if name == "nz":
        eng.upload_nonzero(**kw)
    elif name == "pref":
        eng.upload_preferences(**kw)
    elif name == "loc":
        eng.upload_locality(**kw)
    elif name == "spread":
        eng.upload_spread(**kw, n_zones=8 if half == "node" else None)
    else:
        eng.upload_interpod(**kw)


def _weights(eng, L, op):
    if "weights" in op:
        eng.set_score_weights(*op["weights"])
    if "ratio" in op:
        r = op["ratio"]
        if r[0]:
            eng.set_ratio_priority(r[0], r[1], r[2], r[3])
        else:
            eng.set_ratio_priority(0, em.rr.BIN_PACK, [0] * L, 0)
    if "pw" in op:
        eng.set_node_priority_weights(*op["pw"])
    if "lw" in op:
        eng.set_locality_weights(*op["lw"])
    if "w_spread" in op:
        eng.set_spread_weight(op["w_spread"])
    if "w_ipa" in op:
        eng.set_interpod_weight(op["w_ipa"])


def _round(eng, cfg, how):
    if how == "view":
        r = eng.evaluate(view=True)
    elif how == "async":
        eng.evaluate_async()
        eng.sync()
        r = eng.fetch()
    else:
        r = eng.evaluate()
    out = {f: np.array(getattr(r, f)) for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit",
                                                  "admit_bitmap", "new_denied", "order", "rank")}
    out["max_group"], out["max_finished"] = r.max_group, r.max_finished
    if cfg.get("fit_bitmap"):
        out["fit_rows"] = eng.fit_rows()
    if cfg.get("score"):
        out["score_rows"] = eng.score_rows()
    if cfg.get("filter"):
        out["filter_rows"], out["filter_code"] = eng.filter_rows(), np.array(r.filter_code)
    if cfg.get("topk"):
        out["topk_nodes"], out["topk_scores"] = eng.topk_rows()
    if cfg.get("reasons"):
        out["reason_rows"] = eng.reason_rows()
        out["interpod_rows"] = eng.fetch_interpod_reason_rows()
        out["host_port_rows"] = eng.fetch_host_port_reason_rows()
    if cfg.get("priority_k"):
        out["priority_nodes"], out["priority_scores"] = eng.priority_rows()
    out["lanes"] = eng.fit_lanes()
    return out


def _call(pkg, eng, L, op, cfg):
    """Runs one op on the engine: (error code or None, outputs or None)."""
    k = op["op"]
    try:
        if k == "upload_nodes":
            eng.upload_nodes(op["table"])
        elif k == "update_nodes":
            eng.update_nodes(op["idx"], op["rows"])
        elif k == "upload_groups":
            eng.upload_groups(op["table"])
        elif k == "update_groups":
            eng.update_groups(op["idx"], op["rows"])
        elif k == "upload_pods":
            eng.upload_pods(op["table"])
        elif k == "upload_affinity":
            eng.upload_affinity(op["bits"])
        elif k == "upload_bound":
            eng.upload_bound_pods(op["table"])
        elif k == "side":
            _side(eng, op)
        elif k == "ipf":
            eng.upload_interpod_filter(**{"node" if op["half"] == "node" else "pods": op["cols"]})
        elif k == "ipf_switch":
            eng.set_interpod_filter(op["on"])
        elif k == "placed":
            eng.upload_interpod_placed(*op["cols"])
        elif k == "hp":
            eng.upload_host_ports(**{"node" if op["half"] == "node" else "pods": op["cols"]})
        elif k == "hp_switch":
            eng.set_host_port_filter(op["on"])
        elif k == "weights":
            _weights(eng, L, op)
        elif k == "evaluate":
            return None, _round(eng, cfg, op["how"])
        elif k == "replay":
            w = eng.replay(priority=op["priority"], after_state=False)
            return None, {f: w[f] for f in ("prefilter", "node", "ready")}
        elif k == "preempt":
            r = eng.preempt(op["pods"])
            return None, {"node": r.node, "n_victims": r.n_victims, "n_candidates": r.n_candidates, "victims": r.victims}
        elif k == "preempt_walk":
            r = eng.preempt_walk(op["pods"], gang=op["gang"])
            return None, {"node": r.node, "n_victims": r.n_victims, "n_candidates": r.n_candidates, "victims": r.victims,
                          "outcome": r.outcome, "evicted_by": r.evicted_by}
        else:
            raise ValueError(k)
    except pkg.capi.BsError as ex:
        return ex.code, None
    return None, None


def _first_diff(got, want):
    for key, w in want.items():
        g = got.get(key)
        if key == "lanes":
            g, w = tuple(np.asarray(x) for x in g), tuple(np.asarray(x) for x in w)
            if not all(np.array_equal(a, b) for a, b in zip(g, w)):
                return f"lanes: got {g} want {w}"
            continue
        g, w = np.asarray(g), np.asarray(w)
        if g.shape != w.shape:
            return f"{key}: shape {g.shape} != {w.shape}"
        if not np.array_equal(g, w):
            at = np.argwhere(g != w)[:4].tolist() if g.ndim else []
            return f"{key}: first differing indices {at}"
    return None


def _expect(model, op, cfg):
    if op["op"] == "evaluate":
        return model.expect(cfg)
    if op["op"] == "replay":
        return model.expect_walk(op["priority"], None)
    if op["op"] == "preempt":
        return model.expect_preempt(op["pods"])
    return model.expect_preempt_walk(op["pods"], op["gang"])


def _fresh_agrees(pkg, model, cfg, L, op):
    """A fresh engine loaded with the model's state (tables, sides, weights, both filters' halves and switches, the
    placed side, the bound table): does `op` (a round, walk or preemption; else a round) on it equal the references?"""
    eng = _engine(pkg, L, cfg)
    try:
        eng.upload_nodes(model.nodes)
        if model.aff is not None:
            eng.upload_affinity(model.aff)
        eng.upload_groups(model.groups)
        eng.upload_pods(model.pods)
        for key, cols in model.side.items():
            if cols is not None:
                name, half = key.split("_")
                _side(eng, {"name": name, "half": half, "cols": cols})
        for kind in ("ipf", "hp"):
            for half in ("node", "pod"):
                if getattr(model, kind + "_" + half) is not None:
                    _call(pkg, eng, L, {"op": kind, "half": half, "cols": getattr(model, kind + "_" + half)}, cfg)
        if model.ipf_placed is not None:
            eng.upload_interpod_placed(*model.ipf_placed)
        eng.set_interpod_filter(model.ipf_on)
        eng.set_host_port_filter(model.hp_on)
        if model.bound is not None:
            eng.upload_bound_pods(model.bound)
        _weights(eng, L, dict(weights=model.weights, ratio=model.ratio, pw=model.pw, lw=model.lw,
                              w_spread=model.w_spread, w_ipa=model.w_ipa))
        if op["op"] not in ("evaluate", "replay", "preempt", "preempt_walk"):
            op = {"op": "evaluate", "how": "evaluate"}
        code, got = _call(pkg, eng, L, op, cfg)
        if code is not None:
            return f"fresh engine answered {code}"
        want = _expect(model, op, cfg)
        want.pop("lanes", None)
        got.pop("lanes", None)
        return _first_diff(got, want) is None
    except Exception as ex:  # noqa: BLE001
        return f"fresh engine failed: {ex!r}"
    finally:
        eng.close()


def _run_seed(pkg, cfg, seed):
    ops, _, L = em.generate(seed)
    model = em.Model(L)
    eng = _engine(pkg, L, cfg)
    try:
        for step, op in enumerate(ops):
            want_code = model.apply(op)
            code, got = _call(pkg, eng, L, op, cfg)

            def fail(what):
                log = "\n".join(f"  {i:3d} {em.describe(o)}" for i, o in enumerate(ops[:step + 1]))
                fresh = _fresh_agrees(pkg, model, cfg, L, op) if model.complete() else "n/a (tables missing)"
                pytest.fail(f"seed {seed} step {step}: {what}\nfresh engine with the model's state agrees with the "
                            f"references: {fresh}\nops:\n{log}")

            if code != want_code:
                fail(f"{em.describe(op)} answered {code}, the model predicts {want_code}")
            if got is None or want_code is not None:
                continue
            d = _first_diff(got, _expect(model, op, cfg))
            if d:
                fail(f"{em.describe(op)}: {d}")
    finally:
        eng.close()


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("seed", range(len(em.BURSTS)))
def test_engine_sequences(pkg, oracle, config, seed):
    _run_seed(pkg, CONFIGS[config], seed)
