"""GPU, 2-4 ranks: the group-sharded round on every rank with peers attached, against the unsharded references.

Each rank loads its shard of every case of tests/shard_cases.py (tables and side columns, all six priority weights and
both filters on) into both engine configurations of test_gpu_engine_sequences.CONFIGS, attaches the
peer exchange, and runs shard_cases.ROUNDS rounds with the same group row updates in between.  After each round every
rank checks its own outputs bit-exact against the whole snapshot's references restricted to its shard
(shard_cases.first_diff: the CPU test pins that decomposition), and the gathered bitmap: every rank's bits in its own
range merge into the oracle's admits for all G groups, every slot is that rank's admit bitmap, bits past G and words
past the table's words are 0.  The lane map is reported, not compared (a shard's requests may choose another gang_fit
shape than the whole table's).

Two exchange rules are tested on their own:
- a group table that grows past 32 * words_per_rank after bs_peer_init makes bs_evaluate_async refuse the round on
  every rank (its admits could not all travel), and a smaller table still works with its tail words 0;
- after bs_peer_detach, bs_peer_attach with the old handles and no bs_peer_init starts a new epoch: the first round's
  gathered words are that round's, not the previous epoch's, even for a rank that fetches before its peers arrive.

On a one-GPU box all ranks share cuda:0 (CUDA IPC maps a buffer of another process on the same device, the contexts
time-slice) and the handles travel over gloo; with at least `world` GPUs every rank has its own."""
import os
import pickle
import socket
import sys
import time

import numpy as np
import pytest

import shard_cases as sc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAD = 2   # words_per_rank beyond the table's words: the push's zero fill runs in every round
H1_MESSAGE = ("bs_evaluate: the group table needs 4 admit-bitmap words per rank, but the peer exchange carries 3 "
              "(bs_peer_init with words_per_rank >= 4)")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _setup(rank, world, port, shared_gpu):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import datetime
    import importlib
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = 0 if shared_gpu else rank
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    pkg = importlib.import_module("batch-scheduler_b200")
    return pkg, dist, dev


def _ag(dist, world, obj):
    out = [None] * world
    dist.all_gather_object(out, obj)
    return out


def _engine(pkg, dev, cfg):
    return pkg.Engine(sc.L, dev, fit_bitmap=cfg.get("fit_bitmap", False), score=cfg.get("score", False),
                      filter=cfg.get("filter", False), topk=cfg.get("topk", 0), reasons=cfg.get("reasons", False),
                      priority_k=cfg.get("priority_k", 0))


def _load(eng, m):
    """Every table, side column, both filters' halves and switches, and every weight of the Model m."""
    import test_gpu_engine_sequences as seq
    eng.upload_nodes(m.nodes)
    eng.upload_affinity(m.aff)
    eng.upload_groups(m.groups)
    eng.upload_pods(m.pods)
    for key, cols in m.side.items():
        name, half = key.split("_")
        seq._side(eng, {"name": name, "half": half, "cols": cols})
    eng.upload_interpod_filter(node=m.ipf_node)
    eng.upload_interpod_filter(pods=m.ipf_pod)
    eng.set_interpod_filter(m.ipf_on)
    eng.upload_host_ports(node=m.hp_node, pods=m.hp_pod)
    eng.set_host_port_filter(m.hp_on)
    seq._weights(eng, m.lanes, dict(weights=m.weights, ratio=m.ratio, pw=m.pw, lw=m.lw, w_spread=m.w_spread,
                                    w_ipa=m.w_ipa))


def _gather_diff(words, bitmaps, admit, ranges, G):
    """The first rule the gathered words [world, wpr] break: bitmaps are every rank's own admit bitmap, admit the
    oracle's admits of all G groups."""
    nw = (G + 31) // 32
    merged = np.zeros(G, bool)
    for r, (a0, a1) in enumerate(ranges):
        merged[a0:a1] = sc.admit_bits(words[r], G)[a0:a1]
    want = np.asarray(admit) == sc.S.ADMIT
    if not np.array_equal(merged, want):
        return f"gathered admits: groups {np.flatnonzero(merged != want)[:6].tolist()} differ from the oracle"
    for r, bm in enumerate(bitmaps):
        if not np.array_equal(words[r, :nw], np.asarray(bm)[:nw]):
            return f"rank {r}'s slot is not its admit bitmap: words {np.flatnonzero(words[r, :nw] != bm[:nw])[:6].tolist()}"
    if (words[:, nw:] != 0).any():
        return f"words past the table's {nw} are not 0"
    if G % 32 and (words[:, nw - 1] >> np.uint32(G % 32)).any():
        return f"bits past G = {G} in the last word are not 0"
    return None


def _worker(rank, world, port, data_path, out_dir, shared_gpu):
    pkg, dist, dev = _setup(rank, world, port, shared_gpu)
    import test_gpu_engine_sequences as seq
    with open(data_path, "rb") as f:
        data = pickle.load(f)
    report = []
    for name in sc.CASES:
        d = data[name]
        m = d["model"]
        s, idx, (g0, g1) = sc.shard(m, rank, world)
        ranges = [sc.shard(m, r, world)[2] for r in range(world)]
        G = m.groups.n
        for cfg_name in sorted(seq.CONFIGS):
            cfg = seq.CONFIGS[cfg_name]
            eng = _engine(pkg, dev, cfg)
            try:
                _load(eng, s)
                eng.peer_setup(rank, world, (G + 31) // 32 + PAD, lambda b: _ag(dist, world, b))
                dist.barrier()
                for k in range(sc.ROUNDS):
                    if k:
                        eng.update_groups(*d["updates"][k - 1])
                    got = seq._round(eng, cfg, ("async", "evaluate", "view")[k % 3])
                    lanes = got.pop("lanes")
                    words = eng.gathered_admit()
                    bitmaps = _ag(dist, world, np.asarray(got["admit_bitmap"]))
                    err = sc.first_diff(d["refs"][k], got, idx, g0, g1, d["idle"][k]) or \
                        _gather_diff(words, bitmaps, d["refs"][k]["admit"], ranges, G)
                    assert err is None, f"world {world} rank {rank} case {name} config {cfg_name} round {k}: {err}"
                    report.append(f"world {world} rank {rank} case {name:12s} config {cfg_name:29s} round {k}: "
                                  f"P={len(idx)} groups [{g0}, {g1}) of {G}, lanes kind {lanes[0].tolist()} "
                                  f"unit {lanes[1].tolist()}: every output and the gathered bitmap exact")
                dist.barrier()
                eng.peer_detach()
            finally:
                eng.close()
    with open(os.path.join(out_dir, f"rank{rank}"), "w") as f:
        f.write("\n".join(report) + "\n")
    dist.barrier()
    dist.destroy_process_group()


def _prepare(tmp_path):
    data = {}
    for name in sc.CASES:
        m = sc.case(name)
        ups = sc.group_updates(m)
        refs, idle, cur = [], [], m
        for k in range(sc.ROUNDS):
            if k:
                cur = sc.updated(cur, ups[k - 1])
            refs.append(cur.expect(sc.EVERY_OUTPUT))
            idle.append(sc.idle_groups(cur))
        data[name] = {"model": m, "updates": ups, "refs": refs, "idle": idle}
    path = os.path.join(str(tmp_path), "cases.pkl")
    with open(path, "wb") as f:
        pickle.dump(data, f)
    return path


def _spawn(fn, world, *args):
    import torch
    import torch.multiprocessing as mp
    shared = torch.cuda.device_count() < world
    mp.spawn(fn, args=(world, _free_port(), *args, shared), nprocs=world, join=True)
    return shared


@pytest.mark.parametrize("world", sc.WORLDS)
def test_every_rank_every_output(tmp_path, oracle, world):
    path = _prepare(tmp_path)
    shared = _spawn(_worker, world, path, str(tmp_path))
    print(f"\nworld {world} ({'all ranks on cuda:0' if shared else 'one GPU per rank'}):")
    for r in range(world):
        print(open(os.path.join(str(tmp_path), f"rank{r}")).read(), end="")


# ---- the two exchange rules -----------------------------------------------------------------------------------------

def _h1_worker(rank, world, port, data_path, out_dir, shared_gpu):
    """A group table past 32 * words_per_rank is refused on every rank; a smaller one still works."""
    pkg, dist, dev = _setup(rank, world, port, shared_gpu)
    with open(data_path, "rb") as f:
        d = pickle.load(f)
    m = d["model"]
    s, idx, (g0, g1) = sc.shard(m, rank, world)
    ranges = [sc.shard(m, r, world)[2] for r in range(world)]
    G = m.groups.n
    eng = pkg.Engine(sc.L, dev, fit_bitmap=False, score=False)
    try:
        eng.upload(sc.S.Snapshot(s.nodes, s.pods, s.groups, aff_bits=s.aff))
        eng.peer_setup(rank, world, (G + 31) // 32, lambda b: _ag(dist, world, b))
        dist.barrier()
        eng.evaluate_async()
        eng.sync()
        res = eng.fetch()
        err = _gather_diff(eng.gathered_admit(), _ag(dist, world, res.admit_bitmap), d["admit"], ranges, G)
        assert err is None, f"rank {rank}, the table of {G} groups: {err}"

        big = d["big"]
        eng.upload_groups(big)
        try:
            eng.evaluate_async()
            eng.sync()
            words, res = eng.gathered_admit(), eng.fetch()
            mine = sc.admit_bits(res.admit_bitmap, big.n)
            sent = np.zeros(big.n, bool)
            carried = sc.admit_bits(words[rank], 32 * words.shape[1])
            sent[:len(carried)] = carried
            lost = np.flatnonzero(mine & ~sent)
            outcome = (None, f"the round succeeded; {len(lost)} admitted groups of this rank's bitmap are missing from "
                             f"its gathered slot (groups {lost[:5].tolist()}...)")
        except pkg.capi.BsError as ex:
            outcome = (ex.code, str(ex))
        outcomes = _ag(dist, world, outcome)
        for r, (code, msg) in enumerate(outcomes):
            assert code == pkg.capi.BS_E_STATE, f"rank {r}, a table of {big.n} groups over 3 words per rank: {msg}"
            assert msg.endswith(H1_MESSAGE), f"rank {r}: {msg!r}"

        small = d["small"]
        eng.upload_groups(small)
        eng.evaluate_async()
        eng.sync()
        words, res = eng.gathered_admit(), eng.fetch()
        bitmaps = _ag(dist, world, res.admit_bitmap)
        nw = (small.n + 31) // 32
        for r, bm in enumerate(bitmaps):
            assert np.array_equal(words[r, :nw], bm[:nw]), f"rank {rank}: rank {r}'s slot is not its bitmap"
        assert (words[:, nw:] == 0).all(), f"rank {rank}: words past {nw} are not 0 with {small.n} groups"
        assert not (words[:, nw - 1] >> np.uint32(small.n % 32)).any(), f"rank {rank}: bits past {small.n} are not 0"

        eng.upload_groups(m.groups)   # and the table of the start again
        eng.evaluate_async()
        eng.sync()
        res = eng.fetch()
        err = _gather_diff(eng.gathered_admit(), _ag(dist, world, res.admit_bitmap), d["admit"], ranges, G)
        assert err is None, f"rank {rank}, the table of {G} groups again: {err}"
        dist.barrier()
        eng.peer_detach()
    finally:
        eng.close()
    if rank == 0:
        open(os.path.join(out_dir, "ok_h1"), "w").write("ok")
    dist.barrier()
    dist.destroy_process_group()


def _plain_tail():
    """Case tail with the filters off: these engines load the tables only."""
    m = sc.case("tail")
    m.ipf_on = m.ipf_round = m.hp_on = m.hp_round = False
    return m


def test_group_table_past_words_per_rank_is_refused(tmp_path, oracle):
    m = _plain_tail()
    assert m.groups.n == 77   # 3 words; 117 groups need 4, 40 need 2
    big = _concat(m.groups, m.groups.take(np.arange(40)))
    small = m.groups.take(np.arange(40))
    path = os.path.join(str(tmp_path), "h1.pkl")
    with open(path, "wb") as f:
        pickle.dump({"model": m, "big": big, "small": small, "admit": m.expect({})["admit"]}, f)
    _spawn(_h1_worker, 2, path, str(tmp_path))
    assert os.path.exists(os.path.join(str(tmp_path), "ok_h1"))


def _concat(a, b):
    return type(a)(*(None if getattr(a, f) is None else np.concatenate([getattr(a, f), getattr(b, f)], axis=-1)
                     for f in a.__dataclass_fields__))


def _h2_worker(rank, world, port, data_path, out_dir, shared_gpu):
    """A new epoch by bs_peer_detach and bs_peer_attach with the old handles, without bs_peer_init."""
    import ctypes as C
    pkg, dist, dev = _setup(rank, world, port, shared_gpu)
    with open(data_path, "rb") as f:
        d = pickle.load(f)
    m = d["model"]
    s, idx, (g0, g1) = sc.shard(m, rank, world)
    ranges = [sc.shard(m, r, world)[2] for r in range(world)]
    G = m.groups.n
    wpr = (G + 31) // 32
    eng = pkg.Engine(sc.L, dev, fit_bitmap=False, score=False)
    try:
        eng.upload(sc.S.Snapshot(s.nodes, s.pods, s.groups, aff_bits=s.aff))
        # Engine.peer_setup, keeping the handle blob
        eng._check(eng.lib.bs_peer_init(eng.h, rank, world, wpr))
        buf = (C.c_ubyte * 64)()
        eng._check(eng.lib.bs_peer_handle(eng.h, buf))
        blob = (C.c_ubyte * (64 * world)).from_buffer_copy(b"".join(_ag(dist, world, bytes(buf))))
        eng._check(eng.lib.bs_peer_attach(eng.h, blob))
        eng.peer_world, eng.peer_wpr = world, wpr
        dist.barrier()
        for _ in range(3):   # the last round is odd: its flags are the ones round 1 of the next epoch waits on
            eng.evaluate_async()
        eng.sync()
        res = eng.fetch()
        err = _gather_diff(eng.gathered_admit(), _ag(dist, world, res.admit_bitmap), d["admit"], ranges, G)
        assert err is None, f"rank {rank}, the first epoch: {err}"
        dist.barrier()
        eng.peer_detach()
        dist.barrier()

        eng.upload_groups(d["groups2"])
        eng._check(eng.lib.bs_peer_attach(eng.h, blob))
        dist.barrier()
        if rank == 0:
            eng.evaluate_async()
            early = eng.gathered_admit()   # before the others have evaluated
            want = np.asarray(d["admit2"]) == sc.S.ADMIT
            old = np.asarray(d["admit"]) == sc.S.ADMIT
            for r, (a0, a1) in enumerate(ranges):
                got = sc.admit_bits(early[r], G)[a0:a1]
                stale = "the previous epoch's" if np.array_equal(got, old[a0:a1]) else "neither round's"
                assert np.array_equal(got, want[a0:a1]), \
                    f"rank 0 fetched before its peers arrived and read {stale} words in rank {r}'s slot"
        else:
            time.sleep(0.3)
            eng.evaluate_async()
        eng.sync()
        res = eng.fetch()
        bitmaps = _ag(dist, world, res.admit_bitmap)   # every rank has evaluated
        err = _gather_diff(eng.gathered_admit(), bitmaps, d["admit2"], ranges, G)
        assert err is None, f"rank {rank}, the second epoch after every rank arrived: {err}"
        dist.barrier()
        eng.peer_detach()
    finally:
        eng.close()
    if rank == 0:
        open(os.path.join(out_dir, "ok_h2"), "w").write("ok")
    dist.barrier()
    dist.destroy_process_group()


def test_reattach_without_init_starts_a_new_epoch(tmp_path, oracle):
    world = 3
    m = _plain_tail()
    r0 = m.expect({})
    g2 = m.groups.copy()   # every group flipped: admitted ones wait for 1000 members, the others are fully matched
    admitted = r0["admit"] == sc.S.ADMIT
    g2.min_member = np.where(admitted, 1000, g2.min_member).astype(np.uint32)
    g2.matched = np.where(admitted, 0, g2.min_member).astype(np.uint32)
    g2.scheduled[:] = 0
    m2 = sc.with_groups(m, g2)
    r2 = m2.expect({})
    for r in range(world):   # a stale slot is visible in every rank's range
        a0, a1 = sc.shard(m, r, world)[2]
        assert not np.array_equal(r0["admit"][a0:a1] == sc.S.ADMIT, r2["admit"][a0:a1] == sc.S.ADMIT), r
    path = os.path.join(str(tmp_path), "h2.pkl")
    with open(path, "wb") as f:
        pickle.dump({"model": m, "admit": r0["admit"], "groups2": g2, "admit2": r2["admit"]}, f)
    _spawn(_h2_worker, world, path, str(tmp_path))
    assert os.path.exists(os.path.join(str(tmp_path), "ok_h2"))
