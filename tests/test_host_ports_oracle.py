"""CPU: the two restatements of kube-scheduler v1.17's PodFitsHostPorts predicate agree — tests/pyref_host_ports.py
over the objects and tests/host_ports_ref.c over the packed columns — on the designed cases and on random ones; the
packer's dictionary limits; and the FailedScheduling text of bs_format_fit_error_filters."""
import numpy as np
import pytest

import host_port_cases as cases
import host_ports_ref as hr
import pyref_host_ports as py
from pyref_host_ports import Port


@pytest.mark.parametrize("name,used,wanted,passes", cases.CASES, ids=[c[0] for c in cases.CASES])
def test_designed_cases(name, used, wanted, passes):
    pod, node = py.Pod("p", wanted), py.Node("n", used)
    assert py.verdict(pod, node) == passes
    entries, u, w = py.pack([node], [pod])
    assert hr.passes(entries, u, w).tolist() == [[passes]]


def test_random_objects():
    rng = np.random.default_rng(7)
    ips = ["", "0.0.0.0", "10.0.0.1", "10.0.0.2", "::"]
    protos = ["", "TCP", "UDP", "SCTP"]

    def ports(k):
        return [Port(int(rng.choice([-1, 0, 80, 81, 443])), str(rng.choice(ips)), str(rng.choice(protos)))
                for _ in range(k)]
    for _ in range(30):
        nodes = [py.Node(f"n{i}", ports(int(rng.integers(0, 4)))) for i in range(int(rng.integers(1, 12)))]
        pods = [py.Pod(f"p{i}", ports(int(rng.integers(0, 3)))) for i in range(int(rng.integers(1, 12)))]
        entries, used, want = py.pack(nodes, pods)
        np.testing.assert_array_equal(hr.passes(entries, used, want), py.verdicts(pods, nodes))


def test_dictionary_order_and_pruning():
    nodes = [py.Node("a", [Port(22, "10.0.0.9"), Port(5000)]), py.Node("b", [Port(8080, "10.0.0.2")])]
    pods = [py.Pod("x", [Port(8080, "10.0.0.1"), Port(22)]), py.Pod("y", [Port(22), Port(53, protocol="UDP")])]
    entries, used, want = py.pack(nodes, pods)
    # the pods' triples in order of first appearance, then the node triple that conflicts (22 on 10.0.0.9); 5000 and
    # 8080 on 10.0.0.2 conflict with nothing wanted and are left out
    assert entries.tolist() == [[1, 0, 8080], [0, 0, 22], [0, 1, 53], [2, 0, 22]]
    assert used.tolist() == [0b1000, 0] and want.tolist() == [0b011, 0b110]


def test_dictionary_limit():
    pods = [py.Pod("p", [Port(1000 + k) for k in range(64)])]
    entries, _, want = py.pack([], pods)
    assert len(entries) == 64 and int(want[0]) == (1 << 64) - 1
    with pytest.raises(ValueError):
        py.pack([], [py.Pod("p", [Port(1000 + k) for k in range(65)])])


def _fmt(pkg, row, L, n, **kw):
    return pkg.engine.format_fit_error(row, L, n, **kw)


def test_format_text_and_sort(pkg):
    row = [0, 0, 9, 0, 0, 0, 0, 0]
    msg = _fmt(pkg, row, 4, 30, host_ports=[10])
    # byte-wise sort: "10 ..." before "9 ..."
    assert msg == ("0/30 nodes are available: 10 node(s) didn't have free ports for the requested pod ports, "
                   "9 node(s) didn't match node selector.")
    both = _fmt(pkg, row, 4, 30, interpod=(2, 0, 0), host_ports=[10])
    assert both == ("0/30 nodes are available: 10 node(s) didn't have free ports for the requested pod ports, "
                    "2 node(s) didn't match pod affinity/anti-affinity, "
                    "2 node(s) didn't satisfy existing pods anti-affinity rules, "
                    "9 node(s) didn't match node selector.")
    # a zero count, or no companion, is the message without the entry; the inter-pod one is unchanged
    plain = _fmt(pkg, row, 4, 30)
    assert _fmt(pkg, row, 4, 30, host_ports=[0]) == plain
    assert _fmt(pkg, row, 4, 30, interpod=(2, 0, 0), host_ports=[0]) == _fmt(pkg, row, 4, 30, interpod=(2, 0, 0))
    with pytest.raises(ValueError):
        _fmt(pkg, row, 4, 30, host_ports=[1, 2])


def test_hooked_walk():
    # with no wanted ports the hooked walk is the first-fit walk; with them every placement is free of conflicts on the
    # live masks, and the live masks are the uploaded ones ORed with the placed pods' want masks
    import replay_priority_ref as rpr
    from randsnap import random_snapshot
    snap = random_snapshot(11, P=150, N=120, G=20, L=5, case="mixed")
    cols = hr.random_columns(snap, 3, grouped=0.6, node_bits=1)
    (entries, used), want = cols
    none = hr.replay(snap, ((entries, used), np.zeros_like(want)))
    ff = rpr.replay_first_fit(snap)
    for a, b in zip(none[:3], ff[:3]):
        np.testing.assert_array_equal(a, b)
    pf, node, ready, _, live, _ = hr.replay(snap, cols)
    mask = np.array(used, np.uint64)
    for p, n in enumerate(node):
        if pf[p] == 0 and n >= 0:
            assert hr.passes(entries, mask[n:n + 1], want[p:p + 1])[0, 0]
            mask[n] |= np.uint64(want[p])
    np.testing.assert_array_equal(mask, live)
    assert (node != none[1]).any()
