"""TEST INFRASTRUCTURE — kube-scheduler v1.17's PodFitsHostPorts predicate restated from objects [upstream, from
memory], and a packer from the objects to the engine's columns (include/bsched.h bs_upload_node_host_ports,
bs_upload_pod_host_ports).

verdict() follows HostPortInfo: Add and CheckConflict drop port <= 0, sanitize an empty HostIP to "0.0.0.0" and an
empty protocol to "TCP", and a wanted (ip, protocol, port) conflicts with a used one of the same protocol and port when
either ip is "0.0.0.0" or the ips are equal as strings.  pack() resolves the same objects into the dictionary, the used
masks and the want masks; tests/host_ports_ref.c over those columns and verdict() here must agree.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

ANY = "0.0.0.0"
MAX_ENTRIES = 64


@dataclass
class Port:
    host_port: int
    host_ip: str = ""
    protocol: str = ""
    container_port: int = 0   # not read by the predicate: the API defaults hostPort from it under hostNetwork


@dataclass
class Pod:
    name: str
    ports: list = field(default_factory=list)        # the containers' ports, flattened (init containers excluded)


@dataclass
class Node:
    name: str
    used: list = field(default_factory=list)         # NodeInfo.UsedPorts(), flattened as Port objects


def _sanitize(p: Port):
    return (p.host_ip or ANY, p.protocol or "TCP", p.host_port)


def triples(ports) -> list:
    """The sanitized (ip, protocol, port) set of a port list in order of first appearance, port <= 0 dropped."""
    out = []
    for p in ports:
        if p.host_port <= 0:
            continue
        t = _sanitize(p)
        if t not in out:
            out.append(t)
    return out


def conflict(w, u) -> bool:
    return w[1] == u[1] and w[2] == u[2] and (w[0] == ANY or u[0] == ANY or w[0] == u[0])


def verdict(pod: Pod, node: Node) -> bool:
    """True when the pod passes PodFitsHostPorts on the node."""
    used = triples(node.used)
    return not any(conflict(w, u) for w in triples(pod.ports) for u in used)


def verdicts(pods, nodes) -> np.ndarray:
    return np.array([[verdict(p, n) for n in nodes] for p in pods], bool).reshape(len(pods), len(nodes))


def pack(nodes, pods):
    """(entries [K, 3] int64 (ip id, protocol id, port), used [N] uint64, want [P] uint64).  The dictionary holds the
    pods' wanted triples in order of first appearance, then the nodes' used triples that conflict with any of them
    (a used triple that conflicts with nothing never decides a verdict).  Ip id 0 is "0.0.0.0"; the other ips and the
    protocols are numbered by first appearance.  More than MAX_ENTRIES entries is a ValueError."""
    dic = []
    for p in pods:
        for t in triples(p.ports):
            if t not in dic:
                dic.append(t)
    wanted = list(dic)
    for n in nodes:
        for t in triples(n.used):
            if t not in dic and any(conflict(w, t) for w in wanted):
                dic.append(t)
    if len(dic) > MAX_ENTRIES:
        raise ValueError(f"{len(dic)} host-port entries, more than {MAX_ENTRIES}")
    ips, protos = {ANY: 0}, {}
    entries = np.array([(ips.setdefault(ip, len(ips)), protos.setdefault(pr, len(protos)), port)
                        for ip, pr, port in dic], np.int64).reshape(-1, 3)
    index = {t: k for k, t in enumerate(dic)}

    def mask(ts):
        m = 0
        for t in ts:
            if t in index:
                m |= 1 << index[t]
        return m
    used = np.array([mask(triples(n.used)) for n in nodes], np.uint64)
    want = np.array([mask(triples(p.ports)) for p in pods], np.uint64)
    return entries, used, want
