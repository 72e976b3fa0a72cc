"""TEST INFRASTRUCTURE — designed PodFitsHostPorts cases: (name, node used ports, pod wanted ports, passes).

Each case is one pod against one node; the verdict is what kube-scheduler v1.17's HostPortInfo.CheckConflict gives
[upstream, from memory].
"""
from pyref_host_ports import Port as P

CASES = [
    ("same wildcard both sides", [P(8080)], [P(8080)], False),
    ("wildcard used, specific wanted", [P(8080, "0.0.0.0")], [P(8080, "10.0.0.1")], False),
    ("specific used, wildcard wanted", [P(8080, "10.0.0.1")], [P(8080)], False),
    ("empty ip is the wildcard", [P(8080, "10.0.0.1")], [P(8080, "")], False),
    ("two different specific ips", [P(8080, "10.0.0.1")], [P(8080, "10.0.0.2")], True),
    ("the same specific ip", [P(8080, "10.0.0.1")], [P(8080, "10.0.0.1")], False),
    ("same port over TCP and UDP", [P(53, protocol="UDP")], [P(53, protocol="TCP")], True),
    ("same port, both UDP", [P(53, protocol="UDP")], [P(53, protocol="UDP")], False),
    ("empty protocol is TCP", [P(22, protocol="TCP")], [P(22)], False),
    ("empty protocol is not UDP", [P(22, protocol="UDP")], [P(22)], True),
    ("'::' is not a wildcard", [P(9000, "::")], [P(9000, "10.0.0.1")], True),
    ("'::' against the wildcard", [P(9000, "::")], [P(9000)], False),
    ("port 0 is ignored on the pod", [P(0)], [P(0)], True),
    ("a container port without a host port", [P(0, container_port=80)], [P(0, container_port=80)], True),
    ("negative ports are ignored", [P(-1)], [P(-1)], True),
    ("different ports", [P(8080)], [P(8081)], True),
    ("a pod's own duplicates", [], [P(7000), P(7000)], True),
    ("duplicates against a used port", [P(7000, "10.0.0.3")], [P(7000), P(7000, "0.0.0.0")], False),
    ("one of several wanted conflicts", [P(1, protocol="SCTP")], [P(2), P(1, protocol="SCTP"), P(3)], False),
    ("no wanted ports", [P(8080)], [], True),
]
