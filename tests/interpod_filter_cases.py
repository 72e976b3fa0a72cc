"""TEST INFRASTRUCTURE — hand-built MatchInterPodAffinity cases with their answers written out.

Each case: (name, nodes {name: labels} in order, existing pods, pending pods, answers {pending pod: verdict per node}),
a verdict being "" (passes), "E", "A" or "N" (the step of include/bsched.h bs_set_interpod_filter that fails it).
"""
from pyref_interpod_filter import INVALID, Pod, Term

H = "kubernetes.io/hostname"
Z = "zone"


def _nodes(*zones):
    """n0, n1, ... with a hostname label and the given zone (None: no zone label)."""
    out = {}
    for i, z in enumerate(zones):
        lab = {H: f"n{i}"}
        if z is not None:
            lab[Z] = z
        out[f"n{i}"] = lab
    return out


def _worker(name, job, ns="default", **kw):
    return Pod(name, ns, {"job": job}, **kw)


CASES = [
    # one worker per host: a sibling is bound on n1
    ("one-per-host", _nodes("a", "a", "b"),
     [_worker("w0", "j", node="n1")],
     [_worker("w1", "j", anti=[Term({"job": "j"}, H)])],
     {"w1": ["", "N", ""]}),
    # zone affinity: the parameter server is bound in zone b
    ("ps-zone", _nodes("a", "b", "b", None),
     [Pod("ps", labels={"role": "ps", "job": "j"}, node="n2")],
     [_worker("w", "j", affinity=[Term({"role": "ps", "job": "j"}, Z)])],
     {"w": ["A", "", "", "A"]}),
    # the first-pod exception with self-match: no pod matches the set anywhere, the pod matches it itself
    ("first-pod-self", _nodes("a", "b"),
     [Pod("other", labels={"app": "x"}, node="n0")],
     [_worker("w", "j", affinity=[Term({"job": "j"}, Z)])],
     {"w": ["", ""]}),
    # ... and without self-match: the exception does not apply
    ("first-pod-noself", _nodes("a", "b"),
     [],
     [_worker("w", "j", affinity=[Term({"role": "ps"}, Z)])],
     {"w": ["A", "A"]}),
    # the exception needs an empty pair map: a matching pod on a node with the key exists in zone a
    ("first-pod-map-not-empty", _nodes("a", "b"),
     [_worker("s", "j", node="n0")],
     [_worker("w", "j", affinity=[Term({"job": "j"}, Z)])],
     {"w": ["", "A"]}),
    # a matching pod only on a node without the key leaves the map empty: the exception applies
    ("first-pod-unkeyed", _nodes(None, "b"),
     [_worker("s", "j", node="n0")],
     [_worker("w", "j", affinity=[Term({"job": "j"}, Z)])],
     {"w": ["", ""]}),
    # a two-term set: only pods that match both terms count (p1 matches one term only, in zone a)
    ("two-term-set", _nodes("a", "b", "c"),
     [Pod("p1", labels={"role": "ps"}, node="n0"), Pod("p2", labels={"role": "ps", "tier": "1"}, node="n1")],
     [Pod("w", affinity=[Term({"role": "ps"}, Z), Term({"tier": "1"}, Z)])],
     {"w": ["A", "", "A"]}),
    # a bound pod's anti-affinity blocks its whole zone for a pod without affinity of its own
    ("existing-blocks-zone", _nodes("a", "a", "b", None),
     [Pod("guard", labels={"app": "g"}, node="n0", anti=[Term({"app": "x"}, Z)])],
     [Pod("x", labels={"app": "x"}), Pod("y", labels={"app": "y"})],
     {"x": ["E", "E", "", ""], "y": ["", "", "", ""]}),
    # nodes without the key in each role: existing anti (passes), affinity (fails), anti (passes)
    ("unkeyed-nodes", _nodes(None, "a"),
     [Pod("guard", labels={"app": "g", "job": "j"}, node="n1", anti=[Term({"app": "x"}, Z)])],
     [Pod("x", labels={"app": "x"}), _worker("aff", "k", affinity=[Term({"app": "g"}, Z)]),
      _worker("anti", "k", anti=[Term({"app": "g"}, Z)])],
     {"x": ["", "E"], "aff": ["A", ""], "anti": ["", "N"]}),
    # namespaces: an empty list is the defining pod's namespace, a listed one is taken as listed
    ("namespaces", _nodes("a", "b"),
     [Pod("e1", "other", {"app": "db"}, node="n0"), Pod("e2", "default", {"app": "db"}, node="n1")],
     [Pod("same", "default", anti=[Term({"app": "db"}, Z)]),
      Pod("listed", "default", anti=[Term({"app": "db"}, Z, ["other"])])],
     {"same": ["", "N"], "listed": ["N", ""]}),
    # selectors: nil matches nothing, empty matches everything, invalid matches nothing
    ("selectors", _nodes("a", "b"),
     [Pod("e", labels={"app": "db"}, node="n0")],
     [Pod("nil", anti=[Term(None, Z)]), Pod("empty", anti=[Term({}, Z)]), Pod("invalid", anti=[Term(INVALID, Z)]),
      Pod("nil-aff", affinity=[Term(None, Z)])],
     {"nil": ["", ""], "empty": ["N", ""], "invalid": ["", ""], "nil-aff": ["A", "A"]}),
    # a terminating bound pod still counts
    ("terminating", _nodes("a", "b"),
     [_worker("w0", "j", node="n0", terminating=True)],
     [_worker("w1", "j", anti=[Term({"job": "j"}, Z)])],
     {"w1": ["N", ""]}),
    # two terms on one key: the affinity set needs both, an anti term on the same key
    ("two-terms-one-key", _nodes("a", "b", "c"),
     [Pod("p", labels={"role": "ps", "tier": "1"}, node="n0"), Pod("q", labels={"app": "q"}, node="n1")],
     [Pod("w", affinity=[Term({"role": "ps"}, Z), Term({"tier": "1"}, Z)], anti=[Term({"app": "q"}, Z)]),
      Pod("v", anti=[Term({"app": "q"}, Z), Term({"role": "ps"}, Z)])],
     {"w": ["", "A", "A"], "v": ["N", "N", ""]}),
    # an empty topologyKey: no node carries it; in an affinity set it fails the term, the exception still applies
    ("empty-key", _nodes("a", "b"),
     [Pod("e", labels={"app": "db"}, node="n0")],
     [Pod("aff", affinity=[Term({"app": "db"}, "")]), Pod("self", labels={"app": "s"}, affinity=[Term({"app": "s"}, "")]),
      Pod("anti", anti=[Term({"app": "db"}, "")])],
     {"aff": ["A", "A"], "self": ["", ""], "anti": ["", ""]}),
    # existing anti-affinity comes first: a node failing both steps reports E
    ("order", _nodes("a", "b"),
     [Pod("guard", labels={"app": "g"}, node="n0", anti=[Term({"job": "j"}, Z)]), _worker("s", "j", node="n0")],
     [_worker("w", "j", anti=[Term({"job": "j"}, Z)])],
     {"w": ["E", ""]}),
]

# The message of a reason row with two "Insufficient cpu" nodes and the companion (E, A, N) = (1, 2, 0), 6 nodes:
# the entries sorted as whole strings.
MESSAGE_ROW = ([0, 0, 0, 0, 2, 0, 0, 0], (1, 2, 0), 6)
MESSAGE = ("0/6 nodes are available: 1 node(s) didn't satisfy existing pods anti-affinity rules, "
           "2 Insufficient cpu, 2 node(s) didn't match pod affinity rules, "
           "3 node(s) didn't match pod affinity/anti-affinity.")
