"""TEST INFRASTRUCTURE — seeded objects for the InterPodAffinity tests: node labels, pending pods and bound pods with
pod-affinity terms of every kind, matched to the rows of a random snapshot (pending pod p is the table's pod p, label
set n the table's node n)."""
import numpy as np

import pyref_interpod_priority as pyi

HOST, ZONE, RACK = "kubernetes.io/hostname", "failure-domain.beta.kubernetes.io/zone", "rack"
NAMESPACES = ("a", "b", "c")
APPS = ("web", "db", "cache", "batch")


def node_labels(rng, N, n_zones=3, rack_size=4, unlabelled=0.15):
    out = []
    for n in range(N):
        lab = {HOST: f"node-{n}"}
        if rng.random() >= unlabelled:
            lab[ZONE] = f"zone-{rng.integers(n_zones)}"
        if rng.random() >= unlabelled:
            lab[RACK] = f"rack-{n // rack_size}"
        out.append(lab)
    return out


def random_selector(rng, invalid=0.0):
    r = rng.random()
    if r < 0.1:
        return None
    if r < 0.2:
        return pyi.Selector()
    sel = pyi.Selector()
    if rng.random() < 0.7:
        sel.match_labels["app"] = str(rng.choice(APPS))
    if rng.random() < 0.4:
        op = str(rng.choice(["In", "NotIn", "Exists", "DoesNotExist"]))
        vals = [str(v) for v in rng.choice(["x", "y"], int(rng.integers(1, 3)))] if op in ("In", "NotIn") else []
        sel.match_expressions.append(("tier", op, vals))
    if rng.random() < invalid:
        sel.match_expressions.append(("tier", "In", []))   # fails LabelSelectorAsSelector
    return sel


def random_term(rng, invalid=0.0):
    ns = () if rng.random() < 0.6 else tuple(rng.choice(NAMESPACES, int(rng.integers(1, 3)), replace=False).tolist())
    key = str(rng.choice([HOST, ZONE, ZONE, RACK, ""] if rng.random() < 0.05 else [HOST, ZONE, ZONE, RACK]))
    return pyi.Term(random_selector(rng, invalid), ns, key)


def random_pod(rng, node=None, max_terms=3, invalid=0.0, no_terms=0.3):
    pod = pyi.PodObj(namespace=str(rng.choice(NAMESPACES)), node=node, terminating=bool(rng.random() < 0.1))
    pod.labels = {"app": str(rng.choice(APPS))}
    if rng.random() < 0.5:
        pod.labels["tier"] = str(rng.choice(["x", "y", "z"]))
    if rng.random() < no_terms:
        return pod
    for _ in range(int(rng.integers(0, max_terms + 1))):
        kind = int(rng.integers(0, 3))
        t = random_term(rng, invalid)
        w = int(rng.integers(1, 101))
        if kind == 0:
            pod.required.append(t)
        elif kind == 1:
            pod.preferred.append((w, t))
        else:
            pod.anti.append((w, t))
    return pod


def random_objects(seed, N, P, per_node=3, invalid=0.0, **kw):
    """(pending [P], bound, labels [N]): bound pods in node order, about per_node per node."""
    rng = np.random.default_rng(seed)
    labels = node_labels(rng, N, **kw)
    bound = [random_pod(rng, node=n, invalid=invalid) for n in range(N) for _ in range(int(rng.integers(0, 2 * per_node + 1)))]
    pending = [random_pod(rng, invalid=invalid) for _ in range(P)]
    return pending, bound, labels


def columns(pending, bound, labels, hard=1):
    """((node side), (pod side)) for Engine.upload_interpod and interpod_priority_ref, packed by pyref's rules."""
    pk = pyi.pack(pending, bound, labels, hard)
    return pk["node"], pk["pods"]
