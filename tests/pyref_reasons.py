"""A second, independent restatement of the reason rows (include/bsched.h BS_OUT_REASONS) in pure Python over the
Go-like objects of tests/pyref.py (dict-based ScalarResources, explicit loops), written from core.go without looking
at the C restatement.  Used to cross-check tests/fit_reasons_ref.c on small cases."""
import numpy as np

from pyref import M64, Node, resource_from, single_node_resource


def fit_reasons(snap):
    """[P, 4 + L] reason rows: per pod and node, the guards in the order of core.go:606-617 and :639, then checkFit's
    two predicates (:741-759; a required node-affinity class is part of the selector predicate), then every lane of
    compareResourceAndRequire (:672-699) that fails against singleNodeResource at percent 1.0 (:634-670)."""
    nt, pt = snap.nodes, snap.pods
    L = nt.lanes
    nodes = [Node(nt, i) for i in range(nt.n)]
    aff_bits = getattr(snap, "aff_bits", None)
    aff_class = getattr(pt, "aff_class", None)
    out = np.zeros((pt.n, 4 + L), np.uint32)
    for p in range(pt.n):
        sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
        aff = 0xFFFFFFFF if aff_class is None else int(aff_class[p])
        req = resource_from(pt.req[:, p], int(pt.req_present[p]), L)
        for i, node in enumerate(nodes):
            if node.flags & 0x01 or node.flags & 0x02:      # nil info, nil Node()
                out[p, 1] += 1
                continue
            if node.flags & 0x04:                            # Spec.Unschedulable
                out[p, 0] += 1
                continue
            if node.flags & 0x08:                            # Taints() error
                out[p, 1] += 1
                continue
            labels_ok = (node.labels & sel) == sel
            if aff != 0xFFFFFFFF:
                labels_ok = labels_ok and bool((int(aff_bits[aff, i // 32]) >> (i % 32)) & 1)
            taints_ok = (node.taints & ~tol & M64) == 0
            if not labels_ok:
                out[p, 2] += 1
            if not taints_ok:
                out[p, 3] += 1
            if not (labels_ok and taints_ok):
                continue
            left = single_node_resource(node, sel, tol, 1.0)
            fixed = (("MilliCPU", 0), ("Memory", 1), ("EphemeralStorage", 2), ("AllowedPodNumber", 3))
            for name, d in fixed:
                if getattr(left, name) < getattr(req, name):
                    out[p, 4 + d] += 1
            for k, v in req.ScalarResources.items():
                if k not in left.ScalarResources:
                    if v != 0:
                        out[p, 4 + k] += 1
                elif v > left.ScalarResources[k]:
                    out[p, 4 + k] += 1
    return out
