"""ctypes binding of include/bsched.h (libbsched.so) — the same C ABI the Go cgo shim binds.

No torch types cross this boundary; numpy arrays (or any object exposing a raw pointer)
are passed as plain pointers + sizes.  The library is CUDA-only: loading works on a CPU
box (symbols resolve), bs_create fails with BS_E_NODEVICE.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import build as _build

AFF_NONE = 0xffffffff
BS_OK, BS_E_INVAL, BS_E_NODEVICE, BS_E_CUDA, BS_E_NOMEM, BS_E_RANGE, BS_E_STATE, BS_E_REF_PANIC, BS_E_INDEX, BS_E_PEER = \
    0, -1, -2, -3, -4, -5, -6, -7, -8, -9
CODE_SUCCESS, CODE_ERROR, CODE_UNSCHEDULABLE, CODE_UNSCHEDULABLE_AND_UNRESOLVABLE, CODE_WAIT, CODE_SKIP = range(6)
OUT_FIT_BITMAP, OUT_SCORE, OUT_FILTER, OUT_TOPK, OUT_REASONS, OUT_PRIORITY = 0x1, 0x2, 0x4, 0x8, 0x10, 0x20
# bins of a reason row (BS_OUT_REASONS): [unschedulable, unavailable, selector, taints, lane 0, lane 1, ...]
REASON_UNSCHEDULABLE, REASON_UNAVAILABLE, REASON_SELECTOR, REASON_TAINTS, REASON_LANE0 = range(5)
TOPK_MAX = 32   # BS_TOPK_MAX: longest top-K list
NONZERO_MAX = 1 << 56   # BS_NONZERO_MAX: largest non-zero request a priority column may hold
PREF_NONE = 0xffffffff   # BS_PREF_NONE: pref_class of a pod without preferred node-affinity terms
PREF_TABLE_MAX_BYTES = 1 << 30   # BS_PREF_TABLE_MAX_BYTES: cap of the class x node weight table
IMAGE_NONE = 0xffffffff   # BS_IMAGE_NONE: image_class of a pod without dictionary images
AVOID_NONE = 0xff         # BS_AVOID_NONE: avoid_bit of a pod without an RC / RS controller
IMAGE_SIZE_MAX = 1 << 48  # BS_IMAGE_SIZE_MAX: largest image size in bytes
LOC_CLASS_MAX = 64        # BS_LOC_CLASS_MAX: ids one image class may list
LOC_TABLE_MAX_BYTES = 1 << 30   # BS_LOC_TABLE_MAX_BYTES: cap of the image bit rows and of the class x node IL table
SPREAD_NONE = 0xffffffff  # BS_SPREAD_NONE: spread_class of a pod without selectors
ZONE_NONE = 0xff          # BS_ZONE_NONE: zone of a node without a zone key
SPREAD_ZONE_MAX = 64      # BS_SPREAD_ZONE_MAX: zones of one node side
SPREAD_COUNT_MAX = 1 << 24   # BS_SPREAD_COUNT_MAX: largest selector count
SPREAD_TABLE_MAX_BYTES = 1 << 30   # BS_SPREAD_TABLE_MAX_BYTES: cap of the class x node count table
IPA_NONE = 0xffffffff     # BS_IPA_NONE: class of a pod or bound pod without entries
TOPO_NONE = 0xffffffff    # BS_TOPO_NONE: topo value of a node without the key
IPF_NONE = 0xffffffff     # BS_IPF_NONE: filter class of a pod without entries (passes every node)
IPF_AFFINITY, IPF_ANTI, IPF_EXISTING = range(3)   # BS_IPF_*: roles of a pod's filter class entries
HOSTPORT_MAX = 64         # BS_HOSTPORT_MAX: entries of the host-port dictionary
HOSTPORT_IP_ANY = 0       # BS_HOSTPORT_IP_ANY: ip id of "0.0.0.0"
IPA_KEY_MAX = 64          # BS_IPA_KEY_MAX: topology keys of one node side
IPA_BOUND_MAX = 1 << 24   # BS_IPA_BOUND_MAX: bound pods of one node side
IPA_CLASS_MAX = 64        # BS_IPA_CLASS_MAX: entries of one class
IPA_OWN_MAX = 1 << 16     # BS_IPA_OWN_MAX: largest |own| of one entry
IPA_TERM_MAX_BYTES = 1 << 30    # BS_IPA_TERM_MAX_BYTES: cap of the (term, value) M / S tables
IPA_TABLE_MAX_BYTES = 1 << 30   # BS_IPA_TABLE_MAX_BYTES: cap of the pod class x node raw table
# core.PreemptRemovePod verdicts (bs_remove_code) and the bound-pod flags
REMOVE_ALLOW, REMOVE_OFFLINE_ONLINE, REMOVE_NOT_FOUND, REMOVE_LOCKED, REMOVE_SAME_GROUP = range(5)
BOUND_GROUP_LOCKED = 0x01
BOUND_PDB_VIOLATING = 0x02
# bs_preempt_walk: the flag and the per-preemptor outcomes (bs_walk_outcome)
PREEMPT_GANG = 0x1
WALK_NONE, WALK_NOMINATED, WALK_ROLLED_BACK = range(3)
FILTER_PASS, FILTER_NOT_FOUND, FILTER_NOT_ENOUGH, FILTER_NO_SNAPSHOT, FILTER_REF_PANIC = range(5)
BUF_FIT_BITMAP, BUF_SCORE, BUF_ADMIT_BITMAP, BUF_PREFILTER, BUF_ADMIT, BUF_ORDER, BUF_GATHERED_ADMIT = range(7)
K_NODE_LEFT, K_FIND_MAX, K_CLASS_PREFIX, K_PREFILTER, K_GANG_FIT, K_SORT, K_FILTER, K_PEER, K_REPLAY, K_REASONS, K_COUNT = \
    range(11)
KERNEL_NAMES = ["node_left", "find_max", "class_prefix", "prefilter", "gang_fit", "sort", "filter", "peer", "replay"]


def _p(t):
    return C.POINTER(t)


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("n_lanes", C.c_uint32), ("out_flags", C.c_uint32), ("topk", C.c_uint32)]


class NodeTableC(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("n_lanes", C.c_uint32), ("alloc", C.c_void_p), ("requested", C.c_void_p),
                ("pod_count", C.c_void_p), ("alloc_present", C.c_void_p), ("req_present", C.c_void_p),
                ("label_mask", C.c_void_p), ("taint_mask", C.c_void_p), ("flags", C.c_void_p)]


class PodTableC(C.Structure):
    _fields_ = [("n_pods", C.c_uint32), ("n_lanes", C.c_uint32), ("req", C.c_void_p), ("req_present", C.c_void_p),
                ("gid", C.c_void_p), ("sel_mask", C.c_void_p), ("tol_mask", C.c_void_p), ("priority", C.c_void_p),
                ("ts_ns", C.c_void_p), ("flags", C.c_void_p), ("aff_class", C.c_void_p)]


class GroupTableC(C.Structure):
    _fields_ = [("n_groups", C.c_uint32), ("n_lanes", C.c_uint32), ("min_member", C.c_void_p),
                ("scheduled", C.c_void_p), ("matched", C.c_void_p), ("flags", C.c_void_p), ("min_res", C.c_void_p),
                ("min_res_present", C.c_void_p), ("rep_sel", C.c_void_p), ("rep_tol", C.c_void_p),
                ("creation_ns", C.c_void_p), ("name_rank", C.c_void_p), ("rep_aff_class", C.c_void_p)]


class ResultsC(C.Structure):
    _fields_ = [("prefilter", C.c_void_p), ("feasible_count", C.c_void_p), ("best_node", C.c_void_p),
                ("best_score", C.c_void_p), ("admit", C.c_void_p), ("admit_bitmap", C.c_void_p),
                ("new_denied", C.c_void_p), ("order", C.c_void_p), ("rank", C.c_void_p),
                ("max_group", C.c_int32), ("max_finished", C.c_uint32), ("filter_code", C.c_void_p)]


class ReplayResultC(C.Structure):
    _fields_ = [("prefilter", C.c_void_p), ("node", C.c_void_p), ("ready", C.c_void_p),
                ("node_requested", C.c_void_p), ("node_pod_count", C.c_void_p), ("node_req_present", C.c_void_p),
                ("group_matched", C.c_void_p), ("group_flags", C.c_void_p), ("group_min_res", C.c_void_p),
                ("group_min_res_present", C.c_void_p), ("group_rep_sel", C.c_void_p), ("group_rep_tol", C.c_void_p)]


class BoundTableC(C.Structure):
    _fields_ = [("n_pods", C.c_uint32), ("n_lanes", C.c_uint32), ("node", C.c_void_p), ("req", C.c_void_p),
                ("req_present", C.c_void_p), ("gid", C.c_void_p), ("priority", C.c_void_p), ("start_ns", C.c_void_p),
                ("flags", C.c_void_p)]


class InterpodClassesC(C.Structure):
    _fields_ = [("n_classes", C.c_uint32), ("class_offset", C.c_void_p), ("term", C.c_void_p), ("own", C.c_void_p),
                ("match", C.c_void_p)]


class InterpodNodesC(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("n_keys", C.c_uint32), ("n_values", C.c_void_p), ("topo", C.c_void_p),
                ("n_terms", C.c_uint32), ("term_key", C.c_void_p), ("n_bound", C.c_uint32), ("bound_node", C.c_void_p),
                ("bound_class", C.c_void_p), ("classes", InterpodClassesC)]


class InterpodPodsC(C.Structure):
    _fields_ = [("n_pods", C.c_uint32), ("pod_class", C.c_void_p), ("classes", InterpodClassesC)]


class InterpodFilterPodsC(C.Structure):
    _fields_ = [("n_pods", C.c_uint32), ("pod_class", C.c_void_p), ("n_classes", C.c_uint32),
                ("class_offset", C.c_void_p), ("term", C.c_void_p), ("role", C.c_void_p), ("self_match", C.c_void_p)]


class HostPortNodesC(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("n_entries", C.c_uint32), ("ip", C.c_void_p), ("protocol", C.c_void_p),
                ("port", C.c_void_p), ("used", C.c_void_p)]


class PreemptResultC(C.Structure):
    _fields_ = [("node", C.c_void_p), ("n_victims", C.c_void_p), ("n_candidates", C.c_void_p),
                ("victim_offset", C.c_void_p), ("victims", C.c_void_p), ("victims_cap", C.c_uint32),
                ("victims_total", C.c_uint32)]


class StatusC(C.Structure):
    _fields_ = [("code", C.c_int32), ("reason", C.c_int32), ("group", C.c_int32)]


class PermitResultC(C.Structure):
    _fields_ = [("ready", C.c_int32), ("code", C.c_int32), ("wait_ns", C.c_int64), ("start_signal", C.c_int32),
                ("group", C.c_int32)]


# every symbol include/bsched.h declares: (restype, argtypes)
SYMBOLS = {
    "bs_abi_version": (C.c_int, []),
    "bs_create": (C.c_int, [_p(Config), _p(C.c_void_p)]),
    "bs_destroy": (None, [C.c_void_p]),
    "bs_strerror": (C.c_char_p, [C.c_int]),
    "bs_last_error": (C.c_char_p, [C.c_void_p]),
    "bs_upload_nodes": (C.c_int, [C.c_void_p, _p(NodeTableC)]),
    "bs_update_nodes": (C.c_int, [C.c_void_p, C.c_void_p, _p(NodeTableC)]),
    "bs_update_groups": (C.c_int, [C.c_void_p, C.c_void_p, _p(GroupTableC)]),
    "bs_upload_groups": (C.c_int, [C.c_void_p, _p(GroupTableC)]),
    "bs_upload_pods": (C.c_int, [C.c_void_p, _p(PodTableC)]),
    "bs_upload_affinity": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_set_wait_time": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32]),
    "bs_evaluate": (C.c_int, [C.c_void_p, _p(ResultsC)]),
    "bs_evaluate_async": (C.c_int, [C.c_void_p]),
    "bs_sync": (C.c_int, [C.c_void_p]),
    "bs_fetch": (C.c_int, [C.c_void_p, _p(ResultsC)]),
    "bs_fetch_view": (C.c_int, [C.c_void_p, _p(ResultsC)]),
    "bs_evaluate_view": (C.c_int, [C.c_void_p, _p(ResultsC)]),
    "bs_prefilter": (C.c_int, [C.c_void_p, C.c_uint32, _p(StatusC)]),
    "bs_permit": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _p(PermitResultC)]),
    "bs_less": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "bs_filter": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _p(StatusC)]),
    "bs_state_reset": (C.c_int, [C.c_void_p]),
    "bs_state_remap": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_state_view": (C.c_int, [C.c_void_p, C.c_int64, C.c_uint32, C.c_void_p, C.c_void_p]),
    "bs_permitted_view": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_state_move": (C.c_int, [C.c_void_p, C.c_void_p]),
    "bs_set_pod_ids": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "bs_begin_cycle": (C.c_int, [C.c_void_p, C.c_int64]),
    "bs_permit_at": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int64, _p(PermitResultC)]),
    "bs_expire": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_uint32, _p(C.c_uint32), C.c_void_p, C.c_uint32,
                            _p(C.c_uint32)]),
    "bs_allow_list": (C.c_int, [C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p, C.c_void_p, C.c_uint32, _p(C.c_uint32)]),
    "bs_deny": (C.c_int, [C.c_void_p, C.c_uint32, C.c_int64]),
    "bs_mark_permitted": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int64]),
    "bs_group_state": (C.c_int, [C.c_void_p, C.c_uint32, C.c_int64, _p(C.c_uint32), _p(C.c_int32), _p(C.c_int32)]),
    "bs_format_message": (C.c_int, [_p(StatusC), C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]),
    "bs_node_left": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_float, C.c_void_p, C.c_void_p]),
    "bs_replay": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, _p(ReplayResultC)]),
    "bs_cluster_check": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_float, C.c_void_p, C.c_void_p,
                                   C.c_uint32, C.c_void_p]),
    "bs_upload_bound_pods": (C.c_int, [C.c_void_p, _p(BoundTableC)]),
    "bs_preempt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, _p(PreemptResultC)]),
    "bs_preempt_walk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, _p(PreemptResultC), C.c_void_p,
                                  C.c_void_p]),
    "bs_remove_pod": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, _p(StatusC)]),
    "bs_format_remove_message": (C.c_int, [_p(StatusC), C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]),
    "bs_device_buffer": (C.c_int, [C.c_void_p, C.c_int, _p(C.c_void_p), _p(C.c_size_t)]),
    "bs_stream": (C.c_void_p, [C.c_void_p]),
    "bs_score_pitch": (C.c_uint32, [C.c_void_p]),
    "bs_bitmap_pitch": (C.c_uint32, [C.c_void_p]),
    "bs_fetch_fit_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "bs_fetch_score_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "bs_fetch_filter_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "bs_fetch_topk_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]),
    "bs_fetch_reason_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "bs_format_fit_error": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_char_p, C.c_size_t]),
    "bs_set_score_weights": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]),
    "bs_upload_node_nonzero": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_upload_pod_nonzero": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_fetch_priority_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]),
    "bs_replay_priority": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, _p(ReplayResultC), C.c_void_p]),
    "bs_set_ratio_priority": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                        C.c_void_p, C.c_uint32]),
    "bs_set_node_priority_weights": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "bs_upload_node_preferences": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_upload_pod_preferences": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "bs_set_locality_weights": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "bs_upload_node_locality": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "bs_upload_pod_locality": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    "bs_set_spread_weight": (C.c_int, [C.c_void_p, C.c_uint32]),
    "bs_upload_node_spread": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_upload_pod_spread": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_set_interpod_weight": (C.c_int, [C.c_void_p, C.c_uint32]),
    "bs_upload_node_interpod": (C.c_int, [C.c_void_p, _p(InterpodNodesC)]),
    "bs_upload_pod_interpod": (C.c_int, [C.c_void_p, _p(InterpodPodsC)]),
    "bs_set_interpod_filter": (C.c_int, [C.c_void_p, C.c_int]),
    "bs_upload_node_interpod_filter": (C.c_int, [C.c_void_p, _p(InterpodNodesC)]),
    "bs_upload_pod_interpod_filter": (C.c_int, [C.c_void_p, _p(InterpodFilterPodsC)]),
    "bs_upload_pod_interpod_placed": (C.c_int, [C.c_void_p, _p(InterpodPodsC)]),
    "bs_fetch_interpod_reason_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "bs_format_fit_error_interpod": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_char_p,
                                               C.c_size_t]),
    "bs_set_host_port_filter": (C.c_int, [C.c_void_p, C.c_int]),
    "bs_upload_node_host_ports": (C.c_int, [C.c_void_p, _p(HostPortNodesC)]),
    "bs_upload_pod_host_ports": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_fetch_host_port_reason_rows": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "bs_upload_bound_host_ports": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "bs_format_fit_error_filters": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                              C.c_char_p, C.c_size_t]),
    "bs_peer_init": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]),
    "bs_peer_handle": (C.c_int, [C.c_void_p, C.c_void_p]),
    "bs_peer_attach": (C.c_int, [C.c_void_p, C.c_void_p]),
    "bs_peer_detach": (C.c_int, [C.c_void_p]),
    "bs_peer_join": (C.c_int, [C.c_void_p]),
    "bs_fetch_gathered_admit": (C.c_int, [C.c_void_p, C.c_void_p]),
    "bs_set_profiling": (C.c_int, [C.c_void_p, C.c_int]),
    "bs_kernel_ms": (C.c_int, [C.c_void_p, C.c_int, _p(C.c_float), _p(C.c_uint32)]),
    "bs_launch_count": (C.c_uint64, [C.c_void_p]),
    "bs_fit_shape": (C.c_int, [C.c_void_p, _p(C.c_uint32), _p(C.c_uint32), _p(C.c_uint32)]),
    "bs_fit_lanes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "bs_sort_shape": (C.c_int, [C.c_void_p, _p(C.c_uint32), _p(C.c_uint32), _p(C.c_uint32), _p(C.c_uint32)]),
    "bs_score_memory": (C.c_int, [C.c_void_p, _p(C.c_uint32), _p(C.c_uint32)]),
    "bs_replay_shape": (C.c_int, [C.c_void_p] + [_p(C.c_uint32)] * 8),
}

_lib = None


def load(build_if_missing: bool = True):
    """Loads libbsched.so (building it with nvcc first if it is absent)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if build_if_missing and not os.path.exists(path):
        _build.build()
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: the CUDA extension must be built (no CPU fallback exists)")
    lib = C.CDLL(path)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def ptr(a) -> int:
    """Raw address of a numpy array / torch tensor / int."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return int(a)


class BsError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"bsched error {code}: {msg}")
        self.code = code
