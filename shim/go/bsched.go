// Package gpu — cgo binding of include/bsched.h, the file a maintainer of tenstack/batch-scheduler adds as
// pkg/scheduler/core/gpu/bsched.go (with CGO_ENABLED=1; the reference builds with CGO_ENABLED=0, Makefile:28).
//
// NOT BUILT OR TESTED in the authoring container: there is no Go toolchain there.  The identical ABI is
// exercised from Python (batch-scheduler_b200/capi.py, ctypes) and C++ (csrc/plugin.cpp) by the test suite;
// this file mirrors those call sequences one to one.
package gpu

/*
#cgo CFLAGS: -I${SRCDIR}/../../../../third_party/bsched/include
#cgo LDFLAGS: -L${SRCDIR}/../../../../third_party/bsched/lib -lbsched -lcudart
#include <stdlib.h>
#include "bsched.h"
*/
import "C"

import (
	"fmt"
	"hash/fnv"
	"time"
	"unsafe"
)

// Engine wraps one bs_engine (one GPU).  Thread-safe: the C side serialises calls per handle, as the reference
// calls Less / Permit from several goroutines (batchscheduler.go:165,214).
type Engine struct {
	h     *C.bs_engine
	topk  int // list length of BS_OUT_TOPK, 0 without it
	lanes int // resource lanes of every table: a reason row has 4 + lanes bins
}

// ID turns a pod UID or a "namespace/name" into the 64-bit id the gang-state calls take (FNV-1a, as
// BatchSchedulingPlugin::IdOf does in csrc/plugin.cpp).
func ID(s string) uint64 {
	f := fnv.New64a()
	f.Write([]byte(s))
	return f.Sum64()
}

// New replaces core.NewScheduleOperation (core.go:64-77).
func New(device, lanes int, outFlags uint32) (*Engine, error) { return NewTopK(device, lanes, outFlags, 0) }

// NewTopK is New with each round also keeping every pod's topk best fitting nodes (BS_OUT_TOPK, 1..BS_TOPK_MAX;
// 0 = none), read with TopNodes.
func NewTopK(device, lanes int, outFlags uint32, topk int) (*Engine, error) {
	if topk > 0 {
		outFlags |= C.BS_OUT_TOPK
	}
	cfg := C.bs_config{device: C.int32_t(device), n_lanes: C.uint32_t(lanes), out_flags: C.uint32_t(outFlags),
		topk: C.uint32_t(topk)}
	var h *C.bs_engine
	if rc := C.bs_create(&cfg, &h); rc != 0 {
		return nil, fmt.Errorf("bs_create: %s", C.GoString(C.bs_strerror(rc)))
	}
	return &Engine{h, topk, lanes}, nil
}

// NewPriority is New with each round also keeping every pod's k best fitting nodes under kube-scheduler's resource
// priorities (BS_OUT_PRIORITY, 1..BS_TOPK_MAX), read with PriorityNodes.  outFlags may hold BS_OUT_TOPK too: both
// lists then have length k.
func NewPriority(device, lanes int, outFlags uint32, k int) (*Engine, error) {
	cfg := C.bs_config{device: C.int32_t(device), n_lanes: C.uint32_t(lanes),
		out_flags: C.uint32_t(outFlags | C.BS_OUT_PRIORITY), topk: C.uint32_t(k)}
	var h *C.bs_engine
	if rc := C.bs_create(&cfg, &h); rc != 0 {
		return nil, fmt.Errorf("bs_create: %s", C.GoString(C.bs_strerror(rc)))
	}
	return &Engine{h, k, lanes}, nil
}

func (e *Engine) Close() { C.bs_destroy(e.h) }

func (e *Engine) rc(code C.int) error {
	if code == 0 {
		return nil
	}
	return fmt.Errorf("bsched: %s (%s)", C.GoString(C.bs_strerror(code)), C.GoString(C.bs_last_error(e.h)))
}

// ---- snapshot upload: the packer builds C-malloc'd (or pinned) SoA columns; cgo forbids retaining Go
// pointers, and the engine copies everything during the call.
func (e *Engine) UploadNodes(t *C.bs_node_table) error   { return e.rc(C.bs_upload_nodes(e.h, t)) }
func (e *Engine) UploadGroups(t *C.bs_group_table) error { return e.rc(C.bs_upload_groups(e.h, t)) }
func (e *Engine) UploadPods(t *C.bs_pod_table) error     { return e.rc(C.bs_upload_pods(e.h, t)) }

// UploadAffinity: checkFit beyond the 64 selector bits (required nodeAffinity terms, > 64 selector pairs):
// bits[nClasses][ceil(nNodes/32)], one host-evaluated verdict per (affinity class, node); after UploadNodes.
func (e *Engine) UploadAffinity(nClasses uint32, bits *C.uint32_t) error {
	return e.rc(C.bs_upload_affinity(e.h, C.uint32_t(nClasses), bits))
}

// UpdateNodes / UpdateGroups: between cycles only the rows the informers touched.
func (e *Engine) UpdateNodes(idx []uint32, t *C.bs_node_table) error {
	return e.rc(C.bs_update_nodes(e.h, (*C.uint32_t)(unsafe.Pointer(&idx[0])), t))
}
func (e *Engine) UpdateGroups(idx []uint32, t *C.bs_group_table) error {
	return e.rc(C.bs_update_groups(e.h, (*C.uint32_t)(unsafe.Pointer(&idx[0])), t))
}

// ---- gang state: MatchedPodNodes / PodNameUIDs / pgs.Scheduled / lastDeniedPG / lastPermittedPod live in the
// engine, driven by the caller's clock.
func (e *Engine) StateReset() error { return e.rc(C.bs_state_reset(e.h)) }
func (e *Engine) StateRemap(oldIndex []int32) error {
	return e.rc(C.bs_state_remap(e.h, C.uint32_t(len(oldIndex)), (*C.int32_t)(unsafe.Pointer(&oldIndex[0]))))
}
func (e *Engine) SetPodIDs(uid, name []uint64) error {
	return e.rc(C.bs_set_pod_ids(e.h, (*C.uint64_t)(unsafe.Pointer(&uid[0])), (*C.uint64_t)(unsafe.Pointer(&name[0]))))
}

// BeginCycle writes the tables' view at `now` into the round's inputs (matched counts, SCHEDULED / DENIED,
// PERMITTED_RECENTLY) — the reads of core.go:95-110 and :706-711.
func (e *Engine) BeginCycle(now time.Time) error { return e.rc(C.bs_begin_cycle(e.h, C.int64_t(now.UnixNano()))) }

// Evaluate runs one round: every pending pod's PreFilter verdict, the pod x node fit matrix, the gang
// decisions and the queue order, in one call.
func (e *Engine) Evaluate() error { return e.rc(C.bs_evaluate(e.h, nil)) }

// Round is the whole round read in place: slices over the engine's pinned decision arena (bs_evaluate_view), valid
// until the next Evaluate* / Upload* / Update* on this engine.  Nothing is copied; do not write through them.
type Round struct {
	PreFilter []uint8  // BS_PF_* per pending pod
	Feasible  []uint32 // nodes each pod fits on
	BestNode  []int32  // highest-score node, -1 = none
	Admit     []uint8  // per PodGroup: the gang reaches minMember this round
	Order     []uint32 // queue order (Compare, core.go:368-411)
	Rank      []uint32 // dense rank of each pod in that order
}

func (e *Engine) EvaluateView(nPods, nGroups int) (Round, error) {
	var r C.bs_results
	if err := e.rc(C.bs_evaluate_view(e.h, &r)); err != nil {
		return Round{}, err
	}
	return Round{
		PreFilter: unsafe.Slice((*uint8)(unsafe.Pointer(r.prefilter)), nPods),
		Feasible:  unsafe.Slice((*uint32)(unsafe.Pointer(r.feasible_count)), nPods),
		BestNode:  unsafe.Slice((*int32)(unsafe.Pointer(r.best_node)), nPods),
		Admit:     unsafe.Slice((*uint8)(unsafe.Pointer(r.admit)), nGroups),
		Order:     unsafe.Slice((*uint32)(unsafe.Pointer(r.order)), nPods),
		Rank:      unsafe.Slice((*uint32)(unsafe.Pointer(r.rank)), nPods),
	}, nil
}

// TopNodes returns the top-K lists of pods [pod0, pod0+n) of the last round as dense [n][K] rows: each pod's
// fitting nodes by score descending, then node index ascending, padded with node -1 and score math.MinInt64.
func (e *Engine) TopNodes(pod0, n int) ([]int32, []int64, error) {
	nodes, scores := make([]int32, n*e.topk), make([]int64, n*e.topk)
	if len(nodes) == 0 {
		return nodes, scores, e.rc(C.bs_fetch_topk_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), nil, nil))
	}
	err := e.rc(C.bs_fetch_topk_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), (*C.int32_t)(unsafe.Pointer(&nodes[0])),
		(*C.int64_t)(unsafe.Pointer(&scores[0]))))
	return nodes, scores, err
}

// SetScoreWeights sets the weights of NodeResourcesLeastAllocated, NodeResourcesMostAllocated and
// NodeResourcesBalancedAllocation (default 1, 0, 1) for the next rounds.
func (e *Engine) SetScoreWeights(least, most, balanced uint32) error {
	return e.rc(C.bs_set_score_weights(e.h, C.uint32_t(least), C.uint32_t(most), C.uint32_t(balanced)))
}

// RatioPoint is one point of a RequestedToCapacityRatio shape in engine units: utilization and score both 0..100.
type RatioPoint struct{ Utilization, Score uint32 }

// SetRatioPriority adds kube-scheduler's RequestedToCapacityRatio priority to the priority score with weight `weight`
// (0 = off).  The v1.17 policy file gives shape scores in 0..10: multiply them by 10 before calling.  laneWeights has
// one weight per lane of the engine (lane 3, pods, must be 0); absentWeight is the weight of the resources no node of
// the round has (pods and names that are not a lane of the round).  An invalid setting keeps the previous one.
func (e *Engine) SetRatioPriority(weight uint32, shape []RatioPoint, laneWeights []uint32, absentWeight uint32) error {
	util := make([]C.uint32_t, len(shape))
	score := make([]C.uint32_t, len(shape))
	for i, p := range shape {
		util[i], score[i] = C.uint32_t(p.Utilization), C.uint32_t(p.Score)
	}
	lw := make([]C.uint32_t, len(laneWeights))
	for i, w := range laneWeights {
		lw[i] = C.uint32_t(w)
	}
	var up, sp, lp *C.uint32_t
	if len(shape) > 0 {
		up, sp = &util[0], &score[0]
	}
	if len(lw) > 0 {
		lp = &lw[0]
	}
	return e.rc(C.bs_set_ratio_priority(e.h, C.uint32_t(weight), C.uint32_t(len(shape)), up, sp, C.uint32_t(len(lw)), lp,
		C.uint32_t(absentWeight)))
}

// SetNodePriorityWeights adds kube-scheduler's TaintToleration and preferred NodeAffinity priorities to the priority
// score (0, 0 = off; v1.17's default profile is 1, 1).  While either is non-zero ReplayPriority is refused.
func (e *Engine) SetNodePriorityWeights(taintToleration, nodeAffinity uint32) error {
	return e.rc(C.bs_set_node_priority_weights(e.h, C.uint32_t(taintToleration), C.uint32_t(nodeAffinity)))
}

// UploadNodePreferences: per node the bits of the round's PreferNoSchedule taint dictionary it carries, and the
// class x node table prefWeights[nClasses][n] of summed preferred-term weights.  UploadNodes / UpdateNodes drop it.
func (e *Engine) UploadNodePreferences(preferTaints []uint64, prefWeights []int32) error {
	n := len(preferTaints)
	if n == 0 {
		return e.rc(C.bs_upload_node_preferences(e.h, 0, nil, 0, nil))
	}
	classes := len(prefWeights) / n
	var wp *C.int32_t
	if classes > 0 {
		wp = (*C.int32_t)(unsafe.Pointer(&prefWeights[0]))
	}
	return e.rc(C.bs_upload_node_preferences(e.h, C.uint32_t(n), (*C.uint64_t)(unsafe.Pointer(&preferTaints[0])),
		C.uint32_t(classes), wp))
}

// UploadPodPreferences: per pod the dictionary bits it tolerates and its row of the class table (BS_PREF_NONE for a
// pod without preferred terms).  UploadPods drops it.
func (e *Engine) UploadPodPreferences(preferTol []uint64, prefClass []uint32) error {
	n := len(preferTol)
	if n == 0 || len(prefClass) != n {
		return e.rc(C.bs_upload_pod_preferences(e.h, C.uint32_t(n), nil, nil))
	}
	return e.rc(C.bs_upload_pod_preferences(e.h, C.uint32_t(n), (*C.uint64_t)(unsafe.Pointer(&preferTol[0])),
		(*C.uint32_t)(unsafe.Pointer(&prefClass[0]))))
}

// SetLocalityWeights: kube-scheduler v1.17's ImageLocality and NodePreferAvoidPods weights in the priority lists and
// in ReplayPriority (0, 0 = off; v1.17's default profile is 1, 10000).
func (e *Engine) SetLocalityWeights(imageLocality, preferAvoidPods uint32) error {
	return e.rc(C.bs_set_locality_weights(e.h, C.uint32_t(imageLocality), C.uint32_t(preferAvoidPods)))
}

// A nil slice is a missing part (NULL), an empty one a part without entries (a non-NULL pointer to locDummy).
var locDummy [8]byte

func locP(isNil bool, n int, first func() unsafe.Pointer) unsafe.Pointer {
	if isNil {
		return nil
	}
	if n == 0 {
		return unsafe.Pointer(&locDummy[0])
	}
	return first()
}
func locI64(v []int64) *C.int64_t {
	return (*C.int64_t)(locP(v == nil, len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }))
}
func locU32(v []uint32) *C.uint32_t {
	return (*C.uint32_t)(locP(v == nil, len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }))
}
func locU64(v []uint64) *C.uint64_t {
	return (*C.uint64_t)(locP(v == nil, len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }))
}
func locU8(v []uint8) *C.uint8_t {
	return (*C.uint8_t)(locP(v == nil, len(v), func() unsafe.Pointer { return unsafe.Pointer(&v[0]) }))
}

// UploadNodeLocality: the image dictionary's sizes (bytes, [0, 2^48]) and bit rows imageBits[len(imageSize)][(n+31)/32]
// (bit n%32 of word n/32: node n reports the name), and avoidMask[n], per node the bits of the round's controller
// dictionary that its preferAvoidPods annotation lists.  imageSize and imageBits may both be nil while the
// ImageLocality weight is 0, avoidMask while the NodePreferAvoidPods weight is 0.  Slices of the wrong length are an
// error before anything is passed to C.  UploadNodes / UpdateNodes drop it.
func (e *Engine) UploadNodeLocality(n int, imageSize []int64, imageBits []uint32, avoidMask []uint64) error {
	if (imageSize == nil) != (imageBits == nil) {
		return fmt.Errorf("UploadNodeLocality: imageSize and imageBits must both be given or both be nil")
	}
	if imageSize != nil && len(imageBits) != len(imageSize)*((n+31)/32) {
		return fmt.Errorf("UploadNodeLocality: len(imageBits) = %d, want len(imageSize) * ((n + 31) / 32) = %d",
			len(imageBits), len(imageSize)*((n+31)/32))
	}
	if avoidMask != nil && len(avoidMask) != n {
		return fmt.Errorf("UploadNodeLocality: len(avoidMask) = %d, want n = %d", len(avoidMask), n)
	}
	return e.rc(C.bs_upload_node_locality(e.h, C.uint32_t(n), C.uint32_t(len(imageSize)),
		locI64(imageSize), locU32(imageBits), locU64(avoidMask)))
}

// UploadPodLocality: imageClass[n], each pod's image class (BS_IMAGE_NONE: none), the classes as
// classOffset[nClasses+1] into classImages, and avoidBit[n], each pod's controller bit (BS_AVOID_NONE: none).  The
// three image parts may be nil together while the ImageLocality weight is 0, avoidBit while the NodePreferAvoidPods
// weight is 0.  Slices of the wrong length are an error before anything is passed to C.  UploadPods drops it.
func (e *Engine) UploadPodLocality(n int, imageClass, classOffset, classImages []uint32, avoidBit []uint8) error {
	classes := 0
	if imageClass != nil || classOffset != nil || classImages != nil {
		if imageClass == nil || classOffset == nil || classImages == nil {
			return fmt.Errorf("UploadPodLocality: imageClass, classOffset and classImages must all be given or all be nil")
		}
		if len(imageClass) != n {
			return fmt.Errorf("UploadPodLocality: len(imageClass) = %d, want n = %d", len(imageClass), n)
		}
		if len(classOffset) < 1 || int(classOffset[len(classOffset)-1]) > len(classImages) {
			return fmt.Errorf("UploadPodLocality: classOffset needs nClasses + 1 entries and classImages " +
				"classOffset[nClasses] of them")
		}
		classes = len(classOffset) - 1
	}
	if avoidBit != nil && len(avoidBit) != n {
		return fmt.Errorf("UploadPodLocality: len(avoidBit) = %d, want n = %d", len(avoidBit), n)
	}
	return e.rc(C.bs_upload_pod_locality(e.h, C.uint32_t(n), locU32(imageClass), C.uint32_t(classes), locU32(classOffset),
		locU32(classImages), locU8(avoidBit)))
}

// SetSpreadWeight: kube-scheduler v1.17's SelectorSpread weight in the priority lists (0 = off; v1.17's default
// profile is 1).  ReplayPriority refuses a non-zero weight.
func (e *Engine) SetSpreadWeight(selectorSpread uint32) error {
	return e.rc(C.bs_set_spread_weight(e.h, C.uint32_t(selectorSpread)))
}

// UploadNodeSpread: zone[n], each node's id in the round's zone dictionary of nZones keys (BS_ZONE_NONE: no zone
// key), and counts[classes][n], per class the pods on each node that its selectors match.  Slices of the wrong length
// are an error before anything is passed to C.  UploadNodes / UpdateNodes drop it.
func (e *Engine) UploadNodeSpread(n, nZones int, zone []uint8, counts []int32) error {
	if len(zone) != n {
		return fmt.Errorf("UploadNodeSpread: len(zone) = %d, want n = %d", len(zone), n)
	}
	classes := 0
	if n > 0 {
		if len(counts)%n != 0 {
			return fmt.Errorf("UploadNodeSpread: len(counts) = %d is not a multiple of n = %d", len(counts), n)
		}
		classes = len(counts) / n
	}
	var zp *C.uint8_t
	var cp *C.int32_t
	if n > 0 {
		zp = (*C.uint8_t)(unsafe.Pointer(&zone[0]))
	}
	if len(counts) > 0 {
		cp = (*C.int32_t)(unsafe.Pointer(&counts[0]))
	}
	return e.rc(C.bs_upload_node_spread(e.h, C.uint32_t(n), C.uint32_t(nZones), zp, C.uint32_t(classes), cp))
}

// UploadPodSpread: per pod its row of the count table (BS_SPREAD_NONE for a pod without selectors).  UploadPods
// drops it.
func (e *Engine) UploadPodSpread(spreadClass []uint32) error {
	if len(spreadClass) == 0 {
		return e.rc(C.bs_upload_pod_spread(e.h, 0, nil))
	}
	return e.rc(C.bs_upload_pod_spread(e.h, C.uint32_t(len(spreadClass)),
		(*C.uint32_t)(unsafe.Pointer(&spreadClass[0]))))
}

// SetInterPodAffinityWeight: kube-scheduler v1.17's InterPodAffinity weight in the priority lists (0 = off; v1.17's
// default profile is 1).  ReplayPriority refuses a non-zero weight.
func (e *Engine) SetInterPodAffinityWeight(interPodAffinity uint32) error {
	return e.rc(C.bs_set_interpod_weight(e.h, C.uint32_t(interPodAffinity)))
}

// UploadNodeInterPodAffinity / UploadPodInterPodAffinity: the InterPodAffinity sides (topology values, term keys,
// bound pods and their classes; each pending pod's class), as the packer builds them in C-malloc'd (or pinned)
// columns, like the other tables: cgo forbids passing a Go struct that holds Go pointers.  UploadNodes / UpdateNodes
// drop the node side and UploadPods the pod side.
func (e *Engine) UploadNodeInterPodAffinity(t *C.bs_interpod_nodes) error {
	return e.rc(C.bs_upload_node_interpod(e.h, t))
}
func (e *Engine) UploadPodInterPodAffinity(t *C.bs_interpod_pods) error {
	return e.rc(C.bs_upload_pod_interpod(e.h, t))
}

// MatchInterPodAffinity filter roles and the class of a pod without entries (include/bsched.h BS_IPF_*).
const (
	IPFNone     = uint32(C.BS_IPF_NONE)
	IPFAffinity = uint8(C.BS_IPF_AFFINITY)
	IPFAnti     = uint8(C.BS_IPF_ANTI)
	IPFExisting = uint8(C.BS_IPF_EXISTING)
	IPFClassMax = int(C.BS_IPF_CLASS_MAX)
	IPFBoundMax = uint32(C.BS_IPF_BOUND_MAX)
)

// SetInterPodAffinityFilter: kube-scheduler v1.17's MatchInterPodAffinity filter in every pod's fit set (off by
// default).  While it is on, each Evaluate needs both filter sides, Replay and ReplayPriority need the placed side
// as well (UploadPodInterPodPlaced; they refuse to run without it), and Preempt and PreemptWalk refuse to run.
func (e *Engine) SetInterPodAffinityFilter(on bool) error {
	v := C.int(0)
	if on {
		v = 1
	}
	return e.rc(C.bs_set_interpod_filter(e.h, v))
}

// UploadNodeInterPodFilter / UploadPodInterPodFilter: the filter's sides in C-malloc'd (or pinned) columns.  The node
// side has the layout of the InterPodAffinity node side, own = 1 for a bound pod's required anti-affinity terms.
// UploadNodes / UpdateNodes drop the node side and UploadPods the pod side.
func (e *Engine) UploadNodeInterPodFilter(t *C.bs_interpod_nodes) error {
	return e.rc(C.bs_upload_node_interpod_filter(e.h, t))
}
func (e *Engine) UploadPodInterPodFilter(t *C.bs_interpod_filter_pods) error {
	return e.rc(C.bs_upload_pod_interpod_filter(e.h, t))
}

// UploadPodInterPodPlaced: the filter's placed side, what each pending pod adds to presence once a walk assumes it, in
// the layout of a bound pod's class (own on its anti-affinity terms, match on the terms it matches).  UploadPods drops
// it.
func (e *Engine) UploadPodInterPodPlaced(t *C.bs_interpod_pods) error {
	return e.rc(C.bs_upload_pod_interpod_placed(e.h, t))
}

// FetchInterPodReasonRows: the companion of FetchReasonRows, counts[n][3] (E, A, N) of the nodes that pass every
// other check and fail the filter.
func (e *Engine) FetchInterPodReasonRows(pod0, n uint32, counts []uint32) error {
	if uint64(len(counts)) < uint64(n)*3 {
		return fmt.Errorf("bsched: counts needs n*3 entries")
	}
	var p *C.uint32_t
	if n > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&counts[0]))
	}
	return e.rc(C.bs_fetch_interpod_reason_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), p))
}

// SetHostPortFilter: kube-scheduler v1.17's PodFitsHostPorts filter in every pod's fit set and in the Replay walks
// (off by default).  While it is on, each Evaluate and Replay needs both sides, and Preempt and PreemptWalk apply it
// once UploadBoundHostPorts has given the bound pods' masks (they refuse to run without them).
func (e *Engine) SetHostPortFilter(on bool) error {
	v := C.int(0)
	if on {
		v = 1
	}
	return e.rc(C.bs_set_host_port_filter(e.h, v))
}

// HostPortEntry is one (ip id, protocol id, port) of the dictionary; ip id 0 (BS_HOSTPORT_IP_ANY) is "0.0.0.0".
type HostPortEntry struct {
	IP, Protocol uint32
	Port         int32
}

// UploadNodeHostPorts: the dictionary (at most BS_HOSTPORT_MAX entries) and used[n_nodes], bit k = the node's
// UsedPorts() holds entry k.  UploadNodes / UpdateNodes drop it.
func (e *Engine) UploadNodeHostPorts(entries []HostPortEntry, used []uint64) error {
	k := len(entries)
	ip, proto, port := make([]uint32, k+1), make([]uint32, k+1), make([]int32, k+1)
	for i, x := range entries {
		ip[i], proto[i], port[i] = x.IP, x.Protocol, x.Port
	}
	cip := (*C.uint32_t)(C.malloc(C.size_t(4 * (k + 1))))
	cproto := (*C.uint32_t)(C.malloc(C.size_t(4 * (k + 1))))
	cport := (*C.int32_t)(C.malloc(C.size_t(4 * (k + 1))))
	cused := (*C.uint64_t)(C.malloc(C.size_t(8 * (len(used) + 1))))
	defer C.free(unsafe.Pointer(cip))
	defer C.free(unsafe.Pointer(cproto))
	defer C.free(unsafe.Pointer(cport))
	defer C.free(unsafe.Pointer(cused))
	copy(unsafe.Slice((*uint32)(unsafe.Pointer(cip)), k+1), ip)
	copy(unsafe.Slice((*uint32)(unsafe.Pointer(cproto)), k+1), proto)
	copy(unsafe.Slice((*int32)(unsafe.Pointer(cport)), k+1), port)
	copy(unsafe.Slice((*uint64)(unsafe.Pointer(cused)), len(used)+1), used)
	t := C.bs_host_port_nodes{n_nodes: C.uint32_t(len(used)), n_entries: C.uint32_t(k), ip: cip, protocol: cproto,
		port: cport, used: cused}
	return e.rc(C.bs_upload_node_host_ports(e.h, &t))
}

// UploadPodHostPorts: want[n_pods], bit k = the pod's containers ask for entry k.  UploadPods drops it.
func (e *Engine) UploadPodHostPorts(want []uint64) error {
	if len(want) == 0 {
		return e.rc(C.bs_upload_pod_host_ports(e.h, 0, nil))
	}
	c := (*C.uint64_t)(C.malloc(C.size_t(8 * len(want))))
	defer C.free(unsafe.Pointer(c))
	copy(unsafe.Slice((*uint64)(unsafe.Pointer(c)), len(want)), want)
	return e.rc(C.bs_upload_pod_host_ports(e.h, C.uint32_t(len(want)), c))
}

// UploadBoundHostPorts: ports[n_bound_pods], bit k = bound row v of UploadBoundPods holds exactly entry k of the
// node side's dictionary, what preemption under the filter frees when it evicts the row.  UploadBoundPods and every
// call that drops the bound table drop it; the bits are checked against the node side when a preemption starts.
func (e *Engine) UploadBoundHostPorts(ports []uint64) error {
	if len(ports) == 0 {
		return e.rc(C.bs_upload_bound_host_ports(e.h, 0, nil))
	}
	c := (*C.uint64_t)(C.malloc(C.size_t(8 * len(ports))))
	defer C.free(unsafe.Pointer(c))
	copy(unsafe.Slice((*uint64)(unsafe.Pointer(c)), len(ports)), ports)
	return e.rc(C.bs_upload_bound_host_ports(e.h, C.uint32_t(len(ports)), c))
}

// FetchHostPortReasonRows: the companion of FetchReasonRows, counts[n] of the nodes past the guards with a host-port
// conflict.
func (e *Engine) FetchHostPortReasonRows(pod0, n uint32, counts []uint32) error {
	if uint64(len(counts)) < uint64(n) {
		return fmt.Errorf("bsched: counts needs n entries")
	}
	var p *C.uint32_t
	if n > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&counts[0]))
	}
	return e.rc(C.bs_fetch_host_port_reason_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), p))
}

// UploadNodeNonZero / UploadPodNonZero: the non-zero request columns, nz[2][n] (cpu millicores, then memory bytes):
// per pod the sum over its containers of GetNonzeroRequestForResource(Requests), per node NodeInfo.NonZeroRequest().
// UploadNodes / UpdateNodes drop the node column and UploadPods the pod column: upload them again before Evaluate.
func (e *Engine) UploadNodeNonZero(nz []int64) error {
	n := len(nz) / 2
	if n == 0 {
		return e.rc(C.bs_upload_node_nonzero(e.h, 0, nil))
	}
	return e.rc(C.bs_upload_node_nonzero(e.h, C.uint32_t(n), (*C.int64_t)(unsafe.Pointer(&nz[0]))))
}
func (e *Engine) UploadPodNonZero(nz []int64) error {
	n := len(nz) / 2
	if n == 0 {
		return e.rc(C.bs_upload_pod_nonzero(e.h, 0, nil))
	}
	return e.rc(C.bs_upload_pod_nonzero(e.h, C.uint32_t(n), (*C.int64_t)(unsafe.Pointer(&nz[0]))))
}

// PriorityNodes returns the priority lists of pods [pod0, pod0+n) of the last round (engine from NewPriority) as dense
// [n][K] rows: each pod's fitting nodes by priority score descending, then node index ascending, padded with node -1
// and score math.MinInt64.  Entry 0 is the node to bind or nominate.
func (e *Engine) PriorityNodes(pod0, n int) ([]int32, []int64, error) {
	nodes, scores := make([]int32, n*e.topk), make([]int64, n*e.topk)
	if len(nodes) == 0 {
		return nodes, scores, e.rc(C.bs_fetch_priority_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), nil, nil))
	}
	err := e.rc(C.bs_fetch_priority_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), (*C.int32_t)(unsafe.Pointer(&nodes[0])),
		(*C.int64_t)(unsafe.Pointer(&scores[0]))))
	return nodes, scores, err
}

// Reasons returns the reason rows of pods [pod0, pod0+n) of the last round (engine created with BS_OUT_REASONS) as
// dense [n][4+lanes] counters: bin b of a row = the nodes that reject the pod for reason b (BS_REASON_*).
func (e *Engine) Reasons(pod0, n int) ([]uint32, error) {
	counts := make([]uint32, n*(4+e.lanes))
	if len(counts) == 0 {
		var none C.uint32_t
		return counts, e.rc(C.bs_fetch_reason_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), &none))
	}
	err := e.rc(C.bs_fetch_reason_rows(e.h, C.uint32_t(pod0), C.uint32_t(n), (*C.uint32_t)(unsafe.Pointer(&counts[0]))))
	return counts, err
}

// FitError formats one reason row (4 + lanes counters) as kube-scheduler's FailedScheduling message,
// "0/<nNodes> nodes are available: ...", naming lanes 4.. by scalarNames (nil: "lane<d>").  Needs no engine.
func FitError(counts []uint32, nNodes int, scalarNames []string) (string, error) {
	return FitErrorInterPod(counts, nil, nNodes, scalarNames)
}

// FitErrorInterPod is FitError with the row's MatchInterPodAffinity companion (E, A, N from FetchInterPodReasonRows)
// as further entries (bs_format_fit_error_interpod); a nil interPod is FitError.
func FitErrorInterPod(counts, interPod []uint32, nNodes int, scalarNames []string) (string, error) {
	return FitErrorFilters(counts, interPod, nil, nNodes, scalarNames)
}

// FitErrorFilters is FitError with both filters' companions (nil: absent): interPod as FitErrorInterPod, hostPorts the
// one counter of FetchHostPortReasonRows (bs_format_fit_error_filters).
func FitErrorFilters(counts, interPod, hostPorts []uint32, nNodes int, scalarNames []string) (string, error) {
	lanes := len(counts) - 4
	if lanes < C.BS_FIXED_LANES {
		return "", fmt.Errorf("bs_format_fit_error: a reason row has 4 + lanes bins")
	}
	var ip *C.uint32_t
	if interPod != nil {
		if len(interPod) != 3 {
			return "", fmt.Errorf("bs_format_fit_error_interpod: a companion row has 3 counters")
		}
		ip = (*C.uint32_t)(unsafe.Pointer(&interPod[0]))
	}
	var hp *C.uint32_t
	if hostPorts != nil {
		if len(hostPorts) != 1 {
			return "", fmt.Errorf("bs_format_fit_error_filters: a host-port companion row has 1 counter")
		}
		hp = (*C.uint32_t)(unsafe.Pointer(&hostPorts[0]))
	}
	var names **C.char
	if len(scalarNames) > 0 {
		arr := C.malloc(C.size_t(len(scalarNames)) * C.size_t(unsafe.Sizeof(uintptr(0))))
		defer C.free(arr)
		view := unsafe.Slice((**C.char)(arr), len(scalarNames))
		for i, s := range scalarNames {
			view[i] = C.CString(s)
			defer C.free(unsafe.Pointer(view[i]))
		}
		names = (**C.char)(arr)
	}
	for size := 512; size <= 1<<20; size *= 4 {
		buf := (*C.char)(C.malloc(C.size_t(size)))
		rc := C.bs_format_fit_error_filters((*C.uint32_t)(unsafe.Pointer(&counts[0])), C.uint32_t(lanes), ip, hp,
			C.uint32_t(nNodes), names, buf, C.size_t(size))
		msg := C.GoString(buf)
		C.free(unsafe.Pointer(buf))
		if rc == 0 {
			return msg, nil
		}
	}
	return "", fmt.Errorf("bs_format_fit_error: %s", C.GoString(C.bs_strerror(C.BS_E_INVAL)))
}

// PreFilter mirrors ScheduleOperation.PreFilter(pod) error (core.go:88): nil == pass.
func (e *Engine) PreFilter(pod uint32, nsName, occupiedBy string) error {
	var st C.bs_status
	if err := e.rc(C.bs_prefilter(e.h, C.uint32_t(pod), &st)); err != nil {
		return err
	}
	if st.reason == C.BS_PF_PASS {
		return nil
	}
	buf := (*C.char)(C.malloc(512))
	defer C.free(unsafe.Pointer(buf))
	cn, co := C.CString(nsName), C.CString(occupiedBy)
	defer C.free(unsafe.Pointer(cn))
	defer C.free(unsafe.Pointer(co))
	C.bs_format_message(&st, cn, co, buf, 512)
	return fmt.Errorf("%s", C.GoString(buf)) // the adapter turns it into framework.Unschedulable (batchscheduler.go:104-107)
}

// Bound-pod flags (bs_bound_table.flags): the pod's PodGroup is Scheduled or Running; the pod violates a
// PodDisruptionBudget (filterPodsWithPDBViolation's verdict, which preemption reprieves first and ranks nodes by).
const (
	BoundGroupLocked  = C.BS_BOUND_GROUP_LOCKED
	BoundPDBViolating = C.BS_BOUND_PDB_VIOLATING
)

// UploadBoundPods uploads the pods bound to the snapshot's nodes (NodeInfo.Pods()): what preemption may evict.
// Upload nodes and groups first; either upload, and UpdateNodes, drop the table.
func (e *Engine) UploadBoundPods(t *C.bs_bound_table) error { return e.rc(C.bs_upload_bound_pods(e.h, t)) }

// RemovePod mirrors batchSchedulingPluginExtension.RemovePod (batchscheduler.go:132-144) ->
// core.PreemptRemovePod (core.go:203-260) for pod row `pod` and bound-pod row `bound`: nil == the victim may go.
// victimGroup is "namespace/pgName" of the victim's group (the not-found message names it).
func (e *Engine) RemovePod(pod, bound uint32, podName, victimName, victimGroup string) error {
	var st C.bs_status
	if err := e.rc(C.bs_remove_pod(e.h, C.uint32_t(pod), C.uint32_t(bound), &st)); err != nil {
		return err
	}
	if st.reason == C.BS_REMOVE_ALLOW {
		return nil
	}
	buf := (*C.char)(C.malloc(1024))
	defer C.free(unsafe.Pointer(buf))
	cp, cv, cg := C.CString(podName), C.CString(victimName), C.CString(victimGroup)
	defer C.free(unsafe.Pointer(cp))
	defer C.free(unsafe.Pointer(cv))
	defer C.free(unsafe.Pointer(cg))
	if err := e.rc(C.bs_format_remove_message(&st, cp, cv, cg, buf, 1024)); err != nil {
		return err
	}
	return fmt.Errorf("%s", C.GoString(buf)) // the adapter turns it into framework.Unschedulable (batchscheduler.go:137-141)
}

// Preemption is one preemptor's answer: the snapshot index of the node preemption would pick (-1 none) and the
// bound-pod rows it would evict there: the BoundPDBViolating ones first, then the others, each part most important
// first.
type Preemption struct {
	Node       int32
	Victims    []uint32
	Candidates uint32
}

// Preempt mirrors genericScheduler.Preempt's node and victim choice for every pod row in pods, against the uploaded
// snapshot and bound-pod table (bs_preempt; DESIGN.md §2 "Preemption").
func (e *Engine) Preempt(pods []uint32) ([]Preemption, error) {
	n := len(pods)
	out := make([]Preemption, n)
	if n == 0 {
		return out, nil
	}
	node := make([]int32, n)
	nv := make([]uint32, n)
	cand := make([]uint32, n)
	off := make([]uint32, n+1)
	r := C.bs_preempt_result{node: (*C.int32_t)(unsafe.Pointer(&node[0])), n_victims: (*C.uint32_t)(unsafe.Pointer(&nv[0])),
		n_candidates: (*C.uint32_t)(unsafe.Pointer(&cand[0])), victim_offset: (*C.uint32_t)(unsafe.Pointer(&off[0]))}
	p := (*C.uint32_t)(unsafe.Pointer(&pods[0]))
	rc := C.bs_preempt(e.h, p, C.uint32_t(n), &r)
	var victims []uint32
	if rc == C.BS_E_INVAL && r.victims_total > 0 { // the first call sized the victim list
		victims = make([]uint32, int(r.victims_total))
		r.victims = (*C.uint32_t)(unsafe.Pointer(&victims[0]))
		r.victims_cap = r.victims_total
		rc = C.bs_preempt(e.h, p, C.uint32_t(n), &r)
	}
	if err := e.rc(rc); err != nil {
		return nil, err
	}
	for i := 0; i < n; i++ {
		out[i] = Preemption{Node: node[i], Victims: append([]uint32(nil), victims[off[i]:off[i+1]]...), Candidates: cand[i]}
	}
	return out, nil
}

// WalkOutcome is one preemptor's outcome in PreemptWalk (bs_walk_outcome).
type WalkOutcome uint32

const (
	WalkNone       WalkOutcome = C.BS_WALK_NONE        // no candidate node
	WalkNominated  WalkOutcome = C.BS_WALK_NOMINATED   // nominated to Node; its victims are evicted
	WalkRolledBack WalkOutcome = C.BS_WALK_ROLLED_BACK // a member of its gang unit got no node: the unit was undone
)

// PreemptWalk preempts for the pod rows of pods one after another, as kube-scheduler does one pod per cycle: each
// preemptor sees the evictions and nominations of those before it (bs_preempt_walk; DESIGN.md §2 "Preemption").
// Priorities must not rise along pods.  With gang, the rows of one group must be contiguous, and a group gets nodes
// for all its rows or for none.  evictedBy[v] is the position in pods whose step evicted bound-pod row v, or -1.
func (e *Engine) PreemptWalk(pods []uint32, gang bool, nBound int) (out []Preemption, outcome []WalkOutcome,
	evictedBy []int32, err error) {
	n := len(pods)
	out = make([]Preemption, n)
	outcome = make([]WalkOutcome, n)
	evictedBy = make([]int32, nBound+1)
	node := make([]int32, n+1)
	nv := make([]uint32, n+1)
	cand := make([]uint32, n+1)
	off := make([]uint32, n+1)
	oc := make([]uint32, n+1)
	flags := C.uint32_t(0)
	if gang {
		flags = C.BS_PREEMPT_GANG
	}
	r := C.bs_preempt_result{node: (*C.int32_t)(unsafe.Pointer(&node[0])), n_victims: (*C.uint32_t)(unsafe.Pointer(&nv[0])),
		n_candidates: (*C.uint32_t)(unsafe.Pointer(&cand[0])), victim_offset: (*C.uint32_t)(unsafe.Pointer(&off[0]))}
	var p *C.uint32_t
	if n > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&pods[0]))
	}
	call := func() C.int {
		return C.bs_preempt_walk(e.h, p, C.uint32_t(n), flags, &r, (*C.uint32_t)(unsafe.Pointer(&oc[0])),
			(*C.int32_t)(unsafe.Pointer(&evictedBy[0])))
	}
	rc := call()
	var victims []uint32
	if rc == C.BS_E_INVAL && r.victims_total > 0 { // the first call sized the victim list
		victims = make([]uint32, int(r.victims_total))
		r.victims = (*C.uint32_t)(unsafe.Pointer(&victims[0]))
		r.victims_cap = r.victims_total
		rc = call()
	}
	if err := e.rc(rc); err != nil {
		return nil, nil, nil, err
	}
	for i := 0; i < n; i++ {
		out[i] = Preemption{Node: node[i], Victims: append([]uint32(nil), victims[off[i]:off[i+1]]...), Candidates: cand[i]}
		outcome[i] = WalkOutcome(oc[i])
	}
	return out, outcome, evictedBy[:nBound], nil
}

// Permit mirrors batchSchedulingPlugin.Permit (batchscheduler.go:165-202) with core.Permit's bookkeeping
// (core.go:268-309) against the engine's tables: ready only once len(MatchedPodNodes.Items()) reaches
// MinMember - Status.Scheduled.
func (e *Engine) Permit(pod, node uint32, now time.Time) (code int, wait time.Duration, startSignal bool, err error) {
	var r C.bs_permit_result
	if err = e.rc(C.bs_permit_at(e.h, C.uint32_t(pod), C.uint32_t(node), C.int64_t(now.UnixNano()), &r)); err != nil {
		return
	}
	return int(r.code), time.Duration(r.wait_ns), r.start_signal != 0, nil
}

// Expire is one janitor tick (controller.go:322-333): the uids to Reject ("Group failed",
// batchscheduler.go:347-354) and the evicted groups (deny-listed for 20 s inside the engine).
func (e *Engine) Expire(now time.Time, maxPods, maxGroups int) (rejGroup []uint32, rejUID []uint64, evicted []uint32, err error) {
	rejGroup, rejUID, evicted = make([]uint32, maxPods), make([]uint64, maxPods), make([]uint32, maxGroups)
	var nr, ne C.uint32_t
	err = e.rc(C.bs_expire(e.h, C.int64_t(now.UnixNano()), (*C.uint32_t)(unsafe.Pointer(&rejGroup[0])),
		(*C.uint64_t)(unsafe.Pointer(&rejUID[0])), C.uint32_t(maxPods), &nr,
		(*C.uint32_t)(unsafe.Pointer(&evicted[0])), C.uint32_t(maxGroups), &ne))
	return rejGroup[:nr], rejUID[:nr], evicted[:ne], err
}

// AllowList is StartBatchSchedule's loop (batchscheduler.go:292-344): the waiting pods of a complete gang.
func (e *Engine) AllowList(group uint32, now time.Time, max int) (uids []uint64, nodes []uint32, err error) {
	uids, nodes = make([]uint64, max), make([]uint32, max)
	var n C.uint32_t
	err = e.rc(C.bs_allow_list(e.h, C.uint32_t(group), C.int64_t(now.UnixNano()), (*C.uint64_t)(unsafe.Pointer(&uids[0])),
		(*C.uint32_t)(unsafe.Pointer(&nodes[0])), C.uint32_t(max), &n))
	return uids[:n], nodes[:n], err
}

func (e *Engine) Deny(group uint32, now time.Time) error { // AddToDenyCache core.go:423
	return e.rc(C.bs_deny(e.h, C.uint32_t(group), C.int64_t(now.UnixNano())))
}
func (e *Engine) MarkPermitted(uid uint64, now time.Time) error { // core.go:188
	return e.rc(C.bs_mark_permitted(e.h, C.uint64_t(uid), C.int64_t(now.UnixNano())))
}

// Less mirrors batchSchedulingPlugin.Less (batchscheduler.go:214) for two pods of the evaluated round: a read of
// the rank the device sort produced.  Pods the round has not seen go through ScheduleOperation.Compare as before.
func (e *Engine) Less(a, b uint32) bool { return C.bs_less(e.h, C.uint32_t(a), C.uint32_t(b)) == 1 }

// Replay walks the whole queue (pod rows in pop order) through the reference's cycle — PreFilter on the live
// state, assume onto the first fitting node, Permit — on the device; a what-if that leaves the uploaded tables as
// they are.  The three slices are C-allocated by the caller (len(queue) each).
func (e *Engine) Replay(queue []uint32, prefilter *C.uint8_t, node *C.int32_t, ready *C.uint8_t) error {
	r := C.bs_replay_result{prefilter: prefilter, node: node, ready: ready}
	return e.rc(C.bs_replay(e.h, (*C.uint32_t)(unsafe.Pointer(&queue[0])), C.uint32_t(len(queue)), &r))
}

// ReplayPriority is Replay with kube-scheduler's node choice: each passing pod goes to its best fitting node under the
// resource priorities (SetScoreWeights) on the live state.  Both non-zero columns must be uploaded
// (UploadNodeNonZero, UploadPodNonZero).  nodeNonZeroAfter ([2][n_nodes], C-allocated) may be nil.
func (e *Engine) ReplayPriority(queue []uint32, prefilter *C.uint8_t, node *C.int32_t, ready *C.uint8_t,
	nodeNonZeroAfter *C.int64_t) error {
	r := C.bs_replay_result{prefilter: prefilter, node: node, ready: ready}
	return e.rc(C.bs_replay_priority(e.h, (*C.uint32_t)(unsafe.Pointer(&queue[0])), C.uint32_t(len(queue)), &r,
		nodeNonZeroAfter))
}

// ---- several GPUs: one process per GPU, groups sharded; the admit bitmaps are all-gathered over NVLink peer
// memory at the end of every round.
func (e *Engine) PeerInit(rank, world, words uint32) error {
	return e.rc(C.bs_peer_init(e.h, C.uint32_t(rank), C.uint32_t(world), C.uint32_t(words)))
}
func (e *Engine) PeerHandle() (h [64]byte, err error) {
	err = e.rc(C.bs_peer_handle(e.h, (*C.uchar)(unsafe.Pointer(&h[0]))))
	return
}
func (e *Engine) PeerAttach(handles []byte) error { // world * 64 bytes, exchanged out of band
	return e.rc(C.bs_peer_attach(e.h, (*C.uchar)(unsafe.Pointer(&handles[0]))))
}
func (e *Engine) PeerDetach() error { return e.rc(C.bs_peer_detach(e.h)) }
func (e *Engine) GatheredAdmit(words []uint32) error { // [world][words_per_rank]
	return e.rc(C.bs_fetch_gathered_admit(e.h, (*C.uint32_t)(unsafe.Pointer(&words[0]))))
}
