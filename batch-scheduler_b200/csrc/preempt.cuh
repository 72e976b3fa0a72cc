// preempt.cuh — sm_90a kernels of bs_preempt: for each preemptor, the node kube-scheduler's preemption would pick and
// the victims it would evict there (genericScheduler.Preempt -> selectVictimsOnNode -> pickOneNodeForPreemption,
// k8s v1.17.5 [upstream, from memory]; DESIGN.md §2 "Preemption"), with the plugin's RemovePod rule
// (core.PreemptRemovePod, core.go:203-260) as the gate on every potential victim.
//
// The bound pods of a node are stored as one CSR segment in MoreImportantPod order (priority descending, start time
// ascending, table index ascending), so the potential victims of a preemptor (priority strictly lower) are a SUFFIX
// of the segment.  preempt_prep_kernel builds, per CSR position, the suffix sums of the removable lanes and the
// suffix counts of the rows RemovePod refuses for some preemptor and of the PodDisruptionBudget-violating rows; the
// hot kernel answers "all victims removed" with one binary search and one suffix read per (preemptor, node) and walks
// the suffix only for the pairs that survive that test.  The oracles in the tests mutate a copy of the node instead:
// the two must agree.
//
// Under the PodFitsHostPorts filter (the HP builds) each CSR position also carries its row's host-port mask and the
// suffix OR of those masks.  Removing every potential victim is a set delete on the node's used mask
// (HostPortInfo.Remove: an entry goes even when a more important row lists it too): base = used & ~suf_ports[s].  The
// node is a candidate when (base | nominated) holds no entry the preemptor conflicts with.  Since neither side of that
// OR conflicts afterwards, re-adding row k in the reprieve conflicts exactly when the row's own mask does: a row holding
// a conflicting port is always a victim.
#pragma once
#include "kernels.cuh"

namespace bsk {

// bound-pod table grouped by node (CSR), columns in CSR position order
struct BoundTab {
  const uint32_t* row;      // [N + 1] segment of node n: [row[n], end[n])
  const uint32_t* end;      // [N] segment ends: row + 1, or bs_preempt_walk's live ends (evicted rows leave)
  const int32_t* prio;      // [V]
  const int64_t* start;     // [V]
  const int32_t* gid;       // [V]
  const uint8_t* flags;     // [V] BS_BOUND_*
  const uint32_t* idx;      // [V] bound-table index
  const int64_t* req;       // [L][V] removable amounts: lanes 0-2 and the row's scalar keys, 0 elsewhere
  const int64_t* suf;       // [L][V] sum of req over positions k .. end of the segment
  const uint32_t* suf_online;   // [V] rows without a group label in k .. end
  const uint32_t* suf_bad;      // [V] rows whose group is missing or Scheduled / Running in k .. end
  const uint32_t* suf_vio;      // [V] rows flagged BS_BOUND_PDB_VIOLATING in k .. end
  uint32_t V;
};

// one preemptor, as the host resolves it from the pod table and its fit class
struct PreemptPod {
  uint64_t sel, tol;
  uint32_t pod;   // pod-table index
  uint32_t nz;    // scalar keys requested with a non-zero amount (the class-fit presence rule)
  uint32_t aff;   // affinity class or BS_AFF_NONE
  int32_t prio, gid;
};

// pickOneNodeForPreemption's order over candidate nodes; the smaller key wins.  A candidate without victims wins
// at once (lowest index); otherwise: PDB-violating victims, the priority of the FIRST victim (upstream's "highest",
// which is the first violating victim when there is one), sum of (priority + 2^31), victim count, LATEST earliest
// start among the victims of the true maximum priority (GetEarliestPodStartTime), node index.  node = -1: none.
struct PickKey {
  int64_t sum;
  int64_t start;
  int32_t hp;
  uint32_t nv;
  uint32_t vio;    // victims flagged BS_BOUND_PDB_VIOLATING (numViolatingVictim)
  int32_t node;
  uint32_t cand;   // candidates counted into this key (not part of the order)
};

__device__ __forceinline__ bool pick_less(const PickKey& a, const PickKey& b) {
  if (a.node < 0) return false;
  if (b.node < 0) return true;
  if ((a.nv == 0) != (b.nv == 0)) return a.nv == 0;
  if (a.nv != 0) {
    if (a.vio != b.vio) return a.vio < b.vio;
    if (a.hp != b.hp) return a.hp < b.hp;
    if (a.sum != b.sum) return a.sum < b.sum;
    if (a.nv != b.nv) return a.nv < b.nv;
    if (a.start != b.start) return a.start > b.start;
  }
  return a.node < b.node;
}

__device__ __forceinline__ PickKey pick_min(const PickKey& a, const PickKey& b) {
  PickKey r = pick_less(b, a) ? b : a;
  r.cand = a.cand + b.cand;
  return r;
}

__device__ __forceinline__ PickKey pick_none() {
  PickKey k;
  k.sum = 0; k.start = 0; k.hp = 0; k.nv = 0; k.vio = 0; k.node = -1; k.cand = 0;
  return k;
}

// The suffix sums of the removable lanes and the suffix counts of the online, the missing-or-locked and the
// PDB-violating rows of one node's segment [b, e), walking it from its end.
__device__ __forceinline__ void prep_node(uint32_t b, uint32_t e, const int32_t* gid, const uint8_t* flags,
                                          const int64_t* req, int64_t* suf, uint32_t* suf_online, uint32_t* suf_bad,
                                          uint32_t* suf_vio, uint32_t V, uint32_t L) {
  uint32_t on = 0, bad = 0, vio = 0;
  for (uint32_t k = e; k-- > b;) {
    const int32_t g = gid[k];
    const uint8_t f = flags[k];
    on += g == BS_GID_NONE ? 1u : 0u;
    bad += (g == BS_GID_MISSING || (g >= 0 && (f & BS_BOUND_GROUP_LOCKED))) ? 1u : 0u;
    vio += (f & BS_BOUND_PDB_VIOLATING) ? 1u : 0u;
    suf_online[k] = on;
    suf_bad[k] = bad;
    suf_vio[k] = vio;
  }
  for (uint32_t d = 0; d < L; ++d) {
    int64_t s = 0;
    for (uint32_t k = e; k-- > b;) {
      s += req[(size_t)d * V + k];
      suf[(size_t)d * V + k] = s;
    }
  }
}

// ---------------------------------------------------------------------------
// preempt_prep_kernel — once per bound-table upload, one thread per node: prep_node over the node's segment.
__global__ void preempt_prep_kernel(const uint32_t* __restrict__ row, const int32_t* __restrict__ gid,
                                    const uint8_t* __restrict__ flags, const int64_t* __restrict__ req,
                                    int64_t* __restrict__ suf, uint32_t* __restrict__ suf_online,
                                    uint32_t* __restrict__ suf_bad, uint32_t* __restrict__ suf_vio, uint32_t N,
                                    uint32_t V, uint32_t L) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  prep_node(row[n], row[n + 1], gid, flags, req, suf, suf_online, suf_bad, suf_vio, V, L);
}

// The suffix OR of the host-port masks of one node's segment [b, e).
__device__ __forceinline__ void prep_node_ports(uint32_t b, uint32_t e, const uint64_t* ports, uint64_t* suf_ports) {
  uint64_t m = 0;
  for (uint32_t k = e; k-- > b;) {
    m |= ports[k];
    suf_ports[k] = m;
  }
}

// preempt_ports_prep_kernel — once per bound host-port upload, one thread per node: the masks into CSR order (by_row
// is in bound-table order) and their suffix OR.
__global__ void preempt_ports_prep_kernel(const uint32_t* __restrict__ row, const uint32_t* __restrict__ idx,
                                          const uint64_t* __restrict__ by_row, uint64_t* __restrict__ ports,
                                          uint64_t* __restrict__ suf_ports, uint32_t N) {
  const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  for (uint32_t k = row[n]; k < row[n + 1]; ++k) ports[k] = by_row[idx[k]];
  prep_node_ports(row[n], row[n + 1], ports, suf_ports);
}

struct PreemptArgs {
  NodeTab t;                  // node table (guards, masks, affinity bits, requested lane 3)
  const int64_t* left;        // [L][Npad] node_left_kernel's full-width residuals at percent 1.0 (0 = key absent)
  const uint32_t* left_present;   // [Npad] scalar keys of `left`
  BoundTab b;
  const PreemptPod* pp;       // [n] the preemptors
  const int64_t* preq;        // [L][P] pod-table requests
  const uint32_t* preq_present;   // [P]
  uint32_t P, n;
  uint32_t p0;                // first preemptor of this launch (grid.y covers [p0, p0 + gridDim.y))
  PickKey* tiles;             // [gridDim.y][n_tiles] per-(preemptor, node tile) best keys
  uint32_t n_tiles;
  // reduce + emit
  int32_t* out_node;
  uint32_t* out_nv;
  uint32_t* out_cand;
  const uint32_t* offset;     // [n] exclusive scan of out_nv (emit)
  uint32_t* victims;          // emit output
};
// HP's arguments: a derived type, so that the kernels without the filter keep theirs
struct PreemptHpArgs : PreemptArgs {
  const uint64_t* hp_used;    // [Npad] the bound pods' used masks (bs_preempt_walk: live, evictions delete from it)
  const uint64_t* hp_nom;     // [Npad] the nominated pods' want masks (bs_preempt_walk), null in bs_preempt
  const uint64_t* hp_ports;   // [V] each CSR position's host-port mask
  const uint64_t* hp_suf;     // [V] OR of hp_ports over positions k .. end of the segment
  const uint64_t* hp_conf;    // [n] each preemptor's conflict mask (the OR of its wanted entries')
  const uint64_t* hp_want;    // [n] each preemptor's want mask (bs_preempt_walk's nominations)
};
template <bool HP>
using PreemptArgsOf = std::conditional_t<HP, PreemptHpArgs, PreemptArgs>;

// preemptor slot i's conflict mask, 0 without the filter
template <bool HP>
__device__ __forceinline__ uint64_t hp_conf_of(const PreemptArgsOf<HP>& a, uint32_t i) {
  if constexpr (HP) return a.hp_conf[i];
  else return 0;
}

constexpr int PREEMPT_THREADS = 256;   // nodes per tile of the hot kernel

// The fit predicate of the round (bso_fit_eval / the fit bitmap), on a node from which `freed` (per lane) and
// `count` pods have been removed: left[d] + freed[d] >= req[d] on lanes 0-2 and on the scalar keys both sides have,
// and on the pods lane left + count >= req when requested[3] == 0 (len(Pods()) is the pod count then, core.go:650-653),
// else left >= req (lane 3 of requested is not touched by a removal).  The guards, checkFit and the absent-key rule
// do not change under removal (victims' keys are a subset of the node's): they are the gate.
template <int MAXL>
__device__ __forceinline__ bool fits_freed(const int64_t* left, const int64_t* freed, const int64_t* req,
                                           uint32_t cmask, int64_t pods_left, int64_t pods_req) {
  bool ok = pods_left >= pods_req;
#pragma unroll
  for (int d = 0; d < MAXL; ++d)
    if (d != LANE_PODS && ((cmask >> d) & 1u)) ok &= left[d] + freed[d] >= req[d];
  return ok;
}

template <bool B>
struct BoolC {
  static constexpr bool value = B;
};

// selectVictimsOnNode for preemptor slot i on node n.  Returns false when the node is not a candidate; else the
// key of the node, and with EMIT the victims' bound-table indices at out[0..): the PDB-violating victims first, then
// the others, each part in MoreImportantPod order (filterPodsWithPDBViolation splits the potential victims and the
// violating ones are reprieved first).  HP: under the PodFitsHostPorts filter, with conf the preemptor's conflict mask
// (the header's rule: the node's used mask after the set delete, and each reprieved row's own mask).
template <int MAXL, bool EMIT, bool HP>
__device__ bool select_victims(const PreemptArgsOf<HP>& a, const PreemptPod& q, const int64_t* req, uint32_t rpres,
                               uint32_t n, PickKey& key, uint32_t* out, uint64_t conf) {
  const NodeTab& t = a.t;
  const uint8_t f = t.flags[n];
  // the gate: the pod's fit-class bit (guards core.go:606-617 and :639, checkFit :741-759, absent-key rule :688-690)
  if (node_skipped(f) || (f & BS_NODE_TAINTS_ERR) || !check_fit(t.label[n], t.taint[n], q.sel, q.tol) ||
      !aff_ok(t, q.aff, n) || (q.nz & ~a.left_present[n]) != 0)
    return false;
  const uint32_t beg = a.b.row[n], end = a.b.end[n];
  // potential victims: priority strictly below the preemptor's, a suffix of the segment
  uint32_t lo = beg, hi = end;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (a.b.prio[mid] < q.prio) hi = mid;
    else lo = mid + 1;
  }
  const uint32_t s = lo;
  const bool offline = q.gid != BS_GID_NONE;
  if (s < end) {
    // RemovePod refuses some potential victim -> the node is dropped (upstream aborts its selection)
    if (a.b.suf_bad[s] != 0) return false;
    if (offline && a.b.suf_online[s] != 0) return false;
    if (offline && q.gid >= 0)
      for (uint32_t k = s; k < end; ++k)
        if (a.b.gid[k] == q.gid) return false;
  }
  if constexpr (HP) {   // every potential victim's ports leave; the nominated pods' stay
    const uint64_t nom = a.hp_nom ? a.hp_nom[n] : 0ull;
    const uint64_t base = a.hp_used[n] & ~(s < end ? a.hp_suf[s] : 0ull);
    if ((base | nom) & conf) return false;
  }
  const uint32_t cmask = 0x7u | (rpres & a.left_present[n] & ~0xFu);
  const bool pods_by_count = t.requested[(size_t)LANE_PODS * t.Npad + n] == 0;
  int64_t left[MAXL], freed[MAXL];
#pragma unroll
  for (int d = 0; d < MAXL; ++d) {
    left[d] = d < (int)t.L ? a.left[(size_t)d * t.Npad + n] : 0;
    freed[d] = (d < (int)t.L && s < end) ? a.b.suf[(size_t)d * a.b.V + s] : 0;
  }
  const int64_t pods_left = left[LANE_PODS], pods_req = req[LANE_PODS];
  uint32_t removed = end - s;
  if (!fits_freed<MAXL>(left, freed, req, cmask, pods_left + (pods_by_count ? removed : 0), pods_req)) return false;
  // reprieve, most important first: add each back; keep it when the pod still fits, else it is a victim.  With
  // PDB-violating potential victims, two passes over the suffix: the violating rows, then the others.
  key = pick_none();
  key.node = (int32_t)n;
  key.cand = 1;
  int32_t maxp = 0;   // the highest victim priority so far; key.start is the earliest start among its victims
  // one reprieve step on row k.  SPLIT: the walk is the two-pass one, whose victims are not in priority order, so
  // the start criterion follows the running maximum; in the single pass the first victim has the maximum priority
  // and the earliest start among it.
  auto reprieve = [&](uint32_t k, bool vio, auto split_c) {
    constexpr bool SPLIT = decltype(split_c)::value;
#pragma unroll
    for (int d = 0; d < MAXL; ++d)
      if (d < (int)t.L) freed[d] -= a.b.req[(size_t)d * a.b.V + k];
    --removed;
    if constexpr (HP) {
      if (fits_freed<MAXL>(left, freed, req, cmask, pods_left + (pods_by_count ? removed : 0), pods_req) &&
          (a.hp_ports[k] & conf) == 0)
        return;
    } else {
      if (fits_freed<MAXL>(left, freed, req, cmask, pods_left + (pods_by_count ? removed : 0), pods_req)) return;
    }
#pragma unroll
    for (int d = 0; d < MAXL; ++d)
      if (d < (int)t.L) freed[d] += a.b.req[(size_t)d * a.b.V + k];
    ++removed;
    const int32_t pr = a.b.prio[k];
    if (key.nv == 0) {
      key.hp = pr;
      key.start = a.b.start[k];
      maxp = pr;
    } else if (SPLIT && pr >= maxp) {
      const int64_t st = a.b.start[k];
      if (pr > maxp || st < key.start) key.start = st;
      maxp = pr;
    }
    key.sum += (int64_t)pr + ((int64_t)1 << 31);
    if (SPLIT) key.vio += vio ? 1u : 0u;
    if (EMIT) out[key.nv] = a.b.idx[k];
    ++key.nv;
  };
  if (s == end || a.b.suf_vio[s] == 0) {
    for (uint32_t k = s; k < end; ++k) reprieve(k, false, BoolC<false>{});
  } else {   // the violating rows first, then the others, each in MoreImportantPod order
    for (uint32_t k = s; k < end; ++k)
      if (a.b.flags[k] & BS_BOUND_PDB_VIOLATING) reprieve(k, true, BoolC<true>{});
    for (uint32_t k = s; k < end; ++k)
      if (!(a.b.flags[k] & BS_BOUND_PDB_VIOLATING)) reprieve(k, false, BoolC<true>{});
  }
  return true;
}

template <int MAXL>
__device__ __forceinline__ uint32_t load_req(const PreemptArgs& a, const PreemptPod& q, int64_t* req) {
#pragma unroll
  for (int d = 0; d < MAXL; ++d) req[d] = d < (int)a.t.L ? a.preq[(size_t)d * a.P + q.pod] : 0;
  return a.preq_present[q.pod];
}

// The smallest key of a PREEMPT_THREADS-thread block (pick_min over the warps, then over the warp minima), valid in
// thread 0.
__device__ __forceinline__ PickKey block_pick_min(PickKey key) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    PickKey k2;
    k2.sum = __shfl_down_sync(0xffffffffu, key.sum, o);
    k2.start = __shfl_down_sync(0xffffffffu, key.start, o);
    k2.hp = __shfl_down_sync(0xffffffffu, key.hp, o);
    k2.nv = __shfl_down_sync(0xffffffffu, key.nv, o);
    k2.vio = __shfl_down_sync(0xffffffffu, key.vio, o);
    k2.node = __shfl_down_sync(0xffffffffu, key.node, o);
    k2.cand = __shfl_down_sync(0xffffffffu, key.cand, o);
    key = pick_min(key, k2);
  }
  __shared__ PickKey s_key[PREEMPT_THREADS / 32];
  if ((threadIdx.x & 31) == 0) s_key[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < PREEMPT_THREADS / 32; ++w) key = pick_min(key, s_key[w]);
  return key;
}

// preempt_node_kernel — the hot path: block (tile, preemptor) evaluates PREEMPT_THREADS nodes for one preemptor and
// writes the tile's best key (and its candidate count).  The key is a total order (the node index decides last),
// so the tree below gives the same winner as a walk in node order.  At MAXL 5 the bound holds 64 registers, four
// blocks per SM, without spills (the PDB pass would otherwise take it to 72 and three blocks).
template <int MAXL, bool HP>
__global__ void __launch_bounds__(PREEMPT_THREADS, MAXL <= 5 ? 4 : 1) preempt_node_kernel(PreemptArgsOf<HP> a) {
  const uint32_t i = a.p0 + blockIdx.y;
  const uint32_t n = blockIdx.x * PREEMPT_THREADS + threadIdx.x;
  const PreemptPod q = a.pp[i];
  int64_t req[MAXL];
  const uint32_t rpres = load_req<MAXL>(a, q, req);
  const uint64_t conf = hp_conf_of<HP>(a, i);
  PickKey key = pick_none();
  if (n < a.t.N && !select_victims<MAXL, false, HP>(a, q, req, rpres, n, key, nullptr, conf)) key = pick_none();
  key = block_pick_min(key);
  if (threadIdx.x == 0) a.tiles[(size_t)blockIdx.y * a.n_tiles + blockIdx.x] = key;
}

// preempt_reduce_kernel — one thread per preemptor of the launch: the tiles in node order
__global__ void preempt_reduce_kernel(PreemptArgs a, uint32_t count) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  PickKey r = pick_none();
  for (uint32_t tl = 0; tl < a.n_tiles; ++tl) r = pick_min(r, a.tiles[(size_t)j * a.n_tiles + tl]);
  const uint32_t i = a.p0 + j;
  a.out_node[i] = r.node;
  a.out_nv[i] = r.node >= 0 ? r.nv : 0u;
  a.out_cand[i] = r.cand;
}

// preempt_emit_kernel — one thread per preemptor with a node: the reprieve again on that node, writing the victims
template <int MAXL, bool HP>
__global__ void preempt_emit_kernel(PreemptArgsOf<HP> a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int32_t n = a.out_node[i];
  if (n < 0 || a.out_nv[i] == 0) return;
  const PreemptPod q = a.pp[i];
  int64_t req[MAXL];
  const uint32_t rpres = load_req<MAXL>(a, q, req);
  PickKey key;
  select_victims<MAXL, true, HP>(a, q, req, rpres, (uint32_t)n, key, a.victims + a.offset[i], hp_conf_of<HP>(a, i));
}

// ---------------------------------------------------------------------------
// bs_preempt_walk (DESIGN.md §2 "Preemption"): the preemptors in list order over a private copy of the node and bound
// state.  Step i is preempt_node_kernel for preemptor i against the live state, then preempt_commit_kernel, which
// picks the node, writes the victims, evicts them (the segment is compacted in order and its suffixes rebuilt),
// nominates the preemptor (bs_replay's assume) and rebuilds the node's residuals.  With gang units, every commit of
// the open unit is logged, and the unit's last step undoes the unit from the log when a member got no node.

enum : uint32_t { WALK_NONE = 0, WALK_NOMINATED = 1, WALK_ROLLED_BACK = 2 };   // BS_WALK_*

// the walk's running counters (device memory, zeroed once per call)
struct WalkCtl {
  uint32_t voff;         // victims written so far
  uint32_t unit_first;   // first step of the open unit
  uint32_t unit_voff;    // voff when the open unit began
  uint32_t failed;       // a member of the open unit got no node
  uint32_t n_ent;        // log entries of the open unit
  uint32_t n_rows;       // logged rows of the open unit
};

struct WalkArgs {
  // the live copies behind PreemptArgs' const views (a.b, a.t.requested / req_present / pod_count, a.left)
  uint32_t* end;
  int32_t* prio;
  int64_t* start;
  int32_t* gid;
  uint8_t* flags;
  uint32_t* idx;
  int64_t* req;
  int64_t* suf;
  uint32_t *suf_online, *suf_bad, *suf_vio;
  int64_t* requested;       // [L][Npad]
  uint32_t* req_present;    // [Npad]
  int32_t* pod_count;       // [Npad]
  int64_t* left;            // [L][Npad]
  uint32_t* left_present;   // [Npad]
  int32_t* evicted_by;      // [V] by bound-table index: the step that evicted the row, -1
  uint32_t* outcome;        // [n] WALK_*
  const uint8_t* unit_last; // [n] step i closes its unit
  WalkCtl* ctl;
  // the undo log of the open unit (gang units only; null otherwise): per commit the node, its segment end, victim
  // count and first logged row, and its requested / req_present / pod_count before the commit; per evicted row its
  // position in the segment before the commit and its columns
  uint32_t *ent_node, *ent_end, *ent_nv, *ent_row;
  int64_t* ent_req;         // [L][n]
  uint32_t* ent_rp;
  int32_t* ent_pc;
  uint32_t* row_pos;        // [V]
  int32_t* row_prio;
  int64_t* row_start;
  int32_t* row_gid;
  uint8_t* row_flags;
  uint32_t* row_idx;
  int64_t* row_req;         // [L][V]
  uint32_t n;
};
// HP's live state and its share of the undo log: derived, so that the kernels without the filter keep theirs
struct WalkHpArgs : WalkArgs {
  uint64_t* used;           // [Npad] the bound pods' used masks (PreemptHpArgs::hp_used): evictions set-delete
  uint64_t* nom;            // [Npad] the nominated pods' want masks (PreemptHpArgs::hp_nom): nominations OR in
  uint64_t* ports;          // [V] each live CSR position's mask (PreemptHpArgs::hp_ports)
  uint64_t* suf_ports;      // [V] their suffix OR (PreemptHpArgs::hp_suf)
  uint64_t *ent_used, *ent_nom;   // [n] per commit: the node's two masks before it
  uint64_t* row_ports;      // [V] per logged row: its mask
};
template <bool HP>
using WalkArgsOf = std::conditional_t<HP, WalkHpArgs, WalkArgs>;

// Rebuilds node n's suffixes and residuals from its live segment and its live requested / req_present / pod_count.
__device__ __forceinline__ void walk_refresh_node(const PreemptArgs& a, const WalkArgs& w, uint32_t n) {
  const uint32_t V = a.b.V, L = a.t.L;
  prep_node(a.b.row[n], w.end[n], w.gid, w.flags, w.req, w.suf, w.suf_online, w.suf_bad, w.suf_vio, V, L);
  const uint32_t both = node_left_keys(a.t, n);
  for (uint32_t d = 0; d < L; ++d) {
    bool pres;
    const int64_t v = node_lane_left(a.t, n, both, d, pres);
    w.left[(size_t)d * a.t.Npad + n] = pres ? v : 0;
  }
  w.left_present[n] = both;
}

// Step i's pick, victims, eviction and nomination, and at the end of a failed unit its undo.  One CTA; the tiles of
// preempt_node_kernel are reduced by the whole block, the rest runs on thread 0 (one node's segment).
template <int MAXL, bool HP>
__global__ void __launch_bounds__(PREEMPT_THREADS) preempt_commit_kernel(PreemptArgsOf<HP> a, WalkArgsOf<HP> w,
                                                                         uint32_t i) {
  PickKey key = pick_none();
  for (uint32_t tl = threadIdx.x; tl < a.n_tiles; tl += PREEMPT_THREADS) key = pick_min(key, a.tiles[tl]);
  key = block_pick_min(key);
  if (threadIdx.x != 0) return;
  WalkCtl& c = *w.ctl;
  const uint32_t L = a.t.L, V = a.b.V, Npad = a.t.Npad;
  a.out_cand[i] = key.cand;
  if (key.node < 0) {
    a.out_node[i] = -1;
    a.out_nv[i] = 0;
    w.outcome[i] = WALK_NONE;
    c.failed = 1;
  } else {
    const uint32_t n = (uint32_t)key.node;
    const PreemptPod q = a.pp[i];
    int64_t req[MAXL];
    const uint32_t rpres = load_req<MAXL>(a, q, req);
    uint32_t* vict = a.victims + c.voff;
    PickKey k2;
    select_victims<MAXL, true, HP>(a, q, req, rpres, n, k2, vict, hp_conf_of<HP>(a, i));
    const uint32_t nv = k2.nv;
    a.out_node[i] = (int32_t)n;
    a.out_nv[i] = nv;
    w.outcome[i] = WALK_NOMINATED;
    c.voff += nv;
    for (uint32_t j = 0; j < nv; ++j) w.evicted_by[vict[j]] = (int32_t)i;
    const uint32_t beg = a.b.row[n], end = w.end[n];
    if (w.ent_node) {   // log the node before the commit
      const uint32_t e = c.n_ent++;
      w.ent_node[e] = n;
      w.ent_end[e] = end;
      w.ent_nv[e] = nv;
      w.ent_row[e] = c.n_rows;
      for (uint32_t d = 0; d < L; ++d) w.ent_req[(size_t)d * w.n + e] = w.requested[(size_t)d * Npad + n];
      w.ent_rp[e] = w.req_present[n];
      w.ent_pc[e] = w.pod_count[n];
      if constexpr (HP) {
        w.ent_used[e] = w.used[n];
        w.ent_nom[e] = w.nom[n];
      }
    }
    // evict: the victims leave the segment (order kept) and NodeInfo.RemovePod takes their Requests
    uint32_t dst = beg;
    for (uint32_t k = beg; k < end; ++k) {
      if (w.evicted_by[w.idx[k]] == (int32_t)i) {
        for (uint32_t d = 0; d < L; ++d) w.requested[(size_t)d * Npad + n] -= w.req[(size_t)d * V + k];
        if constexpr (HP) w.used[n] &= ~w.ports[k];   // HostPortInfo.Remove: a set delete
        if (w.ent_node) {
          const uint32_t r = c.n_rows++;
          w.row_pos[r] = k - beg;
          w.row_prio[r] = w.prio[k];
          w.row_start[r] = w.start[k];
          w.row_gid[r] = w.gid[k];
          w.row_flags[r] = w.flags[k];
          w.row_idx[r] = w.idx[k];
          for (uint32_t d = 0; d < L; ++d) w.row_req[(size_t)d * V + r] = w.req[(size_t)d * V + k];
          if constexpr (HP) w.row_ports[r] = w.ports[k];
        }
        continue;
      }
      if (dst != k) {
        w.prio[dst] = w.prio[k];
        w.start[dst] = w.start[k];
        w.gid[dst] = w.gid[k];
        w.flags[dst] = w.flags[k];
        w.idx[dst] = w.idx[k];
        for (uint32_t d = 0; d < L; ++d) w.req[(size_t)d * V + dst] = w.req[(size_t)d * V + k];
        if constexpr (HP) w.ports[dst] = w.ports[k];
      }
      ++dst;
    }
    w.end[n] = dst;
    // nominate: bs_replay's assume (NodeInfo.AddPod): the pod's request on every lane but 3 and its scalar keys
    for (uint32_t d = 0; d < L; ++d)
      if (d != LANE_PODS && (d < 4 || ((rpres >> d) & 1u)))
        w.requested[(size_t)d * Npad + n] += a.preq[(size_t)d * a.P + q.pod];
    w.req_present[n] |= rpres & ~0xFu;
    w.pod_count[n] += 1 - (int32_t)nv;
    walk_refresh_node(a, w, n);
    if constexpr (HP) {   // the nominated pod's ports, kept apart from the bound ones (addNominatedPods' clone)
      w.nom[n] |= a.hp_want[i];
      prep_node_ports(beg, w.end[n], w.ports, w.suf_ports);
    }
  }
  if (!w.unit_last[i]) return;
  if (c.failed && w.ent_node) {   // undo the unit, last commit first
    for (uint32_t e = c.n_ent; e-- > 0;) {
      const uint32_t n = w.ent_node[e], beg = a.b.row[n], nv = w.ent_nv[e], r0 = w.ent_row[e];
      uint32_t src = w.end[n], j = nv;
      for (uint32_t k = w.ent_end[e]; k-- > beg;) {
        if (j > 0 && beg + w.row_pos[r0 + j - 1] == k) {
          const uint32_t r = r0 + --j;
          w.prio[k] = w.row_prio[r];
          w.start[k] = w.row_start[r];
          w.gid[k] = w.row_gid[r];
          w.flags[k] = w.row_flags[r];
          w.idx[k] = w.row_idx[r];
          for (uint32_t d = 0; d < L; ++d) w.req[(size_t)d * V + k] = w.row_req[(size_t)d * V + r];
          if constexpr (HP) w.ports[k] = w.row_ports[r];
          w.evicted_by[w.row_idx[r]] = -1;
        } else if (--src != k) {
          w.prio[k] = w.prio[src];
          w.start[k] = w.start[src];
          w.gid[k] = w.gid[src];
          w.flags[k] = w.flags[src];
          w.idx[k] = w.idx[src];
          for (uint32_t d = 0; d < L; ++d) w.req[(size_t)d * V + k] = w.req[(size_t)d * V + src];
          if constexpr (HP) w.ports[k] = w.ports[src];
        }
      }
      w.end[n] = w.ent_end[e];
      for (uint32_t d = 0; d < L; ++d) w.requested[(size_t)d * Npad + n] = w.ent_req[(size_t)d * w.n + e];
      w.req_present[n] = w.ent_rp[e];
      w.pod_count[n] = w.ent_pc[e];
      walk_refresh_node(a, w, n);
      if constexpr (HP) {
        w.used[n] = w.ent_used[e];
        w.nom[n] = w.ent_nom[e];
        prep_node_ports(beg, w.end[n], w.ports, w.suf_ports);
      }
    }
    for (uint32_t k = c.unit_first; k <= i; ++k) {
      a.out_node[k] = -1;
      a.out_nv[k] = 0;
      w.outcome[k] = WALK_ROLLED_BACK;
    }
    c.voff = c.unit_voff;
  }
  c.unit_first = i + 1;
  c.unit_voff = c.voff;
  c.failed = 0;
  c.n_ent = 0;
  c.n_rows = 0;
}

}  // namespace bsk
