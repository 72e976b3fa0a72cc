/* preempt_walk_ref.c — TEST INFRASTRUCTURE: the CPU restatement of bs_preempt_walk (include/bsched.h), linked against
 * oracle/libbs_oracle.so.  tests/preempt_walk_ref.py compiles and binds it.
 *
 * The walk is restated as the sequential loop over tests/preempt_pdb_ref.c's single-pod preemption (each node a
 * mutated one-node copy, the pick's staged filters), run for one preemptor at a time on a master node state and on
 * the bound pods not yet evicted.  After a pick, the victims leave the master state through preempt_pdb_ref.c's
 * apply() (NodeInfo.RemovePod) and the preemptor is added by the oracle's assume step (bso_replay,
 * oracle/bs_oracle.c: its request on every lane but 3, its scalar keys, one pod more).  A failed gang unit is undone
 * by restoring a copy of the state saved when the unit began.  The engine compacts CSR segments and rebuilds suffix
 * sums instead; the two must agree. */
#include "preempt_pdb_ref.c"

enum { BSW_NONE = 0, BSW_NOMINATED = 1, BSW_ROLLED_BACK = 2 };

/* The walk over pods[0..n).  unit_last[i]: step i closes its unit (every step without gangs); gang: a unit with a
 * member without a node is undone.  Per step: node_out, nv_out, cand_out, outcome; the victims in step order at
 * victims[0 ..) (capacity b->n); evicted_by[b->n]: the step that evicted each row, or -1.  Returns the victim count. */
uint32_t bsw_walk(const bso_nodes* nd0, const bso_pods* pd, const bsp_bound* b, const uint32_t* pods, uint32_t n,
                  const uint8_t* unit_last, int gang, int32_t* node_out, uint32_t* nv_out, uint32_t* cand_out,
                  uint32_t* outcome, uint32_t* victims, int32_t* evicted_by) {
  const uint32_t N = nd0->n, L = nd0->lanes, V = b->n;
  const size_t nl = (size_t)L * N + 1;
  /* the master node state and its copy at the start of the open unit */
  int64_t* req = malloc(nl * 8);
  int64_t* req_save = malloc(nl * 8);
  int32_t* pc = malloc(((size_t)N + 1) * 4);
  int32_t* pc_save = malloc(((size_t)N + 1) * 4);
  uint32_t* rp = malloc(((size_t)N + 1) * 4);
  uint32_t* rp_save = malloc(((size_t)N + 1) * 4);
  int32_t* ev_save = malloc(((size_t)V + 1) * 4);
  memcpy(req, nd0->requested, (size_t)L * N * 8);
  memcpy(pc, nd0->pod_count, (size_t)N * 4);
  memcpy(rp, nd0->req_present, (size_t)N * 4);
  bso_nodes nd = *nd0;
  nd.requested = req;
  nd.pod_count = pc;
  nd.req_present = rp;
  /* the bound pods not yet evicted, in table order, and their table indices */
  const size_t vl = (size_t)L * V + 1;
  uint32_t* l_node = malloc(((size_t)V + 1) * 4);
  int64_t* l_req = malloc(vl * 8);
  uint32_t* l_rp = malloc(((size_t)V + 1) * 4);
  int32_t* l_gid = malloc(((size_t)V + 1) * 4);
  int32_t* l_prio = malloc(((size_t)V + 1) * 4);
  int64_t* l_start = malloc(((size_t)V + 1) * 8);
  uint8_t* l_flags = malloc((size_t)V + 1);
  uint32_t* l_orig = malloc(((size_t)V + 1) * 4);
  uint32_t* vict = malloc(((size_t)V + 1) * 4);
  node_copy c;
  c.aff = malloc((nd.n_aff + 1) * 4);
  for (uint32_t v = 0; v < V; ++v) evicted_by[v] = -1;
  uint32_t voff = 0, voff_save = 0, unit_first = 0;
  int failed = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (i == unit_first && gang) {
      memcpy(req_save, req, (size_t)L * N * 8);
      memcpy(pc_save, pc, (size_t)N * 4);
      memcpy(rp_save, rp, (size_t)N * 4);
      memcpy(ev_save, evicted_by, (size_t)V * 4);
      voff_save = voff;
    }
    uint32_t m = 0;
    for (uint32_t v = 0; v < V; ++v) {
      if (evicted_by[v] >= 0) continue;
      l_node[m] = b->node[v];
      l_rp[m] = b->req_present[v];
      l_gid[m] = b->gid[v];
      l_prio[m] = b->priority[v];
      l_start[m] = b->start_ns[v];
      l_flags[m] = b->flags[v];
      l_orig[m] = v;
      ++m;
    }
    for (uint32_t d = 0; d < L; ++d)
      for (uint32_t k = 0; k < m; ++k) l_req[(size_t)d * m + k] = b->req[(size_t)d * V + l_orig[k]];
    const bsp_bound live = {m, L, l_node, l_req, l_rp, l_gid, l_prio, l_start, l_flags};
    int32_t node;
    uint32_t nv, cand;
    bsp_preempt(&nd, pd, &live, &pods[i], 1, &node, &nv, &cand, vict, m ? m : 1, 1);
    cand_out[i] = cand;
    if (node < 0) {
      node_out[i] = -1;
      nv_out[i] = 0;
      outcome[i] = BSW_NONE;
      failed = 1;
    } else {
      node_out[i] = node;
      nv_out[i] = nv;
      outcome[i] = BSW_NOMINATED;
      /* evict: NodeInfo.RemovePod on the master state */
      copy_node(&c, &nd, (uint32_t)node);
      for (uint32_t j = 0; j < nv; ++j) {
        const uint32_t v = l_orig[vict[j]];
        victims[voff++] = v;
        evicted_by[v] = (int32_t)i;
        apply(&c, b, v, -1);
      }
      for (uint32_t d = 0; d < L; ++d) req[(size_t)d * N + node] = c.requested[d];
      pc[node] = c.pod_count;
      /* nominate: the oracle's assume (NodeInfo.AddPod) */
      const uint32_t p = pods[i];
      for (uint32_t d = 0; d < L; ++d) {
        if (d == 3) continue;   /* the pods lane */
        if (d >= 4 && !(pd->req_present[p] & (1u << d))) continue;
        req[(size_t)d * N + node] += pd->req[(size_t)d * pd->n + p];
        if (d >= 4) rp[node] |= 1u << d;
      }
      pc[node] += 1;
    }
    if (!unit_last[i]) continue;
    if (gang && failed) {
      memcpy(req, req_save, (size_t)L * N * 8);
      memcpy(pc, pc_save, (size_t)N * 4);
      memcpy(rp, rp_save, (size_t)N * 4);
      memcpy(evicted_by, ev_save, (size_t)V * 4);
      voff = voff_save;
      for (uint32_t k = unit_first; k <= i; ++k) {
        node_out[k] = -1;
        nv_out[k] = 0;
        outcome[k] = BSW_ROLLED_BACK;
      }
    }
    failed = 0;
    unit_first = i + 1;
  }
  free(c.aff); free(vict); free(l_orig); free(l_flags); free(l_start); free(l_prio); free(l_gid); free(l_rp);
  free(l_req); free(l_node); free(ev_save); free(rp_save); free(rp); free(pc_save); free(pc); free(req_save); free(req);
  return voff;
}
