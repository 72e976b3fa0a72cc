/* host_ports_ref.c — TEST INFRASTRUCTURE: the CPU restatement of kube-scheduler v1.17's PodFitsHostPorts predicate as
 * the engine applies it (include/bsched.h bs_set_host_port_filter), on the packed columns of bs_upload_node_host_ports
 * and bs_upload_pod_host_ports.  No conflict masks: for each (pod, node) it compares every wanted entry with every used
 * entry.  bsr_hp_choose / bsr_hp_assumed are a chooser / assume hook pair for tests/replay_priority_ref.c's
 * bsr_replay_choose: they wrap another pair (first fit, priority, ratio) and add the filter on a live copy of the used
 * masks.  tests/host_ports_ref.py compiles it into a library of its own. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include "bs_oracle.h"
#include "bs_ref.h"

#define BSR_HP_IP_ANY 0u

typedef struct {
  uint32_t n_entries;
  const uint32_t* ip;        /* [n_entries] */
  const uint32_t* protocol;  /* [n_entries] */
  const int32_t* port;       /* [n_entries] */
} bsr_hp_dict;

static int entries_conflict(const bsr_hp_dict* d, uint32_t w, uint32_t u) {
  if (d->protocol[w] != d->protocol[u] || d->port[w] != d->port[u]) return 0;
  return d->ip[w] == BSR_HP_IP_ANY || d->ip[u] == BSR_HP_IP_ANY || d->ip[w] == d->ip[u];
}

/* 1 when a pod wanting `want` passes a node using `used` */
int bsr_hp_pass(const bsr_hp_dict* d, uint64_t want, uint64_t used) {
  for (uint32_t w = 0; w < d->n_entries; ++w) {
    if (!((want >> w) & 1u)) continue;
    for (uint32_t u = 0; u < d->n_entries; ++u)
      if (((used >> u) & 1u) && entries_conflict(d, w, u)) return 0;
  }
  return 1;
}

/* out[p * n_nodes + n] = bsr_hp_pass of pod p on node n */
void bsr_hp_matrix(const bsr_hp_dict* d, const uint64_t* want, uint32_t n_pods, const uint64_t* used, uint32_t n_nodes,
                   uint8_t* out) {
  for (uint32_t p = 0; p < n_pods; ++p)
    for (uint32_t n = 0; n < n_nodes; ++n) out[(size_t)p * n_nodes + n] = (uint8_t)bsr_hp_pass(d, want[p], used[n]);
}

/* The hook pair's state: the wrapped pair and its context, the dictionary, the live used masks [n_nodes] (updated on
 * every assume) and the pods' want masks [n_pods]. */
typedef struct {
  bsr_choose_fn inner;
  bsr_assumed_fn inner_assumed;   /* may be NULL */
  void* inner_ctx;
  bsr_hp_dict dict;
  uint64_t* live;
  const uint64_t* want;
} bsr_hp_ctx;

/* The wrapped chooser over the nodes without a port conflict: the others are flagged unschedulable while it runs, so
 * that bso_fit_eval skips them, and get their flags back before the walk goes on. */
int32_t bsr_hp_choose(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p) {
  const bsr_hp_ctx* c = (const bsr_hp_ctx*)ctx;
  uint8_t* saved = (uint8_t*)malloc(nd->n ? nd->n : 1);
  for (uint32_t n = 0; n < nd->n; ++n) {
    saved[n] = nd->flags[n];
    if (!bsr_hp_pass(&c->dict, c->want[p], c->live[n])) nd->flags[n] |= BSO_NODE_UNSCHEDULABLE;
  }
  const int32_t r = c->inner(c->inner_ctx, nd, pd, p);
  for (uint32_t n = 0; n < nd->n; ++n) nd->flags[n] = saved[n];
  free(saved);
  return r;
}

/* NodeInfo.AddPod adds the pod's ports to the node's UsedPorts */
void bsr_hp_assumed(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n) {
  const bsr_hp_ctx* c = (const bsr_hp_ctx*)ctx;
  c->live[n] |= c->want[p];
  if (c->inner_assumed) c->inner_assumed(c->inner_ctx, nd, pd, p, n);
}
