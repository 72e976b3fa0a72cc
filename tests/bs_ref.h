/* bs_ref.h — TEST INFRASTRUCTURE: the declarations the C restatements share.  tests/native.py compiles every
 * restatement into one library, so each of these has one definition there, checked against this header. */
#ifndef BS_REF_H
#define BS_REF_H

#include <stdint.h>

#include "bs_oracle.h"

/* tests/priority_ref.c: the weighted score of one (requested, capacity) pair per resource, int64 wrapping */
int64_t bsr_priority_score(int64_t r_cpu, int64_t c_cpu, int64_t r_mem, int64_t c_mem, uint32_t w_least, uint32_t w_most,
                           uint32_t w_balanced);

/* tests/replay_priority_ref.c: the node choice of the hooked walk (a node where bso_fit_eval holds on the live tables,
 * or -1), and the hook told which node the pod was assumed onto */
typedef int32_t (*bsr_choose_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p);
typedef void (*bsr_assumed_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n);

/* tests/replay_priority_ref.c: bso_replay with the node choice `choose` (assumed may be NULL); tables mutated in place
 * as bso_replay does */
int bsr_replay_choose(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue, uint32_t n_queue,
                      uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out, bsr_choose_fn choose,
                      bsr_assumed_fn assumed, void* ctx);

#endif
