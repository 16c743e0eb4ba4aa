/* hived_multictx.h — the batches of several contexts on one GPU in one launch.
 *
 * One cluster's batch keeps only a few SMs busy: the device program runs one CTA per group of virtual clusters (at most
 * 16), one CTA per SM.  A process that drives several independent clusters on one device (several Kubernetes clusters
 * served from one host, what-if replays of one trace against quota variants, replicas) can run their batches together:
 * hived_process_events_many launches one kernel in which every listed context gets CTAs of its own.  Contexts share
 * no state, so each batch gives exactly — results, pool, return code, running result hash, counters, last error, host
 * bookkeeping — what hived_process_events(ctx, ...) on that context alone would have given, and the order of the list
 * does not matter.
 *
 * Threads: the caller holds every listed context (the single-writer rule of hived.h).  Contexts that are not listed
 * keep taking turns on the device through the ordinary calls.
 *
 * Concurrent contexts (HIVED_OPT_CONCURRENT, hived.h) may be listed like any other: the call first stops the resident
 * per-call kernel of each listed context (the caller holds it, so none of its calls is in flight) and its next per-call
 * operation starts a new one.  Concurrent contexts that are not listed keep answering their own threads' calls and
 * running their batches during the joint call; the launch leaves one SM per concurrent context of the device to them, so
 * a list may need one more round than it would on an otherwise idle device, and it waits until its largest round's CTAs
 * can all be resident beside their running batches.
 */
#ifndef HIVED_MULTICTX_H_
#define HIVED_MULTICTX_H_
#include "hived.h"
#ifdef __cplusplus
extern "C" {
#endif

#define HIVED_MANY_MAX 16 /* contexts per call */

typedef struct hived_batch {
  hived_ctx* ctx;
  const hived_event_t* events; int32_t n;                 /* as for hived_process_events */
  const uint32_t* suggested_pool; int64_t suggested_words;
  hived_result_t* res; int32_t* pool; int64_t pool_cap;
  int32_t rc;          /* out: what hived_process_events(ctx, ...) would have returned */
  int32_t reserved;
  int64_t pool_used;   /* out: words of `pool` the batch filled */
} hived_batch_t;

/* Runs every batch of the list.  Returns
 *   0                   every batch ran; read each batch's rc;
 *   HIVED_ERR_BAD_SPEC  nothing ran and no context changed: k < 1 or k > HIVED_MANY_MAX, a NULL ctx, a ctx listed twice,
 *                       contexts on different devices, or a ctx staged for a multi-GPU partition (hived_mg_stage,
 *                       hived_multigpu.h);
 *   HIVED_ERR_PLATFORM  the launch failed; every rc is set to it.
 * Contexts whose VC count exceeds what fits on the device next to the others run in further launches of the same
 * call; the results do not depend on that. */
int hived_process_events_many(hived_batch_t* batches, int32_t k);

#ifdef __cplusplus
}
#endif
#endif
