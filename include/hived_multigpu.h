/* hived_multigpu.h — one calm batch of events partitioned over several GPUs (SURVEY.md §8 row e).
 *
 * The reference runs ONE scheduler instance (pkg/internal/types.go:64-71: every SchedulerAlgorithm call is made
 * under the scheduler lock, pkg/scheduler/scheduler.go:149), so there is no reference interface for this: these
 * entry points sit next to the ABI of hived.h, which stays the drop-in surface.
 *
 * Model: every rank (one process per GPU) creates the SAME scheduler (hived_create with the same spec) and brings it
 * to the same state.  Rank r owns the virtual clusters v with v % world == r and runs one CTA per owned VC.  VCs
 * interact only through the chain-wide buddy free lists and counters (the "cluster-wide state", a few MB); an
 * event that may touch them — the first gang of a VC in a preassigned cell (buddy allocation,
 * cell_allocation.go:233-287) or the release of the last one (:384-397) — must run at its position in the batch
 * order.  Protocol, driven by the caller (bench.py / tests use torch.distributed for the two collectives):
 *
 *   hived_mg_stage(ctx, events, n, pool_cap, rank, world)        every rank, the whole batch
 *   H = W                               the horizon: an event index; windows of W events keep the VCs moving together
 *   loop:
 *     hived_mg_run_window(ctx, H, &stop) every rank runs its events below H; a CTA whose next event may touch the
 *                                       cluster-wide state parks BEFORE it: stop = the first such event of the rank,
 *                                       0x7fffffff = every owned event below H has run
 *     E = allreduce_min(stop)           (collective #1)
 *     E == 0x7fffffff:                  H >= n: leave the loop; else H += W, next round
 *     owner of E: hived_mg_solo(ctx, E); hived_mg_export_shared(ctx, buf)
 *     broadcast(buf, src = owner)       (collective #2, hived_mg_shared_bytes() bytes of device memory)
 *     everyone else: hived_mg_import_shared(ctx, buf)
 *   hived_mg_finish(ctx)
 *   (hived_mg_run = hived_mg_run_window with H = infinity: correct, but a CTA then runs on to ITS next such event
 *   while every other one is parked at theirs — one VC at a time.)
 *   hived_bench_fetch_results()         rank r holds the results of ITS events (the other records are all-zero)
 *
 * Every event of every rank before E is complete when E runs, and E is complete before any later event that may
 * touch the cluster-wide state: the sequential contract holds, results are identical to a single-GPU run (the
 * chain hash over the merged results — hived_mg_chain_hash — is the witness).  Only calm batches are accepted
 * (SCHEDULE / DELETE_ALLOCATED events, every node healthy, one guaranteed priority, no recovery): the regime in
 * which the single-GPU engine runs VC-parallel (hived_engine.hpp Engine::route).  hived_mg_stage refuses with
 * HIVED_ERR_BAD_SPEC, and changes nothing, a batch with any other event type, an event with a suggested-node set
 * (suggested_off >= 0: no rank holds a suggested-node pool), more than one priority (or an opportunistic one), a
 * group id scheduled under two VCs, or an event of an unknown VC; and any batch on a context with a bad node or a
 * recovered pod.
 * After the run a rank's physical-cell state and its views (hived_debug_view_hash_vc) are authoritative for its own
 * VCs only.                                                                                                       */
#ifndef HIVED_MULTIGPU_H_
#define HIVED_MULTIGPU_H_
#include "hived.h"
#ifdef __cplusplus
extern "C" {
#endif
int hived_mg_stage(hived_ctx*, const hived_event_t* events, int32_t n, int64_t pool_cap, int32_t rank, int32_t world);
int hived_mg_reset(hived_ctx*);   /* the staged batch once more (after hived_bench_restore_state): cursors and results cleared */
int hived_mg_run(hived_ctx*, int32_t* stop_event);
int hived_mg_run_window(hived_ctx*, int32_t horizon, int32_t* stop_event);
int hived_mg_solo(hived_ctx*, int32_t event_index);
int64_t hived_mg_shared_bytes(hived_ctx*);
int hived_mg_export_shared(hived_ctx*, void* device_buffer);       /* device pointer on the context's GPU */
int hived_mg_import_shared(hived_ctx*, const void* device_buffer);
int hived_mg_finish(hived_ctx*);
/* chain hash (hived_hash.h) over the SCHEDULE results of the whole batch, event i taken from rank (vc % world)'s
 * fetched results and pool; equals hived_result_hash() of a single-GPU run started from the same hash seed */
int hived_mg_chain_hash(const hived_event_t* events, int32_t n, int32_t world, const hived_result_t* const* res,
                        const int32_t* const* pools, uint64_t seed, uint64_t* out);
#ifdef __cplusplus
}
#endif
#endif
