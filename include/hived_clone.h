/* hived_clone.h — an independent copy of a live scheduler context, for what-if runs, on the same GPU or another.
 *
 * Recovery (hived_add_allocated_pod for every bound pod) restores placements only: it loses the state that depends on
 * history — the persisted order of every cluster view (it breaks first-fit ties), the order of the free, bad-free and
 * doomed-bad lists with their stale entries and duplicates, the erased groups that cells still name, lazy-preempted and
 * preempting groups, the running result hash and the work counters — and it marks the context as recovered, which
 * keeps every later batch on one CTA.  A clone keeps all of it: "if these pending gangs arrived now, which would bind,
 * wait or preempt", K clones each trying another ordering or priority policy in one hived_process_events_many call
 * (hived_multictx.h), or a copy on a second GPU for replay or replica work.
 *
 * Threads: the caller holds `src` (the single-writer rule of hived.h), so no call of `src` is in flight; `src` is not
 * changed in any observable way.  The clone is a context like any other: it takes turns on its device as a context
 * created by hived_create with the same flags does, and may be driven by another thread than `src` from the moment it
 * is returned.
 */
#ifndef HIVED_CLONE_H_
#define HIVED_CLONE_H_
#include "hived.h"
#ifdef __cplusplus
extern "C" {
#endif

/* A new context that answers every later call exactly as `src` would have answered it.
 * It copies all of src's state: results, pool, return codes, result hash, stats and path counters, inspect outputs, and
 * the debug view / bookkeeping hashes.  Afterwards the two share nothing.
 *   device: CUDA ordinal for the clone (as hived_options_t.device), -1 = src's device.  The copy to another device
 *           needs no peer access and changes no device or process setting.
 *   flags:  HIVED_OPT_* for the clone (HIVED_OPT_NO_RESULT_HASH stops the clone's running hash where src's stands).
 *           Capacities (max_groups, max_pods, max_group_leaves, max_group_pods) are src's.
 * The clone starts with an empty last error, a fresh turn counter, kernel-timing and launch counters (hived_bench.h)
 * at zero and no state saved by hived_bench_save_state.
 * Returns 0 and *out, or creates nothing, sets *out = NULL and names the reason in hived_create_error():
 *   HIVED_ERR_BAD_SPEC   src is staged for a multi-GPU partition (hived_mg_stage, hived_multigpu.h);
 *   HIVED_ERR_CAPACITY   a HIVED_OPT_CONCURRENT clone past HIVED_CONCURRENT_MAX on its device, or out of device memory;
 *   HIVED_ERR_NO_DEVICE  no usable CUDA device;
 *   HIVED_ERR_PLATFORM   a copy failed. */
int hived_clone(hived_ctx* src, int32_t device, int32_t flags, hived_ctx** out);

#ifdef __cplusplus
}
#endif
#endif
