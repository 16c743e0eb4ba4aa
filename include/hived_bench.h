/* hived_bench.h — measurement hooks exported by libhived_cuda.so next to the ABI of hived.h.
 * They exist so that bench.py can (a) time the kernel with the batch already resident in HBM and
 * (b) rewind the scheduler state between timed steps.  Not part of the reference-facing surface. */
#ifndef HIVED_BENCH_H_
#define HIVED_BENCH_H_
#include "hived.h"
#ifdef __cplusplus
extern "C" {
#endif
int hived_bench_save_state(hived_ctx*);     /* device-to-device copy of every mutable array */
int hived_bench_restore_state(hived_ctx*);
int hived_bench_stage_events(hived_ctx*, const hived_event_t* events, int32_t n, int64_t pool_cap); /* H2D once */
int hived_bench_run_staged(hived_ctx*);     /* one kernel launch over the staged batch; nothing crosses PCIe */
/* the staged batches of k contexts in one joint launch (hived_multictx.h); each context's hived_bench_last_kernel_ms
   then reports the joint launch.  HIVED_ERR_BAD_SPEC for a list hived_process_events_many refuses */
int hived_bench_run_staged_many(hived_ctx* const* ctxs, int32_t k);
int hived_bench_fetch_results(hived_ctx*, hived_result_t* res, int32_t* pool, int64_t pool_cap, int64_t* pool_used);
int hived_bench_flush_l2(hived_ctx*);       /* overwrite a buffer larger than L2 */
/* out[0..15): SM cycles of the leader warps in {view pass, leaf search, v->p mapping, result emission, commit, delete,
 * all events, waiting at shared sections}, the number of shared sections entered, then cycles / events of
 * {Schedule of a pod of an existing gang, delete of a pod that is not the gang's last, commit of such a pod} */
int hived_bench_phase_cycles(hived_ctx*, int64_t* out);
int hived_bench_debug_cycles(hived_ctx*, int64_t* out); /* out[0..16): scratch cycle counters used in profiling sessions */
/* out[0..12): events by path — [0] scheduling passes answered by the bucketed cluster view, [1] full view passes,
   [2] bucket rebuilds, [3] nodes moved between buckets, [4]/[5] gang commits fast/general, [6]/[7] gang releases
   fast/general, [8]/[9] virtual->physical mappings fast/general; returns the number of counters */
int hived_bench_path_counters(hived_ctx*, int64_t* out);
double hived_bench_last_kernel_ms(hived_ctx*);   /* CUDA-event time of the last launch, on its stream */
double hived_bench_total_kernel_ms(hived_ctx*);
int64_t hived_bench_kernel_launches(hived_ctx*);
/* calls of this context (hived_create and hived_destroy included) that took the library's process-wide device lock,
   i.e. took turns with the other contexts of the process (include/hived.h "Threads"); 0 in the host builds */
int64_t hived_bench_turns(hived_ctx*);
int hived_bench_num_ctas(hived_ctx*);            /* CTAs the last batch ran on (VC-parallel execution) */
int hived_bench_set_result_hash(hived_ctx*, int on); /* toggle the running parity hash (HIVED_OPT_NO_RESULT_HASH) */
#ifdef __cplusplus
}
#endif
#endif
