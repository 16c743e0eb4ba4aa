/* Per-call throughput of K threads on one GPU, each driving its own full-size C3 context, with HIVED_OPT_CONCURRENT
 * (every context's calls on a resident kernel of its own) and without it (the contexts take turns on the device).
 *
 * Every context gets the spec and the half-full fill of percall_latency.c (all nodes healthy, 300 8-GPU pods per VC),
 * saved with hived_bench_save_state.  One run = every context rewound to that state, then K pthreads released at once,
 * each doing `calls` rounds of hived_process_events(n = 1, SCHEDULE) + hived_delete_allocated_pod on its own context.
 * For every K the runs alternate flag on / flag off, `reps` times.  Every context's result hash after a run must equal
 * that of the same rounds run single-threaded on a context without the flag.  Prints one JSON line.
 *
 *   gcc -O2 -pthread -I include -o concurrent_calls profiles/micro/concurrent_calls.c -L hivedscheduler_b200/csrc \
 *       -lhived_cuda -Wl,-rpath,$PWD/hivedscheduler_b200/csrc
 *   ./concurrent_calls c3.spec [ks=1,2,4,8,16] [calls=2000] [reps=2]       (profiles/micro/concurrent_calls.py does this)
 */
#define _POSIX_C_SOURCE 200809L
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "hived.h"
#include "hived_bench.h"

#define KMAX HIVED_CONCURRENT_MAX

static double now_us(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e6 + ts.tv_nsec / 1e3;
}
static int cmp(const void* a, const void* b) { double x = *(const double*)a, y = *(const double*)b; return x < y ? -1 : x > y; }

static int g_vcs, g_fill, g_calls;

static hived_ctx* make(const char* spec, int flags) {
  hived_options_t opt;
  memset(&opt, 0, sizeof opt);
  opt.max_groups = 1 << 16; opt.max_pods = 1 << 18; opt.max_group_leaves = 64; opt.max_group_pods = 8; opt.flags = flags;
  hived_ctx* ctx = NULL;
  int rc = hived_create(spec, &opt, &ctx);
  if (rc) { fprintf(stderr, "hived_create: %d %s\n", rc, hived_create_error()); exit(1); }
  const int nodes = hived_num_nodes(ctx);
  g_vcs = hived_num_vcs(ctx);
  g_fill = 300 * g_vcs;
  const int nev = nodes + g_fill;
  hived_event_t* ev = (hived_event_t*)calloc((size_t)nev, sizeof *ev);
  hived_result_t* res = (hived_result_t*)calloc((size_t)nev, sizeof *res);
  const long long cap = 3ll * 8 * nev + 4096;
  int32_t* pool = (int32_t*)calloc((size_t)cap, 4);
  for (int i = 0; i < nodes; i++) { ev[i].type = HIVED_EV_NODE_HEALTH; ev[i].arg0 = i; ev[i].arg1 = 1; ev[i].suggested_off = -1; }
  for (int i = 0; i < g_fill; i++) {
    hived_event_t* e = &ev[nodes + i];
    e->type = HIVED_EV_SCHEDULE; e->phase = HIVED_PHASE_FILTERING; e->suggested_off = -1;
    e->spec.pod = i; e->spec.group = i; e->spec.vc = i % g_vcs; e->spec.priority = 0; e->spec.pinned = -1; e->spec.leaf_type = 0;
    e->spec.leaf_num = 8; e->spec.flags = HIVED_SPEC_IGNORE_SUGGESTED; e->spec.n_members = 1;
    e->spec.member_leaf_num[0] = 8; e->spec.member_pod_num[0] = 1;
  }
  rc = hived_process_events(ctx, ev, nev, NULL, 0, res, pool, cap);
  if (rc) { fprintf(stderr, "fill: %d %s\n", rc, hived_last_error(ctx)); exit(1); }
  hived_bench_save_state(ctx);
  free(ev); free(res); free(pool);
  return ctx;
}

typedef struct {
  hived_ctx* ctx;
  pthread_barrier_t* go;
  double* lat;  /* 2 * g_calls per-call latencies */
  uint64_t hash;
  int failed;
} Job;

static void* rounds(void* arg) {
  Job* j = (Job*)arg;
  hived_event_t one;
  hived_result_t r1;
  int32_t pool[64];
  if (j->go) pthread_barrier_wait(j->go);
  for (int k = 0; k < g_calls; k++) {
    const int id = g_fill + k % 1000;
    memset(&one, 0, sizeof one);
    one.type = HIVED_EV_SCHEDULE; one.phase = HIVED_PHASE_FILTERING; one.suggested_off = -1;
    one.spec.pod = id; one.spec.group = id; one.spec.vc = k % g_vcs; one.spec.priority = 0; one.spec.pinned = -1; one.spec.leaf_type = 0;
    one.spec.leaf_num = 8; one.spec.flags = HIVED_SPEC_IGNORE_SUGGESTED; one.spec.n_members = 1;
    one.spec.member_leaf_num[0] = 8; one.spec.member_pod_num[0] = 1;
    const double t0 = now_us();
    int rc = hived_process_events(j->ctx, &one, 1, NULL, 0, &r1, pool, 64);
    const double t1 = now_us();
    if (rc || r1.kind != HIVED_KIND_BIND) { j->failed = 1; break; }
    rc = hived_delete_allocated_pod(j->ctx, id, 8, r1.pod_index);
    const double t2 = now_us();
    if (rc) { j->failed = 1; break; }
    j->lat[2 * k] = t1 - t0;
    j->lat[2 * k + 1] = t2 - t1;
  }
  j->hash = hived_result_hash(j->ctx);
  return NULL;
}

/* one run of K threads; returns its wall time in seconds and appends the latencies */
static double run(hived_ctx** ctxs, int K, double* lat, uint64_t ref, int* mismatches) {
  Job jobs[KMAX];
  pthread_t th[KMAX];
  pthread_barrier_t go;
  pthread_barrier_init(&go, NULL, (unsigned)K + 1);
  for (int i = 0; i < K; i++) {
    hived_bench_restore_state(ctxs[i]);
    jobs[i] = (Job){ctxs[i], &go, lat + (size_t)i * 2 * g_calls, 0, 0};
    pthread_create(&th[i], NULL, rounds, &jobs[i]);
  }
  pthread_barrier_wait(&go);
  const double t0 = now_us();
  for (int i = 0; i < K; i++) pthread_join(th[i], NULL);
  const double wall = (now_us() - t0) / 1e6;
  pthread_barrier_destroy(&go);
  for (int i = 0; i < K; i++) {
    if (jobs[i].failed) { fprintf(stderr, "a call failed (K = %d)\n", K); exit(1); }
    if (jobs[i].hash != ref) (*mismatches)++;
  }
  return wall;
}

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: %s spec-file [ks] [calls] [reps]\n", argv[0]); return 2; }
  int ks[8], nk = 0, kmax = 0;
  for (char* s = strtok(argc > 2 ? argv[2] : (char[]){"1,2,4,8,16"}, ","); s && nk < 8; s = strtok(NULL, ",")) {
    ks[nk] = atoi(s);
    if (ks[nk] < 1 || ks[nk] > KMAX) { fprintf(stderr, "K must be 1..%d\n", KMAX); return 2; }
    if (ks[nk] > kmax) kmax = ks[nk];
    nk++;
  }
  g_calls = argc > 3 ? atoi(argv[3]) : 2000;
  const int reps = argc > 4 ? atoi(argv[4]) : 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  fseek(f, 0, SEEK_END);
  long len = ftell(f);
  fseek(f, 0, SEEK_SET);
  char* spec = (char*)malloc((size_t)len + 1);
  if (fread(spec, 1, (size_t)len, f) != (size_t)len) return 2;
  spec[len] = 0;
  fclose(f);
  hived_ctx* on[KMAX];
  hived_ctx* off[KMAX];
  for (int i = 0; i < kmax; i++) { on[i] = make(spec, HIVED_OPT_CONCURRENT); off[i] = make(spec, 0); }
  /* the reference: the same rounds single-threaded, without the flag */
  double* lat = (double*)malloc(sizeof(double) * (size_t)KMAX * 2 * g_calls * (size_t)reps);
  Job ref = {off[0], NULL, lat, 0, 0};
  hived_bench_restore_state(off[0]);
  rounds(&ref);
  if (ref.failed) { fprintf(stderr, "the reference run failed\n"); return 1; }
  printf("{\"what\": \"K threads, one full-size C3 context each, rounds of hived_process_events(n = 1) + "
         "hived_delete_allocated_pod\", \"backend\": \"%s\", \"calls_per_thread\": %d, \"reps\": %d, "
         "\"reference_hash\": \"%016llx\", \"by_k\": {", hived_backend(), 2 * g_calls, reps, (unsigned long long)ref.hash);
  int allOk = 1;
  for (int ki = 0; ki < nk; ki++) {
    const int K = ks[ki];
    const size_t per = (size_t)K * 2 * g_calls;
    double* latOn = (double*)malloc(sizeof(double) * per * (size_t)reps);
    double* latOff = (double*)malloc(sizeof(double) * per * (size_t)reps);
    double wallOn = 0, wallOff = 0;
    int bad = 0;
    for (int r = 0; r < reps; r++) {  /* alternating */
      wallOn += run(on, K, latOn + per * (size_t)r, ref.hash, &bad);
      wallOff += run(off, K, latOff + per * (size_t)r, ref.hash, &bad);
    }
    const size_t n = per * (size_t)reps;
    qsort(latOn, n, sizeof(double), cmp);
    qsort(latOff, n, sizeof(double), cmp);
    if (bad) allOk = 0;
    printf("%s\"%d\": {\"concurrent\": {\"calls_per_s\": %.0f, \"p50_us\": %.2f, \"p99_us\": %.2f}, "
           "\"taking_turns\": {\"calls_per_s\": %.0f, \"p50_us\": %.2f, \"p99_us\": %.2f}, \"speedup\": %.2f, "
           "\"hash_mismatches\": %d}", ki ? ", " : "", K, n / wallOn, latOn[n / 2], latOn[(size_t)(n * 0.99)], n / wallOff,
           latOff[n / 2], latOff[(size_t)(n * 0.99)], wallOff / wallOn, bad);
    free(latOn);
    free(latOff);
  }
  printf("}, \"every_context_matches_the_single_threaded_run\": %s}\n", allOk ? "true" : "false");
  for (int i = 0; i < kmax; i++) { hived_destroy(on[i]); hived_destroy(off[i]); }
  return allOk ? 0 : 1;
}
