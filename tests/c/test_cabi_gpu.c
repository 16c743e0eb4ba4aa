/* Plain-C driver of the drop-in boundary (include/hived.h) — no Python, no ctypes: what a cgo shim does, in C.
 *
 * usage: test_cabi_gpu <HIVEDSPEC file of config C1>
 * C1 (SURVEY.md section 8c): 2 nodes x 4 K80, chain 2-K80-NODE, one VC "default" owning the whole chain.  Four one-GPU
 * pods (own group each, priority 0, leafCellType K80) through Schedule -> AddAllocatedPod, like filterRoutine
 * (reference pkg/scheduler/scheduler.go:516-523): all four must bind to node 10.151.41.23 with leaf cell indices
 * 0, 1, 2, 3, cell chain 2-K80-NODE, preassigned cell type 2-K80-NODE.  Then DeleteAllocatedPod for each and the
 * groups must be gone.  Exit code 0 = all checks passed.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "hived.h"

#define CHECK(cond, ...)                                        \
  do {                                                          \
    if (!(cond)) {                                              \
      fprintf(stderr, "FAILED %s:%d: ", __FILE__, __LINE__);    \
      fprintf(stderr, __VA_ARGS__);                             \
      fprintf(stderr, "\n");                                    \
      return 1;                                                 \
    }                                                           \
  } while (0)

static char* slurp(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) return NULL;
  fseek(f, 0, SEEK_END);
  long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  char* buf = (char*)malloc((size_t)n + 1);
  if (fread(buf, 1, (size_t)n, f) != (size_t)n) { fclose(f); free(buf); return NULL; }
  buf[n] = 0;
  fclose(f);
  return buf;
}

static int find_id(hived_ctx* ctx, int32_t (*num)(hived_ctx*), const char* (*name)(hived_ctx*, int32_t), const char* want) {
  for (int32_t i = 0; i < num(ctx); i++)
    if (strcmp(name(ctx, i), want) == 0) return i;
  return -1;
}

int main(int argc, char** argv) {
  CHECK(argc == 2, "usage: %s <spec file>", argv[0]);
  char* spec = slurp(argv[1]);
  CHECK(spec != NULL, "cannot read %s", argv[1]);
  hived_options_t opt;
  memset(&opt, 0, sizeof opt);
  opt.max_groups = 16; opt.max_pods = 16; opt.max_group_leaves = 8; opt.max_group_pods = 8;
  hived_ctx* ctx = NULL;
  int rc = hived_create(spec, &opt, &ctx);
  CHECK(rc == 0, "hived_create: %d %s", rc, hived_create_error());
  if (!getenv("HIVED_TEST_ANY_BACKEND")) CHECK(strcmp(hived_backend(), "cuda-sm90a") == 0, "not the CUDA library: %s", hived_backend());
  const int vc = find_id(ctx, hived_num_vcs, hived_vc_name, "default");
  const int k80 = find_id(ctx, hived_num_leaf_types, hived_leaf_type_name, "K80");
  const int node23 = find_id(ctx, hived_num_nodes, hived_node_name, "10.151.41.23");
  const int chain = find_id(ctx, hived_num_chains, hived_chain_name, "2-K80-NODE");
  const int ctype = find_id(ctx, hived_num_cell_types, hived_cell_type_name, "2-K80-NODE");
  CHECK(vc >= 0 && k80 >= 0 && node23 >= 0 && chain >= 0 && ctype >= 0, "id tables incomplete");
  /* every node starts bad (hived_algorithm.go:453-464); healthy nodes arrive in ascending id order */
  for (int32_t n = 0; n < hived_num_nodes(ctx); n++) CHECK(hived_set_node_health(ctx, n, 1) == 0, "set_node_health");

  uint32_t all_nodes[1] = {0xffffffffu};
  int32_t pool[256];
  hived_result_t res;
  hived_bind_info_t infos[4];
  int32_t leaves[4][3];
  for (int p = 0; p < 4; p++) {
    hived_pod_spec_t sp;
    memset(&sp, 0, sizeof sp);
    sp.pod = p; sp.group = p; sp.vc = vc; sp.priority = 0; sp.pinned = -1; sp.leaf_type = k80; sp.leaf_num = 1;
    sp.flags = HIVED_SPEC_IGNORE_SUGGESTED;
    sp.n_members = 1; sp.member_leaf_num[0] = 1; sp.member_pod_num[0] = 1;
    rc = hived_schedule(ctx, &sp, all_nodes, HIVED_PHASE_PREEMPTING, &res, pool, 256);
    CHECK(rc == 0, "hived_schedule pod %d: %d %s", p, rc, hived_last_error(ctx));
    CHECK(res.kind == HIVED_KIND_BIND, "pod %d: kind %d", p, res.kind);
    CHECK(res.node == node23 && res.chain == chain && res.this_n == 1 && res.n_leaves == 1, "pod %d: node %d chain %d", p, res.node, res.chain);
    CHECK(pool[res.this_off] == node23 && pool[res.this_off + 1] == p && pool[res.this_off + 2] == ctype,
          "pod %d: leaf triple (%d, %d, %d), wanted (%d, %d, %d)", p, pool[res.this_off], pool[res.this_off + 1], pool[res.this_off + 2], node23, p, ctype);
    /* AddAllocatedPod with the PodBindInfo just produced */
    hived_bind_info_t* bi = &infos[p];
    memset(bi, 0, sizeof *bi);
    bi->node = res.node; bi->first_leaf = pool[res.this_off + 1]; bi->chain = res.chain; bi->has_preassigned = 1;
    bi->n_members = 1; bi->member_leaf_num[0] = 1; bi->member_pod_num[0] = 1; bi->n_leaves = 1;
    memcpy(leaves[p], pool + res.leaf_off, 3 * sizeof(int32_t));
    rc = hived_add_allocated_pod(ctx, &sp, bi, leaves[p], res.pod_index);
    CHECK(rc == 0, "hived_add_allocated_pod pod %d: %d %s", p, rc, hived_last_error(ctx));
    hived_group_info_t gi;
    CHECK(hived_get_group(ctx, p, &gi) == 0 && gi.state == HIVED_GROUP_ALLOCATED && gi.vc == vc, "pod %d: group state %d", p, gi.state);
  }
  /* a fifth GPU on the same node fits too (node has 4: the next pod goes to the other node) */
  {
    hived_pod_spec_t sp;
    memset(&sp, 0, sizeof sp);
    sp.pod = 4; sp.group = 4; sp.vc = vc; sp.priority = 0; sp.pinned = -1; sp.leaf_type = k80; sp.leaf_num = 1;
    sp.flags = HIVED_SPEC_IGNORE_SUGGESTED; sp.n_members = 1; sp.member_leaf_num[0] = 1; sp.member_pod_num[0] = 1;
    rc = hived_schedule(ctx, &sp, all_nodes, HIVED_PHASE_PREEMPTING, &res, pool, 256);
    CHECK(rc == 0 && res.kind == HIVED_KIND_BIND && res.node != node23, "fifth pod: rc %d kind %d node %d", rc, res.kind, res.node);
  }
  /* an unknown VC is a user error (HTTP 400 in the reference) and changes nothing */
  {
    hived_pod_spec_t sp;
    memset(&sp, 0, sizeof sp);
    sp.pod = 5; sp.group = 5; sp.vc = -1; sp.priority = 0; sp.pinned = -1; sp.leaf_type = k80; sp.leaf_num = 1;
    sp.n_members = 1; sp.member_leaf_num[0] = 1; sp.member_pod_num[0] = 1;
    rc = hived_schedule(ctx, &sp, all_nodes, HIVED_PHASE_PREEMPTING, &res, pool, 256);
    CHECK(rc == HIVED_ERR_UNKNOWN_VC, "unknown VC: rc %d", rc);
  }
  for (int p = 0; p < 4; p++) {
    rc = hived_delete_allocated_pod(ctx, p, 1, 0);
    CHECK(rc == 0, "hived_delete_allocated_pod %d: %d %s", p, rc, hived_last_error(ctx));
    hived_group_info_t gi;
    CHECK(hived_get_group(ctx, p, &gi) == 0 && gi.state == HIVED_GROUP_NONE, "pod %d: group still there (%d)", p, gi.state);
  }
  /* everything is free again: the first pod lands where it landed before */
  {
    hived_pod_spec_t sp;
    memset(&sp, 0, sizeof sp);
    sp.pod = 6; sp.group = 6; sp.vc = vc; sp.priority = 0; sp.pinned = -1; sp.leaf_type = k80; sp.leaf_num = 1;
    sp.flags = HIVED_SPEC_IGNORE_SUGGESTED; sp.n_members = 1; sp.member_leaf_num[0] = 1; sp.member_pod_num[0] = 1;
    rc = hived_schedule(ctx, &sp, all_nodes, HIVED_PHASE_PREEMPTING, &res, pool, 256);
    CHECK(rc == 0 && res.kind == HIVED_KIND_BIND && res.node == node23 && pool[res.this_off + 1] == 0, "after delete: rc %d kind %d node %d", rc, res.kind, res.node);
  }
  hived_destroy(ctx);
  free(spec);
  printf("test_cabi_gpu: ok\n");
  return 0;
}
