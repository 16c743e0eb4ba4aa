/*
 * hived.h — C ABI of the CUDA-native HiveD scheduling hot path (libhived_cuda.so).
 *
 * The reference (microsoft/hivedscheduler, Go) has no FFI.  This header is the contract a cgo shim
 * binds so that a Go type implementing internal.SchedulerAlgorithm
 * (reference pkg/internal/types.go:76-100) can delegate every method of
 * algorithm.HivedAlgorithm (reference pkg/algorithm/hived_algorithm.go:40-363) to the CUDA
 * backend.  The shim keeps what the reference keeps in Go: YAML (de)serialisation of the pod
 * annotations and the string<->id interning described below.  See INTEGRATION.md for the cgo stub.
 *
 * Threads: a context is used by one thread at a time (the reference serialises every SchedulerAlgorithm call behind
 *   its algorithmLock, hived_algorithm.go:104, and the shims keep that lock).  Different contexts may be driven by
 *   different threads; contexts that live on the same GPU take turns there (the device-side view of a context's state
 *   sits in the device's constant bank, one context at a time: a process-wide lock inside the library).  To run the
 *   batches of several contexts on one GPU at the same time, hand them to one call: hived_multictx.h.
 * Conventions
 *   - plain C, ints and pointers only, no callbacks, nothing retained after a call returns;
 *   - every buffer is caller-owned; results are written into caller-provided arrays;
 *   - return code: 0 ok; 1..99 user errors (the reference panics with a 4xx api.WebServerError,
 *     pkg/internal/utils.go:316-326); >=100 platform errors (plain Go panic).  A failing call leaves
 *     the scheduler state unchanged (pkg/internal/types.go:58-61).  hived_last_error() has the text;
 *   - single writer: callers serialise all calls on one ctx (the reference's algorithmLock,
 *     hived_algorithm.go:104).
 *
 * Id spaces (identical in every implementation of this ABI, defined by the spec text alone)
 *   - cell type ids : ascending byte order over {cellTypes keys} U {leaf cell types};
 *   - leaf type ids : ascending byte order of leaf cell type names;
 *   - chain ids     : ascending byte order of chain names (a chain = top-level physical cell type);
 *   - VC ids        : ascending byte order of VC names;
 *   - pinned ids    : ascending byte order of pinnedCellId strings;
 *   - node ids      : order of first appearance in a pre-order walk of physicalCells;
 *   - physical cell ids: for chain in id order, for level 1..top, construction (pre-order) order
 *     (= fullCellList[chain][level], reference pkg/algorithm/config.go:185-203);
 *   - virtual cell ids: for VC in id order: non-pinned chains in id order then pinned cells in id
 *     order; inside each: level 1..top, construction order (config.go:282-317).
 *   Group ids and pod ids are interned by the caller (dense, < the capacities in hived_options_t).
 *   Id lifetime: a group id may be handed to another group once hived_get_group reports HIVED_GROUP_NONE for it AND
 *   `referenced` == 0 (after the DeleteAllocatedPod / DeleteUnallocatedPod that removed its last pod; `referenced` = cells
 *   still point at the erased object, which the reference can reach and erase BY NAME later: the name keeps its id until
 *   then, so that a re-created group of that name is the one that is hit — and no other), a pod id once the pod has been deleted
 *   AND hived_delete_allocated_pod_ex reported it as the removed occupant (see there);
 *   the shims recycle them that way (hivedscheduler_b200/algorithm.py, integration/pkg/algorithm/cuda_backend.go), so a
 *   long-running scheduler never meets HIVED_ERR_CAPACITY.  Batch callers (hived_process_events) number the gangs of
 *   one batch themselves.
 *
 * Order canonicalisation of the reference's Go-map iteration sites (SURVEY.md section 8c): chains
 * of one leaf type are tried in DESCENDING name order (the order the reference's own test pins,
 * hived_algorithm_test.go:634-643); leaf types, VCs and affinity-group members ascending.
 *
 * HIVEDSPEC text (hived_create): whitespace separated tokens, one record per line
 *   HIVEDSPEC 1
 *   celltypes <n>            then n lines: <name> <childCellType> <childCellNumber> <isNodeLevel 0|1>
 *   physicalcells <n_top>    then the cells in pre-order: <depth> <cellType> <fullAddress> <pinnedCellId|-> <nChildren>
 *   virtualclusters <n>      then per VC: "vc <name> <nVirtualCells> <nPinned>", nVirtualCells lines
 *                            "<cellTypePath a.b.c> <cellNumber>", nPinned lines "<pinnedCellId>"
 *   end
 * It is the reference's api.Config after api.NewConfig defaulting (pkg/api/config.go:87-167).
 */
#ifndef HIVED_H_
#define HIVED_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HIVED_MAX_MEMBERS 8

/* internal cell priorities, reference pkg/algorithm/constants.go:30-35 */
#define HIVED_MAX_GUARANTEED_PRIORITY 1000
#define HIVED_OPPORTUNISTIC_PRIORITY (-1)
#define HIVED_FREE_PRIORITY (-2)

/* internal.SchedulingPhase, reference pkg/internal/types.go:102-114 */
#define HIVED_PHASE_FILTERING 0
#define HIVED_PHASE_PREEMPTING 1

/* which member of internal.PodScheduleResult is set, pkg/internal/types.go:132-136 */
#define HIVED_KIND_WAIT 0
#define HIVED_KIND_BIND 1
#define HIVED_KIND_PREEMPT 2

/* cell states, constants.go:43-58 ; group states, constants.go:62-70 */
#define HIVED_CELL_FREE 0
#define HIVED_CELL_USED 1
#define HIVED_CELL_RESERVING 2
#define HIVED_CELL_RESERVED 3
#define HIVED_GROUP_NONE 0
#define HIVED_GROUP_ALLOCATED 1
#define HIVED_GROUP_PREEMPTING 2
#define HIVED_GROUP_BEING_PREEMPTED 3

/* wait reasons (PodWaitInfo.Reason strings of the reference; the shim formats them):
 *   base code | scope.  topology_aware_scheduler.go:268-306, intra_vc_scheduler.go:112,
 *   hived_algorithm.go:935-941, 975 */
#define HIVED_WAIT_NONE 0                 /* "" (e.g. no chain was searched) */
#define HIVED_WAIT_INSUFFICIENT 1         /* "insufficient capacity" */
#define HIVED_WAIT_BAD_NODE 2             /* "have to use at least one bad node <wait_cell>" */
#define HIVED_WAIT_NON_SUGGESTED_NODE 3   /* "have to use at least one non-suggested node <wait_cell>" */
#define HIVED_WAIT_MAPPING 4              /* "Mapping the virtual placement would need to use at least one bad [or non-suggested] node" */
#define HIVED_WAIT_NO_SCHEDULER 5         /* "" + scope suffix: VC has no scheduler for the chain */
#define HIVED_WAIT_SCOPE_VC 16            /* "... when scheduling in VC <vc>" */
#define HIVED_WAIT_SCOPE_PHYSICAL 32      /* "... when scheduling in physical cluster" */

/* user errors (HTTP 400 in the reference) */
#define HIVED_ERR_UNKNOWN_VC 1            /* hived_algorithm.go:855-870 */
#define HIVED_ERR_UNKNOWN_PINNED_CELL 2   /* hived_algorithm.go:859-861 */
#define HIVED_ERR_OPPORTUNISTIC_PINNED 3  /* hived_algorithm.go:862-864 */
#define HIVED_ERR_LEAF_TYPE_NOT_IN_CLUSTER 4 /* hived_algorithm.go:783-787 */
#define HIVED_ERR_LEAF_TYPE_NOT_IN_VC 5   /* hived_algorithm.go:823-827 */
#define HIVED_ERR_TOO_MANY_PODS 6         /* hived_algorithm.go:683-687 */
#define HIVED_ERR_BAD_SPEC 7              /* pkg/internal/utils.go:256-287 */
#define HIVED_ERR_UNKNOWN_GROUP 8         /* hived_algorithm.go:316-320 */
/* platform errors */
#define HIVED_ERR_PLATFORM 100            /* "VC Safety Broken", "Assert Failure", ... */
#define HIVED_ERR_BAD_CONFIG 101          /* ParseConfig / initCellNums panics, hived_algorithm.go:369-409 */
#define HIVED_ERR_CAPACITY 102            /* an id or size exceeds hived_options_t */
#define HIVED_ERR_NO_DEVICE 103           /* CUDA device / driver unavailable: there is no CPU fallback */

typedef struct hived_ctx hived_ctx;

typedef struct hived_options {
  int32_t max_groups;       /* affinity-group ids are < max_groups */
  int32_t max_pods;         /* pod ids are < max_pods */
  int32_t max_group_leaves; /* max sum(leafCellNumber*podNumber) over a group's members */
  int32_t max_group_pods;   /* max sum(podNumber) over a group's members */
  int32_t device;           /* CUDA device ordinal (ignored by the CPU oracle) */
  int32_t flags;            /* HIVED_OPT_* */
  int32_t reserved[2];
} hived_options_t;
#define HIVED_OPT_NO_RESULT_HASH 1 /* do not maintain hived_result_hash (a parity witness, ~4 CPU cycles per result byte) */

/* api.PodSchedulingSpec after internal.ExtractPodSchedulingSpec (pkg/api/types.go:78-99,
 * pkg/internal/utils.go:230-289), strings interned. */
#define HIVED_SPEC_LAZY_PREEMPTION 1
#define HIVED_SPEC_IGNORE_SUGGESTED 2
typedef struct hived_pod_spec {
  int32_t pod;        /* interned pod UID */
  int32_t group;      /* interned AffinityGroup.Name */
  int32_t vc;         /* VC id; -1 = name not known to the library */
  int32_t priority;   /* -1 .. 1000 */
  int32_t pinned;     /* pinned cell id; -1 = "" (none); -2 = unknown id string */
  int32_t leaf_type;  /* leaf type id; -1 = "" (any); -2 = unknown type string */
  int32_t leaf_num;   /* LeafCellNumber of this pod */
  int32_t flags;      /* HIVED_SPEC_* */
  int32_t n_members;
  int32_t member_leaf_num[HIVED_MAX_MEMBERS];
  int32_t member_pod_num[HIVED_MAX_MEMBERS];
} hived_pod_spec_t;

/* internal.PodScheduleResult (pkg/internal/types.go:132-136) with api.PodBindInfo
 * (pkg/api/types.go:101-118) flattened.  Variable-length parts live in the caller's int32 pool:
 *   leaves : pool[leaf_off + 3*k + 0..2] = node id, leaf cell index, preassigned cell type id
 *            (-1 = ""), for members ascending by leaf number, pods in index order, leaves in order;
 *   victims: pool[victim_off + 2*k + 0..1] = pod id, node id — ALL victims on ALL nodes; the shim
 *            picks one node like generatePodPreemptInfo (pkg/algorithm/utils.go:81-105). */
typedef struct hived_result {
  int32_t kind;        /* HIVED_KIND_* */
  int32_t error;       /* batch mode: the event's return code (0 ok) */
  int32_t wait_code;   /* HIVED_WAIT_* | scope */
  int32_t wait_cell;   /* physical cell id named by the wait reason, or -1 */
  int32_t chain;       /* PodBindInfo.CellChain (chain id) */
  int32_t pod_index;   /* SCHEDULE: index of this pod among those with the same leaf number;
                          DELETE_ALLOCATED: the pod id that occupied the cleared slot, -1 = nothing cleared
                          (see hived_delete_allocated_pod_ex) */
  int32_t node;        /* PodBindInfo.Node (node id) */
  int32_t this_off;    /* this pod's slice of the leaves (LeafCellIsolation = the leaf indices) */
  int32_t this_n;
  int32_t n_members;
  int32_t member_leaf_num[HIVED_MAX_MEMBERS];
  int32_t member_pod_num[HIVED_MAX_MEMBERS];
  int32_t leaf_off;
  int32_t n_leaves;
  int32_t victim_off;
  int32_t n_victims;
  int32_t has_virtual; /* 0 when the placement has no virtual part (opportunistic) */
  int32_t incomplete;  /* 1: some leaf cells of the (allocated) group's placement are no longer in the cluster spec —
                          their triples are (HIVED_NIL_CELL x3), node/chain are -1 when this pod's first cell is one of
                          them.  The shim completes those pods' placements from the other pods' bind-info annotations
                          (retrieveMissingPodPlacement, utils.go:250-265: the annotations live on the pod objects) */
} hived_result_t;
#define HIVED_NIL_CELL (-2)

/* api.PodBindInfo as parsed from the pod-bind-info annotation by the shim
 * (internal.ExtractPodBindInfo, pkg/internal/utils.go:199-212).  leaves: 3 ints per leaf as in
 * hived_result_t but node id -1 = node name unknown, type id -2 = unknown type string. */
typedef struct hived_bind_info {
  int32_t node;          /* PodBindInfo.Node */
  int32_t first_leaf;    /* PodBindInfo.LeafCellIsolation[0] */
  int32_t chain;         /* PodBindInfo.CellChain; -1 = unknown chain name */
  int32_t has_preassigned; /* 0 when PreassignedCellTypes is absent (old annotations) */
  int32_t n_members;
  int32_t member_leaf_num[HIVED_MAX_MEMBERS]; /* len(PodPlacements[0].PhysicalLeafCellIndices) */
  int32_t member_pod_num[HIVED_MAX_MEMBERS];  /* len(PodPlacements) */
  int32_t n_leaves;
  int32_t reserved;
} hived_bind_info_t;

/* One element of an ordered batch (hived_process_events).  The batch is equivalent to the calls one by one, in order;
 * every event reports its own return code in hived_result_t.error (a user or platform error of ONE event does not
 * stop the batch: that event changed nothing — validated before it mutates — and the following ones run; only
 * HIVED_ERR_CAPACITY is also returned by the call itself, and hived_last_error names the first failing event). */
#define HIVED_EV_SCHEDULE 0           /* Schedule; on a bind result immediately AddAllocatedPod with that
                                         PodBindInfo (the filterRoutine sequence, pkg/scheduler/scheduler.go:516-523) */
#define HIVED_EV_DELETE_ALLOCATED 1   /* DeleteAllocatedPod(group=spec.group, leaf_num=spec.leaf_num, pod_index=arg0); spec.vc is
                                         not needed: the event runs with the VC its group was scheduled under */
#define HIVED_EV_DELETE_UNALLOCATED 2 /* DeleteUnallocatedPod(group, pod) */
#define HIVED_EV_NODE_HEALTH 3        /* node arg0 becomes healthy (arg1=1) / bad (arg1=0) */
typedef struct hived_event {
  int32_t type;
  int32_t phase;
  int32_t arg0;
  int32_t arg1;
  int64_t suggested_off; /* word offset into the batch's suggested-node bitmap pool; -1 = every node suggested */
  hived_pod_spec_t spec;
} hived_event_t;

typedef struct hived_group_info {
  int32_t state;        /* HIVED_GROUP_* (NONE = not in affinityGroups) */
  int32_t vc;
  int32_t priority;
  int32_t has_virtual;  /* 0 after lazy preemption (virtualLeafCellPlacement == nil) */
  int32_t n_preempting_pods;
  int32_t referenced;   /* state == NONE only: 1 = an erased object of this id is still named by cells (keep the id) */
  int32_t reserved[2];
} hived_group_info_t;

typedef struct hived_cell_status {
  int32_t priority;
  int32_t state;     /* HIVED_CELL_* */
  int32_t healthy;
  int32_t peer;      /* bound virtual cell id (physical record) / physical cell id (virtual record), -1 none */
  int32_t level;
  int32_t chain;
  int32_t parent;    /* same id space, -1 for a top cell */
  int32_t flags;     /* physical: bit0 split, bit1 pinned, bit2 in the free list; virtual: bit0 preassigned (no parent) */
} hived_cell_status_t;

/* per-decision work counters for the roofline arithmetic (SURVEY.md section 8d) */
typedef struct hived_stats {
  int64_t schedule_events;
  int64_t bind_results;
  int64_t wait_results;
  int64_t preempt_results;
  int64_t view_nodes_scanned;  /* sum over passes of N_view */
  int64_t leaves_committed;    /* leaf cells allocated + released */
  int64_t free_cells_scanned;  /* candidates filtered by getUsablePhysicalCells */
  int64_t pods_placed;         /* pods placed by new-group searches (leaf search runs) */
  int64_t algorithmic_bytes;   /* formula of SURVEY.md section 8d, accumulated */
} hived_stats_t;

/* ---- lifecycle: algorithm.NewHivedAlgorithm (hived_algorithm.go:108-145).  Every node starts bad
 * (initBadNodes :453-464); report healthy nodes with hived_set_node_health. */
int hived_create(const char* spec_text, const hived_options_t* opt, hived_ctx** out);
void hived_destroy(hived_ctx* ctx);
const char* hived_last_error(hived_ctx* ctx);       /* valid until the next call on ctx */
const char* hived_create_error(void);               /* text of the last failed hived_create */
const char* hived_backend(void);                    /* "cuda-sm90a"  | "cpu-oracle" */

/* ---- interning tables */
int32_t hived_num_nodes(hived_ctx*);       const char* hived_node_name(hived_ctx*, int32_t id);
int32_t hived_num_chains(hived_ctx*);      const char* hived_chain_name(hived_ctx*, int32_t id);
int32_t hived_num_vcs(hived_ctx*);         const char* hived_vc_name(hived_ctx*, int32_t id);
int32_t hived_num_leaf_types(hived_ctx*);  const char* hived_leaf_type_name(hived_ctx*, int32_t id);
int32_t hived_num_pinned(hived_ctx*);      const char* hived_pinned_name(hived_ctx*, int32_t id);
int32_t hived_num_cell_types(hived_ctx*);  const char* hived_cell_type_name(hived_ctx*, int32_t id);
int32_t hived_num_physical_cells(hived_ctx*);
int32_t hived_num_virtual_cells(hived_ctx*);
const char* hived_physical_cell_address(hived_ctx*, int32_t cell);
const char* hived_virtual_cell_address(hived_ctx*, int32_t cell);
/* first id and count of the VC's preassigned (top) cells of a chain at a level:
 * vcSchedulers[vc].getNonPinnedPreassignedCells()[chain][level] (intra_vc_scheduler.go:84-86) */
int hived_vc_preassigned_cells(hived_ctx*, int32_t vc, int32_t chain, int32_t level,
                               int32_t* cells, int32_t cap, int32_t* n);

/* ---- internal.SchedulerAlgorithm (pkg/internal/types.go:76-100) */
/* AddNode/UpdateNode/DeleteNode -> setHealthyNode/setBadNode (hived_algorithm.go:147-178, 467-498) */
int hived_set_node_health(hived_ctx*, int32_t node, int32_t healthy);
/* Schedule (hived_algorithm.go:180-224).  suggested: bit i set = node id i is in suggestedNodes;
 * NULL = every node.  pool receives the variable-length parts of *res. */
int hived_schedule(hived_ctx*, const hived_pod_spec_t* spec, const uint32_t* suggested,
                   int32_t phase, hived_result_t* res, int32_t* pool, int32_t pool_cap);
/* AddAllocatedPod (hived_algorithm.go:247-270).  pod_index = getAllocatedPodIndex(info, leaf_num)
 * (utils.go:291-304), computed by the shim from the annotation; leaves as in hived_bind_info_t. */
int hived_add_allocated_pod(hived_ctx*, const hived_pod_spec_t* spec, const hived_bind_info_t* info,
                            const int32_t* leaves, int32_t pod_index);
/* DeleteAllocatedPod (hived_algorithm.go:272-296).  The reference clears allocatedPods[leaf_num][pod_index] WHOEVER sits
 * there (:287).  _ex also reports that occupant: *removed_pod = its pod id, -1 when the call cleared nothing (unknown
 * group, pod_index -1, empty slot).  A shim may recycle its pod's id only when *removed_pod is that pod; otherwise the
 * pod object can still be named by the library (the group object it was added to has been replaced under the same
 * name — the reference keeps such objects alive through cell.usingGroup) and must be kept.  In a batch the same value
 * is hived_result_t.pod_index of the DELETE_ALLOCATED event. */
int hived_delete_allocated_pod(hived_ctx*, int32_t group, int32_t leaf_num, int32_t pod_index);
int hived_delete_allocated_pod_ex(hived_ctx*, int32_t group, int32_t leaf_num, int32_t pod_index, int32_t* removed_pod);
/* DeleteUnallocatedPod (hived_algorithm.go:229-245); AddUnallocatedPod is a no-op in the reference */
int hived_delete_unallocated_pod(hived_ctx*, int32_t group, int32_t pod);

/* ---- throughput entry point: an ordered batch, equivalent to issuing the events one by one.
 * res[i] describes event i (kind/error are set for every event type); pool is shared, offsets in
 * res[i] index it; suggested_pool backs hived_event_t.suggested_off (may be NULL). */
int hived_process_events(hived_ctx*, const hived_event_t* events, int32_t n,
                         const uint32_t* suggested_pool, int64_t suggested_words,
                         hived_result_t* res, int32_t* pool, int64_t pool_cap);

/* ---- inspect: GetAffinityGroup / GetClusterStatus raw material (hived_algorithm.go:298-363) */
int hived_get_group(hived_ctx*, int32_t group, hived_group_info_t* out);
/* AlgoAffinityGroup.ToAffinityGroup (types.go:187-214) in ids.  phys / virt: the leaf cells of the placement in
 * (member ascending by leaf number, pod, leaf) order, -1 = nil (a cell that left the spec / no virtual placement);
 * pods: one slot per pod in (member, pod) order, the allocated pod id or -1; preempting: ids of the preempting pods
 * (ascending).  Arrays shorter than the counts in *out are filled up to their capacity. */
typedef struct hived_group_placement {
  int32_t state;        /* HIVED_GROUP_*; NONE = the group does not exist (everything else is 0) */
  int32_t n_members;
  int32_t member_leaf_num[HIVED_MAX_MEMBERS];
  int32_t member_pod_num[HIVED_MAX_MEMBERS];
  int32_t n_leaves;
  int32_t n_pods;
  int32_t n_preempting;
  int32_t has_virtual;
  int32_t lazy_preempted; /* lazyPreemptionStatus != nil */
  int32_t reserved;
} hived_group_placement_t;
int hived_get_group_placement(hived_ctx*, int32_t group, hived_group_placement_t* out, int32_t* phys, int32_t* virt,
                              int32_t leaf_cap, int32_t* pods, int32_t pod_cap, int32_t* preempting, int32_t preempting_cap);
/* GetAllAffinityGroups: ids of the groups that exist (allocated or preempting), ascending; returns how many there are */
int32_t hived_list_groups(hived_ctx*, int32_t* ids, int32_t cap);
/* static description of a cell (api.CellStatus minus the mutable fields; cell.go:144-177, 326-363) */
typedef struct hived_cell_info {
  int32_t cell_type;     /* id in the cell type table */
  int32_t is_node_level;
  int32_t leaf_type;     /* leaf cell type of the chain */
  int32_t node;          /* physical leaf: node id; otherwise -1 */
  int32_t leaf_index;    /* physical leaf: its index inside the node; otherwise -1 */
  int32_t vc;            /* virtual cell: VC id; physical: -1 */
  int32_t preassigned;   /* virtual cell: id of its preassigned (top) cell; physical: -1 */
  int32_t pinned;        /* pinned cell id of a pinned physical cell / of a virtual cell in a pinned cell, else -1 */
} hived_cell_info_t;
int hived_physical_cell_info(hived_ctx*, int32_t cell, hived_cell_info_t* out);
int hived_virtual_cell_info(hived_ctx*, int32_t cell, hived_cell_info_t* out);
int hived_snapshot_physical(hived_ctx*, hived_cell_status_t* out, int32_t cap);
int hived_snapshot_virtual(hived_ctx*, hived_cell_status_t* out, int32_t cap);
int hived_get_stats(hived_ctx*, hived_stats_t* out);
/* FNV-1a over every SCHEDULE result processed so far (SURVEY.md section 8d parity hash) */
uint64_t hived_result_hash(hived_ctx*);

#ifdef __cplusplus
}
#endif
#endif /* HIVED_H_ */
