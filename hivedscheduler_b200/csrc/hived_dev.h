// Device-resident state of the CUDA-native HiveD scheduling path: one POD struct of raw pointers
// into HBM (flat int32 SoA, see DESIGN.md "Data layout").  Static arrays come from FlatTopo
// (hived_topo.hpp); mutable arrays are the scheduler state that the reference keeps in its
// pointer forest (pkg/algorithm/cell.go:58-142,315-324; hived_algorithm.go:40-105).
#pragma once
#include <cstdint>

namespace hived {

#if defined(__CUDACC__)
#define HIVED_HD __host__ __device__ __forceinline__
#else
#define HIVED_HD inline
#endif

// An affinity group's scalars live in ONE 128-byte record (a decision touches a group it has not seen for
// a while: one L2 round trip instead of eight).  Word layout: 0 state, 1 vc, 2 priority, 3 flags,
// 4 #members, 5 #preempting pods, 8..15 member leaf numbers, 16..23 member pod numbers, 24..27 the lean lane's unit
// decomposition, 28 (ghost records) the id the ghost came from + 1, 29 (live records; survives re-creation) the ghost
// slot + 1 that last took this id's object over.
constexpr int GROUP_HDR_WORDS = 32;
// Records [maxGroups, maxGroups + GHOST_GROUPS) of the group tables hold GHOSTS: a group that the reference erases from
// its name map while cells still point at the object (cell.usingGroup), see Core::ghostify.  Never visible by id.
constexpr int GHOST_GROUPS = 64;
constexpr int GH_ORIGIN = 28, GH_LINK = 29;
constexpr int DELTA_SLOTS = 4;          // (priority, difference) pairs per cell, see noteDelta
constexpr int DELTA_EMPTY = -1000000;
constexpr int BK_STRIDE = 33;  // buckets of a bucketed cluster view: used-leaf counts 0..32
template <int OFF>
struct GroupFld {
  int32_t* b;
  HIVED_HD int32_t& operator[](long long g) const { return b[g * GROUP_HDR_WORDS + OFF]; }
};
template <int BASE>
struct GroupMemFld {  // indexed by g * 8 + m like the flat arrays it replaces
  int32_t* b;
  HIVED_HD int32_t& operator[](long long i) const { return b[(i >> 3) * GROUP_HDR_WORDS + BASE + (i & 7)]; }
};

// X(name): static int32 array copied verbatim from FlatTopo::name
#define HIVED_STATIC_ARRAYS(X)                                                                         \
  X(p_parent) X(p_child0) X(p_nchild) X(p_level) X(p_chain) X(p_leaf0) X(p_nleaf) X(p_node)           \
  X(p_leafidx) X(p_flags) X(p_nodes_off) X(p_nodes_cnt) X(nodes_flat) X(p_anc) X(v_anc)                                \
  X(v_parent) X(v_child0) X(v_nchild) X(v_level) X(v_chain) X(v_leaf0) X(v_nleaf) X(v_vc) X(v_pre)    \
  X(v_vset) X(v_flags) X(v_pretype) X(v_prelevel)                                                      \
  X(chain_top) X(chain_leaftype) X(chain_lvl_type) X(chain_lvl_leafnum) X(chain_lvl_nchild)           \
  X(p_lvl_base) X(p_lvl_cnt) X(chain_in_vc) X(lt_off) X(lt_cnt) X(lt_chains)                           \
  X(vs_vc) X(vs_chain) X(vs_pinned) X(vs_top) X(v_lvl_base) X(v_lvl_cnt) X(vc_chain_vset)             \
  X(vc_pinned_vset) X(pre_off) X(pre_cnt) X(pre_list) X(vc_chain_counter) X(pin_pcell) X(pin_vcell)   \
  X(pin_vc) X(s_off) X(s_n) X(s_cross) X(s_chain) X(s_virtual) X(s_maxleaf) X(s_level) X(s_vc) X(s_fast) X(s_cell0) X(s_leaf0) X(vset_sched) X(opp_sched) \
  X(ncl_off) X(ncl_cnt) X(ncl_list) X(fl_base) X(fl_cap) X(dm_base) X(dm_cap)

// Y(name, count, init): mutable int32 array of `count` elements filled with `init`
// (count expressions may use the Dev size fields through `S.`)
#define HIVED_MUTABLE_ARRAYS(Y)                                                                        \
  Y(p_prio, S.NP, -2) Y(p_state, S.NP, 0) Y(p_healthy, S.NP, 1) Y(p_vcell, S.NP, -1) Y(p_split, S.NP, 0) \
  Y(p_using, S.NP, -1) Y(p_resv, S.NP, -1) Y(p_usedopp, S.NP, 0) Y(p_flpos, S.NP, -1)                  \
  Y(p_bfpos, S.NP, -1) Y(p_dmpos, S.NP, -1) Y(p_dmvc, S.NP, -1)                                        \
  Y(v_prio, S.NV, -2) Y(v_state, S.NV, 0) Y(v_healthy, S.NV, 1) Y(v_pcell, S.NV, -1)                   \
  Y(vcFree, S.nVCs * S.nChains * MAXL, 0) Y(allVCFree, S.nChains * MAXL, 0)                            \
  Y(totalLeft, S.nChains * MAXL, 0) Y(allVCDoomed, S.nChains * MAXL, 0)                                \
  Y(fl_data, S.flTotal, -1) Y(fl_len, S.nChains * MAXL, 0) Y(fl_dup, S.nChains * MAXL, 0) Y(bf_data, S.flTotal, -1)                   \
  Y(bf_len, S.nChains * MAXL, 0) Y(dm_data, S.dmTotal, -1) Y(dm_len, S.nVCs * S.nChains * MAXL, 0)     \
  Y(cv, S.cvTotal, -1) Y(node_bad, S.nNodes, 0)                                                        \
  Y(g_hdr, (int64_t)(S.maxGroups + GHOST_GROUPS) * GROUP_HDR_WORDS, 0)                                                  \
  Y(g_phys, (int64_t)(S.maxGroups + GHOST_GROUPS) * S.LS, -1) Y(g_virt, (int64_t)(S.maxGroups + GHOST_GROUPS) * S.LS, -1)                \
  Y(g_pods, (int64_t)(S.maxGroups + GHOST_GROUPS) * S.PS, -1)                                                           \
  Y(g_pre, (int64_t)(S.maxGroups + GHOST_GROUPS) * S.PS, -1) Y(pod_node, S.maxPods, -1) \
  Y(vx_of, S.NV, -1) Y(vx_stamp, S.NV, 0) Y(binding, S.NV, -1)                                         \
  /* bucketed cluster views (hived_core.h, "incremental cluster view") */                              \
  Y(bk_valid, S.nScheds, 0) Y(bk_ndirty, S.nScheds, 0) Y(bk_head, S.nScheds * BK_STRIDE, -1)           \
  Y(bk_tail, S.nScheds * BK_STRIDE, -1) Y(bk_cnt, S.nScheds * BK_STRIDE, 0)                            \
  Y(bk_hseq, S.nScheds * BK_STRIDE, -1) Y(bk_tseq, S.nScheds * BK_STRIDE, 0)                           \
  Y(vn_next, S.NV, -1) Y(vn_prev, S.NV, -1) Y(vn_seq, S.NV, 0) Y(vn_u, S.NV, 0) Y(vn_dirty, S.NV, 0)   \
  Y(bk_dl, S.cvTotal, -1) Y(nbad, 4, 0)                                                                \
  /* where the reference's incremental used-leaf counters differ from the leaf priorities (hived_core.h noteDelta): */ \
  /* up to DELTA_SLOTS (priority, difference) pairs per cell; s_anom counts the anomalies of a view                  */ \
  Y(v_dprio, S.NV * DELTA_SLOTS, DELTA_EMPTY) Y(v_dcnt, S.NV * DELTA_SLOTS, 0)                         \
  Y(p_dprio, S.NP * DELTA_SLOTS, DELTA_EMPTY) Y(p_dcnt, S.NP * DELTA_SLOTS, 0) Y(s_anom, S.nScheds, 0)

// Z(name, count): scratch of one scheduling decision — one private copy per CTA (struct Scratch)
#define HIVED_SCRATCH_ARRAYS(Z)                                                                        \
  Z(sfl_data, S.flTotal) Z(sfl_len, MAXL)                                                              \
  Z(vx_cell, S.VX) Z(vx_child, S.VX) Z(vx_last, S.VX) Z(vx_next, S.VX) Z(vx_nch, S.VX)                 \
  Z(pa_list, S.LS) Z(np_head, S.LS) Z(np_cnt, S.LS)                                                    \
  Z(pl_v, S.LS) Z(pl_p, S.LS) Z(pl_v2, S.LS) Z(pl_p2, S.LS)                                            \
  Z(cand, S.PS * MAX_NODE_LEAVES) Z(cand_len, S.PS) Z(cand_node, S.PS)                                 \
  Z(pod_need, S.PS) Z(pod_pos, S.PS) Z(pod_cell, S.PS) Z(pod_unit, S.PS)                               \
  Z(mc0, S.maxLevelCount + MAX_FANOUT) Z(mcbuf, MAXL * MAX_FANOUT)                                     \
  Z(mcpick, MAXL * MAX_FANOUT) Z(mccells, MAXL * MAX_FANOUT)                                           \
  Z(lz_group, S.LS) Z(lz_save, (int64_t)S.LZ * (S.LS + 1)) Z(ba_buf, (int64_t)MAXL * S.maxLevelCount)  \
  Z(tmp_list, S.maxLevelCount + MAX_FANOUT)                                                            \
  Z(vw_cell, S.maxViewN) Z(vw_info, S.maxViewN) Z(vw_ordA, S.maxViewN) Z(vw_ordB, S.maxViewN) Z(vw_sinfo, S.maxViewN)

struct Scratch {
#define Z(name, count) int32_t* name;
  HIVED_SCRATCH_ARRAYS(Z)
#undef Z
};

struct DevSizes {
  int32_t NP, NV, nChains, nVCs, nLeafTypes, nPinned, nNodes, nVsets, nScheds;
  int32_t flTotal, dmTotal, cvTotal, maxGroups, maxPods, LS, PS, VX, LZ;
  int32_t maxLevelCount, maxViewN, bitmapWords, maxLevels, maxNodeLeaves, AS, directLeaf;
};

struct Dev {
  DevSizes S;
#define X(name) const int32_t* name;
  HIVED_STATIC_ARRAYS(X)
#undef X
#define Y(name, count, init) int32_t* name;
  HIVED_MUTABLE_ARRAYS(Y)
#undef Y
  GroupFld<0> g_state; GroupFld<1> g_vc; GroupFld<2> g_prio; GroupFld<3> g_flags; GroupFld<4> g_nmem; GroupFld<5> g_npre;
  GroupMemFld<8> g_mem_leaf; GroupMemFld<16> g_mem_pods;
  long long* stats;        // [ST_COUNT] counters, see ST_* below
  int32_t* epoch;          // [MAX_CTAS] per-CTA stamp for vx_stamp
  const Scratch* scratch;  // [nCta] private scratch arrays of every CTA
  int32_t* progress;       // [MAX_CTAS] index of the event each CTA is working on (multi-CTA ordering)
};

enum {
  ST_VIEW_NODES = 0, ST_LEAVES = 1, ST_FREE_CELLS = 2, ST_PODS = 3, ST_SCHEDULE = 4, ST_BIND = 5, ST_WAIT = 6,
  ST_PREEMPT = 7, ST_PRIO_MASK = 8 /* bit (p+1) for small priorities, else bit 62 */,
  /* SM cycles spent per phase (leader warp), for profiles/ */
  ST_CYC_VIEW = 9, ST_CYC_LEAF = 10, ST_CYC_MAP = 11, ST_CYC_EMIT = 12, ST_CYC_COMMIT = 13, ST_CYC_DELETE = 14, ST_CYC_TOTAL = 15,
  ST_CYC_WAIT = 16 /* spinning at the entry of a shared section (VC-parallel mode) */, ST_SHARED_SECTIONS = 17,
  ST_CYC_SCHED_EXISTING = 18, ST_N_SCHED_EXISTING = 19, ST_CYC_DELETE_POD = 20, ST_N_DELETE_POD = 21,
  ST_CYC_COMMIT_POD = 22, ST_N_COMMIT_POD = 23,
  ST_DBG0 = 24 /* 16 scratch cycle counters for profiling sessions (hived_bench_debug_cycles) */,
  /* which path the events took (always counted; hived_bench_path_counters) */
  ST_PATH0 = 40, PC_FAST_VIEW = 0 /* scheduling passes answered by the bucketed view */, PC_GENERAL_VIEW = 1 /* full view passes */,
  PC_BK_REBUILD = 2, PC_BK_MOVERS = 3, PC_FAST_COMMIT = 4, PC_GENERAL_COMMIT = 5, PC_FAST_DELETE = 6, PC_GENERAL_DELETE = 7,
  PC_FAST_MAP = 8, PC_GENERAL_MAP = 9, PC_POD_LEAN = 10, PC_COUNT = 12,
  ST_COUNT = 40 + PC_COUNT
};

constexpr int MAX_CTAS = 32;

// group flags
enum { GF_LAZY_ENABLE = 1, GF_HAS_VIRTUAL = 2, GF_LAZY_PREEMPTED = 4 };

}  // namespace hived
