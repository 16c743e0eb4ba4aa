// MIT License
//
// cuda_backend.go — drop-in file for microsoft/hivedscheduler, pkg/algorithm.
//
// CudaHivedAlgorithm implements internal.SchedulerAlgorithm (pkg/internal/types.go:76-100) over the C ABI of
// include/hived.h (libhived_cuda.so, the CUDA-native scheduling path).  It keeps in Go exactly what the reference
// keeps in Go around HivedAlgorithm: the pod-annotation YAML (internal.ExtractPodSchedulingSpec /
// ExtractPodBindInfo, pkg/internal/utils.go:199-289), the string <-> id interning, the materialisation of
// api.PodBindInfo / PodWaitInfo / PodPreemptInfo and of the inspect objects.  Everything below the interface —
// rows a1..a21 of the hot path — runs in the library.
//
// Selected at the reference's single construction site, pkg/scheduler/scheduler.go:149 (see scheduler.go.patch in
// this directory's parent).  hivedscheduler_b200/algorithm.py is the same shim in Python; it is the one the parity
// tests drive (this image has no Go toolchain), and this file follows it function by function.
package algorithm

/*
#cgo CFLAGS: -I${SRCDIR}/../../third_party/hived-b200/include
#cgo LDFLAGS: -L${SRCDIR}/../../third_party/hived-b200 -lhived_cuda
#include <stdlib.h>
#include "hived.h"
*/
import "C"

import (
	"fmt"
	"math/rand"
	"sort"
	"strings"
	"sync"
	"unsafe"

	"github.com/microsoft/hivedscheduler/pkg/api"
	"github.com/microsoft/hivedscheduler/pkg/internal"
	core "k8s.io/api/core/v1"
	meta "k8s.io/apimachinery/pkg/apis/meta/v1"
	"k8s.io/apimachinery/pkg/types"
	"k8s.io/klog"
)

// interner hands out dense ids for names and takes them back: the library's group / pod tables are dense and
// bounded (hived_options_t), so an id is recycled once its owner is gone (include/hived.h, "Id lifetime").
type interner struct {
	ids   map[string]C.int32_t
	names []string
	free  []C.int32_t
}

func newInterner() *interner { return &interner{ids: map[string]C.int32_t{}} }

func (t *interner) intern(name string) C.int32_t {
	if id, ok := t.ids[name]; ok {
		return id
	}
	var id C.int32_t
	if n := len(t.free); n > 0 {
		id = t.free[n-1]
		t.free = t.free[:n-1]
		t.names[id] = name
	} else {
		id = C.int32_t(len(t.names))
		t.names = append(t.names, name)
	}
	t.ids[name] = id
	return id
}

func (t *interner) lookup(name string) (C.int32_t, bool) {
	id, ok := t.ids[name]
	return id, ok
}

func (t *interner) release(name string) {
	if id, ok := t.ids[name]; ok {
		delete(t.ids, name)
		t.names[id] = ""
		t.free = append(t.free, id)
	}
}

func (t *interner) name(id C.int32_t) string {
	if id >= 0 && int(id) < len(t.names) {
		return t.names[id]
	}
	return ""
}

const (
	cudaMaxGroups      = 1 << 17
	cudaMaxPods        = 1 << 20
	cudaMaxGroupLeaves = 512
	cudaMaxGroupPods   = 64
)

// CudaHivedAlgorithm is the CUDA-backed implementation of internal.SchedulerAlgorithm.
type CudaHivedAlgorithm struct {
	ctx *C.hived_ctx
	// the reference's algorithmLock (hived_algorithm.go:104): the library is single-writer
	lock sync.RWMutex

	nodeNames, chainNames, vcNames, leafTypeNames, pinnedNames, cellTypeNames []string
	nodeIDs, chainIDs, vcIDs, leafTypeIDs, pinnedIDs, cellTypeIDs             map[string]C.int32_t

	groups *interner             // AffinityGroup.Name -> group id
	pods   *interner             // Pod.UID -> pod id
	podObj map[C.int32_t]*core.Pod // victims and allocated pods come back as pod ids

	// the "every node is suggested" bitmap, built once (hived_algorithm.go:190-193 builds a string set per call)
	bitmapWords int
	pool        []C.int32_t
	// LazyPreemptionStatus: the library reports THAT a group was lazy-preempted; the time it was first seen so is
	// kept here, the preemptor's name is not carried below the ABI (DESIGN.md section 7)
	lazyInfo map[string]*api.LazyPreemptionStatus
}

// NewCudaHivedAlgorithm mirrors NewHivedAlgorithm (hived_algorithm.go:108-145): it panics on an invalid config.
func NewCudaHivedAlgorithm(sConfig *api.Config) *CudaHivedAlgorithm {
	spec := C.CString(toHivedSpec(sConfig))
	defer C.free(unsafe.Pointer(spec))
	opt := C.hived_options_t{
		max_groups: cudaMaxGroups, max_pods: cudaMaxPods,
		max_group_leaves: cudaMaxGroupLeaves, max_group_pods: cudaMaxGroupPods,
		flags: C.HIVED_OPT_NO_RESULT_HASH,
	}
	var ctx *C.hived_ctx
	if rc := C.hived_create(spec, &opt, &ctx); rc != 0 {
		panic(fmt.Errorf("NewCudaHivedAlgorithm failed (%d): %s", int(rc), C.GoString(C.hived_create_error())))
	}
	h := &CudaHivedAlgorithm{
		ctx: ctx, groups: newInterner(), pods: newInterner(),
		podObj: map[C.int32_t]*core.Pod{}, lazyInfo: map[string]*api.LazyPreemptionStatus{},
	}
	table := func(n C.int32_t, name func(C.int32_t) *C.char) ([]string, map[string]C.int32_t) {
		names := make([]string, int(n))
		ids := make(map[string]C.int32_t, int(n))
		for i := C.int32_t(0); i < n; i++ {
			names[i] = C.GoString(name(i))
			ids[names[i]] = i
		}
		return names, ids
	}
	h.nodeNames, h.nodeIDs = table(C.hived_num_nodes(ctx), func(i C.int32_t) *C.char { return C.hived_node_name(ctx, i) })
	h.chainNames, h.chainIDs = table(C.hived_num_chains(ctx), func(i C.int32_t) *C.char { return C.hived_chain_name(ctx, i) })
	h.vcNames, h.vcIDs = table(C.hived_num_vcs(ctx), func(i C.int32_t) *C.char { return C.hived_vc_name(ctx, i) })
	h.leafTypeNames, h.leafTypeIDs = table(C.hived_num_leaf_types(ctx), func(i C.int32_t) *C.char { return C.hived_leaf_type_name(ctx, i) })
	h.pinnedNames, h.pinnedIDs = table(C.hived_num_pinned(ctx), func(i C.int32_t) *C.char { return C.hived_pinned_name(ctx, i) })
	h.cellTypeNames, h.cellTypeIDs = table(C.hived_num_cell_types(ctx), func(i C.int32_t) *C.char { return C.hived_cell_type_name(ctx, i) })
	h.bitmapWords = (len(h.nodeNames) + 31) / 32
	h.pool = make([]C.int32_t, 3*cudaMaxGroupLeaves+2*4096+64)
	return h
}

// Close releases the device context (the reference's object has no counterpart: it lives as long as the process).
func (h *CudaHivedAlgorithm) Close() {
	h.lock.Lock()
	defer h.lock.Unlock()
	if h.ctx != nil {
		C.hived_destroy(h.ctx)
		h.ctx = nil
	}
}

// toHivedSpec serialises *api.Config (after api.NewConfig defaulting, pkg/api/config.go:87-167) into the HIVEDSPEC
// text documented in include/hived.h (config.py::to_spec_text is the same function).
func toHivedSpec(c *api.Config) string {
	var b strings.Builder
	tok := func(s string) string {
		if s == "" || strings.ContainsAny(s, " \t\r\n") {
			panic(fmt.Errorf("names in the scheduler config must be non-empty and free of whitespace: %q", s))
		}
		return s
	}
	b.WriteString("HIVEDSPEC 1\n")
	var ctNames []string
	for name := range c.PhysicalCluster.CellTypes {
		ctNames = append(ctNames, string(name))
	}
	sort.Strings(ctNames)
	fmt.Fprintf(&b, "celltypes %d\n", len(ctNames))
	for _, name := range ctNames {
		ct := c.PhysicalCluster.CellTypes[api.CellType(name)]
		isNode := 0
		if ct.IsNodeLevel {
			isNode = 1
		}
		fmt.Fprintf(&b, "%s %s %d %d\n", tok(name), tok(string(ct.ChildCellType)), ct.ChildCellNumber, isNode)
	}
	fmt.Fprintf(&b, "physicalcells %d\n", len(c.PhysicalCluster.PhysicalCells))
	var emit func(cell *api.PhysicalCellSpec, depth int)
	emit = func(cell *api.PhysicalCellSpec, depth int) {
		pid := string(cell.PinnedCellId)
		if pid == "" {
			pid = "-"
		}
		fmt.Fprintf(&b, "%d %s %s %s %d\n", depth, tok(string(cell.CellType)), tok(string(cell.CellAddress)), tok(pid), len(cell.CellChildren))
		for i := range cell.CellChildren {
			emit(&cell.CellChildren[i], depth+1)
		}
	}
	for i := range c.PhysicalCluster.PhysicalCells {
		emit(&c.PhysicalCluster.PhysicalCells[i], 0)
	}
	var vcNames []string
	for vcn := range c.VirtualClusters {
		vcNames = append(vcNames, string(vcn))
	}
	sort.Strings(vcNames)
	fmt.Fprintf(&b, "virtualclusters %d\n", len(vcNames))
	for _, vcn := range vcNames {
		spec := c.VirtualClusters[api.VirtualClusterName(vcn)]
		fmt.Fprintf(&b, "vc %s %d %d\n", tok(vcn), len(spec.VirtualCells), len(spec.PinnedCells))
		for _, v := range spec.VirtualCells {
			fmt.Fprintf(&b, "%s %d\n", tok(string(v.CellType)), v.CellNumber)
		}
		for _, p := range spec.PinnedCells {
			fmt.Fprintf(&b, "%s\n", tok(string(p.PinnedCellId)))
		}
	}
	b.WriteString("end\n")
	return b.String()
}

// raise turns a library return code into the reference's error convention (pkg/internal/types.go:58-61): 1..99 are
// user errors (HTTP 400, internal.NewBadRequestError), >= 100 platform errors (plain panic).
func (h *CudaHivedAlgorithm) raise(rc C.int) {
	msg := C.GoString(C.hived_last_error(h.ctx))
	if rc >= 1 && rc < 100 {
		panic(internal.NewBadRequestError(msg))
	}
	panic(fmt.Errorf("panic (%d): %s", int(rc), msg))
}

// raiseForPod is raise for a Schedule call: user errors carry the reference's own message text (the names live above
// the ABI, the library only knows ids) — hived_algorithm.go:684-686, 785-787, 824-826, 858-868.
func (h *CudaHivedAlgorithm) raiseForPod(rc C.int, s *api.PodSchedulingSpec, sp *C.hived_pod_spec_t, pod *core.Pod) {
	key := internal.Key(pod)
	switch int(rc) {
	case C.HIVED_ERR_UNKNOWN_VC:
		panic(internal.NewBadRequestError(fmt.Sprintf("[%v]: VC %v does not exists!", key, s.VirtualCluster)))
	case C.HIVED_ERR_UNKNOWN_PINNED_CELL:
		panic(internal.NewBadRequestError(fmt.Sprintf("[%v]: VC %v does not have pinned cell %v", key, s.VirtualCluster, s.PinnedCellId)))
	case C.HIVED_ERR_OPPORTUNISTIC_PINNED:
		panic(internal.NewBadRequestError(fmt.Sprintf("[%v]: opportunistic pod not supported to use pinned cell %v", key, s.PinnedCellId)))
	case C.HIVED_ERR_LEAF_TYPE_NOT_IN_CLUSTER:
		panic(internal.NewBadRequestError(fmt.Sprintf(
			"[%v]: Pod requesting leaf cell type %v which the whole cluster does not have", key, s.LeafCellType)))
	case C.HIVED_ERR_LEAF_TYPE_NOT_IN_VC:
		panic(internal.NewBadRequestError(fmt.Sprintf(
			"[%v]: Pod requesting leaf cell type %v which VC %v does not have", key, s.LeafCellType, s.VirtualCluster)))
	case C.HIVED_ERR_TOO_MANY_PODS:
		var gp C.hived_group_placement_t
		total := int32(0)
		if C.hived_get_group_placement(h.ctx, sp.group, &gp, nil, nil, 0, nil, 0, nil, 0) == 0 {
			for i := 0; i < int(gp.n_members); i++ {
				if int32(gp.member_leaf_num[i]) == s.LeafCellNumber {
					total += int32(gp.member_pod_num[i])
				}
			}
		}
		panic(internal.NewBadRequestError(fmt.Sprintf(
			"Requesting more pods than the configured number for %v leaf cells (%v pods) in affinity group %v",
			s.LeafCellNumber, total, s.AffinityGroup.Name)))
	}
	h.raise(rc)
}

func (h *CudaHivedAlgorithm) toSpec(s *api.PodSchedulingSpec, pod *core.Pod) C.hived_pod_spec_t {
	var sp C.hived_pod_spec_t
	sp.pod = h.pods.intern(string(pod.UID))
	sp.group = h.groups.intern(s.AffinityGroup.Name)
	sp.vc = -1
	if id, ok := h.vcIDs[string(s.VirtualCluster)]; ok {
		sp.vc = id
	}
	sp.priority = C.int32_t(s.Priority)
	sp.pinned = -1
	if s.PinnedCellId != "" {
		sp.pinned = -2
		if id, ok := h.pinnedIDs[string(s.PinnedCellId)]; ok {
			sp.pinned = id
		}
	}
	sp.leaf_type = -1
	if s.LeafCellType != "" {
		sp.leaf_type = -2
		if id, ok := h.leafTypeIDs[s.LeafCellType]; ok {
			sp.leaf_type = id
		}
	}
	sp.leaf_num = C.int32_t(s.LeafCellNumber)
	if s.LazyPreemptionEnable {
		sp.flags |= C.HIVED_SPEC_LAZY_PREEMPTION
	}
	if s.IgnoreK8sSuggestedNodes {
		sp.flags |= C.HIVED_SPEC_IGNORE_SUGGESTED
	}
	if len(s.AffinityGroup.Members) > C.HIVED_MAX_MEMBERS {
		panic(internal.NewBadRequestError(fmt.Sprintf("affinity group has more than %d members", C.HIVED_MAX_MEMBERS)))
	}
	sp.n_members = C.int32_t(len(s.AffinityGroup.Members))
	for i, m := range s.AffinityGroup.Members {
		sp.member_leaf_num[i] = C.int32_t(m.LeafCellNumber)
		sp.member_pod_num[i] = C.int32_t(m.PodNumber)
	}
	return sp
}

// suggestedBitmap: suggestedNodes []string -> node bitmap (the reference builds a string set, :190-193)
func (h *CudaHivedAlgorithm) suggestedBitmap(suggestedNodes []string) []C.uint32_t {
	n := h.bitmapWords
	if n == 0 {
		n = 1
	}
	words := make([]C.uint32_t, n)
	for _, name := range suggestedNodes {
		if id, ok := h.nodeIDs[name]; ok {
			words[id>>5] |= 1 << (uint(id) & 31)
		}
	}
	return words
}

// waitReason rebuilds PodWaitInfo.Reason (topology_aware_scheduler.go:268-306, intra_vc_scheduler.go:112,
// hived_algorithm.go:935-941, 975) from the code and cell the library returns
func (h *CudaHivedAlgorithm) waitReason(res *C.hived_result_t, s *api.PodSchedulingSpec) string {
	code := int(res.wait_code)
	base := code & 15
	addr := ""
	if res.wait_cell >= 0 {
		addr = C.GoString(C.hived_physical_cell_address(h.ctx, res.wait_cell))
	}
	if base == C.HIVED_WAIT_MAPPING {
		kind := "bad or non-suggested"
		if s.IgnoreK8sSuggestedNodes {
			kind = "bad"
		}
		return fmt.Sprintf("Mapping the virtual placement would need to use at least one %s node", kind)
	}
	reason := ""
	switch base {
	case C.HIVED_WAIT_INSUFFICIENT:
		reason = "insufficient capacity"
	case C.HIVED_WAIT_BAD_NODE:
		reason = fmt.Sprintf("have to use at least one bad node %s", addr)
	case C.HIVED_WAIT_NON_SUGGESTED_NODE:
		reason = fmt.Sprintf("have to use at least one non-suggested node %s", addr)
	}
	if code&C.HIVED_WAIT_SCOPE_VC != 0 {
		reason = fmt.Sprintf("%s when scheduling in VC %s", reason, s.VirtualCluster)
	} else if code&C.HIVED_WAIT_SCOPE_PHYSICAL != 0 {
		reason = fmt.Sprintf("%s when scheduling in physical cluster", reason)
	}
	return reason
}

// retrieveMissingPodPlacement is the reference's function of the same name (pkg/algorithm/utils.go:250-265): the
// placement of a pod whose cells left the cluster spec comes from the bind-info annotation of the group's pods.
func (h *CudaHivedAlgorithm) retrieveMissingPodPlacement(gid C.int32_t, leafCellNum int32, podIndex int32) (api.PodPlacementInfo, string) {
	var gp C.hived_group_placement_t
	pods := make([]C.int32_t, cudaMaxGroupPods)
	C.hived_get_group_placement(h.ctx, gid, &gp, nil, nil, 0, &pods[0], cudaMaxGroupPods, nil, 0)
	n := int(gp.n_pods)
	if n > cudaMaxGroupPods {
		n = cudaMaxGroupPods
	}
	for _, pid := range pods[:n] {
		pod := h.podObj[pid]
		if pid < 0 || pod == nil {
			continue
		}
		if _, ok := pod.Annotations[api.AnnotationKeyPodBindInfo]; !ok {
			continue
		}
		info := internal.ExtractPodBindInfo(pod)
		for _, mbi := range info.AffinityGroupBindInfo {
			if leafCellNum == int32(len(mbi.PodPlacements[0].PhysicalLeafCellIndices)) {
				return mbi.PodPlacements[podIndex], info.CellChain
			}
		}
	}
	panic(fmt.Sprintf("No allocated pod found in an allocated group %v when retrieving placement for pod %v with leaf cell number %v",
		h.groups.name(gid), podIndex, leafCellNum))
}

// bindInfo rebuilds api.PodBindInfo from the result record and the leaf triples in the pool
// (generatePodScheduleResult / generateAffinityGroupBindInfo, pkg/algorithm/utils.go:38-171)
func (h *CudaHivedAlgorithm) bindInfo(res *C.hived_result_t, gid C.int32_t) *api.PodBindInfo {
	k := int(res.leaf_off)
	agbi := make([]api.AffinityGroupMemberBindInfo, int(res.n_members))
	chain := ""
	curM := -1
	for m := 0; m < int(res.n_members); m++ {
		ln, pn := int(res.member_leaf_num[m]), int(res.member_pod_num[m])
		pps := make([]api.PodPlacementInfo, pn)
		for pi := 0; pi < pn; pi++ {
			pp := api.PodPlacementInfo{
				PhysicalLeafCellIndices: make([]int32, ln),
				PreassignedCellTypes:    make([]api.CellType, ln),
			}
			for j := 0; j < ln; j++ {
				nid, li, t := h.pool[k], h.pool[k+1], h.pool[k+2]
				k += 3
				if nid == C.HIVED_NIL_CELL && li == C.HIVED_NIL_CELL && t == C.HIVED_NIL_CELL {
					var got api.PodPlacementInfo
					got, chain = h.retrieveMissingPodPlacement(gid, int32(ln), int32(pi))
					pp = api.PodPlacementInfo{
						PhysicalNode:            got.PhysicalNode,
						PhysicalLeafCellIndices: append([]int32(nil), got.PhysicalLeafCellIndices...),
						PreassignedCellTypes:    append([]api.CellType(nil), got.PreassignedCellTypes...),
					}
					continue
				}
				if pp.PhysicalNode == "" && nid >= 0 {
					pp.PhysicalNode = h.nodeNames[nid]
				}
				pp.PhysicalLeafCellIndices[j] = int32(li)
				if t >= 0 {
					pp.PreassignedCellTypes[j] = api.CellType(h.cellTypeNames[t])
				}
			}
			pps[pi] = pp
		}
		if curM < 0 && ln == int(res.this_n) {
			curM = m
		}
		agbi[m] = api.AffinityGroupMemberBindInfo{PodPlacements: pps}
	}
	mine := agbi[curM].PodPlacements[int(res.pod_index)]
	if res.chain >= 0 { // utils.go:163-165: the chain of the pod's first cell when that cell exists
		chain = h.chainNames[res.chain]
	}
	return &api.PodBindInfo{
		Node:                  mine.PhysicalNode,
		LeafCellIsolation:     append([]int32(nil), mine.PhysicalLeafCellIndices...),
		CellChain:             chain,
		AffinityGroupBindInfo: agbi,
	}
}

// victimsOnOneRandomNode is generatePodPreemptInfo (pkg/algorithm/utils.go:81-105): the library returns ALL victims
// on ALL nodes (pod id, node id); K8s preempts on one node at a time, picked at random like the reference does.
func (h *CudaHivedAlgorithm) victimsOnOneRandomNode(res *C.hived_result_t, pod *core.Pod) *internal.PodPreemptInfo {
	byNode := map[C.int32_t][]*core.Pod{}
	var nodesHavingVictims []C.int32_t
	for k := 0; k < int(res.n_victims); k++ {
		pid, nid := h.pool[int(res.victim_off)+2*k], h.pool[int(res.victim_off)+2*k+1]
		if _, seen := byNode[nid]; !seen {
			nodesHavingVictims = append(nodesHavingVictims, nid)
		}
		byNode[nid] = append(byNode[nid], h.podObj[pid])
	}
	nodeToPreempt := nodesHavingVictims[rand.Int31n(int32(len(nodesHavingVictims)))]
	var victimKeys []string
	for _, v := range byNode[nodeToPreempt] {
		victimKeys = append(victimKeys, internal.Key(v))
	}
	klog.Infof("[%v]: need to preempt pods %v", internal.Key(pod), victimKeys)
	return &internal.PodPreemptInfo{VictimPods: byNode[nodeToPreempt]}
}

// ---------------------------------------------------------------------------------------------------------------
// internal.SchedulerAlgorithm
// ---------------------------------------------------------------------------------------------------------------

// Schedule — hived_algorithm.go:180-224.
func (h *CudaHivedAlgorithm) Schedule(pod *core.Pod, suggestedNodes []string, phase internal.SchedulingPhase) internal.PodScheduleResult {
	h.lock.Lock()
	defer h.lock.Unlock()

	klog.Infof("[%v]: Scheduling pod in %v phase...", internal.Key(pod), phase)
	s := internal.ExtractPodSchedulingSpec(pod)
	sp := h.toSpec(s, pod)
	h.podObj[sp.pod] = pod
	bitmap := h.suggestedBitmap(suggestedNodes)
	ph := C.int32_t(C.HIVED_PHASE_FILTERING)
	if phase == internal.PreemptingPhase {
		ph = C.HIVED_PHASE_PREEMPTING
	}
	var res C.hived_result_t
	rc := C.hived_schedule(h.ctx, &sp, (*C.uint32_t)(unsafe.Pointer(&bitmap[0])), ph, &res, &h.pool[0], C.int32_t(len(h.pool)))
	if rc != 0 {
		h.raiseForPod(rc, s, &sp, pod)
	}
	switch res.kind {
	case C.HIVED_KIND_WAIT:
		return internal.PodScheduleResult{PodWaitInfo: &internal.PodWaitInfo{Reason: h.waitReason(&res, s)}}
	case C.HIVED_KIND_PREEMPT:
		return internal.PodScheduleResult{PodPreemptInfo: h.victimsOnOneRandomNode(&res, pod)}
	default:
		return internal.PodScheduleResult{PodBindInfo: h.bindInfo(&res, sp.group)}
	}
}

// AddUnallocatedPod — hived_algorithm.go:226-227 (a no-op in the reference).
func (h *CudaHivedAlgorithm) AddUnallocatedPod(pod *core.Pod) {}

// DeleteUnallocatedPod — hived_algorithm.go:229-245.
func (h *CudaHivedAlgorithm) DeleteUnallocatedPod(pod *core.Pod) {
	h.lock.Lock()
	defer h.lock.Unlock()

	s := internal.ExtractPodSchedulingSpec(pod)
	gid, ok := h.groups.lookup(s.AffinityGroup.Name)
	if !ok {
		return // never seen: nothing is preempting under that name
	}
	pid := h.pods.intern(string(pod.UID))
	if rc := C.hived_delete_unallocated_pod(h.ctx, gid, pid); rc != 0 {
		h.raise(rc)
	}
	h.releasePod(pod, pid)
	h.releaseGroupIfGone(s.AffinityGroup.Name, gid)
}

// toBindInfo flattens api.PodBindInfo (from the pod-bind-info annotation) for hived_add_allocated_pod
func (h *CudaHivedAlgorithm) toBindInfo(info *api.PodBindInfo) (C.hived_bind_info_t, []C.int32_t) {
	var bi C.hived_bind_info_t
	bi.node, bi.chain = -1, -1
	if id, ok := h.nodeIDs[info.Node]; ok {
		bi.node = id
	}
	bi.first_leaf = C.int32_t(info.LeafCellIsolation[0])
	if id, ok := h.chainIDs[info.CellChain]; ok {
		bi.chain = id
	}
	if len(info.AffinityGroupBindInfo) > C.HIVED_MAX_MEMBERS {
		panic(fmt.Errorf("bind info has too many members"))
	}
	bi.n_members = C.int32_t(len(info.AffinityGroupBindInfo))
	bi.has_preassigned = 1
	var flat []C.int32_t
	for m, gms := range info.AffinityGroupBindInfo {
		bi.member_leaf_num[m] = C.int32_t(len(gms.PodPlacements[0].PhysicalLeafCellIndices))
		bi.member_pod_num[m] = C.int32_t(len(gms.PodPlacements))
		for _, pl := range gms.PodPlacements {
			if pl.PreassignedCellTypes == nil { // old annotations (hived_algorithm.go:1260-1263)
				bi.has_preassigned = 0
			}
			nid := C.int32_t(-1)
			if id, ok := h.nodeIDs[pl.PhysicalNode]; ok {
				nid = id
			}
			for j, li := range pl.PhysicalLeafCellIndices {
				t := C.int32_t(-1)
				if pl.PreassignedCellTypes != nil && pl.PreassignedCellTypes[j] != "" {
					t = -2
					if id, ok := h.cellTypeIDs[string(pl.PreassignedCellTypes[j])]; ok {
						t = id
					}
				}
				flat = append(flat, nid, C.int32_t(li), t)
			}
		}
	}
	bi.n_leaves = C.int32_t(len(flat) / 3)
	if len(flat) == 0 {
		flat = []C.int32_t{0}
	}
	return bi, flat
}

// getAllocatedPodIndex — pkg/algorithm/utils.go:291-304 (unchanged logic, on the annotation).
func cudaGetAllocatedPodIndex(info *api.PodBindInfo, leafCellNum int32) int32 {
	for _, gms := range info.AffinityGroupBindInfo {
		if int32(len(gms.PodPlacements[0].PhysicalLeafCellIndices)) == leafCellNum {
			for podIndex, placement := range gms.PodPlacements {
				if placement.PhysicalNode == info.Node {
					for _, idx := range placement.PhysicalLeafCellIndices {
						if idx == info.LeafCellIsolation[0] {
							return int32(podIndex)
						}
					}
				}
			}
		}
	}
	return -1
}

// AddAllocatedPod — hived_algorithm.go:247-270 (createAllocatedAffinityGroup :981-1041 runs in the library).
func (h *CudaHivedAlgorithm) AddAllocatedPod(pod *core.Pod) {
	h.lock.Lock()
	defer h.lock.Unlock()

	klog.Infof("[%v]: Adding allocated pod...", internal.Key(pod))
	s := internal.ExtractPodSchedulingSpec(pod)
	info := internal.ExtractPodBindInfo(pod)
	sp := h.toSpec(s, pod)
	h.podObj[sp.pod] = pod
	bi, leaves := h.toBindInfo(info)
	podIndex := cudaGetAllocatedPodIndex(info, s.LeafCellNumber)
	if rc := C.hived_add_allocated_pod(h.ctx, &sp, &bi, &leaves[0], C.int32_t(podIndex)); rc != 0 {
		h.raise(rc)
	}
}

// DeleteAllocatedPod — hived_algorithm.go:272-296 (deleteAllocatedAffinityGroup :1043-1070 runs in the library).
func (h *CudaHivedAlgorithm) DeleteAllocatedPod(pod *core.Pod) {
	h.lock.Lock()
	defer h.lock.Unlock()

	klog.Infof("[%v]: Deleting allocated pod...", internal.Key(pod))
	s := internal.ExtractPodSchedulingSpec(pod)
	info := internal.ExtractPodBindInfo(pod)
	gid, ok := h.groups.lookup(s.AffinityGroup.Name)
	if !ok {
		return // "Group %v not found when deleting pod" in the reference
	}
	podIndex := cudaGetAllocatedPodIndex(info, s.LeafCellNumber)
	removed := C.int32_t(-1)
	if rc := C.hived_delete_allocated_pod_ex(h.ctx, gid, C.int32_t(s.LeafCellNumber), C.int32_t(podIndex), &removed); rc != 0 {
		h.raise(rc)
	}
	// The reference clears the slot whoever sits there (hived_algorithm.go:287).  Only when that was THIS pod has it
	// left the library's tables; otherwise it can still come back as a preemption victim (its group object was replaced
	// under the same name and lives on through cell.usingGroup): its object and id are kept (hived.h "Id lifetime").
	if pid, ok := h.pods.lookup(string(pod.UID)); ok && pid == removed {
		h.releasePod(pod, pid)
	}
	h.releaseGroupIfGone(s.AffinityGroup.Name, gid)
}

// releasePod / releaseGroupIfGone: ids go back to the interners once their owner is gone, so that a long-running
// scheduler never runs into the dense tables' capacities (include/hived.h, "Id lifetime").
func (h *CudaHivedAlgorithm) releasePod(pod *core.Pod, pid C.int32_t) {
	delete(h.podObj, pid)
	h.pods.release(string(pod.UID))
}

func (h *CudaHivedAlgorithm) releaseGroupIfGone(name string, gid C.int32_t) {
	var gi C.hived_group_info_t
	C.hived_get_group(h.ctx, gid, &gi)
	// (referenced: cells still point at the erased object, which can be erased by name later — the name keeps its id)
	if gi.state == C.HIVED_GROUP_NONE && gi.referenced == 0 {
		h.groups.release(name)
		delete(h.lazyInfo, name)
	}
}

func (h *CudaHivedAlgorithm) setNodeHealth(name string, healthy bool) {
	id, ok := h.nodeIDs[name]
	if !ok {
		return // a node that is not in the cluster config: the reference's loops find no cell for it
	}
	v := C.int32_t(0)
	if healthy {
		v = 1
	}
	if rc := C.hived_set_node_health(h.ctx, id, v); rc != 0 {
		h.raise(rc)
	}
}

// AddNode / UpdateNode / DeleteNode — hived_algorithm.go:147-178.
func (h *CudaHivedAlgorithm) AddNode(node *core.Node) {
	h.lock.Lock()
	defer h.lock.Unlock()
	h.setNodeHealth(node.Name, internal.IsNodeHealthy(node))
}

func (h *CudaHivedAlgorithm) UpdateNode(oldNode, newNode *core.Node) {
	h.lock.Lock()
	defer h.lock.Unlock()
	if oldHealthy := internal.IsNodeHealthy(oldNode); oldHealthy != internal.IsNodeHealthy(newNode) {
		h.setNodeHealth(newNode.Name, !oldHealthy)
	}
}

func (h *CudaHivedAlgorithm) DeleteNode(node *core.Node) {
	h.lock.Lock()
	defer h.lock.Unlock()
	h.setNodeHealth(node.Name, false)
}

// ---------------------------------------------------------------------------------------------------------------
// inspect
// ---------------------------------------------------------------------------------------------------------------

var cudaGroupStates = map[C.int32_t]api.AffinityGroupState{1: "Allocated", 2: "Preempting", 3: "BeingPreempted"}
var cudaCellStates = map[C.int32_t]api.CellState{0: "Free", 1: "Used", 2: "Reserving", 3: "Reserved"}

// affinityGroup is AlgoAffinityGroup.ToAffinityGroup (pkg/algorithm/types.go:187-214); nil when the group is gone
func (h *CudaHivedAlgorithm) affinityGroup(gid C.int32_t, name string) *api.AffinityGroup {
	var gp C.hived_group_placement_t
	phys := make([]C.int32_t, cudaMaxGroupLeaves)
	virt := make([]C.int32_t, cudaMaxGroupLeaves)
	pods := make([]C.int32_t, cudaMaxGroupPods)
	pre := make([]C.int32_t, cudaMaxGroupPods)
	if rc := C.hived_get_group_placement(h.ctx, gid, &gp, &phys[0], &virt[0], cudaMaxGroupLeaves, &pods[0], cudaMaxGroupPods,
		&pre[0], cudaMaxGroupPods); rc != 0 {
		h.raise(rc)
	}
	if gp.state == C.HIVED_GROUP_NONE {
		return nil
	}
	var gi C.hived_group_info_t
	C.hived_get_group(h.ctx, gid, &gi)
	g := &api.AffinityGroup{ObjectMeta: api.ObjectMeta{Name: name}}
	if gi.vc >= 0 {
		g.Status.VC = api.VirtualClusterName(h.vcNames[gi.vc])
	}
	g.Status.Priority = int32(gi.priority)
	g.Status.State = cudaGroupStates[gp.state]
	nl := int(gp.n_leaves)
	if nl > cudaMaxGroupLeaves {
		nl = cudaMaxGroupLeaves
	}
	var info C.hived_cell_info_t
	for k := 0; k < nl; k++ {
		if phys[k] >= 0 { // nodeToLeafCellIndices, types.go:223-237
			C.hived_physical_cell_info(h.ctx, phys[k], &info)
			if g.Status.PhysicalPlacement == nil {
				g.Status.PhysicalPlacement = map[string][]int32{}
			}
			node := h.nodeNames[info.node]
			g.Status.PhysicalPlacement[node] = append(g.Status.PhysicalPlacement[node], int32(info.leaf_index))
		}
		if gp.has_virtual != 0 && virt[k] >= 0 { // preassignedCellToLeafCells, types.go:244-259
			C.hived_virtual_cell_info(h.ctx, virt[k], &info)
			if g.Status.VirtualPlacement == nil {
				g.Status.VirtualPlacement = map[api.CellAddress][]api.CellAddress{}
			}
			preAddr := api.CellAddress(C.GoString(C.hived_virtual_cell_address(h.ctx, info.preassigned)))
			g.Status.VirtualPlacement[preAddr] = append(g.Status.VirtualPlacement[preAddr],
				api.CellAddress(C.GoString(C.hived_virtual_cell_address(h.ctx, virt[k]))))
		}
	}
	np := int(gp.n_pods)
	if np > cudaMaxGroupPods {
		np = cudaMaxGroupPods
	}
	for _, pid := range pods[:np] {
		if pid >= 0 {
			g.Status.AllocatedPods = append(g.Status.AllocatedPods, types.UID(h.pods.name(pid)))
		}
	}
	npre := int(gp.n_preempting)
	if npre > cudaMaxGroupPods {
		npre = cudaMaxGroupPods
	}
	for _, pid := range pre[:npre] {
		g.Status.PreemptingPods = append(g.Status.PreemptingPods, types.UID(h.pods.name(pid)))
	}
	if gp.lazy_preempted != 0 {
		st, ok := h.lazyInfo[name]
		if !ok {
			st = &api.LazyPreemptionStatus{PreemptionTime: meta.Now()}
			h.lazyInfo[name] = st
		}
		g.Status.LazyPreemptionStatus = st
	}
	return g
}

// GetAllAffinityGroups — hived_algorithm.go:298-307.
func (h *CudaHivedAlgorithm) GetAllAffinityGroups() api.AffinityGroupList {
	h.lock.RLock()
	defer h.lock.RUnlock()

	ags := api.AffinityGroupList{}
	n := int(C.hived_list_groups(h.ctx, nil, 0))
	if n == 0 {
		return ags
	}
	ids := make([]C.int32_t, n)
	n = int(C.hived_list_groups(h.ctx, &ids[0], C.int32_t(len(ids))))
	if n > len(ids) {
		n = len(ids)
	}
	for _, gid := range ids[:n] {
		if g := h.affinityGroup(gid, h.groups.name(gid)); g != nil {
			ags.Items = append(ags.Items, *g)
		}
	}
	return ags
}

// GetAffinityGroup — hived_algorithm.go:309-321.
func (h *CudaHivedAlgorithm) GetAffinityGroup(name string) api.AffinityGroup {
	h.lock.RLock()
	defer h.lock.RUnlock()

	if gid, ok := h.groups.lookup(name); ok {
		if g := h.affinityGroup(gid, name); g != nil {
			return *g
		}
	}
	panic(internal.NewBadRequestError(fmt.Sprintf(
		"Affinity group %v does not exist since it is not allocated or preempting", name)))
}

// statusForest rebuilds both api status forests (the reference keeps them mirrored on every cell,
// cell.go:141-204, 298-312, 401-419) from one snapshot of each side.
func (h *CudaHivedAlgorithm) statusForest() (api.PhysicalClusterStatus, map[api.VirtualClusterName]api.VirtualClusterStatus) {
	np, nv := int(C.hived_num_physical_cells(h.ctx)), int(C.hived_num_virtual_cells(h.ctx))
	ps := make([]C.hived_cell_status_t, np+1)
	vs := make([]C.hived_cell_status_t, nv+1)
	if rc := C.hived_snapshot_physical(h.ctx, &ps[0], C.int32_t(np)); rc != 0 {
		h.raise(rc)
	}
	if rc := C.hived_snapshot_virtual(h.ctx, &vs[0], C.int32_t(nv)); rc != 0 {
		h.raise(rc)
	}
	cellStatus := func(i int, physical bool) (api.CellStatus, api.VirtualClusterName) {
		var info C.hived_cell_info_t
		var st C.hived_cell_status_t
		var addr string
		if physical {
			C.hived_physical_cell_info(h.ctx, C.int32_t(i), &info)
			addr = C.GoString(C.hived_physical_cell_address(h.ctx, C.int32_t(i)))
			st = ps[i]
		} else {
			C.hived_virtual_cell_info(h.ctx, C.int32_t(i), &info)
			addr = C.GoString(C.hived_virtual_cell_address(h.ctx, C.int32_t(i)))
			st = vs[i]
		}
		cs := api.CellStatus{CellAddress: api.CellAddress(addr), CellState: cudaCellStates[st.state], CellPriority: int32(st.priority)}
		if info.leaf_type >= 0 {
			cs.LeafCellType = h.leafTypeNames[info.leaf_type]
		}
		if info.cell_type >= 0 {
			cs.CellType = api.CellType(h.cellTypeNames[info.cell_type])
		}
		cs.IsNodeLevel = info.is_node_level != 0
		cs.CellHealthiness = api.CellHealthy
		if st.healthy == 0 {
			cs.CellHealthiness = api.CellBad
		}
		vc := api.VirtualClusterName("")
		if !physical {
			vc = api.VirtualClusterName(h.vcNames[info.vc])
		}
		return cs, vc
	}
	P := make([]*api.PhysicalCellStatus, np)
	V := make([]*api.VirtualCellStatus, nv)
	vcOf := make([]api.VirtualClusterName, nv)
	for i := 0; i < np; i++ {
		cs, _ := cellStatus(i, true)
		P[i] = &api.PhysicalCellStatus{CellStatus: cs}
	}
	for i := 0; i < nv; i++ {
		cs, vc := cellStatus(i, false)
		V[i] = &api.VirtualCellStatus{CellStatus: cs}
		vcOf[i] = vc
	}
	// the embedded peer copies carry the peer's current status without children (cell.go:266-283, 401-419)
	for i := 0; i < np; i++ {
		if peer := int(ps[i].peer); peer >= 0 {
			P[i].VC = vcOf[peer]
			P[i].VirtualCell = &api.VirtualCellStatus{CellStatus: V[peer].CellStatus}
		}
	}
	for i := 0; i < nv; i++ {
		if peer := int(vs[i].peer); peer >= 0 {
			V[i].PhysicalCell = &api.PhysicalCellStatus{CellStatus: P[peer].CellStatus, VC: vcOf[i]}
		}
	}
	for i := 0; i < np; i++ { // ids: cells of one (chain, level) are contiguous in construction order
		if par := int(ps[i].parent); par >= 0 {
			P[par].CellChildren = append(P[par].CellChildren, P[i])
		}
	}
	for i := 0; i < nv; i++ {
		if par := int(vs[i].parent); par >= 0 {
			V[par].CellChildren = append(V[par].CellChildren, V[i])
		}
	}
	var physTop api.PhysicalClusterStatus
	for i := 0; i < np; i++ {
		if ps[i].parent < 0 {
			physTop = append(physTop, P[i])
		}
	}
	virtTop := map[api.VirtualClusterName]api.VirtualClusterStatus{}
	for _, vcn := range h.vcNames {
		virtTop[api.VirtualClusterName(vcn)] = api.VirtualClusterStatus{}
	}
	for i := 0; i < nv; i++ {
		if vs[i].parent < 0 {
			virtTop[vcOf[i]] = append(virtTop[vcOf[i]], V[i])
		}
	}
	return physTop, virtTop
}

// GetClusterStatus — hived_algorithm.go:323-336.
func (h *CudaHivedAlgorithm) GetClusterStatus() api.ClusterStatus {
	h.lock.RLock()
	defer h.lock.RUnlock()
	p, v := h.statusForest()
	return api.ClusterStatus{PhysicalCluster: p, VirtualClusters: v}
}

// GetPhysicalClusterStatus — hived_algorithm.go:338-343.
func (h *CudaHivedAlgorithm) GetPhysicalClusterStatus() api.PhysicalClusterStatus {
	h.lock.RLock()
	defer h.lock.RUnlock()
	p, _ := h.statusForest()
	return p
}

// GetAllVirtualClustersStatus — hived_algorithm.go:345-354.
func (h *CudaHivedAlgorithm) GetAllVirtualClustersStatus() map[api.VirtualClusterName]api.VirtualClusterStatus {
	h.lock.RLock()
	defer h.lock.RUnlock()
	_, v := h.statusForest()
	return v
}

// GetVirtualClusterStatus — hived_algorithm.go:356-363.
func (h *CudaHivedAlgorithm) GetVirtualClusterStatus(vcn api.VirtualClusterName) api.VirtualClusterStatus {
	h.lock.RLock()
	defer h.lock.RUnlock()
	if _, ok := h.vcIDs[string(vcn)]; !ok {
		panic(internal.NewBadRequestError(fmt.Sprintf("VC %v not found", vcn)))
	}
	_, v := h.statusForest()
	return v[vcn]
}

var _ internal.SchedulerAlgorithm = (*CudaHivedAlgorithm)(nil)
