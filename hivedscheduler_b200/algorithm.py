"""Host-side mirror of the reference's plugin boundary for the scheduling hot path.

``HivedAlgorithm`` implements the method set of Go's ``internal.SchedulerAlgorithm``
(reference pkg/internal/types.go:76-100; sole implementation ``algorithm.HivedAlgorithm``,
pkg/algorithm/hived_algorithm.go:40-363) on top of the C ABI of include/hived.h.  It does exactly
what a cgo shim would keep in Go (INTEGRATION.md): YAML (de)serialisation of the pod annotations
(pkg/internal/utils.go:172-289), string<->id interning, and materialising ``PodBindInfo`` /
wait-reason strings from ids.  Every scheduling decision is computed by the library behind the ABI
— ``libhived_cuda.so`` for the product.  There is no CPU fallback: if the CUDA library is missing
construction fails loudly (``MissingExtension``).
"""
from __future__ import annotations

import copy
import ctypes as C
import random
from typing import Any, Dict, List, Optional

import yaml

from . import _cabi
from .config import to_spec_text

# pkg/api/constants.go:34-62
GROUP_NAME = "hivedscheduler.microsoft.com"
ANNOTATION_POD_SCHEDULING_SPEC = GROUP_NAME + "/pod-scheduling-spec"
ANNOTATION_POD_LEAF_CELL_ISOLATION = GROUP_NAME + "/pod-leaf-cell-isolation"
ANNOTATION_POD_BIND_INFO = GROUP_NAME + "/pod-bind-info"
MAX_GUARANTEED_PRIORITY = 1000
MIN_GUARANTEED_PRIORITY = 0
OPPORTUNISTIC_PRIORITY = -1

# pkg/internal/types.go:102-114
FILTERING_PHASE = "Filtering"
PREEMPTING_PHASE = "Preempting"


class WebServerError(Exception):
    """api.WebServerError (pkg/api/types.go:124-139); 4xx = user error, >=500 = platform error."""

    def __init__(self, code: int, message: str):
        super().__init__("Code: %d, Message: %s" % (code, message))
        self.code = code
        self.message = message


class PlatformError(Exception):
    """A plain Go panic of the reference (e.g. "VC Safety Broken")."""


def new_bad_request_error(message: str) -> WebServerError:  # pkg/internal/utils.go:316-318
    return WebServerError(400, message)


class Pod:
    """The fields of core.Pod the algorithm reads (name, namespace, UID, annotations, Spec.NodeName)."""

    def __init__(self, name: str, namespace: str = "default", uid: Optional[str] = None,
                 annotations: Optional[Dict[str, str]] = None, node_name: str = ""):
        self.name = name
        self.namespace = namespace
        self.uid = uid if uid is not None else name
        self.annotations = annotations if annotations is not None else {}
        self.node_name = node_name

    def deep_copy(self) -> "Pod":
        return Pod(self.name, self.namespace, self.uid, dict(self.annotations), self.node_name)

    def key(self) -> str:  # internal.Key
        return "%s(%s/%s)" % (self.uid, self.namespace, self.name)


class PodScheduleResult:
    """internal.PodScheduleResult (pkg/internal/types.go:132-136)."""

    def __init__(self):
        self.pod_wait_info: Optional[Dict[str, Any]] = None      # {"reason": str}
        self.pod_preempt_info: Optional[Dict[str, Any]] = None   # {"victim_pods": [Pod]}
        self.pod_bind_info: Optional[Dict[str, Any]] = None      # api.PodBindInfo as a dict


def to_yaml(obj: Any) -> str:
    return yaml.safe_dump(obj, default_flow_style=False, sort_keys=False)


def convert_old_annotation(annotation: str) -> str:  # pkg/internal/utils.go:188-197
    for old, new in (("gpuType", "leafCellType"), ("gpuNumber", "leafCellNumber"),
                     ("gpuIsolation", "leafCellIsolation"), ("physicalGpuIndices", "physicalLeafCellIndices")):
        annotation = annotation.replace(old, new)
    return annotation


def extract_pod_scheduling_spec(pod: Pod) -> Dict[str, Any]:
    """internal.ExtractPodSchedulingSpec (pkg/internal/utils.go:230-289): every failure is a 400."""
    pfx = "Pod annotation %s: " % ANNOTATION_POD_SCHEDULING_SPEC
    try:
        annotation = convert_old_annotation(pod.annotations.get(ANNOTATION_POD_SCHEDULING_SPEC, ""))
        if annotation == "":
            raise ValueError(pfx + "Annotation does not exist or is empty")
        raw = yaml.safe_load(annotation) or {}
        s = {
            "virtualCluster": raw.get("virtualCluster") or "",
            "priority": int(raw.get("priority") or 0),
            "pinnedCellId": raw.get("pinnedCellId") or "",
            "leafCellType": raw.get("leafCellType") or "",
            "leafCellNumber": int(raw.get("leafCellNumber") or 0),
            "gangReleaseEnable": bool(raw.get("gangReleaseEnable") or False),
            "lazyPreemptionEnable": bool(raw.get("lazyPreemptionEnable") or False),
            "ignoreK8sSuggestedNodes": True if raw.get("ignoreK8sSuggestedNodes") is None
            else bool(raw.get("ignoreK8sSuggestedNodes")),
            "affinityGroup": raw.get("affinityGroup"),
        }
        if s["affinityGroup"] is None:
            s["affinityGroup"] = {"name": "%s/%s" % (pod.namespace, pod.name),
                                  "members": [{"podNumber": 1, "leafCellNumber": s["leafCellNumber"]}]}
        ag = s["affinityGroup"]
        ag = {"name": ag.get("name") or "",
              "members": [{"podNumber": int(m.get("podNumber") or 0), "leafCellNumber": int(m.get("leafCellNumber") or 0)}
                          for m in (ag.get("members") or [])]}
        s["affinityGroup"] = ag
        if s["virtualCluster"] == "":
            raise ValueError(pfx + "VirtualCluster is empty")
        if s["priority"] < OPPORTUNISTIC_PRIORITY:
            raise ValueError(pfx + "Priority is less than %d" % OPPORTUNISTIC_PRIORITY)
        if s["priority"] > MAX_GUARANTEED_PRIORITY:
            raise ValueError(pfx + "Priority is greater than %d" % MAX_GUARANTEED_PRIORITY)
        if s["leafCellNumber"] <= 0:
            raise ValueError(pfx + "LeafCellNumber is non-positive")
        if ag["name"] == "":
            raise ValueError(pfx + "AffinityGroup.Name is empty")
        in_group = False
        for m in ag["members"]:
            if m["podNumber"] <= 0:
                raise ValueError(pfx + "AffinityGroup.Members has non-positive PodNumber")
            if m["leafCellNumber"] <= 0:
                raise ValueError(pfx + "AffinityGroup.Members has non-positive LeafCellNumber")
            if m["leafCellNumber"] == s["leafCellNumber"]:
                in_group = True
        if not in_group:
            raise ValueError(pfx + "AffinityGroup.Members does not contains current Pod")
        return s
    except WebServerError:
        raise
    except Exception as e:  # AsBadRequestPanic
        raise new_bad_request_error(str(e))


def extract_pod_bind_info(pod: Pod) -> Dict[str, Any]:  # pkg/internal/utils.go:199-212
    annotation = convert_old_annotation(pod.annotations.get(ANNOTATION_POD_BIND_INFO, ""))
    if annotation == "":
        raise PlatformError("Pod does not contain or contains empty annotation: %s" % ANNOTATION_POD_BIND_INFO)
    return yaml.safe_load(annotation)


def new_binding_pod(pod: Pod, pod_bind_info: Dict[str, Any]) -> Pod:  # pkg/internal/utils.go:172-186
    binding = pod.deep_copy()
    binding.node_name = pod_bind_info["node"]
    binding.annotations[ANNOTATION_POD_LEAF_CELL_ISOLATION] = ",".join(str(i) for i in pod_bind_info["leafCellIsolation"])
    binding.annotations[ANNOTATION_POD_BIND_INFO] = to_yaml(pod_bind_info)
    return binding


def get_allocated_pod_index(info: Dict[str, Any], leaf_cell_num: int) -> int:  # pkg/algorithm/utils.go:291-304
    for gms in info.get("affinityGroupBindInfo") or []:
        pps = gms["podPlacements"]
        if len(pps[0]["physicalLeafCellIndices"]) == leaf_cell_num:
            for pod_index, placement in enumerate(pps):
                if placement["physicalNode"] == info["node"] and \
                        info["leafCellIsolation"][0] in placement["physicalLeafCellIndices"]:
                    return pod_index
    return -1


class _Interner:
    """name -> dense id, with the ids taken back once their owner is gone (the library's group / pod tables are dense
    and bounded by hived_options_t: a long-running scheduler must not run out of them; include/hived.h "Id lifetime")."""

    def __init__(self):
        self.ids: Dict[str, int] = {}
        self.names: List[str] = []
        self.free: List[int] = []

    def intern(self, name: str) -> int:
        i = self.ids.get(name)
        if i is None:
            if self.free:
                i = self.free.pop()
                self.names[i] = name
            else:
                i = len(self.names)
                self.names.append(name)
            self.ids[name] = i
        return i

    def release(self, name: str) -> None:
        i = self.ids.pop(name, None)
        if i is not None:
            self.names[i] = ""
            self.free.append(i)


class HivedAlgorithm:
    """internal.SchedulerAlgorithm over the C ABI (see module docstring).

    ``lib``: a ctypes library implementing include/hived.h; default = the in-tree CUDA library.
    """

    DEFAULT_OPTIONS = dict(max_groups=1 << 17, max_pods=1 << 20, max_group_leaves=512, max_group_pods=64, device=0)

    def __init__(self, config: Dict[str, Any], lib: Optional[C.CDLL] = None, **options: int):
        self._lib = lib if lib is not None else _cabi.load_cuda_library()
        opts = dict(self.DEFAULT_OPTIONS)
        opts.update(options)
        self._opt = _cabi.Options(**opts)
        self._ctx = C.c_void_p()
        spec = to_spec_text(config).encode()
        rc = self._lib.hived_create(spec, C.byref(self._opt), C.byref(self._ctx))
        if rc != 0:
            msg = (self._lib.hived_create_error() or b"").decode()
            self._ctx = None
            raise PlatformError("NewHivedAlgorithm failed (%d): %s" % (rc, msg))
        lib_ = self._lib

        def table(num, name):
            return [name(self._ctx, i).decode() for i in range(num(self._ctx))]

        self.node_names = table(lib_.hived_num_nodes, lib_.hived_node_name)
        self.chain_names = table(lib_.hived_num_chains, lib_.hived_chain_name)
        self.vc_names = table(lib_.hived_num_vcs, lib_.hived_vc_name)
        self.leaf_type_names = table(lib_.hived_num_leaf_types, lib_.hived_leaf_type_name)
        self.pinned_names = table(lib_.hived_num_pinned, lib_.hived_pinned_name)
        self.cell_type_names = table(lib_.hived_num_cell_types, lib_.hived_cell_type_name)
        self._node_ids = {n: i for i, n in enumerate(self.node_names)}
        self._chain_ids = {n: i for i, n in enumerate(self.chain_names)}
        self._vc_ids = {n: i for i, n in enumerate(self.vc_names)}
        self._leaf_type_ids = {n: i for i, n in enumerate(self.leaf_type_names)}
        self._pinned_ids = {n: i for i, n in enumerate(self.pinned_names)}
        self._cell_type_ids = {n: i for i, n in enumerate(self.cell_type_names)}
        self._groups = _Interner()
        self._pods = _Interner()
        self._pod_objs: Dict[int, Pod] = {}
        self._pool_cap = 3 * int(self._opt.max_group_leaves) + 2 * 4096 + 64
        self._pool = (C.c_int32 * self._pool_cap)()
        self._rand = random.Random(0)
        self._bitmap_words = (len(self.node_names) + 31) // 32
        # request ingest (include/hived_ingest.h): the product library interns the node names itself; the CPU checker
        # (oracle, tests only) does not export the helpers and gets the plain-Python statement below
        self._ingest = None
        if hasattr(lib_, "hived_ingest_create"):
            from .ingest import Ingest
            self._ingest = Ingest(lib_, self._ctx)

    def close(self):
        if getattr(self, "_ingest", None):
            self._ingest.close()
            self._ingest = None
        if getattr(self, "_ctx", None):
            self._lib.hived_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def clone(self, device: Optional[int] = None, concurrent: bool = False) -> "HivedAlgorithm":
        """A second scheduler that answers every later call exactly as this one would (include/hived_clone.h), for
        what-if runs: the library's state is copied into a new context (``device``: its CUDA ordinal, default this
        one's; ``concurrent``: HIVED_OPT_CONCURRENT), and the state this shim keeps above the ABI — the name <-> id
        tables with their recycled ids, the pod objects it keeps for victims and missing placements, the random
        state that picks a preemption's node — is copied too.  The two share nothing afterwards."""
        flags = (int(self._opt.flags) & ~_cabi.OPT_CONCURRENT) | (_cabi.OPT_CONCURRENT if concurrent else 0)
        ctx = C.c_void_p()
        rc = _cabi.bind_clone(self._lib).hived_clone(self._ctx, -1 if device is None else device, flags, C.byref(ctx))
        if rc != 0:
            raise PlatformError("hived_clone failed (%d): %s" % (rc, (self._lib.hived_create_error() or b"").decode()))
        h = copy.copy(self)  # the cluster's name tables, shared read-only
        h._ctx = ctx
        h._opt = _cabi.Options.from_buffer_copy(self._opt)
        h._opt.flags = flags
        if device is not None:
            h._opt.device = device
        h._groups, h._pods = copy.deepcopy(self._groups), copy.deepcopy(self._pods)
        h._pod_objs = dict(self._pod_objs)
        h._pool = (C.c_int32 * self._pool_cap)()
        h._rand = random.Random()
        h._rand.setstate(self._rand.getstate())
        h._ingest = None
        if self._ingest is not None:
            from .ingest import Ingest
            h._ingest = Ingest(self._lib, ctx)
        return h

    # ---------------------------------------------------------------- helpers
    @property
    def backend(self) -> str:
        return self._lib.hived_backend().decode()

    def _raise(self, rc: int, s: Dict[str, Any] = None, pod: "Pod" = None):
        """Library return code -> the reference's panic.  User errors (1..99) carry the reference's own message text
        (the names live above the ABI: the library only knows ids), the one its HTTP 400 body would show."""
        msg = (self._lib.hived_last_error(self._ctx) or b"").decode()
        if 1 <= rc < 100:
            raise new_bad_request_error(self._user_error_message(rc, s, pod) or msg)
        raise PlatformError("panic (%d): %s" % (rc, msg))

    def _user_error_message(self, rc: int, s: Dict[str, Any], pod: "Pod"):
        if s is None:
            return None
        key = "[%s]: " % pod.key() if pod is not None else ""
        vc, pinned, leaf_type = s["virtualCluster"], s["pinnedCellId"], s["leafCellType"]
        if rc == 1:    # validateSchedulingRequest, hived_algorithm.go:858-859
            return key + "VC %s does not exists!" % vc
        if rc == 2:    # :861-862
            return key + "VC %s does not have pinned cell %s" % (vc, pinned)
        if rc == 3:    # :863-864
            return key + "opportunistic pod not supported to use pinned cell %s" % pinned
        if rc == 4:    # scheduleNewAffinityGroup, :785-787
            return key + "Pod requesting leaf cell type %s which the whole cluster does not have" % leaf_type
        if rc == 5:    # scheduleAffinityGroupForLeafCellType, :824-826 (the type the search was trying: the spec's own)
            return key + "Pod requesting leaf cell type %s which VC %s does not have" % (leaf_type, vc)
        if rc == 6:    # schedulePodFromExistingGroup, :684-686: g.totalPodNums of the group as first created
            name = s["affinityGroup"]["name"]
            total = 0
            gid = self._groups.ids.get(name)
            if gid is not None:
                gp = _cabi.GroupPlacement()
                self._lib.hived_get_group_placement(self._ctx, gid, C.byref(gp), None, None, 0, None, 0, None, 0)
                total = sum(gp.member_pod_num[i] for i in range(gp.n_members) if gp.member_leaf_num[i] == s["leafCellNumber"])
            return ("Requesting more pods than the configured number for %d leaf cells (%d pods) in affinity group %s"
                    % (s["leafCellNumber"], total, name))
        return None

    def _spec_struct(self, s: Dict[str, Any], pod: Pod) -> _cabi.PodSpec:
        sp = _cabi.PodSpec()
        sp.pod = self._pods.intern(pod.uid)
        sp.group = self._groups.intern(s["affinityGroup"]["name"])
        sp.vc = self._vc_ids.get(s["virtualCluster"], -1)
        sp.priority = s["priority"]
        sp.pinned = -1 if s["pinnedCellId"] == "" else self._pinned_ids.get(s["pinnedCellId"], -2)
        sp.leaf_type = -1 if s["leafCellType"] == "" else self._leaf_type_ids.get(s["leafCellType"], -2)
        sp.leaf_num = s["leafCellNumber"]
        sp.flags = (_cabi.SPEC_LAZY_PREEMPTION if s["lazyPreemptionEnable"] else 0) | \
                   (_cabi.SPEC_IGNORE_SUGGESTED if s["ignoreK8sSuggestedNodes"] else 0)
        members = s["affinityGroup"]["members"]
        if len(members) > _cabi.HIVED_MAX_MEMBERS:
            raise new_bad_request_error("affinity group has more than %d members" % _cabi.HIVED_MAX_MEMBERS)
        sp.n_members = len(members)
        for i, m in enumerate(members):
            sp.member_leaf_num[i] = m["leafCellNumber"]
            sp.member_pod_num[i] = m["podNumber"]
        return sp

    def _suggested_bitmap(self, suggested_nodes: List[str]):
        """suggestedNodes []string -> node bitmap (the reference builds a string set, hived_algorithm.go:190-193)."""
        if self._ingest is not None:
            # one buffer for the C helper (a ctypes array of 8192 char* costs more than the whole decode)
            joined = '","'.join(suggested_nodes)
            if '\\' not in joined and joined.count('"') == 2 * max(0, len(suggested_nodes) - 1):
                return self._ingest.node_names_json(('["' + joined + '"]').encode() if suggested_nodes else b"[]")[0]
        words = (C.c_uint32 * max(1, self._bitmap_words))()
        ids = self._node_ids
        for n in suggested_nodes:
            i = ids.get(n)
            if i is not None:
                words[i >> 5] |= (1 << (i & 31))
        return words

    def _wait_reason(self, res: _cabi.Result, s: Dict[str, Any]) -> str:
        code = res.wait_code
        base = code & 15
        addr = ""
        if res.wait_cell >= 0:
            addr = (self._lib.hived_physical_cell_address(self._ctx, res.wait_cell) or b"").decode()
        if base == _cabi.WAIT_MAPPING:
            kind = "bad" if s["ignoreK8sSuggestedNodes"] else "bad or non-suggested"
            return "Mapping the virtual placement would need to use at least one %s node" % kind
        reason = {0: "", _cabi.WAIT_INSUFFICIENT: "insufficient capacity",
                  _cabi.WAIT_BAD_NODE: "have to use at least one bad node %s" % addr,
                  _cabi.WAIT_NON_SUGGESTED_NODE: "have to use at least one non-suggested node %s" % addr,
                  _cabi.WAIT_NO_SCHEDULER: ""}[base]
        if code & _cabi.WAIT_SCOPE_VC:
            reason = "%s when scheduling in VC %s" % (reason, s["virtualCluster"])
        elif code & _cabi.WAIT_SCOPE_PHYSICAL:
            reason = "%s when scheduling in physical cluster" % reason
        return reason

    def _retrieve_missing_pod_placement(self, gid: int, leaf_cell_num: int, pod_index: int):
        """retrieveMissingPodPlacement (pkg/algorithm/utils.go:250-265): the placement of a pod whose cells left the
        spec, from the bind-info annotation of the group's allocated pods (first non-nil pod, members ascending)."""
        gp = _cabi.GroupPlacement()
        pcap = int(self._opt.max_group_pods)
        pods = (C.c_int32 * pcap)()
        self._lib.hived_get_group_placement(self._ctx, gid, C.byref(gp), None, None, 0, pods, pcap, None, 0)
        for pid in pods[:min(gp.n_pods, pcap)]:
            pod = self._pod_objs.get(pid) if pid >= 0 else None
            if pod is None or ANNOTATION_POD_BIND_INFO not in pod.annotations:
                continue
            info = extract_pod_bind_info(pod)
            for mbi in info["affinityGroupBindInfo"]:
                if leaf_cell_num == len(mbi["podPlacements"][0]["physicalLeafCellIndices"]):
                    return mbi["podPlacements"][pod_index], info["cellChain"]
        raise PlatformError("No allocated pod found in an allocated group %s when retrieving placement for pod %d with "
                            "leaf cell number %d" % (self._groups.names[gid], pod_index, leaf_cell_num))

    def _bind_info_from_result(self, res: _cabi.Result, pool, gid: int = -1) -> Dict[str, Any]:
        """generatePodScheduleResult / generateAffinityGroupBindInfo output (pkg/algorithm/utils.go:38-171).  Leaf cells
        the library reports as nil (hived_result_t.incomplete: they left the cluster spec) make the pod's placement
        come from the other pods' annotations, exactly in the reference's order: the retrieved PodPlacementInfo
        replaces the pod's whole entry at every nil cell, later cells that still exist overwrite their own slot."""
        k = res.leaf_off
        agbi = []
        chain = ""
        cur_m = None
        for m in range(res.n_members):
            ln, pn = res.member_leaf_num[m], res.member_pod_num[m]
            pps = []
            for pi in range(pn):
                pp = {"physicalNode": "", "physicalLeafCellIndices": [0] * ln, "preassignedCellTypes": [""] * ln}
                for j in range(ln):
                    nid, li, t = pool[k], pool[k + 1], pool[k + 2]
                    k += 3
                    if nid == _cabi.NIL_CELL and li == _cabi.NIL_CELL and t == _cabi.NIL_CELL:
                        got, chain = self._retrieve_missing_pod_placement(gid, ln, pi)
                        pp = {"physicalNode": got["physicalNode"],
                              "physicalLeafCellIndices": list(got["physicalLeafCellIndices"]),
                              "preassignedCellTypes": list(got["preassignedCellTypes"])}
                        continue
                    if pp["physicalNode"] == "":
                        pp["physicalNode"] = self.node_names[nid] if nid >= 0 else ""
                    pp["physicalLeafCellIndices"][j] = li
                    pp["preassignedCellTypes"][j] = "" if t < 0 else self.cell_type_names[t]
                pps.append(pp)
            if cur_m is None and ln == res.this_n:
                cur_m = m
            agbi.append({"podPlacements": pps})
        mine = agbi[cur_m]["podPlacements"][res.pod_index]
        if res.chain >= 0:  # utils.go:163-165: the chain of the pod's first cell when that cell exists
            chain = self.chain_names[res.chain]
        return {"node": mine["physicalNode"], "leafCellIsolation": list(mine["physicalLeafCellIndices"]),
                "cellChain": chain, "affinityGroupBindInfo": agbi}

    def _bind_info_struct(self, info: Dict[str, Any]):
        bi = _cabi.BindInfo()
        bi.node = self._node_ids.get(info["node"], -1)
        bi.first_leaf = info["leafCellIsolation"][0]
        bi.chain = self._chain_ids.get(info.get("cellChain", ""), -1)
        agbi = info.get("affinityGroupBindInfo") or []
        if len(agbi) > _cabi.HIVED_MAX_MEMBERS:
            raise PlatformError("bind info has too many members")
        bi.n_members = len(agbi)
        flat: List[int] = []
        has_pre = 1
        for m, gms in enumerate(agbi):
            pps = gms["podPlacements"]
            bi.member_leaf_num[m] = len(pps[0]["physicalLeafCellIndices"])
            bi.member_pod_num[m] = len(pps)
            for pl in pps:
                types = pl.get("preassignedCellTypes")
                if types is None:
                    has_pre = 0
                nid = self._node_ids.get(pl["physicalNode"], -1)
                for j, li in enumerate(pl["physicalLeafCellIndices"]):
                    t = -1
                    if types is not None:
                        t = -1 if types[j] in ("", None) else self._cell_type_ids.get(types[j], -2)
                    flat += [nid, li, t]
        bi.has_preassigned = has_pre
        bi.n_leaves = len(flat) // 3
        arr = (C.c_int32 * max(1, len(flat)))(*flat)
        return bi, arr

    # ---------------------------------------------------------------- internal.SchedulerAlgorithm
    def Schedule(self, pod: Pod, suggested_nodes: List[str], phase: str) -> PodScheduleResult:
        """hived_algorithm.go:180-224."""
        s = extract_pod_scheduling_spec(pod)
        sp = self._spec_struct(s, pod)
        self._pod_objs[sp.pod] = pod
        bitmap = self._suggested_bitmap(suggested_nodes)
        res = _cabi.Result()
        rc = self._lib.hived_schedule(self._ctx, C.byref(sp), bitmap,
                                      _cabi.PHASE_PREEMPTING if phase == PREEMPTING_PHASE else _cabi.PHASE_FILTERING,
                                      C.byref(res), self._pool, self._pool_cap)
        if rc != 0:
            self._raise(rc, s, pod)
        out = PodScheduleResult()
        if res.kind == _cabi.KIND_WAIT:
            out.pod_wait_info = {"reason": self._wait_reason(res, s)}
        elif res.kind == _cabi.KIND_PREEMPT:
            # generatePodPreemptInfo (utils.go:81-105): victims of ONE random node
            by_node: Dict[int, List[Pod]] = {}
            for k in range(res.n_victims):
                pid, nid = self._pool[res.victim_off + 2 * k], self._pool[res.victim_off + 2 * k + 1]
                by_node.setdefault(nid, []).append(self._pod_objs[pid])
            node = self._rand.choice(sorted(by_node))
            out.pod_preempt_info = {"victim_pods": by_node[node],
                                    "all_victims": [p for n in sorted(by_node) for p in by_node[n]]}
        else:
            out.pod_bind_info = self._bind_info_from_result(res, self._pool, sp.group)
        return out

    def AddUnallocatedPod(self, pod: Pod) -> None:  # hived_algorithm.go:226-227
        return None

    def DeleteUnallocatedPod(self, pod: Pod) -> None:  # hived_algorithm.go:229-245
        s = extract_pod_scheduling_spec(pod)
        name = s["affinityGroup"]["name"]
        gid = self._groups.ids.get(name)
        if gid is None:
            return  # never seen: nothing is preempting under that name
        rc = self._lib.hived_delete_unallocated_pod(self._ctx, gid, self._pods.intern(pod.uid))
        if rc != 0:
            self._raise(rc)
        self._release_pod(pod)
        self._release_group_if_gone(name, gid)

    def _release_pod(self, pod: Pod) -> None:
        pid = self._pods.ids.get(pod.uid)
        if pid is not None:
            self._pod_objs.pop(pid, None)
            self._pods.release(pod.uid)

    def _release_group_if_gone(self, name: str, gid: int) -> None:
        """The id of a group that no longer exists goes back to the interner (include/hived.h "Id lifetime")."""
        gi = _cabi.GroupInfo()
        self._lib.hived_get_group(self._ctx, gid, C.byref(gi))
        if gi.state == _cabi.GROUP_NONE and not gi.referenced:
            self._groups.release(name)

    def AddAllocatedPod(self, pod: Pod) -> None:  # hived_algorithm.go:247-270
        s = extract_pod_scheduling_spec(pod)
        info = extract_pod_bind_info(pod)
        sp = self._spec_struct(s, pod)
        self._pod_objs[sp.pod] = pod
        bi, leaves = self._bind_info_struct(info)
        pod_index = get_allocated_pod_index(info, s["leafCellNumber"])
        rc = self._lib.hived_add_allocated_pod(self._ctx, C.byref(sp), C.byref(bi), leaves, pod_index)
        if rc != 0:
            self._raise(rc)

    def DeleteAllocatedPod(self, pod: Pod) -> None:  # hived_algorithm.go:272-296
        s = extract_pod_scheduling_spec(pod)
        info = extract_pod_bind_info(pod)
        pod_index = get_allocated_pod_index(info, s["leafCellNumber"])
        name = s["affinityGroup"]["name"]
        gid = self._groups.ids.get(name)
        if gid is None:
            return  # "Group %v not found when deleting pod" in the reference
        removed = C.c_int32(-1)
        rc = self._lib.hived_delete_allocated_pod_ex(self._ctx, gid, s["leafCellNumber"], pod_index, C.byref(removed))
        if rc != 0:
            self._raise(rc)
        # The reference clears the slot whoever sits there (:287).  Only when that was THIS pod has it left the
        # library's tables: otherwise (its group object was replaced under the same name and lives on through
        # cell.usingGroup, or the slot held another pod) the pod can still come back as a preemption victim, so its
        # object and id are kept (include/hived.h "Id lifetime").
        if removed.value == self._pods.ids.get(pod.uid, -2):
            self._release_pod(pod)
        self._release_group_if_gone(name, gid)

    # AddNode / UpdateNode / DeleteNode (hived_algorithm.go:147-178); node = {"name":..., "healthy": bool}
    def AddNode(self, node: Dict[str, Any]) -> None:
        if node.get("healthy", True):
            self.setHealthyNode(node["name"])
        else:
            self.setBadNode(node["name"])

    def UpdateNode(self, old_node: Dict[str, Any], new_node: Dict[str, Any]) -> None:
        if bool(old_node.get("healthy", True)) != bool(new_node.get("healthy", True)):
            self.AddNode(new_node)

    def DeleteNode(self, node: Dict[str, Any]) -> None:
        self.setBadNode(node["name"])

    def setBadNode(self, name: str) -> None:  # hived_algorithm.go:466-481
        rc = self._lib.hived_set_node_health(self._ctx, self._node_ids.get(name, -1), 0)
        if rc != 0:
            self._raise(rc)

    def setHealthyNode(self, name: str) -> None:  # hived_algorithm.go:483-498
        rc = self._lib.hived_set_node_health(self._ctx, self._node_ids.get(name, -1), 1)
        if rc != 0:
            self._raise(rc)

    # ---------------------------------------------------------------- inspect (raw material)
    def group_info(self, name: str) -> Optional[Dict[str, Any]]:
        """h.affinityGroups[name] essentials; None when the group does not exist."""
        gi = _cabi.GroupInfo()
        gid = self._groups.ids.get(name)
        if gid is None:
            return None
        self._lib.hived_get_group(self._ctx, gid, C.byref(gi))
        if gi.state == _cabi.GROUP_NONE:
            return None
        return {"state": {1: "Allocated", 2: "Preempting", 3: "BeingPreempted"}[gi.state],
                "vc": self.vc_names[gi.vc] if gi.vc >= 0 else "", "priority": gi.priority,
                "has_virtual_placement": bool(gi.has_virtual), "preempting_pods": gi.n_preempting_pods}

    # ---------------------------------------------------------------- inspect (api objects, as JSON-shaped dicts)
    _GROUP_STATE = {1: "Allocated", 2: "Preempting", 3: "BeingPreempted"}
    _CELL_STATE = {0: "Free", 1: "Used", 2: "Reserving", 3: "Reserved"}

    def _affinity_group(self, gid: int, name: str) -> Optional[Dict[str, Any]]:
        """AlgoAffinityGroup.ToAffinityGroup (types.go:187-214); None when the group does not exist.
        Placement maps are filled in (member ascending, pod, leaf) order (the reference ranges over a Go map)."""
        gp = _cabi.GroupPlacement()
        lcap, pcap = int(self._opt.max_group_leaves), int(self._opt.max_group_pods)
        phys, virt = (C.c_int32 * lcap)(), (C.c_int32 * lcap)()
        pods, pre = (C.c_int32 * pcap)(), (C.c_int32 * pcap)()
        rc = self._lib.hived_get_group_placement(self._ctx, gid, C.byref(gp), phys, virt, lcap, pods, pcap, pre, pcap)
        if rc != 0:
            self._raise(rc)
        if gp.state == _cabi.GROUP_NONE:
            return None
        gi = _cabi.GroupInfo()
        self._lib.hived_get_group(self._ctx, gid, C.byref(gi))
        status: Dict[str, Any] = {"vc": self.vc_names[gi.vc] if gi.vc >= 0 else "", "priority": gi.priority,
                                  "state": self._GROUP_STATE[gp.state]}
        pp: Dict[str, List[int]] = {}
        vp: Dict[str, List[str]] = {}
        info = _cabi.CellInfo()
        for k in range(min(gp.n_leaves, lcap)):
            if phys[k] >= 0:  # nodeToLeafCellIndices, types.go:223-237
                self._lib.hived_physical_cell_info(self._ctx, phys[k], C.byref(info))
                pp.setdefault(self.node_names[info.node], []).append(info.leaf_index)
            if gp.has_virtual and virt[k] >= 0:  # preassignedCellToLeafCells, types.go:244-259
                self._lib.hived_virtual_cell_info(self._ctx, virt[k], C.byref(info))
                pre_addr = (self._lib.hived_virtual_cell_address(self._ctx, info.preassigned) or b"").decode()
                vp.setdefault(pre_addr, []).append((self._lib.hived_virtual_cell_address(self._ctx, virt[k]) or b"").decode())
        if pp:
            status["physicalPlacement"] = pp
        if gp.has_virtual and vp:
            status["virtualPlacement"] = vp
        allocated = [self._pod_objs[p].uid if p in self._pod_objs else self._pods.names[p]
                     for p in pods[:min(gp.n_pods, pcap)] if p >= 0]
        if allocated:
            status["allocatedPods"] = allocated
        preempting = [self._pod_objs[p].uid if p in self._pod_objs else self._pods.names[p]
                      for p in pre[:min(gp.n_preempting, pcap)]]
        if preempting:
            status["preemptingPods"] = preempting
        if gp.lazy_preempted:
            # the library records THAT the group was lazy-preempted; preemptor name and time live in the shim
            status["lazyPreemptionStatus"] = {"preemptor": "", "preemptionTime": None}
        return {"metadata": {"name": name}, "status": status}

    def GetAffinityGroup(self, name: str) -> Dict[str, Any]:  # hived_algorithm.go:309-321
        gid = self._groups.ids.get(name)
        g = self._affinity_group(gid, name) if gid is not None else None
        if g is None:
            raise new_bad_request_error(
                "Affinity group %s does not exist since it is not allocated or preempting" % name)
        return g

    def GetAllAffinityGroups(self) -> Dict[str, Any]:  # hived_algorithm.go:298-307
        cap = self._lib.hived_list_groups(self._ctx, None, 0)
        ids = (C.c_int32 * max(1, cap))()
        n = self._lib.hived_list_groups(self._ctx, ids, cap)
        items = []
        for gid in ids[:min(n, cap)]:
            g = self._affinity_group(gid, self._groups.names[gid] if gid < len(self._groups.names) else "g%d" % gid)
            if g is not None:
                items.append(g)
        return {"items": items}

    def _cell_status(self, snap, i: int, physical: bool) -> Dict[str, Any]:
        """api.CellStatus of cell i (cell.go:144-177, 326-363 + the setters that keep it current)."""
        info = _cabi.CellInfo()
        if physical:
            self._lib.hived_physical_cell_info(self._ctx, i, C.byref(info))
            addr = self._lib.hived_physical_cell_address(self._ctx, i)
        else:
            self._lib.hived_virtual_cell_info(self._ctx, i, C.byref(info))
            addr = self._lib.hived_virtual_cell_address(self._ctx, i)
        st = snap[i]
        out: Dict[str, Any] = {}
        if info.leaf_type >= 0:
            out["leafCellType"] = self.leaf_type_names[info.leaf_type]
        out["cellType"] = self.cell_type_names[info.cell_type] if info.cell_type >= 0 else ""
        if info.is_node_level:
            out["isNodeLevel"] = True
        out["cellAddress"] = (addr or b"").decode()
        out["cellState"] = self._CELL_STATE[st.state]
        out["cellHealthiness"] = "Healthy" if st.healthy else "Bad"
        out["cellPriority"] = st.priority
        if not physical:
            out["_vc"] = self.vc_names[info.vc]
        return out

    def _status_forest(self):
        """Both api status forests from one snapshot of each side.  The embedded peer copies (VirtualCell inside a
        physical status and PhysicalCell inside a virtual one, cell.go:266-283, 401-419) are the peer's current
        status without children — the reference refreshes its copies on every priority/state/health change."""
        ps, vs = self.physical_snapshot(), self.virtual_snapshot()
        np_, nv = len(ps), len(vs)
        P = [self._cell_status(ps, i, True) for i in range(np_)]
        V = [self._cell_status(vs, i, False) for i in range(nv)]
        vc_of = [v.pop("_vc") for v in V]
        flat_p = [dict(x) for x in P]
        flat_v = [dict(x) for x in V]
        for i in range(np_):
            peer = ps[i].peer
            if peer >= 0:
                P[i]["vc"] = vc_of[peer]
                P[i]["virtualCell"] = dict(flat_v[peer])
        for i in range(nv):
            peer = vs[i].peer
            if peer >= 0:
                V[i]["physicalCell"] = dict(flat_p[peer], vc=vc_of[i])
        for side, snap in ((P, ps), (V, vs)):
            for i in range(len(side)):  # ids are assigned parents-after-children per level; children in id order
                par = snap[i].parent
                if par >= 0:
                    side[par].setdefault("cellChildren", []).append(side[i])
        phys_top = [P[i] for i in range(np_) if ps[i].parent < 0]
        virt_top: Dict[str, List[Dict[str, Any]]] = {vc: [] for vc in self.vc_names}
        for i in range(nv):
            if vs[i].parent < 0:
                virt_top[vc_of[i]].append(V[i])
        return phys_top, virt_top

    def GetClusterStatus(self) -> Dict[str, Any]:  # hived_algorithm.go:323-336
        p, v = self._status_forest()
        return {"physicalCluster": p, "virtualClusters": v}

    def GetPhysicalClusterStatus(self) -> List[Dict[str, Any]]:  # hived_algorithm.go:338-343
        return self._status_forest()[0]

    def GetAllVirtualClustersStatus(self) -> Dict[str, List[Dict[str, Any]]]:  # hived_algorithm.go:345-354
        return self._status_forest()[1]

    def GetVirtualClusterStatus(self, vcn: str) -> List[Dict[str, Any]]:  # hived_algorithm.go:356-363
        if vcn not in self._vc_ids:
            raise new_bad_request_error("VC %s not found" % vcn)
        return self._status_forest()[1][vcn]

    def physical_snapshot(self) -> List[_cabi.CellStatus]:
        n = self._lib.hived_num_physical_cells(self._ctx)
        arr = (_cabi.CellStatus * n)()
        rc = self._lib.hived_snapshot_physical(self._ctx, arr, n)
        if rc != 0:
            self._raise(rc)
        return arr

    def virtual_snapshot(self) -> List[_cabi.CellStatus]:
        n = self._lib.hived_num_virtual_cells(self._ctx)
        arr = (_cabi.CellStatus * n)()
        rc = self._lib.hived_snapshot_virtual(self._ctx, arr, n)
        if rc != 0:
            self._raise(rc)
        return arr

    def vc_preassigned_cells(self, vc: str, chain: str, level: int) -> List[int]:
        cap = 4096
        cells = (C.c_int32 * cap)()
        n = C.c_int32()
        self._lib.hived_vc_preassigned_cells(self._ctx, self._vc_ids[vc], self._chain_ids[chain], level, cells, cap,
                                             C.byref(n))
        return list(cells[:n.value])

    def physical_cell_address(self, cell: int) -> str:
        return (self._lib.hived_physical_cell_address(self._ctx, cell) or b"").decode()

    def physical_leaf_status(self, node: str, leaf_index: int) -> Optional[_cabi.CellStatus]:
        """Status of the physical leaf cell <node>/<leaf index> (first chain that has it)."""
        snap = self.physical_snapshot()
        n = len(snap)
        for i in range(n):
            if snap[i].level == 1:
                addr = self.physical_cell_address(i)
                parts = addr.split("/")
                if parts[-1] == str(leaf_index) and node in parts:
                    return snap[i]
        return None

    def stats(self) -> Dict[str, int]:
        st = _cabi.Stats()
        self._lib.hived_get_stats(self._ctx, C.byref(st))
        return {f: getattr(st, f) for f, _ in _cabi.Stats._fields_}

    def result_hash(self) -> int:
        return int(self._lib.hived_result_hash(self._ctx))

    # raw handles for the batch path (hivedscheduler_b200.trace / bench.py)
    @property
    def ctx(self):
        return self._ctx

    @property
    def lib(self):
        return self._lib
