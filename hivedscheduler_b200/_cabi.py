"""ctypes binding of include/hived.h — the same binding serves libhived_cuda.so (the product) and,
in tests/bench only, oracle/libhived_oracle.so (the CPU checker)."""
from __future__ import annotations

import ctypes as C
import os

HIVED_MAX_MEMBERS = 8

KIND_WAIT, KIND_BIND, KIND_PREEMPT = 0, 1, 2
PHASE_FILTERING, PHASE_PREEMPTING = 0, 1
EV_SCHEDULE, EV_DELETE_ALLOCATED, EV_DELETE_UNALLOCATED, EV_NODE_HEALTH = 0, 1, 2, 3
SPEC_LAZY_PREEMPTION, SPEC_IGNORE_SUGGESTED = 1, 2
CELL_FREE, CELL_USED, CELL_RESERVING, CELL_RESERVED = 0, 1, 2, 3
GROUP_NONE, GROUP_ALLOCATED, GROUP_PREEMPTING, GROUP_BEING_PREEMPTED = 0, 1, 2, 3
WAIT_INSUFFICIENT, WAIT_BAD_NODE, WAIT_NON_SUGGESTED_NODE, WAIT_MAPPING, WAIT_NO_SCHEDULER = 1, 2, 3, 4, 5
WAIT_SCOPE_VC, WAIT_SCOPE_PHYSICAL = 16, 32
ERR_PLATFORM = 100

_M = C.c_int32 * HIVED_MAX_MEMBERS


NIL_CELL = -2  # HIVED_NIL_CELL


class Options(C.Structure):
    _fields_ = [("max_groups", C.c_int32), ("max_pods", C.c_int32), ("max_group_leaves", C.c_int32),
                ("max_group_pods", C.c_int32), ("device", C.c_int32), ("flags", C.c_int32), ("reserved", C.c_int32 * 2)]


class PodSpec(C.Structure):
    _fields_ = [("pod", C.c_int32), ("group", C.c_int32), ("vc", C.c_int32), ("priority", C.c_int32),
                ("pinned", C.c_int32), ("leaf_type", C.c_int32), ("leaf_num", C.c_int32), ("flags", C.c_int32),
                ("n_members", C.c_int32), ("member_leaf_num", _M), ("member_pod_num", _M)]


class Result(C.Structure):
    _fields_ = [("kind", C.c_int32), ("error", C.c_int32), ("wait_code", C.c_int32), ("wait_cell", C.c_int32),
                ("chain", C.c_int32), ("pod_index", C.c_int32), ("node", C.c_int32), ("this_off", C.c_int32),
                ("this_n", C.c_int32), ("n_members", C.c_int32), ("member_leaf_num", _M), ("member_pod_num", _M),
                ("leaf_off", C.c_int32), ("n_leaves", C.c_int32), ("victim_off", C.c_int32),
                ("n_victims", C.c_int32), ("has_virtual", C.c_int32), ("incomplete", C.c_int32)]


class BindInfo(C.Structure):
    _fields_ = [("node", C.c_int32), ("first_leaf", C.c_int32), ("chain", C.c_int32),
                ("has_preassigned", C.c_int32), ("n_members", C.c_int32), ("member_leaf_num", _M),
                ("member_pod_num", _M), ("n_leaves", C.c_int32), ("reserved", C.c_int32)]


class Event(C.Structure):
    _fields_ = [("type", C.c_int32), ("phase", C.c_int32), ("arg0", C.c_int32), ("arg1", C.c_int32),
                ("suggested_off", C.c_int64), ("spec", PodSpec)]


class GroupInfo(C.Structure):
    _fields_ = [("state", C.c_int32), ("vc", C.c_int32), ("priority", C.c_int32), ("has_virtual", C.c_int32),
                ("n_preempting_pods", C.c_int32), ("referenced", C.c_int32), ("reserved", C.c_int32 * 2)]


class GroupPlacement(C.Structure):
    _fields_ = [("state", C.c_int32), ("n_members", C.c_int32), ("member_leaf_num", _M), ("member_pod_num", _M),
                ("n_leaves", C.c_int32), ("n_pods", C.c_int32), ("n_preempting", C.c_int32), ("has_virtual", C.c_int32),
                ("lazy_preempted", C.c_int32), ("reserved", C.c_int32)]


class CellInfo(C.Structure):
    _fields_ = [("cell_type", C.c_int32), ("is_node_level", C.c_int32), ("leaf_type", C.c_int32), ("node", C.c_int32),
                ("leaf_index", C.c_int32), ("vc", C.c_int32), ("preassigned", C.c_int32), ("pinned", C.c_int32)]


class CellStatus(C.Structure):
    _fields_ = [("priority", C.c_int32), ("state", C.c_int32), ("healthy", C.c_int32), ("peer", C.c_int32),
                ("level", C.c_int32), ("chain", C.c_int32), ("parent", C.c_int32), ("flags", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("schedule_events", C.c_int64), ("bind_results", C.c_int64), ("wait_results", C.c_int64),
                ("preempt_results", C.c_int64), ("view_nodes_scanned", C.c_int64),
                ("leaves_committed", C.c_int64), ("free_cells_scanned", C.c_int64), ("pods_placed", C.c_int64),
                ("algorithmic_bytes", C.c_int64)]


# every symbol include/hived.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("hived_create", C.c_int, [C.c_char_p, C.POINTER(Options), C.POINTER(_P)]),
    ("hived_destroy", None, [_P]),
    ("hived_last_error", C.c_char_p, [_P]),
    ("hived_create_error", C.c_char_p, []),
    ("hived_backend", C.c_char_p, []),
    ("hived_num_nodes", C.c_int32, [_P]), ("hived_node_name", C.c_char_p, [_P, C.c_int32]),
    ("hived_num_chains", C.c_int32, [_P]), ("hived_chain_name", C.c_char_p, [_P, C.c_int32]),
    ("hived_num_vcs", C.c_int32, [_P]), ("hived_vc_name", C.c_char_p, [_P, C.c_int32]),
    ("hived_num_leaf_types", C.c_int32, [_P]), ("hived_leaf_type_name", C.c_char_p, [_P, C.c_int32]),
    ("hived_num_pinned", C.c_int32, [_P]), ("hived_pinned_name", C.c_char_p, [_P, C.c_int32]),
    ("hived_num_cell_types", C.c_int32, [_P]), ("hived_cell_type_name", C.c_char_p, [_P, C.c_int32]),
    ("hived_num_physical_cells", C.c_int32, [_P]), ("hived_num_virtual_cells", C.c_int32, [_P]),
    ("hived_physical_cell_address", C.c_char_p, [_P, C.c_int32]),
    ("hived_virtual_cell_address", C.c_char_p, [_P, C.c_int32]),
    ("hived_vc_preassigned_cells", C.c_int,
     [_P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32)]),
    ("hived_set_node_health", C.c_int, [_P, C.c_int32, C.c_int32]),
    ("hived_schedule", C.c_int,
     [_P, C.POINTER(PodSpec), C.POINTER(C.c_uint32), C.c_int32, C.POINTER(Result), C.POINTER(C.c_int32), C.c_int32]),
    ("hived_add_allocated_pod", C.c_int,
     [_P, C.POINTER(PodSpec), C.POINTER(BindInfo), C.POINTER(C.c_int32), C.c_int32]),
    ("hived_delete_allocated_pod", C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32]),
    ("hived_delete_allocated_pod_ex", C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]),
    ("hived_delete_unallocated_pod", C.c_int, [_P, C.c_int32, C.c_int32]),
    ("hived_process_events", C.c_int,
     [_P, C.POINTER(Event), C.c_int32, C.POINTER(C.c_uint32), C.c_int64, C.POINTER(Result),
      C.POINTER(C.c_int32), C.c_int64]),
    ("hived_get_group", C.c_int, [_P, C.c_int32, C.POINTER(GroupInfo)]),
    ("hived_get_group_placement", C.c_int,
     [_P, C.c_int32, C.POINTER(GroupPlacement), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
      C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), C.c_int32]),
    ("hived_list_groups", C.c_int32, [_P, C.POINTER(C.c_int32), C.c_int32]),
    ("hived_physical_cell_info", C.c_int, [_P, C.c_int32, C.POINTER(CellInfo)]),
    ("hived_virtual_cell_info", C.c_int, [_P, C.c_int32, C.POINTER(CellInfo)]),
    ("hived_snapshot_physical", C.c_int, [_P, C.POINTER(CellStatus), C.c_int32]),
    ("hived_snapshot_virtual", C.c_int, [_P, C.POINTER(CellStatus), C.c_int32]),
    ("hived_get_stats", C.c_int, [_P, C.POINTER(Stats)]),
    ("hived_result_hash", C.c_uint64, [_P]),
]

HIVED_MANY_MAX = 16


class Batch(C.Structure):
    """hived_batch_t (include/hived_multictx.h)."""
    _fields_ = [("ctx", _P), ("events", C.POINTER(Event)), ("n", C.c_int32),
                ("suggested_pool", C.POINTER(C.c_uint32)), ("suggested_words", C.c_int64),
                ("res", C.POINTER(Result)), ("pool", C.POINTER(C.c_int32)), ("pool_cap", C.c_int64),
                ("rc", C.c_int32), ("reserved", C.c_int32), ("pool_used", C.c_int64)]


def bind_many(lib: C.CDLL) -> C.CDLL:
    """Type hived_process_events_many (include/hived_multictx.h) on a library loaded with load_library."""
    lib.hived_process_events_many.restype = C.c_int
    lib.hived_process_events_many.argtypes = [C.POINTER(Batch), C.c_int32]
    return lib


_HERE = os.path.dirname(os.path.abspath(__file__))
CUDA_LIB_PATH = os.path.join(_HERE, "csrc", "libhived_cuda.so")


class MissingExtension(RuntimeError):
    pass


def load_library(path: str) -> C.CDLL:
    """dlopen a library implementing include/hived.h and type every declared symbol."""
    if not os.path.exists(path):
        raise MissingExtension(
            "%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback for the product path)" % path)
    lib = C.CDLL(path)
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the library does not export the symbol
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


def load_cuda_library() -> C.CDLL:
    # HIVED_CUDA_LIB: another BUILD of the same CUDA library (the profiling variant with SM-cycle counters, -DHIVED_PROFILE)
    return load_library(os.environ.get("HIVED_CUDA_LIB") or CUDA_LIB_PATH)
