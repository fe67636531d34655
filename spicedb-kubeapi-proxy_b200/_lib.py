"""ctypes binding of libzgpu.so (include/zgpu.h). No torch types cross this boundary."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)

NO_PERMISSION, HAS_PERMISSION, ITEM_ERROR = 1, 2, 255
SREL_NONE, SREL_WILDCARD = 0xFFFF, 0xFFFE
NO_OBJECT = 0xFFFFFFFF
OP_TOUCH, OP_CREATE, OP_DELETE = 0, 1, 2
PRECOND_MUST_MATCH, PRECOND_MUST_NOT_MATCH = 1, 2
E2BIG = -7
READ_CURSOR_BYTES = 32  # sizeof(zg_read_cursor)
MAX_LOOKUP_PAGE = 1 << 24  # ids of one lookup_resources_page: its buffers are allocated for the limit
WILDCARDS_INCLUDE, WILDCARDS_EXCLUDE = 0, 1  # zg_lookup_subjects wildcard_option

CHECK_DTYPE = np.dtype(
    [("res", "<u4"), ("subj", "<u4"), ("perm", "<u2"), ("stype", "<u2"), ("srel", "<u2"), ("flags", "<u2")]
)
TUPLE_DTYPE = np.dtype(
    [("res", "<u4"), ("subj", "<u4"), ("rel", "<u2"), ("stype", "<u2"), ("srel", "<u2"), ("flags", "<u2")]
)

EDEPTH = -9
EXPAND_UNION, EXPAND_INTERSECTION, EXPAND_EXCLUSION, EXPAND_LEAF = 1, 2, 3, 4  # zg_expand_node.op
EXPAND_REQUEST_DTYPE = np.dtype([("perm", "<u2"), ("pad", "<u2"), ("res", "<u4")])
EXPAND_NODE_DTYPE = np.dtype([("request", "<u4"), ("parent", "<u4"), ("rank", "<u4"), ("object", "<u4"), ("slot", "<u2"),
                              ("op", "<u2"), ("n_subjects", "<u4"), ("subjects", "<u8")])
EXPAND_SUBJECT_DTYPE = np.dtype([("id", "<u4"), ("type", "<u2"), ("srel", "<u2")])
_EXPAND_OP = {EXPAND_UNION: "U", EXPAND_INTERSECTION: "I", EXPAND_EXCLUSION: "X", EXPAND_LEAF: "L"}


def parse_expand_lines(lines):
    """zg_expand_permission_tree_str's lines -> nested tree: {"op": U|I|X|L, "object": "type:id", "relation": str,
    "subjects": ["type:id", "type:id#rel", "type:*", ...], "children": [...]}."""
    root, stack = None, []
    for line in lines:
        depth, op, node, *subjects = line.split(" ")
        obj, _, rel = node.rpartition("#")
        n = {"op": op, "object": obj, "relation": rel, "subjects": subjects, "children": []}
        depth = int(depth)
        del stack[depth:]
        if stack:
            stack[-1]["children"].append(n)
        else:
            root = n
        stack.append(n)
    return root


class ZgpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"zgpu error {code}: {msg}")
        self.code = code


class _Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("flags", C.c_uint32), ("subquery_capacity", C.c_uint64),
                ("work_budget", C.c_uint32), ("shard_rank", C.c_uint16), ("shard_count", C.c_uint16),
                ("n_devices", C.c_uint32), ("n_shards", C.c_uint32)]


class _RelStr(C.Structure):
    _fields_ = [(n, C.c_char_p) for n in ("res_type", "res_id", "relation", "subj_type", "subj_id", "subj_rel")]


class _UpdateStr(C.Structure):
    _fields_ = [("rel", _RelStr), ("expires_at", C.c_uint32), ("op", C.c_uint32)]


class _Precond(C.Structure):
    _fields_ = [("op", C.c_uint32), ("filter", _RelStr)]


class _FilterEx(C.Structure):
    _fields_ = [("f", _RelStr), ("res_id_prefix", C.c_char_p)]


class _PrecondEx(C.Structure):
    _fields_ = [("op", C.c_uint32), ("filter", _FilterEx)]


class _ImportGroup(C.Structure):
    _fields_ = [("res_type", C.c_char_p), ("relation", C.c_char_p), ("subj_type", C.c_char_p), ("subj_rel", C.c_char_p),
                ("res_ids", C.c_char_p), ("res_off", C.c_void_p), ("subj_ids", C.c_char_p), ("subj_off", C.c_void_p),
                ("expires_at", C.c_void_p), ("n", C.c_uint64)]


class _ListTemplate(C.Structure):
    _fields_ = [(k, C.c_char_p) for k in ("res_type", "permission", "subj_type", "subj_id", "subj_rel", "req_name",
                                          "req_namespace")] + [("id_kind", C.c_uint32), ("flags", C.c_uint32)]


ID_NAME, ID_NAMESPACED_NAME = 0, 1
TPL_CLEAR_NAMESPACE = 1


class _Stats(C.Structure):
    _fields_ = [("checks", C.c_uint64), ("launches", C.c_uint64), ("passes", C.c_uint64), ("tuples", C.c_uint64),
                ("snapshot_bytes", C.c_uint64), ("revision", C.c_uint64), ("last_alg_bytes", C.c_uint64),
                ("last_kernel_ms", C.c_double), ("coalesced_launches", C.c_uint64), ("coalesced_requests", C.c_uint64),
                ("stack_spills", C.c_uint64), ("memo_batches", C.c_uint64), ("split_batches", C.c_uint64),
                ("delta_publishes", C.c_uint64), ("full_publishes", C.c_uint64), ("last_publish_ms", C.c_double),
                ("streamed_calls", C.c_uint64), ("lookup_batches", C.c_uint64), ("lookups_batched", C.c_uint64),
                ("devices", C.c_uint64), ("shards", C.c_uint64), ("last_levels", C.c_uint64),
                ("last_subqueries", C.c_uint64), ("last_round_trips", C.c_uint64), ("flat_slots", C.c_uint64),
                ("flat_residual", C.c_uint64)]


class _Update(C.Structure):
    _fields_ = [("res", C.c_uint32), ("subj", C.c_uint32), ("rel", C.c_uint16), ("stype", C.c_uint16),
                ("srel", C.c_uint16), ("flags", C.c_uint16), ("expires_at", C.c_uint32), ("op", C.c_uint32)]


UPDATE_DTYPE = np.dtype([("res", "<u4"), ("subj", "<u4"), ("rel", "<u2"), ("stype", "<u2"), ("srel", "<u2"),
                         ("flags", "<u2"), ("expires_at", "<u4"), ("op", "<u4")])


class _ListItem(C.Structure):
    _fields_ = [("begin", C.c_uint64), ("end", C.c_uint64), ("name_off", C.c_uint64), ("ns_off", C.c_uint64),
                ("name_len", C.c_uint32), ("ns_len", C.c_uint32), ("flags", C.c_uint32), ("reserved", C.c_uint32)]


LIST_ITEM_DTYPE = np.dtype([("begin", "<u8"), ("end", "<u8"), ("name_off", "<u8"), ("ns_off", "<u8"),
                            ("name_len", "<u4"), ("ns_len", "<u4"), ("flags", "<u4"), ("reserved", "<u4")])
ITEM_IS_OBJECT, ITEM_HAS_METADATA, ITEM_HAS_OBJECT, ITEM_RAW_NAMES = 1, 2, 4, 8
LIST_ITEMS, LIST_TABLE_ROWS, LIST_PROTOBUF, LIST_PROTOBUF_OBJECT = 0, 1, 2, 3
LIST_EMPTY_AS_NULL = 1


def library_path() -> str:
    # ZGPU_LIB selects an alternative build of the same sources (tuning experiments)
    return os.environ.get("ZGPU_LIB") or os.path.join(_HERE, "libzgpu.so")


def build_library(force: bool = False) -> str:
    """nvcc-compile csrc/ into libzgpu.so for sm_90a (cross-compiles without a GPU)."""
    so = library_path()
    csrc = os.path.join(_HERE, "csrc")
    # the Makefile holds the architecture and compiler flags: a change there rebuilds too
    srcs = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cc", ".h", ".cuh")) or f == "Makefile"]
    srcs.append(os.path.join(_ROOT, "include", "zgpu.h"))
    stale = not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if os.environ.get("ZGPU_LIB"):
        stale = force = False  # explicitly chosen library: use as is
    if force or stale:
        if not os.path.exists("/usr/local/cuda/bin/nvcc"):
            if os.path.exists(so):
                return so
            raise ZgpuError(-4, "libzgpu.so is missing and nvcc is not available to build it")
        # several ranks (torchrun) or test workers may import at once: one builds, the others wait
        import fcntl

        with open(os.path.join(csrc, ".build.lock"), "w") as lock:
            fcntl.flock(lock, fcntl.LOCK_EX)
            try:
                still_stale = not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
                if force or still_stale:
                    r = subprocess.run(["make", "-C", csrc], capture_output=True, text=True)
                    if r.returncode != 0:
                        raise ZgpuError(-4, "building libzgpu.so failed:\n" + r.stdout[-2000:] + r.stderr[-4000:])
            finally:
                fcntl.flock(lock, fcntl.LOCK_UN)
    return so


_LIB = None

_SIGS = {
    "zg_engine_create": (C.c_int, [C.POINTER(_Config), C.POINTER(C.c_void_p)]),
    "zg_engine_destroy": (None, [C.c_void_p]),
    "zg_last_error": (C.c_char_p, []),
    "zg_build_info": (C.c_char_p, []),
    "zg_last_error_copy": (C.c_size_t, [C.c_char_p, C.c_size_t]),
    "zg_clear_relationships": (C.c_int, [C.c_void_p]),
    "zg_load_schema": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "zg_num_types": (C.c_int, [C.c_void_p]),
    "zg_num_slots": (C.c_int, [C.c_void_p]),
    "zg_type_id": (C.c_int, [C.c_void_p, C.c_char_p]),
    "zg_slot_id": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p]),
    "zg_slot_type": (C.c_int, [C.c_void_p, C.c_int]),
    "zg_slot_is_permission": (C.c_int, [C.c_void_p, C.c_int]),
    "zg_slot_name": (C.c_char_p, [C.c_void_p, C.c_int]),
    "zg_type_name": (C.c_char_p, [C.c_void_p, C.c_int]),
    "zg_intern_object": (C.c_uint32, [C.c_void_p, C.c_int, C.c_char_p]),
    "zg_find_object": (C.c_uint32, [C.c_void_p, C.c_int, C.c_char_p]),
    "zg_object_name": (C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_char_p, C.c_size_t]),
    "zg_load_tuples": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]),
    "zg_apply_updates": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "zg_publish": (C.c_int, [C.c_void_p]),
    "zg_num_tuples": (C.c_uint64, [C.c_void_p]),
    "zg_set_clock": (None, [C.c_void_p, C.c_int64]),
    "zg_write_relationships": (C.c_int, [C.c_void_p, C.POINTER(_UpdateStr), C.c_uint64, C.POINTER(_Precond), C.c_uint64]),
    "zg_import_relationships": (C.c_int, [C.c_void_p, C.POINTER(_ImportGroup), C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_import_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_import_last_times": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_delete_relationships": (C.c_int, [C.c_void_p, C.POINTER(_RelStr), C.POINTER(_Precond), C.c_uint64,
                                          C.POINTER(C.c_uint64)]),
    "zg_collect_expired": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(C.c_uint64)]),
    "zg_retire_unused_names": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "zg_name_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_object_capacity": (C.c_uint64, [C.c_void_p, C.c_int]),
    "zg_debug_set_resolve_hook": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "zg_read_relationships": (C.c_int, [C.c_void_p, C.POINTER(_RelStr), C.c_char_p, C.c_size_t,
                                        C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]),
    "zg_read_relationships_page": (C.c_int, [C.c_void_p, C.POINTER(_RelStr), C.c_uint64, C.c_void_p, C.c_char_p,
                                             C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "zg_delete_relationships_limited": (C.c_int, [C.c_void_p, C.POINTER(_RelStr), C.POINTER(_Precond), C.c_uint64,
                                                  C.c_uint64, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]),
    "zg_page_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_read_relationships_ex": (C.c_int, [C.c_void_p, C.POINTER(_FilterEx), C.c_char_p, C.c_size_t,
                                           C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]),
    "zg_read_relationships_page_ex": (C.c_int, [C.c_void_p, C.POINTER(_FilterEx), C.c_uint64, C.c_void_p, C.c_char_p,
                                                C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "zg_delete_relationships_limited_ex": (C.c_int, [C.c_void_p, C.POINTER(_FilterEx), C.POINTER(_PrecondEx), C.c_uint64,
                                                     C.c_uint64, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]),
    "zg_write_relationships_ex": (C.c_int, [C.c_void_p, C.POINTER(_UpdateStr), C.c_uint64, C.POINTER(_PrecondEx),
                                            C.c_uint64]),
    "zg_prefix_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_watch_read": (C.c_int, [C.c_void_p, C.c_uint64, C.c_char_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t),
                                C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "zg_check_bulk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "zg_check_bulk_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "zg_check_bulk_str": (C.c_int, [C.c_void_p, C.POINTER(_RelStr), C.c_uint64, C.c_void_p]),
    "zg_resolve_checks": (C.c_int, [C.c_void_p, C.POINTER(_RelStr), C.c_uint64, C.c_void_p]),
    "zg_resolve_checks_packed": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "zg_check_bulk_packed": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "zg_lookup_resources": (C.c_int, [C.c_void_p, C.c_uint16, C.c_uint16, C.c_uint16, C.c_uint32, C.c_uint16,
                                      C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_lookup_resources_str": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p,
                                          C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]),
    "zg_lookup_resources_page": (C.c_int, [C.c_void_p, C.c_uint16, C.c_uint16, C.c_uint16, C.c_uint32, C.c_uint16,
                                           C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p,
                                           C.c_void_p, C.POINTER(C.c_int32)]),
    "zg_lookup_resources_page_str": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p,
                                               C.c_uint64, C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t),
                                               C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "zg_lookup_page_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_lookup_subjects": (C.c_int, [C.c_void_p, C.c_uint16, C.c_uint32, C.c_uint16, C.c_uint16, C.c_uint32, C.c_void_p,
                                     C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_int32)]),
    "zg_lookup_subjects_str": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint32,
                                         C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]),
    "zg_lookup_subjects_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_expand_permission_trees": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                                             C.POINTER(C.c_uint64), C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_expand_permission_tree_str": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t,
                                                C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]),
    "zg_expand_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_expand_last_times": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_handle_lookup_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_handle_subjects_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_filter_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_closure_index_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_closure_index_info": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "zg_closure_signature_info": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "zg_closure_signature_copy": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_closure_table_info": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "zg_closure_table_copy": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "zg_closure_index_copy": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "zg_flat_record_info": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p]),
    "zg_flat_record_copy": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_resolve_checks_packed_device": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "zg_check_bulk_packed_ingress": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "zg_intern_objects_packed": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "zg_ingress_counters": (C.c_int, [C.c_void_p, C.c_void_p]),
    "zg_shard_route_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "zg_shard_pass_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(C.c_uint64)]),
    "zg_shard_fold_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int]),
    "zg_shard_unroute_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "zg_shard_lookup_begin_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64,
                                            C.c_void_p]),
    "zg_shard_lookup_expand_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p,
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "zg_shard_lookup_candidates_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_shard_lookup_route_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p]),
    "zg_shard_lookup_finish_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                             C.POINTER(C.c_uint64)]),
    "zg_shard_pass_nowild_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(C.c_uint64)]),
    "zg_shard_subjects_begin_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                              C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]),
    "zg_shard_subjects_expand_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p,
                                               C.POINTER(C.c_int)]),
    "zg_shard_subjects_admit_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]),
    "zg_shard_subjects_candidates_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_shard_subjects_verdicts_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                                 C.POINTER(C.c_uint64)]),
    "zg_shard_subjects_nowild_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p,
                                               C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_shard_subjects_route_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p]),
    "zg_shard_subjects_finish_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "zg_debug_row": (C.c_int, [C.c_void_p, C.c_uint16, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                               C.POINTER(C.c_uint64)]),
    "zg_debug_shard_row": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint16, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64,
                                     C.POINTER(C.c_uint64)]),
    "zg_host_alloc": (C.c_void_p, [C.c_size_t]),
    "zg_host_free": (None, [C.c_void_p]),
    "zg_list_scan": (C.c_int64, [C.c_char_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                 C.POINTER(C.c_uint64)]),
    "zg_list_filter": (C.c_int, [C.c_char_p, C.c_size_t, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint64,
                                 C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "zg_list_resolve": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_uint64, C.POINTER(_ListTemplate),
                                  C.c_void_p, C.c_void_p]),
    "zg_list_postfilter": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.POINTER(_ListTemplate), C.c_uint32,
                                     C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "zg_list_keep_allowed": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_uint64, C.c_uint32, C.c_char_p,
                                       C.c_char_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_void_p]),
    "zg_list_prefilter": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_uint32, C.POINTER(_ListTemplate), C.c_void_p,
                                    C.c_size_t, C.POINTER(C.c_size_t)]),
    "zg_stats_get": (C.c_int, [C.c_void_p, C.POINTER(_Stats)]),
    "zg_count_alg_bytes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "zg_phase_clocks": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
}


def exported_symbols():
    """Names include/zgpu.h declares; tests assert the .so exports each of them."""
    return sorted(_SIGS)


def lib():
    """Loads libzgpu.so. There is NO fallback: a missing library is an error."""
    global _LIB
    if _LIB is None:
        so = build_library()
        L = C.CDLL(so)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)  # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def _b(s):
    if s is None:
        return None
    return s.encode() if isinstance(s, str) else s


def _relstr(rt, rid, rel, st, sid, srel):
    return _RelStr(_b(rt), _b(rid), _b(rel), _b(st), _b(sid), _b(srel or ""))


def split_rel(rel: str):
    """'type:id#rel@stype:sid[#srel]' (pkg/rules/rules.go:1050 grammar) -> 6-tuple."""
    left, right = rel.split("@", 1)
    rt, rest = left.split(":", 1)
    rid, r = rest.rsplit("#", 1)
    st, srest = right.split(":", 1)
    sid, _, srel = srest.partition("#")
    return rt, rid, r, st, sid, srel


def list_scan(body: bytes, mode: int = LIST_ITEMS):
    """zg_list_scan: (items structured array, items_begin, items_end), or None when the body has no
    top-level "items" ("rows" with LIST_TABLE_ROWS) array. LIST_PROTOBUF: a protobuf-encoded <Kind>List
    (items = whole `items` entries, items_begin = offset of raw's length, items_end = end of raw).
    Raises ZgpuError(-1) on a malformed body."""
    L = lib()
    ib, ie = C.c_uint64(0), C.c_uint64(0)
    cap = len(body) // 128 + 16  # an item is rarely shorter; untouched pages of the buffer cost nothing
    while True:
        items = np.empty(cap, dtype=LIST_ITEM_DTYPE)
        n = L.zg_list_scan(body, len(body), mode, items.ctypes.data, cap, C.byref(ib), C.byref(ie))
        if n == -7:
            cap *= 4
            continue
        if n < 0:
            raise ZgpuError(int(n), "malformed list body")
        if ie.value == 0:
            return None
        return items[:n], ib.value, ie.value


def list_filter(body: bytes, items: np.ndarray, keep: np.ndarray, items_begin: int, items_end: int,
                flags: int = 0) -> bytes:
    """zg_list_filter: the body with only the kept items, every other byte untouched."""
    L = lib()
    items = np.ascontiguousarray(items, dtype=LIST_ITEM_DTYPE)
    keep = np.ascontiguousarray(keep, dtype=np.uint8)
    out = np.empty(len(body) + 8, dtype=np.uint8)  # the filtered body is never longer than body + 2
    need = C.c_size_t(0)
    rc = L.zg_list_filter(body, len(body), items.ctypes.data, len(items), keep.ctypes.data, items_begin, items_end,
                          flags, out.ctypes.data, out.size, C.byref(need))
    if rc != 0:
        raise ZgpuError(rc, "zg_list_filter failed")
    return out[:need.value].tobytes()


class PinnedArray:
    """numpy view over zg_host_alloc memory (freed with the object)."""

    def __init__(self, shape, dtype):
        self.dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * self.dtype.itemsize
        self._L = lib()
        self.ptr = self._L.zg_host_alloc(max(n, 1))
        if not self.ptr:
            raise ZgpuError(-8, "zg_host_alloc failed")
        buf = (C.c_uint8 * max(n, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(shape))).reshape(shape)

    def __del__(self):
        if getattr(self, "ptr", None):
            self.array = None
            self._L.zg_host_free(self.ptr)
            self.ptr = None


class Engine:
    """One zg_engine: schema + relationship store + published CSR snapshot in HBM."""

    def __init__(self, schema: str | None = None, device: int = -1, subquery_capacity: int = 0, work_budget: int = 0,
                 host_only: bool = False, forward_only: bool = False, shard_rank: int = 0, shard_count: int = 0,
                 n_devices: int = 0, n_shards: int = 0, handle_lookups: bool = False, handle_subjects: bool = False):
        """host_only=True builds schema/store/snapshot without a GPU (CPU unit tests of
        the host logic); every check/lookup on such an engine raises ZgpuError. n_shards=S > 1: this one handle
        holds the S shards of an object-hash sharded store (zg_config.n_shards); handle_lookups=True
        (ZG_FLAG_HANDLE_LOOKUPS) makes it answer LookupResources and the list pre-filter too, handle_subjects=True
        (ZG_FLAG_HANDLE_SUBJECTS) LookupSubjects."""
        self._L = lib()
        flags = ((1 if host_only else 0) | (2 if forward_only else 0) | (4 if handle_lookups else 0)
                 | (8 if handle_subjects else 0))
        cfg = _Config(device, flags, subquery_capacity, work_budget, shard_rank, shard_count, n_devices & 0xFFFFFFFF,
                      n_shards)
        h = C.c_void_p()
        rc = self._L.zg_engine_create(C.byref(cfg), C.byref(h))
        if rc:
            raise ZgpuError(rc, self._L.zg_last_error().decode())
        self._h = h
        if schema is not None:
            self.load_schema(schema)

    def close(self):
        if getattr(self, "_h", None):
            self._L.zg_engine_destroy(self._h)
            self._h = None

    __del__ = close

    def _ck(self, rc):
        if rc:
            raise ZgpuError(rc, self._L.zg_last_error().decode())

    # -- schema ---------------------------------------------------------------
    def load_schema(self, text: str):
        b = _b(text)
        self._ck(self._L.zg_load_schema(self._h, b, len(b)))

    def type_id(self, name):
        return self._L.zg_type_id(self._h, _b(name))

    def slot_id(self, type_name, rel):
        return self._L.zg_slot_id(self._h, self.type_id(type_name), _b(rel))

    def slot_table(self):
        L, h = self._L, self._h
        return [
            (s, L.zg_type_name(h, L.zg_slot_type(h, s)).decode(), L.zg_slot_name(h, s).decode(),
             bool(L.zg_slot_is_permission(h, s)))
            for s in range(L.zg_num_slots(h))
        ]

    def intern(self, type_name, object_id):
        return self._L.zg_intern_object(self._h, self.type_id(type_name), _b(object_id))

    def find(self, type_name, object_id):
        return self._L.zg_find_object(self._h, self.type_id(type_name), _b(object_id))

    def object_name(self, type_name, oid: int) -> str:
        """zg_object_name: the name of id `oid`; ZgpuError(ZG_EINVAL) when it has none."""
        buf = C.create_string_buffer(1 << 12)
        rc = self._L.zg_object_name(self._h, self.type_id(type_name), oid, buf, len(buf))
        if rc < 0:
            self._ck(rc)
        return buf.value.decode()

    # -- store ----------------------------------------------------------------
    def load_tuples(self, tuples: np.ndarray, expires: np.ndarray | None = None):
        t = np.ascontiguousarray(tuples, dtype=TUPLE_DTYPE)
        ex = None if expires is None else np.ascontiguousarray(expires, dtype=np.uint32)
        self._ck(self._L.zg_load_tuples(self._h, t.ctypes.data, None if ex is None else ex.ctypes.data, t.size))

    def add_bulk(self, type_name, rel, subj_type, res, subj, srel=None, wildcard=False):
        """Bulk TOUCH of relationships sharing (relation, subject type, subject relation)."""
        res = np.ascontiguousarray(res, dtype=np.uint32)
        t = np.zeros(res.size, dtype=TUPLE_DTYPE)
        t["res"] = res
        t["subj"] = 0 if wildcard else np.ascontiguousarray(subj, dtype=np.uint32)
        t["rel"] = self.slot_id(type_name, rel)
        t["stype"] = self.type_id(subj_type)
        t["srel"] = SREL_WILDCARD if wildcard else (SREL_NONE if srel is None else self.slot_id(subj_type, srel))
        self.load_tuples(t)

    def publish(self):
        self._ck(self._L.zg_publish(self._h))

    def apply_updates(self, updates: np.ndarray):
        """zg_apply_updates: interned CREATE / TOUCH / DELETE (UPDATE_DTYPE); visible after publish()."""
        u = np.ascontiguousarray(updates, dtype=UPDATE_DTYPE)
        self._ck(self._L.zg_apply_updates(self._h, u.ctypes.data, u.size))

    def num_tuples(self):
        return self._L.zg_num_tuples(self._h)

    def set_clock(self, unix_seconds: int):
        self._L.zg_set_clock(self._h, int(unix_seconds))

    def write_relationships(self, updates, preconditions=()):
        """updates: [(op, 'type:id#rel@stype:sid[#srel]', expires_at)];
        preconditions: [(op, {filter fields})]"""
        n = len(updates)
        arr = (_UpdateStr * max(n, 1))()
        keep = []
        for i, (op, rel, exp) in enumerate(updates):
            parts = [_b(x) for x in split_rel(rel)]
            keep.append(parts)
            arr[i] = _UpdateStr(_RelStr(*parts), int(exp), int(op))
        if self._any_prefix(f for _, f in preconditions):
            self._ck(self._L.zg_write_relationships_ex(self._h, arr, n, self._preconds_ex(preconditions), len(preconditions)))
            return
        pre = (_Precond * max(len(preconditions), 1))()
        for i, (op, f) in enumerate(preconditions):
            pre[i] = _Precond(int(op), self._filter(f))
        self._ck(self._L.zg_write_relationships(self._h, arr, n, pre, len(preconditions)))

    def import_relationships(self, groups) -> int:
        """zg_import_relationships: ImportBulkRelationships, all-or-nothing, published once. groups: iterable of
        (res_type, relation, subj_type, subj_rel, res_ids, subj_ids, expires) with res_ids / subj_ids lists of ids
        (str or bytes; "*" = the wildcard subject) and expires None or a list of unix seconds (0 = none). Returns how
        many relationships were imported."""
        groups = list(groups)
        arr = (_ImportGroup * max(len(groups), 1))()
        keep = []  # buffers must outlive the call
        for i, (rt, rel, st, srel, res_ids, subj_ids, expires) in enumerate(groups):
            rblob, roff = self.pack_ids(res_ids)
            sblob, soff = self.pack_ids(subj_ids)
            if len(res_ids) != len(subj_ids):
                raise ValueError("res_ids and subj_ids differ in length")
            ex = None if expires is None else np.ascontiguousarray(expires, dtype=np.uint32)
            if ex is not None and ex.size != len(res_ids):
                raise ValueError("expires and res_ids differ in length")
            rblob, sblob = rblob or b"\0", sblob or b"\0"
            parts = (_b(rt), _b(rel), _b(st), _b(srel or ""), rblob, sblob)
            keep.append((parts, roff, soff, ex))
            arr[i] = _ImportGroup(parts[0], parts[1], parts[2], parts[3], rblob, roff.ctypes.data, sblob, soff.ctypes.data,
                                  None if ex is None else ex.ctypes.data, len(res_ids))
        n = C.c_uint64(0)
        self._ck(self._L.zg_import_relationships(self._h, arr, len(groups), C.byref(n)))
        return n.value

    @staticmethod
    def import_groups(rels):
        """[(relationship text 'type:id#rel@stype:sid[#srel]', expires_at)] -> import_relationships groups: one group
        per class in order of first appearance, items in the order given within a group. The call order of the import
        is that of the groups, so it equals the given order when each class's relationships are contiguous."""
        groups = {}
        for rel, exp in rels:
            rt, rid, r, st, sid, srel = split_rel(rel)
            g = groups.setdefault((rt, r, st, srel), ([], [], []))
            g[0].append(rid)
            g[1].append(sid)
            g[2].append(int(exp))
        return [(rt, r, st, srel, res, subj, ex if any(ex) else None) for (rt, r, st, srel), (res, subj, ex) in groups.items()]

    def import_counters(self) -> dict:
        """zg_import_counters: successful imports on the device / on the host, relationships imported, name
        occurrences the store had, names interned new."""
        out = np.zeros(5, dtype=np.uint64)
        self._ck(self._L.zg_import_counters(self._h, out.ctypes.data))
        return dict(zip(("device", "host", "relationships", "names_found", "names_new"), (int(x) for x in out)))

    def import_last_times(self) -> dict:
        """zg_import_last_times: the last successful import's steps in milliseconds."""
        out = np.zeros(7, dtype=np.float64)
        self._ck(self._L.zg_import_last_times(self._h, out.ctypes.data))
        return dict(zip(("names", "sort", "duplicates", "host", "index", "build", "total"), (float(x) for x in out)))

    @staticmethod
    def _filter(f):
        return _RelStr(_b(f.get("res_type", "")), _b(f.get("res_id", "")), _b(f.get("rel", "")),
                       _b(f.get("subj_type", "")), _b(f.get("subj_id", "")), _b(f.get("subj_rel", "")))

    # A filter dict's "res_id_prefix" (optional_resource_id_prefix) goes through the _ex calls, and only when set: a
    # filter without one takes the calls it always took.
    @staticmethod
    def _any_prefix(filters) -> bool:
        return any(f.get("res_id_prefix") for f in filters)

    @classmethod
    def _filter_ex(cls, f):
        return _FilterEx(cls._filter(f), _b(f.get("res_id_prefix") or ""))

    @classmethod
    def _preconds_ex(cls, preconditions):
        pre = (_PrecondEx * max(len(preconditions), 1))()
        for i, (op, f) in enumerate(preconditions):
            pre[i] = _PrecondEx(int(op), cls._filter_ex(f))
        return pre

    def delete_relationships(self, flt: dict, preconditions=()):
        if self._any_prefix([flt, *(f for _, f in preconditions)]):
            return self.delete_relationships_limited(flt, preconditions)[0]
        pre = (_Precond * max(len(preconditions), 1))()
        for i, (op, f) in enumerate(preconditions):
            pre[i] = _Precond(int(op), self._filter(f))
        n = C.c_uint64(0)
        f = self._filter(flt)
        self._ck(self._L.zg_delete_relationships(self._h, C.byref(f), pre, len(preconditions), C.byref(n)))
        return n.value

    def collect_expired(self, before: int) -> int:
        """zg_collect_expired: removes every relationship whose expiration is set and <= before (unix seconds, not
        later than the engine's clock); returns how many. Answers at clocks >= before do not change."""
        n = C.c_uint64(0)
        self._ck(self._L.zg_collect_expired(self._h, int(before), C.byref(n)))
        return n.value

    def read_relationships(self, **flt):
        """ReadRelationships: the matching lines, sorted. flt: res_type, res_id, res_id_prefix, rel, subj_type,
        subj_id, subj_rel."""
        ex = self._any_prefix([flt])
        f = self._filter_ex(flt) if ex else self._filter(flt)
        read = self._L.zg_read_relationships_ex if ex else self._L.zg_read_relationships
        cap = 1 << 16
        while True:
            buf = C.create_string_buffer(cap)
            need, n = C.c_size_t(0), C.c_uint64(0)
            rc = read(self._h, C.byref(f), buf, cap, C.byref(need), C.byref(n))
            if rc == E2BIG:
                cap = need.value + 16
                continue
            self._ck(rc)
            return [l for l in buf.value.decode().split("\n") if l]

    def read_relationships_page(self, limit: int, cursor: bytes | None = None, **flt):
        """zg_read_relationships_page -> (lines, expires, cursors, next, more): the first `limit` relationships matching
        the filter after `cursor` (None: from the start) in the page order, their expirations (0 = none), the cursor
        after each line, the cursor after the page and whether more follow. Cursors are opaque bytes."""
        ex = self._any_prefix([flt])
        f = self._filter_ex(flt) if ex else self._filter(flt)
        page = self._L.zg_read_relationships_page_ex if ex else self._L.zg_read_relationships_page
        after = None if cursor is None else C.create_string_buffer(bytes(cursor), READ_CURSOR_BYTES)
        cap = max(1 << 16, min(int(limit), 1 << 18) * 64)  # a line rarely takes more: no second run of the page
        while True:
            buf = C.create_string_buffer(cap)
            need, n, more = C.c_size_t(0), C.c_uint64(0), C.c_int32(0)
            rows = min(int(limit), cap // 8 + 1)  # a line takes at least 8 bytes
            exp = np.zeros(rows, dtype=np.uint32)
            curs = C.create_string_buffer(rows * READ_CURSOR_BYTES)
            nxt = C.create_string_buffer(READ_CURSOR_BYTES)
            rc = page(self._h, C.byref(f), int(limit), after, buf, cap, C.byref(need), C.byref(n), exp.ctypes.data, curs,
                      nxt, C.byref(more))
            if rc == E2BIG:
                cap = need.value + 16
                continue
            self._ck(rc)
            k = n.value
            lines = [l for l in buf.value.decode().split("\n") if l]
            raw = curs.raw
            cursors = [raw[i * READ_CURSOR_BYTES:(i + 1) * READ_CURSOR_BYTES] for i in range(k)]
            return lines, exp[:k].tolist(), cursors, nxt.raw, bool(more.value)

    def iter_relationships(self, limit: int, **flt):
        """Every relationship matching the filter, read page by page (`limit` per page) in the page order."""
        cursor = None
        while True:
            lines, _, _, cursor, more = self.read_relationships_page(limit, cursor, **flt)
            yield from lines
            if not more:
                return

    def delete_relationships_limited(self, flt: dict, preconditions=(), limit: int = 0, allow_partial: bool = False):
        """zg_delete_relationships_limited -> (deleted, partial). limit 0 deletes every match; otherwise more than
        `limit` matches raise ZgpuError(ZG_EPRECOND) unless allow_partial, which deletes the first `limit` of them in
        the page order and returns partial=True."""
        if self._any_prefix([flt, *(f for _, f in preconditions)]):
            n, partial = C.c_uint64(0), C.c_int32(0)
            f = self._filter_ex(flt)
            self._ck(self._L.zg_delete_relationships_limited_ex(self._h, C.byref(f), self._preconds_ex(preconditions),
                                                                len(preconditions), int(limit), 1 if allow_partial else 0,
                                                                C.byref(n), C.byref(partial)))
            return n.value, bool(partial.value)
        pre = (_Precond * max(len(preconditions), 1))()
        for i, (op, f) in enumerate(preconditions):
            pre[i] = _Precond(int(op), self._filter(f))
        n, partial = C.c_uint64(0), C.c_int32(0)
        f = self._filter(flt)
        self._ck(self._L.zg_delete_relationships_limited(self._h, C.byref(f), pre, len(preconditions), int(limit),
                                                         1 if allow_partial else 0, C.byref(n), C.byref(partial)))
        return n.value, bool(partial.value)

    def page_counters(self) -> dict:
        """zg_page_counters: pages served on the device / by the host store, entries the device windows covered,
        device launches."""
        out = np.zeros(4, dtype=np.uint64)
        self._ck(self._L.zg_page_counters(self._h, out.ctypes.data))
        return dict(zip(("device_pages", "host_pages", "scanned", "launches"), (int(x) for x in out)))

    PREFIX_COUNTERS = ("device_filters", "host_filters", "names_scanned", "matched", "launches", "mirror_syncs")

    def prefix_counters(self) -> dict:
        """zg_prefix_counters: prefix filters answered on the device / by the host store, names the device scanned,
        resources it matched, launches of the prefix scans and their match lists, names-mirror syncs that uploaded."""
        out = np.zeros(len(self.PREFIX_COUNTERS), dtype=np.uint64)
        self._ck(self._L.zg_prefix_counters(self._h, out.ctypes.data))
        return {k: int(v) for k, v in zip(self.PREFIX_COUNTERS, out)}

    # -- hot path ---------------------------------------------------------------
    def watch_read(self, since_revision: int, res_type: str = ""):
        """-> ([(revision, op_name, relationship text, expires_at)], through_revision)."""
        cap = 1 << 16
        while True:
            buf = C.create_string_buffer(cap)
            need, n, through = C.c_size_t(0), C.c_uint64(0), C.c_uint64(0)
            rc = self._L.zg_watch_read(self._h, since_revision, _b(res_type), buf, cap, C.byref(need), C.byref(n),
                                       C.byref(through))
            if rc == -7:
                cap = need.value
                continue
            self._ck(rc)
            out = []
            for line in buf.value.decode().splitlines():
                parts = line.split(" ")
                out.append((int(parts[0]), parts[1], parts[2], int(parts[3]) if len(parts) > 3 else 0))
            return out, through.value

    def check_bulk(self, items: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """CheckBulkPermissions on interned items (HOST buffers; copies inside the call)."""
        items = np.ascontiguousarray(items, dtype=CHECK_DTYPE)
        if out is None:
            out = np.empty(items.size, dtype=np.uint8)
        self._ck(self._L.zg_check_bulk(self._h, items.ctypes.data, items.size, out.ctypes.data))
        return out

    def check_bulk_ptr(self, items_ptr: int, n: int, out_ptr: int):
        """Raw HOST pointers (e.g. pinned buffers from PinnedArray)."""
        self._ck(self._L.zg_check_bulk(self._h, items_ptr, n, out_ptr))

    def check_bulk_device(self, d_items_ptr: int, n: int, d_out_ptr: int, stream: int = 0):
        """DEVICE pointers (e.g. torch tensors' data_ptr()) on a cudaStream_t handle."""
        self._ck(self._L.zg_check_bulk_device(self._h, d_items_ptr, n, d_out_ptr, stream))

    @staticmethod
    def _relstr_array(rels):
        n = len(rels)
        arr = (_RelStr * max(n, 1))()
        keep = []  # the bytes objects must outlive the call
        for i, r in enumerate(rels):
            parts = [_b(x) for x in (split_rel(r) if isinstance(r, str) else r)]
            keep.append(parts)
            arr[i] = _RelStr(*parts)
        return arr, keep

    def check_bulk_str(self, rels) -> np.ndarray:
        n = len(rels)
        arr, _keep = self._relstr_array(rels)
        out = np.empty(n, dtype=np.uint8)
        self._ck(self._L.zg_check_bulk_str(self._h, arr, n, out.ctypes.data))
        return out

    @staticmethod
    def list_template(res_type, permission, subj_type, subj_id, subj_rel="", id_kind=ID_NAMESPACED_NAME, req_name="",
                      req_namespace="", clear_namespace=False):
        return _ListTemplate(_b(res_type), _b(permission), _b(subj_type), _b(subj_id), _b(subj_rel or ""), _b(req_name),
                             _b(req_namespace), id_kind, TPL_CLEAR_NAMESPACE if clear_namespace else 0)

    def list_resolve(self, body: bytes, items: np.ndarray, tpl: "_ListTemplate"):
        """-> (interned checks, checked mask) for the scanned items; no GPU work."""
        items = np.ascontiguousarray(items, dtype=LIST_ITEM_DTYPE)
        out = np.zeros(len(items), dtype=CHECK_DTYPE)
        checked = np.zeros(len(items), dtype=np.uint8)
        self._ck(self._L.zg_list_resolve(self._h, body, len(body), items.ctypes.data, len(items), C.byref(tpl),
                                         out.ctypes.data, checked.ctypes.data))
        return out, checked

    def list_postfilter(self, body: bytes, templates) -> bytes:
        """zg_list_postfilter: the whole post-filter of a list body in one call."""
        arr = (_ListTemplate * max(len(templates), 1))(*templates)
        out = np.empty(len(body) + 8, dtype=np.uint8)
        need = C.c_size_t(0)
        self._ck(self._L.zg_list_postfilter(self._h, body, len(body), arr, len(templates), out.ctypes.data, out.size,
                                            C.byref(need)))
        return out[:need.value].tobytes()

    def list_keep_allowed(self, body: bytes, items: np.ndarray, res_type: str, allowed_ids: np.ndarray, mode: int = LIST_ITEMS,
                          req_namespace: str = "", self_name: str | None = None) -> np.ndarray:
        """keep mask of the scanned items given the (ascending) object ids a LookupResources returned; no GPU work."""
        items = np.ascontiguousarray(items, dtype=LIST_ITEM_DTYPE)
        allowed = np.ascontiguousarray(allowed_ids, dtype=np.uint32)
        keep = np.zeros(len(items), dtype=np.uint8)
        self._ck(self._L.zg_list_keep_allowed(self._h, body, len(body), items.ctypes.data, len(items), mode, _b(res_type),
                                              _b(req_namespace), allowed.ctypes.data, allowed.size, _b(self_name),
                                              keep.ctypes.data))
        return keep

    def list_prefilter(self, body: bytes, tpl: "_ListTemplate", mode: int = LIST_ITEMS) -> bytes:
        """zg_list_prefilter: LookupResources + scan + keep + splice in one call."""
        out = np.empty(len(body) + 8, dtype=np.uint8)
        need = C.c_size_t(0)
        self._ck(self._L.zg_list_prefilter(self._h, body, len(body), mode, C.byref(tpl), out.ctypes.data, out.size,
                                           C.byref(need)))
        return out[:need.value].tobytes()

    @staticmethod
    def pack_ids(ids):
        """[str] -> (blob, offsets[n+1]) as the packed entry points take them."""
        enc = [_b(i) for i in ids]
        off = np.zeros(len(enc) + 1, dtype=np.uint32)
        np.cumsum([len(x) for x in enc], out=off[1:])
        return b"".join(enc), off

    def _packed_call(self, fn, res_type, relation, subj_type, subj_rel, res_ids, subjects, out):
        blob, off = self.pack_ids(res_ids)
        if isinstance(subjects, (str, bytes)):
            sblob, soff = _b(subjects), None
        else:
            sblob, so = self.pack_ids(subjects)
            soff = so.ctypes.data
            sblob = sblob or b"\0"
        self._ck(fn(self._h, _b(res_type), _b(relation), _b(subj_type), _b(subj_rel or ""), blob or b"\0", off.ctypes.data,
                    sblob, soff, len(res_ids), out.ctypes.data))
        return out

    def resolve_checks_packed(self, res_type, relation, subj_type, res_ids, subjects, subj_rel="") -> np.ndarray:
        """`subjects`: one id (str) for all items, or a list of n ids."""
        return self._packed_call(self._L.zg_resolve_checks_packed, res_type, relation, subj_type, subj_rel, res_ids, subjects,
                                 np.zeros(len(res_ids), dtype=CHECK_DTYPE))

    def check_bulk_packed(self, res_type, relation, subj_type, res_ids, subjects, subj_rel="") -> np.ndarray:
        return self._packed_call(self._L.zg_check_bulk_packed, res_type, relation, subj_type, subj_rel, res_ids, subjects,
                                 np.empty(len(res_ids), dtype=np.uint8))

    def check_bulk_packed_ingress(self, res_type, relation, subj_type, res_ids, subjects, subj_rel="") -> np.ndarray:
        """check_bulk_packed with the ids resolved on the GPU (one launch sequence, outside the batcher)."""
        return self._packed_call(self._L.zg_check_bulk_packed_ingress, res_type, relation, subj_type, subj_rel, res_ids,
                                 subjects, np.empty(len(res_ids), dtype=np.uint8))

    def resolve_checks_packed_device(self, res_type, relation, subj_type, d_res_ids: int, d_res_off: int, n: int,
                                     d_out: int, subjects=None, d_subj_off: int = 0, subj_rel="", stream: int = 0):
        """zg_resolve_checks_packed_device: DEVICE pointers as ints (blob, n + 1 u32 offsets, n zg_check out). `subjects`:
        the one subject (str) for every item, or the device pointer of the per-item subject blob with d_subj_off."""
        one = isinstance(subjects, (str, bytes))
        self._ck(self._L.zg_resolve_checks_packed_device(
            self._h, _b(res_type), _b(relation), _b(subj_type), _b(subj_rel or ""), d_res_ids, d_res_off,
            _b(subjects) if one else subjects, None if one else d_subj_off, n, d_out, stream))

    def intern_packed(self, type_name, ids) -> np.ndarray:
        """zg_intern_objects_packed: the ids of the names (str or bytes), interning the new ones."""
        blob, off = self.pack_ids(ids)
        out = np.empty(len(ids), dtype=np.uint32)
        self._ck(self._L.zg_intern_objects_packed(self._h, self.type_id(type_name), blob or b"\0", off.ctypes.data, len(ids),
                                                  out.ctypes.data))
        return out

    def ingress_counters(self) -> dict:
        out = np.zeros(5, dtype=np.uint64)
        self._ck(self._L.zg_ingress_counters(self._h, out.ctypes.data))
        return {"names": int(out[0]), "device_bytes": int(out[1]), "sync_uploads": int(out[2]), "rebuilds": int(out[3]),
                "items_resolved": int(out[4])}

    def resolve_checks(self, rels) -> np.ndarray:
        """Strings -> interned zg_check items (no GPU work); feed them to check_bulk."""
        n = len(rels)
        arr, _keep = self._relstr_array(rels)
        out = np.zeros(n, dtype=CHECK_DTYPE)
        self._ck(self._L.zg_resolve_checks(self._h, arr, n, out.ctypes.data))
        return out

    def lookup_resources_ids(self, res_type, perm, subj_type, subj, srel=None) -> np.ndarray:
        sr = SREL_NONE if srel is None else self.slot_id(subj_type, srel)
        cap = 1 << 14
        while True:  # on ZG_E2BIG the library keeps the answer: the retry only copies it
            out = np.empty(cap, dtype=np.uint32)
            n = C.c_uint64(0)
            rc = self._L.zg_lookup_resources(self._h, self.type_id(res_type), self.slot_id(res_type, perm),
                                             self.type_id(subj_type), int(subj), sr, out.ctypes.data, cap, C.byref(n))
            if rc == E2BIG:
                cap = int(n.value)
                continue
            self._ck(rc)
            return out[: n.value].copy()

    def lookup_resources_str(self, res_type, perm, subj_type, subj_id, subj_rel=""):
        cap = 1 << 16
        while True:
            buf = C.create_string_buffer(cap)
            need, n = C.c_size_t(0), C.c_uint64(0)
            rc = self._L.zg_lookup_resources_str(self._h, _b(res_type), _b(perm), _b(subj_type), _b(subj_id),
                                                 _b(subj_rel or ""), buf, cap, C.byref(need), C.byref(n))
            if rc == E2BIG:
                cap = need.value + 16
                continue
            self._ck(rc)
            return [l for l in buf.value.decode().split("\n") if l]

    def lookup_resources_page(self, res_type, perm, subj_type, subj, srel=None, limit: int = 1000,
                              after: bytes | None = None):
        """zg_lookup_resources_page -> (ids, cursors, next, more): the first `limit` ids (ascending) of the
        LookupResources answer after the cursor `after` (None: from the start), the cursor after each id, the cursor
        after the page and whether more follow. Cursors are opaque bytes."""
        rt = self.type_id(res_type)
        sr = SREL_NONE if srel is None else self.slot_id(subj_type, srel)
        rows = min(int(limit), MAX_LOOKUP_PAGE)
        a = None if after is None else C.create_string_buffer(bytes(after), READ_CURSOR_BYTES)
        out = np.empty(rows, dtype=np.uint32)
        curs, nxt = C.create_string_buffer(rows * READ_CURSOR_BYTES), C.create_string_buffer(READ_CURSOR_BYTES)
        n, more = C.c_uint64(0), C.c_int32(0)
        self._ck(self._L.zg_lookup_resources_page(self._h, rt, self.slot_id(res_type, perm), self.type_id(subj_type),
                                                  int(subj), sr, rows, a, out.ctypes.data, C.byref(n), curs, nxt,
                                                  C.byref(more)))
        k, raw = n.value, curs.raw
        return (out[:k].copy(), [raw[i * READ_CURSOR_BYTES:(i + 1) * READ_CURSOR_BYTES] for i in range(k)], nxt.raw,
                bool(more.value))

    def lookup_resources_page_str(self, res_type, perm, subj_type, subj_id, subj_rel="", limit: int = 1000,
                                  after: bytes | None = None):
        """zg_lookup_resources_page_str -> (names, cursors, next, more), as lookup_resources_page."""
        rows = min(int(limit), MAX_LOOKUP_PAGE)
        a = None if after is None else C.create_string_buffer(bytes(after), READ_CURSOR_BYTES)
        cap = max(1 << 16, min(rows, 1 << 18) * 64)  # a name rarely takes more: no second run of the page
        while True:
            buf = C.create_string_buffer(cap)
            curs, nxt = C.create_string_buffer(rows * READ_CURSOR_BYTES), C.create_string_buffer(READ_CURSOR_BYTES)
            need, n, more = C.c_size_t(0), C.c_uint64(0), C.c_int32(0)
            rc = self._L.zg_lookup_resources_page_str(self._h, _b(res_type), _b(perm), _b(subj_type), _b(subj_id),
                                                      _b(subj_rel or ""), rows, a, buf, cap, C.byref(need),
                                                      C.byref(n), curs, nxt, C.byref(more))
            if rc == E2BIG:
                cap = need.value + 16
                continue
            self._ck(rc)
            k, raw = n.value, curs.raw
            names = [l for l in buf.value.decode().split("\n") if l]
            return names, [raw[i * READ_CURSOR_BYTES:(i + 1) * READ_CURSOR_BYTES] for i in range(k)], nxt.raw, bool(more.value)

    def iter_lookup_resources(self, res_type, perm, subj_type, subj, srel=None, limit: int = 1000):
        """Every id of the LookupResources answer, looked up page by page (`limit` per page), ascending."""
        cursor = None
        while True:
            ids, _, cursor, more = self.lookup_resources_page(res_type, perm, subj_type, subj, srel, limit, cursor)
            yield from (int(i) for i in ids)
            if not more:
                return

    def lookup_page_counters(self) -> dict:
        """zg_lookup_page_counters: pages answered by windowed verification / cut from a whole answer (sharded handle),
        candidates after the cursor, candidates verified, verification windows."""
        out = np.zeros(5, dtype=np.uint64)
        self._ck(self._L.zg_lookup_page_counters(self._h, out.ctypes.data))
        return dict(zip(("windowed_pages", "cut_pages", "after_cursor", "verified", "windows"), (int(x) for x in out)))

    def lookup_subjects_ids(self, res_type, res, perm, subj_type, srel=None, wildcards=WILDCARDS_INCLUDE, cap=1 << 14):
        """LookupSubjects by ids -> (ids ascending, wildcard: bool, excluded ids ascending)."""
        sr = SREL_NONE if srel is None else self.slot_id(subj_type, srel)
        p = self.slot_id(res_type, perm)
        ex_cap = cap
        while True:  # ZG_E2BIG reports both required sizes
            out, ex = np.empty(cap, dtype=np.uint32), np.empty(ex_cap, dtype=np.uint32)
            n, nx, wild = C.c_uint64(0), C.c_uint64(0), C.c_int32(0)
            rc = self._L.zg_lookup_subjects(self._h, p & 0xFFFF, int(res), self.type_id(subj_type) & 0xFFFF, sr & 0xFFFF,
                                            int(wildcards), out.ctypes.data, cap, C.byref(n), ex.ctypes.data, ex_cap,
                                            C.byref(nx), C.byref(wild))
            if rc == E2BIG:
                cap, ex_cap = max(cap, int(n.value)), max(ex_cap, int(nx.value))
                continue
            self._ck(rc)
            return out[: n.value].copy(), bool(wild.value), ex[: nx.value].copy()

    def lookup_subjects_str(self, res_type, res_id, perm, subj_type, subj_rel="", wildcards=WILDCARDS_INCLUDE, cap=1 << 16):
        """LookupSubjects by names -> (subject ids, wildcard: bool, excluded subject ids) in internal-id order."""
        while True:
            buf = C.create_string_buffer(cap)
            need, n = C.c_size_t(0), C.c_uint64(0)
            rc = self._L.zg_lookup_subjects_str(self._h, _b(res_type), _b(res_id), _b(perm), _b(subj_type), _b(subj_rel or ""),
                                                int(wildcards), buf, cap, C.byref(need), C.byref(n))
            if rc == E2BIG:
                cap = need.value + 16
                continue
            self._ck(rc)
            lines = [l for l in buf.value.decode().split("\n") if l]
            if "*" in lines:
                at = lines.index("*")
                return lines[:at], True, [l[1:] for l in lines[at + 1:]]
            return lines, False, []

    def lookup_subjects_counters(self) -> dict:
        out = np.zeros(3, dtype=np.uint64)
        self._ck(self._L.zg_lookup_subjects_counters(self._h, out.ctypes.data))
        return {"walks": int(out[0]), "fallbacks": int(out[1]), "items_verified": int(out[2])}

    def expand_permission_trees(self, requests, node_cap=1 << 12, subj_cap=1 << 14):
        """ExpandPermissionTree by ids. requests: [(res_type, res id or NO_OBJECT, relation or permission)]. Returns one
        entry per request: its tree, or the ZgpuError it failed with (ZG_EDEPTH). A tree node is {"op": U|I|X|L,
        "type": str, "object": int, "relation": str, "subjects": [(type, id, srel)], "children": [...]}, children in
        rank order, a subject's srel None (plain), "*" (wildcard, id 0) or the userset's relation name."""
        reqs = np.zeros(len(requests), dtype=EXPAND_REQUEST_DTYPE)
        for i, (rt, res, perm) in enumerate(requests):
            p = self.slot_id(rt, perm)
            if p < 0:
                raise ZgpuError(-1, f"relation/permission `{perm}` not found under definition `{rt}`")
            reqs[i] = (p, 0, int(res))
        return self.expand_trees_from(reqs.size, *self.expand_permission_arrays(reqs, node_cap, subj_cap))

    def expand_permission_arrays(self, reqs, node_cap=1 << 12, subj_cap=1 << 14, out=None):
        """zg_expand_permission_trees on EXPAND_REQUEST_DTYPE requests -> (status, nodes, subjects) arrays. out: (nodes,
        subjects) arrays to answer into (views of them are returned) while they are large enough."""
        reqs = np.ascontiguousarray(reqs, dtype=EXPAND_REQUEST_DTYPE)
        status = np.zeros(max(len(reqs), 1), dtype=np.int32)
        while True:  # ZG_E2BIG reports both required sizes
            if out is not None and out[0].size >= node_cap and out[1].size >= subj_cap:
                nodes, subj = out
                node_cap, subj_cap = nodes.size, subj.size
            else:
                nodes, subj = np.zeros(node_cap, dtype=EXPAND_NODE_DTYPE), np.zeros(subj_cap, dtype=EXPAND_SUBJECT_DTYPE)
            nn, ns = C.c_uint64(0), C.c_uint64(0)
            rc = self._L.zg_expand_permission_trees(self._h, reqs.ctypes.data, len(reqs), status.ctypes.data,
                                                    nodes.ctypes.data, node_cap, C.byref(nn), subj.ctypes.data, subj_cap,
                                                    C.byref(ns))
            if rc == E2BIG:
                node_cap, subj_cap = max(node_cap, int(nn.value)), max(subj_cap, int(ns.value))
                continue
            self._ck(rc)
            return status, nodes[: nn.value], subj[: ns.value]

    def expand_trees_from(self, n_requests, status, nodes, subj):
        """zg_expand_permission_trees' arrays -> the nested trees of expand_permission_trees."""
        slots = self.slot_table()
        tnames = [self._L.zg_type_name(self._h, t).decode() for t in range(self._L.zg_num_types(self._h))]
        out = [ZgpuError(int(status[i]), "ExpandPermissionTree: the tree passes the maximum depth")
               if status[i] else None for i in range(n_requests)]
        built = []
        for nd in nodes:
            _, t, rel, _ = slots[int(nd["slot"])]
            b = int(nd["subjects"])
            n = {"op": _EXPAND_OP[int(nd["op"])], "type": t, "object": int(nd["object"]), "relation": rel, "children": [],
                 "subjects": [(tnames[int(x["type"])], int(x["id"]),
                               None if x["srel"] == SREL_NONE else "*" if x["srel"] == SREL_WILDCARD else slots[int(x["srel"])][2])
                              for x in subj[b: b + int(nd["n_subjects"])]], "_rank": int(nd["rank"])}
            built.append(n)
            if nd["parent"] == 0xFFFFFFFF:
                out[int(nd["request"])] = n
            else:
                built[int(nd["parent"])]["children"].append(n)
        for n in built:
            n["children"].sort(key=lambda c: c["_rank"])
        for n in built:
            del n["_rank"]
        return out

    def expand_permission_tree_str(self, res_type, res_id, perm, cap=1 << 16):
        """ExpandPermissionTree by names -> the lines of zg_expand_permission_tree_str (parse_expand_lines nests them)."""
        while True:
            buf = C.create_string_buffer(cap)
            need, n = C.c_size_t(0), C.c_uint64(0)
            rc = self._L.zg_expand_permission_tree_str(self._h, _b(res_type), _b(res_id), _b(perm), buf, cap, C.byref(need),
                                                       C.byref(n))
            if rc == E2BIG:
                cap = need.value + 16
                continue
            self._ck(rc)
            return [l for l in buf.value.decode().split("\n") if l]

    def expand_counters(self) -> dict:
        out = np.zeros(4, dtype=np.uint64)
        self._ck(self._L.zg_expand_counters(self._h, out.ctypes.data))
        return dict(zip(("trees", "levels", "nodes", "subjects"), (int(x) for x in out)))

    def expand_last_times(self) -> np.ndarray:
        """Per level of the last expand call: (count, scan, emit) device milliseconds."""
        n = C.c_uint64(0)
        out = np.zeros(3 * 64, dtype=np.float64)
        self._ck(self._L.zg_expand_last_times(self._h, out.ctypes.data, out.size, C.byref(n)))
        return out[: n.value].reshape(-1, 3)

    CLOSURE_INDEX_COUNTERS = ("indexed", "over_budget", "entries", "device_bytes", "builds", "last_build_us", "failures")

    def closure_index_counters(self) -> dict:
        """Closure indexes of the two-level steps in the published snapshot (zg_closure_index_counters)."""
        out = np.zeros(len(self.CLOSURE_INDEX_COUNTERS), dtype=np.uint64)
        self._ck(self._L.zg_closure_index_counters(self._h, out.ctypes.data))
        return {k: int(v) for k, v in zip(self.CLOSURE_INDEX_COUNTERS, out)}

    def closure_index_info(self, pair: int = 0) -> dict:
        """Built flag, entry width in bytes, entries and device bytes of closure index `pair` (zg_closure_index_info)."""
        out = np.zeros(4, dtype=np.uint64)
        self._ck(self._L.zg_closure_index_info(self._h, pair, out.ctypes.data))
        return {k: int(v) for k, v in zip(("built", "width", "entries", "device_bytes"), out)}

    def closure_index(self, pair: int = 0):
        """(row_ptr, col) of closure index `pair` of the published snapshot (zg_closure_index_copy)."""
        nr, ne = C.c_uint64(0), C.c_uint64(0)
        rc = self._L.zg_closure_index_copy(self._h, pair, None, 0, None, 0, C.byref(nr), C.byref(ne))
        if rc != E2BIG:
            self._ck(rc)
        row_ptr, col = np.empty(nr.value + 1, dtype=np.uint32), np.empty(max(ne.value, 1), dtype=np.uint32)
        self._ck(self._L.zg_closure_index_copy(self._h, pair, row_ptr.ctypes.data, row_ptr.size, col.ctypes.data, col.size,
                                               C.byref(nr), C.byref(ne)))
        return row_ptr, col[: ne.value]

    def closure_signature_info(self, pair: int = 0) -> dict:
        """Built flag, words per row, bits per entry, device bytes and last build time (device microseconds) of the
        signatures of closure index `pair` (zg_closure_signature_info)."""
        out = np.zeros(5, dtype=np.uint64)
        self._ck(self._L.zg_closure_signature_info(self._h, pair, out.ctypes.data))
        return {k: int(v) for k, v in zip(("built", "words", "k", "device_bytes", "build_us"), out)}

    def closure_signature(self, pair: int = 0):
        """Signatures of closure index `pair`: uint64 array of shape (rows, words per row) (zg_closure_signature_copy)."""
        words = self.closure_signature_info(pair)["words"]
        n = C.c_uint64(0)
        rc = self._L.zg_closure_signature_copy(self._h, pair, None, 0, C.byref(n))
        if rc != E2BIG:
            self._ck(rc)
        out = np.empty(max(n.value, 1), dtype=np.uint64)
        self._ck(self._L.zg_closure_signature_copy(self._h, pair, out.ctypes.data, out.size, C.byref(n)))
        return out[: n.value].reshape(-1, max(words, 1))

    def closure_table_info(self, pair: int = 0) -> dict:
        """Built flag, buckets, slots per bucket, device bytes and last build time (device microseconds) of the set
        table of closure index `pair` (zg_closure_table_info)."""
        out = np.zeros(5, dtype=np.uint64)
        self._ck(self._L.zg_closure_table_info(self._h, pair, out.ctypes.data))
        return {k: int(v) for k, v in zip(("built", "buckets", "slots", "device_bytes", "build_us"), out)}

    def closure_table(self, pair: int = 0):
        """Set table of closure index `pair`: (uint64 header per row, uint16 array of shape (buckets, 4))
        (zg_closure_table_copy)."""
        nr, nb = C.c_uint64(0), C.c_uint64(0)
        rc = self._L.zg_closure_table_copy(self._h, pair, None, 0, None, 0, C.byref(nr), C.byref(nb))
        if rc != E2BIG:
            self._ck(rc)
        hdr = np.empty(max(nr.value, 1), dtype=np.uint64)
        tab = np.empty(max(nb.value, 1), dtype=np.uint64)
        self._ck(self._L.zg_closure_table_copy(self._h, pair, hdr.ctypes.data, hdr.size, tab.ctypes.data, tab.size,
                                               C.byref(nr), C.byref(nb)))
        return hdr[: nr.value], tab[: nb.value].view(np.uint16).reshape(-1, 4)

    def flat_record_info(self, k: int = 0) -> dict:
        """Built flag, edge class, objects, device bytes, rows kept on the offsets path and last build time (device
        microseconds) of range records `k` (zg_flat_record_info)."""
        out = np.zeros(6, dtype=np.uint64)
        self._ck(self._L.zg_flat_record_info(self._h, k, out.ctypes.data))
        return {k: int(v) for k, v in zip(("built", "cls", "objects", "device_bytes", "long_rows", "build_us"), out)}

    def flat_records(self, k: int = 0):
        """Range records `k`: uint16 array of shape (objects, slots per record) (zg_flat_record_copy)."""
        n = C.c_uint64(0)
        rc = self._L.zg_flat_record_copy(self._h, k, None, 0, C.byref(n))
        if rc != E2BIG:
            self._ck(rc)
        out = np.empty(max(n.value, 1), dtype=np.uint16)
        self._ck(self._L.zg_flat_record_copy(self._h, k, out.ctypes.data, out.size, C.byref(n)))
        objects = self.flat_record_info(k)["objects"]
        return out[: n.value].reshape(objects, -1) if objects else out[:0].reshape(0, 1)

    HANDLE_LOOKUP_COUNTERS = ("rounds", "levels", "round_trips", "frontier_entries", "candidates", "halvings", "fallbacks")

    def handle_lookup_counters(self) -> dict:
        """Cumulative LookupResources counters of a sharded handle with handle_lookups (zg_handle_lookup_counters)."""
        out = np.zeros(len(self.HANDLE_LOOKUP_COUNTERS), dtype=np.uint64)
        self._ck(self._L.zg_handle_lookup_counters(self._h, out.ctypes.data))
        return {k: int(v) for k, v in zip(self.HANDLE_LOOKUP_COUNTERS, out)}

    HANDLE_SUBJECTS_COUNTERS = ("lookups", "levels", "host_waits", "inbox_entries", "candidates", "nowild_items",
                                "fallbacks")

    def handle_subjects_counters(self) -> dict:
        """Cumulative LookupSubjects counters of a sharded handle with handle_subjects (zg_handle_subjects_counters)."""
        out = np.zeros(len(self.HANDLE_SUBJECTS_COUNTERS), dtype=np.uint64)
        self._ck(self._L.zg_handle_subjects_counters(self._h, out.ctypes.data))
        return {k: int(v) for k, v in zip(self.HANDLE_SUBJECTS_COUNTERS, out)}

    FILTER_COUNTERS = ("device_filters", "host_filters", "device_relationships", "by_resource", "by_subject", "by_scan")

    def filter_counters(self) -> dict:
        """Cumulative counters of the relationship filters of reads, deletes by filter and preconditions: answered from
        the snapshot on the device or by the host scan (zg_filter_counters)."""
        out = np.zeros(len(self.FILTER_COUNTERS), dtype=np.uint64)
        self._ck(self._L.zg_filter_counters(self._h, out.ctypes.data))
        return {k: int(v) for k, v in zip(self.FILTER_COUNTERS, out)}

    def retire_unused_names(self) -> int:
        """zg_retire_unused_names: retires every interned name no relationship in the store and no retained watch
        change mentions; returns how many. Their ids are handed to new names, lowest first."""
        n = C.c_uint64(0)
        self._ck(self._L.zg_retire_unused_names(self._h, C.byref(n)))
        return n.value

    NAME_COUNTERS = ("named", "retired", "free_ids", "id_extent", "arena_bytes", "retired_device", "retired_host")

    def name_counters(self) -> dict:
        """Interned names, retirements, free ids, the id extent and the host arena bytes (zg_name_counters)."""
        out = np.zeros(len(self.NAME_COUNTERS), dtype=np.uint64)
        self._ck(self._L.zg_name_counters(self._h, out.ctypes.data))
        return {k: int(v) for k, v in zip(self.NAME_COUNTERS, out)}

    _HOOK = C.CFUNCTYPE(None, C.c_void_p)

    def set_resolve_hook(self, fn):
        """Tests only (zg_debug_set_resolve_hook): fn() runs inside the string checks and lookups between resolving their
        names and answering; None removes it."""
        self._resolve_hook = None if fn is None else self._HOOK(lambda _arg: fn())
        self._ck(self._L.zg_debug_set_resolve_hook(self._h, self._resolve_hook, None))

    def object_capacity(self, type_name) -> int:
        """The object capacity of a type in the last layout (zg_object_capacity)."""
        return int(self._L.zg_object_capacity(self._h, self.type_id(type_name)))

    # -- sharded store (dist.DeviceShardedChecker drives these) --------------------
    # every pointer is a device address on this engine's GPU (ints, e.g. tensor.data_ptr())
    def shard_route_dev(self, d_items: int, n: int, level: int, n_dest: int, d_routed: int, d_src: int) -> list:
        counts = (C.c_uint64 * n_dest)()
        self._ck(self._L.zg_shard_route_dev(self._h, d_items or None, n, level, n_dest, d_routed or None, d_src or None, counts))
        return [int(c) for c in counts]

    def shard_pass_dev(self, d_queries: int, n: int, level: int) -> int:
        ns = C.c_uint64(0)
        self._ck(self._L.zg_shard_pass_dev(self._h, d_queries or None, n, level, C.byref(ns)))
        return ns.value

    def shard_fold_dev(self, level: int, d_child_vals: int, d_src: int, n_sub: int, d_out: int, final_codes: bool):
        self._ck(self._L.zg_shard_fold_dev(self._h, level, d_child_vals or None, d_src or None, n_sub, d_out or None,
                                           1 if final_codes else 0))

    def shard_unroute_dev(self, d_src: int, d_val: int, n: int, d_out: int):
        self._ck(self._L.zg_shard_unroute_dev(self._h, d_src or None, d_val or None, n, d_out or None))

    # sharded LookupResources (dist.DeviceShardedLookup drives these): one round of <= 64 lookups at a time
    def shard_lookup_begin_dev(self, res_types, protos, home, walk_cap: int, d_seeds: int):
        """res_types (uint16), protos (CHECK_DTYPE: subj, perm, stype, srel), home (uint8): host arrays of k."""
        rt = np.ascontiguousarray(res_types, dtype=np.uint16)
        pr = np.ascontiguousarray(protos, dtype=CHECK_DTYPE)
        hm = np.ascontiguousarray(home, dtype=np.uint8)
        self._ck(self._L.zg_shard_lookup_begin_dev(self._h, rt.ctypes.data, pr.ctypes.data, hm.ctypes.data, rt.size, walk_cap,
                                                   d_seeds or None))

    def shard_lookup_expand_dev(self, d_front: int, n_in: int, level: int, d_next: int):
        """-> (new frontier entries, overflow)"""
        n, ovf = C.c_uint64(0), C.c_int(0)
        self._ck(self._L.zg_shard_lookup_expand_dev(self._h, d_front or None, n_in, level, d_next or None, C.byref(n),
                                                    C.byref(ovf)))
        return n.value, bool(ovf.value)

    def shard_lookup_candidates_dev(self, exhaustive: bool, d_items: int, cap: int) -> int:
        """d_items == 0: the capacity needed; else the candidates written."""
        n = C.c_uint64(0)
        self._ck(self._L.zg_shard_lookup_candidates_dev(self._h, 1 if exhaustive else 0, d_items or None, cap, C.byref(n)))
        return n.value

    def shard_lookup_route_dev(self, d_codes: int, n: int, n_dest: int, d_routed: int) -> list:
        counts = (C.c_uint64 * n_dest)()
        self._ck(self._L.zg_shard_lookup_route_dev(self._h, d_codes or None, n, n_dest, d_routed or None, counts))
        return [int(c) for c in counts]

    def shard_lookup_finish_dev(self, d_keys: int, n: int, d_ids: int, k: int):
        """-> (answers per lookup of the round, error mask)"""
        per = (C.c_uint64 * max(k, 1))()
        mask = C.c_uint64(0)
        self._ck(self._L.zg_shard_lookup_finish_dev(self._h, d_keys or None, n, d_ids or None, per, C.byref(mask)))
        return [int(per[i]) for i in range(k)], mask.value

    def shard_pass_nowild_dev(self, d_queries: int, n: int, level: int) -> int:
        """shard_pass_dev with every wildcard relationship invisible (LookupSubjects' second verification)."""
        ns = C.c_uint64(0)
        self._ck(self._L.zg_shard_pass_nowild_dev(self._h, d_queries or None, n, level, C.byref(ns)))
        return ns.value

    # sharded LookupSubjects (dist.DeviceShardedLookup.lookup_subjects drives these): one round of <= 64 lookups at a time
    def shard_subjects_begin_dev(self, res_types, reqs, options, home, walk_cap: int, d_front: int) -> int:
        """res_types (uint16), reqs (CHECK_DTYPE: res, perm, stype, srel), options (uint32 ZG_WILDCARDS_*), home (uint8):
        host arrays of k. -> entries of this rank's level-0 frontier."""
        rt = np.ascontiguousarray(res_types, dtype=np.uint16)
        rq = np.ascontiguousarray(reqs, dtype=CHECK_DTYPE)
        op = np.ascontiguousarray(options, dtype=np.uint32)
        hm = np.ascontiguousarray(home, dtype=np.uint8)
        n = C.c_uint64(0)
        self._ck(self._L.zg_shard_subjects_begin_dev(self._h, rt.ctypes.data, rq.ctypes.data, op.ctypes.data, hm.ctypes.data,
                                                     rq.size, walk_cap, d_front or None, C.byref(n)))
        return n.value

    def shard_subjects_expand_dev(self, d_front: int, n_in: int, n_dest: int, d_routed: int):
        """-> (entries per destination rank, overflow)"""
        counts = (C.c_uint64 * n_dest)()
        ovf = C.c_int(0)
        self._ck(self._L.zg_shard_subjects_expand_dev(self._h, d_front or None, n_in, n_dest, d_routed or None, counts,
                                                      C.byref(ovf)))
        return [int(c) for c in counts], bool(ovf.value)

    def shard_subjects_admit_dev(self, d_in: int, n_in: int, d_next: int) -> int:
        n = C.c_uint64(0)
        self._ck(self._L.zg_shard_subjects_admit_dev(self._h, d_in or None, n_in, d_next or None, C.byref(n)))
        return n.value

    def shard_subjects_candidates_dev(self, exhaustive: bool, d_items: int, cap: int) -> int:
        """d_items == 0: the capacity needed; else the candidates written."""
        n = C.c_uint64(0)
        self._ck(self._L.zg_shard_subjects_candidates_dev(self._h, 1 if exhaustive else 0, d_items or None, cap, C.byref(n)))
        return n.value

    def shard_subjects_verdicts_dev(self, d_codes: int, n: int):
        """-> (granted mask, failed mask) of this rank's items"""
        g, f = C.c_uint64(0), C.c_uint64(0)
        self._ck(self._L.zg_shard_subjects_verdicts_dev(self._h, d_codes or None, n, C.byref(g), C.byref(f)))
        return g.value, f.value

    def shard_subjects_nowild_dev(self, d_codes: int, n: int, granted: int, failed: int, d_items: int, cap: int) -> int:
        m = C.c_uint64(0)
        self._ck(self._L.zg_shard_subjects_nowild_dev(self._h, d_codes or None, n, granted, failed, d_items or None, cap,
                                                      C.byref(m)))
        return m.value

    def shard_subjects_route_dev(self, d_codes: int, n: int, n_dest: int, d_routed: int) -> list:
        counts = (C.c_uint64 * n_dest)()
        self._ck(self._L.zg_shard_subjects_route_dev(self._h, d_codes or None, n, n_dest, d_routed or None, counts))
        return [int(c) for c in counts]

    def shard_subjects_finish_dev(self, d_keys: int, n: int, d_ids: int, k: int):
        """-> (listed ids per lookup, excluded ids per lookup) of the round"""
        listed, excluded = (C.c_uint64 * max(k, 1))(), (C.c_uint64 * max(k, 1))()
        self._ck(self._L.zg_shard_subjects_finish_dev(self._h, d_keys or None, n, d_ids or None, listed, excluded))
        return [int(listed[i]) for i in range(k)], [int(excluded[i]) for i in range(k)]

    def debug_row(self, type_name, rel, res, cls=0, reverse=False, shard=None) -> np.ndarray:
        """Forward row (resource `res`, class) or, reverse=True, the reverse row of subject `res`; shard=k: that row in
        shard k of a sharded handle."""
        if reverse:
            cls |= 0x80000000
        cap = 1 << 10
        while True:
            out = np.empty(cap, dtype=np.uint32)
            n = C.c_uint64(0)
            slot = self.slot_id(type_name, rel)
            if shard is None:
                rc = self._L.zg_debug_row(self._h, slot, int(res), int(cls), out.ctypes.data, cap, C.byref(n))
            else:
                rc = self._L.zg_debug_shard_row(self._h, int(shard), slot, int(res), int(cls), out.ctypes.data, cap,
                                                C.byref(n))
            if rc == E2BIG:
                cap = int(n.value)
                continue
            self._ck(rc)
            return out[: n.value].copy()

    # -- measurement ------------------------------------------------------------
    def stats(self) -> dict:
        s = _Stats()
        self._ck(self._L.zg_stats_get(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in _Stats._fields_}

    def count_alg_bytes(self, items: np.ndarray) -> int:
        items = np.ascontiguousarray(items, dtype=CHECK_DTYPE)
        b = C.c_uint64(0)
        self._ck(self._L.zg_count_alg_bytes(self._h, items.ctypes.data, items.size, C.byref(b)))
        return b.value

    PHASES = ("admission", "root_visit", "l2_meet", "l1_meet", "pop_loop")

    def phase_clocks(self) -> dict:
        """Cumulative check-kernel cycles per phase (a library built with -DZG_PHASE_CLOCKS=1 only)."""
        c = (C.c_uint64 * len(self.PHASES))()
        self._ck(self._L.zg_phase_clocks(self._h, c))
        return dict(zip(self.PHASES, (int(x) for x in c)))
