"""ctypes binding of the kernel emulator (tests/emu/emu_main.cc): the product's kernels.cuh executed by a CPU SIMT
emulator. TEST INFRASTRUCTURE ONLY -- never imported by the product, never linked into libzgpu.so."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_CSRC = os.path.join(_ROOT, "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None

CHECK_DTYPE = np.dtype([("res", "<u4"), ("subj", "<u4"), ("perm", "<u2"), ("stype", "<u2"), ("srel", "<u2"), ("flags", "<u2")])
TUPLE_DTYPE = np.dtype([("res", "<u4"), ("subj", "<u4"), ("rel", "<u2"), ("stype", "<u2"), ("srel", "<u2"), ("flags", "<u2")])
SREL_NONE, SREL_WILDCARD = 0xFFFF, 0xFFFE


class Opts(C.Structure):
    _fields_ = [("invert", C.c_int32), ("memo_after", C.c_uint32), ("memo_entries", C.c_uint32), ("subq_cap", C.c_uint64),
                ("budget", C.c_uint32), ("now", C.c_uint32), ("grid", C.c_uint32), ("spill_cap", C.c_uint32),
                ("streamed", C.c_uint32)]


def default_opts(**kw):
    o = Opts(1, 2048, 8192, 1 << 16, 1 << 20, 0, 2, 4096, 0)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def build() -> str:
    extra = os.environ.get("ZGPU_EMU_CFLAGS", "").split()  # tuning macros of kernels.cuh (-DZG_PHASE_CLOCKS=1 ...)
    so = os.path.join(_HERE, "libzgemu" + ("_" + "".join(c if c.isalnum() else "_" for c in "".join(extra)) if extra else "") + ".so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", *extra, "-I", _HERE,
                        os.path.join(_HERE, "emu_main.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.emu_create.restype = C.c_void_p
        L.emu_create.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
        L.emu_destroy.argtypes = [C.c_void_p]
        L.emu_type_id.argtypes = [C.c_void_p, C.c_char_p]
        L.emu_slot_id.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
        L.emu_load.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_size_t]
        L.emu_publish.argtypes = [C.c_void_p]
        L.emu_stat.restype = C.c_uint64
        L.emu_stat.argtypes = [C.c_void_p, C.c_int]
        L.emu_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(Opts), C.c_int]
        L.emu_lookup_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(Opts), C.c_uint64,
                                       C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
        L.emu_set_shard.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.emu_shard_route.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.emu_shard_pass.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(Opts), C.POINTER(C.c_uint64)]
        L.emu_shard_fold.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int]
        L.emu_unroute.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.emu_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_size_t]
        L.emu_journal_start.argtypes = [C.c_void_p]
        L.emu_merge_and_verify.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        _LIB = L
    return _LIB


UPDATE_DTYPE = np.dtype([("res", "<u4"), ("subj", "<u4"), ("rel", "<u2"), ("stype", "<u2"), ("srel", "<u2"),
                         ("flags", "<u2"), ("expires_at", "<u4"), ("op", "<u4")])


class EmuEngine:
    """Same surface as zgpu.Engine / oracle.pyoracle.Oracle where the workload generators need it."""

    def __init__(self, schema: str, shard_rank: int = 0, shard_count: int = 1):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}  # (type, name) -> id, for string-driven tests
        self.shard_opts = default_opts()
        if shard_count > 1:
            self._L.emu_set_shard(self._h, shard_rank, shard_count)

    # the four device-resident shard calls of zgpu.Engine, over host memory (pointers = CPU tensor data_ptr())
    def shard_route_dev(self, d_items, n, level, n_dest, d_routed, d_src):
        counts = (C.c_uint64 * n_dest)()
        if self._L.emu_shard_route(self._h, d_items or None, n, level, n_dest, d_routed or None, d_src or None, counts):
            raise RuntimeError("emu_shard_route failed")
        return [int(c) for c in counts]

    def shard_pass_dev(self, d_queries, n, level):
        ns = C.c_uint64(0)
        rc = self._L.emu_shard_pass(self._h, d_queries or None, n, level, C.byref(self.shard_opts), C.byref(ns))
        if rc:
            raise RuntimeError(f"emu_shard_pass rc={rc}")
        return ns.value

    def shard_fold_dev(self, level, d_child_vals, d_src, n_sub, d_out, final_codes):
        if self._L.emu_shard_fold(self._h, level, d_child_vals or None, d_src or None, n_sub, d_out or None, 1 if final_codes else 0):
            raise RuntimeError("emu_shard_fold failed")

    def shard_unroute_dev(self, d_src, d_val, n, d_out):
        if self._L.emu_unroute(self._h, d_src or None, d_val or None, n, d_out or None):
            raise RuntimeError("emu_unroute failed")

    def close(self):
        if getattr(self, "_h", None):
            self._L.emu_destroy(self._h)
            self._h = None

    __del__ = close

    def type_id(self, name):
        return self._L.emu_type_id(self._h, name.encode())

    def slot_id(self, type_name, rel):
        return self._L.emu_slot_id(self._h, self.type_id(type_name), rel.encode())

    def load_tuples(self, t, expires=None):
        t = np.ascontiguousarray(t, dtype=TUPLE_DTYPE)
        ex = None if expires is None else np.ascontiguousarray(expires, dtype=np.uint32)
        err = C.create_string_buffer(512)
        if self._L.emu_load(self._h, t.ctypes.data, None if ex is None else ex.ctypes.data, t.size, err, 512):
            raise RuntimeError(err.value.decode())

    def add_bulk(self, type_name, rel, subj_type, res, subj, srel=None, wildcard=False):
        res = np.ascontiguousarray(res, dtype=np.uint32)
        t = np.zeros(res.size, dtype=TUPLE_DTYPE)
        t["res"] = res
        t["subj"] = 0 if wildcard else np.ascontiguousarray(subj, dtype=np.uint32)
        t["rel"] = self.slot_id(type_name, rel)
        t["stype"] = self.type_id(subj_type)
        t["srel"] = SREL_WILDCARD if wildcard else (SREL_NONE if srel is None else self.slot_id(subj_type, srel))
        self.load_tuples(t)

    def publish(self):
        if self._L.emu_publish(self._h):
            raise RuntimeError("emu_publish failed")
        self._L.emu_journal_start(self._h)

    def apply_updates(self, ups):
        u = np.ascontiguousarray(ups, dtype=UPDATE_DTYPE)
        err = C.create_string_buffer(512)
        if self._L.emu_apply(self._h, u.ctypes.data, u.size, err, 512):
            raise RuntimeError(err.value.decode())

    def merge_and_verify(self) -> int:
        """Incremental publish under the emulator, then every array against a fresh host build. 0 = identical,
        1 = needs a rebuild (layout changed); raises on a mismatch."""
        err = C.create_string_buffer(512)
        rc = self._L.emu_merge_and_verify(self._h, err, 512)
        if rc < 0:
            raise RuntimeError(f"merge rc={rc}: {err.value.decode()}")
        if rc == 1:
            self.publish()
        return rc

    def check_bulk(self, items, opts=None, count=False):
        items = np.ascontiguousarray(items, dtype=CHECK_DTYPE)
        out = np.zeros(items.size, dtype=np.uint8)
        o = opts or default_opts()
        rc = self._L.emu_check(self._h, items.ctypes.data, items.size, out.ctypes.data, C.byref(o), 1 if count else 0)
        if rc:
            raise RuntimeError(f"emu_check rc={rc}")
        return out

    def stat(self, name):
        return self._L.emu_stat(self._h, ["alg_bytes", "spills", "memo_batches", "passes", "splits", "flags"].index(name))

    def lookup_batch(self, reqs, opts=None, batch_cap=1 << 16):
        """reqs: [(res_type_id, perm_slot, stype_id, subj, srel_slot)] -> list of id arrays (or None on EDEPTH)."""
        K = len(reqs)
        rts = np.array([r[0] for r in reqs], dtype=np.uint16)
        protos = np.zeros(K, dtype=CHECK_DTYPE)
        for i, r in enumerate(reqs):
            protos["perm"][i], protos["stype"][i], protos["subj"][i], protos["srel"][i] = r[1], r[2], r[3], r[4]
        cap = 1 << 20
        out = np.zeros(cap, dtype=np.uint32)
        counts = np.zeros(K, dtype=np.uint64)
        rcs = np.zeros(K, dtype=np.int32)
        o = opts or default_opts()
        rc = self._L.emu_lookup_batch(self._h, rts.ctypes.data, protos.ctypes.data, K, C.byref(o), batch_cap, out.ctypes.data, cap,
                                      counts.ctypes.data, rcs.ctypes.data)
        if rc:
            raise RuntimeError(f"emu_lookup_batch rc={rc}")
        res, off = [], 0
        for i in range(K):
            res.append(None if rcs[i] else out[off:off + int(counts[i])].copy())
            off += int(counts[i])
        return res

    # ---- string-driven helpers (randgen relationships "type:id#rel@stype:sid[#srel]") ----
    def _id(self, t, name, create):
        key = (t, name)
        if key not in self._names:
            if not create:
                return None
            self._names[key] = sum(1 for k in self._names if k[0] == t)
        return self._names[key]

    def write_rels(self, rels, split_rel):
        t = np.zeros(len(rels), dtype=TUPLE_DTYPE)
        for i, r in enumerate(rels):
            rt, rid, rel, st, sid, srel = split_rel(r)
            t["rel"][i] = self.slot_id(rt, rel)
            t["stype"][i] = self.type_id(st)
            t["res"][i] = self._id(rt, rid, True)
            if sid == "*":
                t["srel"][i], t["subj"][i] = SREL_WILDCARD, 0
            else:
                t["srel"][i] = self.slot_id(st, srel) if srel else SREL_NONE
                t["subj"][i] = self._id(st, sid, True)
        self.load_tuples(t)

    def items_from_strings(self, checks, split_rel):
        items = np.zeros(len(checks), dtype=CHECK_DTYPE)
        for i, q in enumerate(checks):
            rt, rid, perm, st, sid, srel = split_rel(q)
            items["perm"][i] = self.slot_id(rt, perm) & 0xFFFF
            items["stype"][i] = self.type_id(st)
            items["srel"][i] = (self.slot_id(st, srel) & 0xFFFF) if srel else SREL_NONE
            if srel and self.slot_id(st, srel) < 0:
                items["perm"][i] = 0xFFFF  # unknown subject relation: an invalid item, as zg_resolve_checks makes it
            r, u = self._id(rt, rid, False), self._id(st, sid, False)
            items["res"][i] = 0xFFFFFFFF if r is None else r
            items["subj"][i] = u if u is not None else (0xFFFFFFFF if (r is None and rt == st and rid == sid) else 0xFFFFFFFE)
        return items
