"""ctypes binding of tests/emu/emu_shard_subjects.cc: the sharded LookupSubjects round (device.cu
Device::shard_subjects_* and shard_pass_nowild_dev) run by the CPU SIMT emulator over the product's kernels.cuh. TEST
INFRASTRUCTURE ONLY -- never imported by the product, never linked into libzgpu.so. The library also carries every entry
point of the emulator driver (emu_main.cc is compiled into it), so EmuEngine below is emu.EmuEngine over this library,
with the shard_pass_nowild_dev and shard_subjects_*_dev methods of zgpu.Engine: dist.DeviceShardedLookup drives
emulated shards with CPU tensors."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import emu as _emu
from emu import CHECK_DTYPE, SREL_NONE, SREL_WILDCARD, TUPLE_DTYPE, default_opts  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None
_DRIVER = ["emu_create", "emu_destroy", "emu_type_id", "emu_slot_id", "emu_load", "emu_publish", "emu_stat", "emu_check",
           "emu_set_shard", "emu_shard_route", "emu_shard_pass", "emu_shard_fold", "emu_unroute", "emu_apply",
           "emu_journal_start", "emu_merge_and_verify"]


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_shard_subjects.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_shard_subjects.cc", "emu_subjects.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        tmp = f"{so}.{os.getpid()}.tmp"  # concurrent test processes must never load a half-written library
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_shard_subjects.cc"), os.path.join(_CSRC, "schema.cc"),
                        os.path.join(_CSRC, "store.cc"), "-o", tmp], check=True)
        os.replace(tmp, so)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        base = _emu.lib()  # the driver's signatures, declared once in emu.py
        for name in _DRIVER:
            fn, ref = getattr(L, name), getattr(base, name)
            fn.argtypes, fn.restype = ref.argtypes, ref.restype
        vp, u64, pu64 = C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)
        L.emu_ss_release.argtypes = [vp]
        L.emu_ss_pass_nowild.argtypes = [vp, vp, u64, C.c_int, C.POINTER(_emu.Opts), pu64]
        L.emu_ss_begin.argtypes = [vp, vp, vp, vp, vp, C.c_uint32, u64, vp, pu64]
        L.emu_ss_expand.argtypes = [vp, vp, u64, C.c_uint32, vp, vp, C.POINTER(C.c_int)]
        L.emu_ss_admit.argtypes = [vp, vp, u64, vp, pu64]
        L.emu_ss_candidates.argtypes = [vp, C.c_int, vp, u64, pu64]
        L.emu_ss_verdicts.argtypes = [vp, vp, u64, pu64, pu64]
        L.emu_ss_nowild.argtypes = [vp, vp, u64, u64, u64, vp, u64, pu64]
        L.emu_ss_route.argtypes = [vp, vp, u64, C.c_uint32, vp, vp]
        L.emu_ss_finish.argtypes = [vp, vp, u64, vp, vp, vp]
        L.emu_ss_replica_marks.argtypes = [vp, C.c_uint16, C.c_uint32, C.c_uint16, C.c_uint16, C.c_uint16, u64, pu64]
        _LIB = L
    return _LIB


class EmuEngine(_emu.EmuEngine):
    """emu.EmuEngine driven through this library, plus the sharded LookupSubjects calls."""

    def __init__(self, schema: str, shard_rank: int = 0, shard_count: int = 1):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = default_opts()
        if shard_count > 1:
            self._L.emu_set_shard(self._h, shard_rank, shard_count)

    def close(self):
        if getattr(self, "_h", None):
            self._L.emu_ss_release(self._h)
        super().close()

    __del__ = close

    def _ck(self, rc, what):
        if rc:
            raise RuntimeError(f"{what} rc={rc}")

    def shard_pass_nowild_dev(self, d_queries, n, level):
        ns = C.c_uint64(0)
        self._ck(self._L.emu_ss_pass_nowild(self._h, d_queries or None, n, level, C.byref(self.shard_opts), C.byref(ns)),
                 "emu_ss_pass_nowild")
        return ns.value

    def shard_subjects_begin_dev(self, res_types, reqs, options, home, walk_cap, d_front):
        rt = np.ascontiguousarray(res_types, dtype=np.uint16)
        rq = np.ascontiguousarray(reqs, dtype=CHECK_DTYPE)
        op = np.ascontiguousarray(options, dtype=np.uint32)
        hm = np.ascontiguousarray(home, dtype=np.uint8)
        n = C.c_uint64(0)
        self._ck(self._L.emu_ss_begin(self._h, rt.ctypes.data, rq.ctypes.data, op.ctypes.data, hm.ctypes.data, rq.size, walk_cap,
                                      d_front or None, C.byref(n)), "emu_ss_begin")
        return n.value

    def shard_subjects_expand_dev(self, d_front, n_in, n_dest, d_routed):
        counts = (C.c_uint64 * n_dest)()
        ovf = C.c_int(0)
        self._ck(self._L.emu_ss_expand(self._h, d_front or None, n_in, n_dest, d_routed or None, counts, C.byref(ovf)),
                 "emu_ss_expand")
        return [int(c) for c in counts], bool(ovf.value)

    def shard_subjects_admit_dev(self, d_in, n_in, d_next):
        n = C.c_uint64(0)
        self._ck(self._L.emu_ss_admit(self._h, d_in or None, n_in, d_next or None, C.byref(n)), "emu_ss_admit")
        return n.value

    def shard_subjects_candidates_dev(self, exhaustive, d_items, cap):
        n = C.c_uint64(0)
        self._ck(self._L.emu_ss_candidates(self._h, 1 if exhaustive else 0, d_items or None, cap, C.byref(n)), "emu_ss_candidates")
        return n.value

    def shard_subjects_verdicts_dev(self, d_codes, n):
        g, f = C.c_uint64(0), C.c_uint64(0)
        self._ck(self._L.emu_ss_verdicts(self._h, d_codes or None, n, C.byref(g), C.byref(f)), "emu_ss_verdicts")
        return g.value, f.value

    def shard_subjects_nowild_dev(self, d_codes, n, granted, failed, d_items, cap):
        m = C.c_uint64(0)
        self._ck(self._L.emu_ss_nowild(self._h, d_codes or None, n, granted, failed, d_items or None, cap, C.byref(m)),
                 "emu_ss_nowild")
        return m.value

    def shard_subjects_route_dev(self, d_codes, n, n_dest, d_routed):
        counts = (C.c_uint64 * n_dest)()
        self._ck(self._L.emu_ss_route(self._h, d_codes or None, n, n_dest, d_routed or None, counts), "emu_ss_route")
        return [int(c) for c in counts]

    def shard_subjects_finish_dev(self, d_keys, n, d_ids, k):
        listed, excluded = (C.c_uint64 * max(k, 1))(), (C.c_uint64 * max(k, 1))()
        self._ck(self._L.emu_ss_finish(self._h, d_keys or None, n, d_ids or None, listed, excluded), "emu_ss_finish")
        return [int(listed[i]) for i in range(k)], [int(excluded[i]) for i in range(k)]

    def replica_marks(self, res_type_id, res, perm, stype, srel=SREL_NONE, walk_cap=1 << 16):
        """Objects a replica's forward walk marks for this lookup (this engine must not be sharded)."""
        n = C.c_uint64(0)
        self._ck(self._L.emu_ss_replica_marks(self._h, res_type_id, int(res), perm, stype, srel, walk_cap, C.byref(n)),
                 "emu_ss_replica_marks")
        return n.value
