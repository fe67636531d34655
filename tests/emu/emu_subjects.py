"""ctypes binding of tests/emu/emu_subjects.cc: LookupSubjects' launch sequence (forward walk, fallback fill, the
no-wildcards verification) run by the CPU SIMT emulator over the product's kernels.cuh. TEST INFRASTRUCTURE ONLY --
never imported by the product, never linked into libzgpu.so. The library also carries every entry point of the
emulator driver (emu_main.cc is compiled into it), so EmuEngine below is emu.EmuEngine over this library."""
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
           "emu_lookup_batch", "emu_set_shard", "emu_shard_route", "emu_shard_pass", "emu_shard_fold", "emu_unroute",
           "emu_apply", "emu_journal_start", "emu_merge_and_verify"]


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_subjects.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_subjects.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_subjects.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        base = _emu.lib()  # the driver's signatures, declared once in emu.py
        for name in _DRIVER:
            fn, ref = getattr(L, name), getattr(base, name)
            fn.argtypes, fn.restype = ref.argtypes, ref.restype
        L.emu_lookup_subjects.argtypes = [C.c_void_p, C.c_uint16, C.c_uint32, C.c_uint16, C.c_uint16, C.c_uint16, C.c_int,
                                          C.c_int, C.c_uint64, C.POINTER(_emu.Opts), C.c_void_p, C.c_uint64, C.c_void_p]
        _LIB = L
    return _LIB


class EmuEngine(_emu.EmuEngine):
    """emu.EmuEngine driven through this library, plus LookupSubjects."""

    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = default_opts()

    def lookup_subjects_ids(self, res_type_id, res, perm, stype, srel=SREL_NONE, include_wildcard=True, force_fallback=False,
                            walk_cap=1 << 16, opts=None):
        """device.cu lookup_subjects under the emulator -> (concrete ids, wildcard entry present, excluded ids, info);
        raises RuntimeError("EDEPTH") when a subject cannot be decided."""
        cap = 1 << 20
        out = np.zeros(cap, dtype=np.uint32)
        info = np.zeros(5, dtype=np.uint64)
        o = opts or default_opts()
        rc = self._L.emu_lookup_subjects(self._h, res_type_id, int(res), perm, stype, srel, 1 if include_wildcard else 0,
                                         1 if force_fallback else 0, walk_cap, C.byref(o), out.ctypes.data, cap, info.ctypes.data)
        if rc == -9:
            raise RuntimeError("EDEPTH")
        if rc:
            raise RuntimeError(f"emu_lookup_subjects rc={rc}")
        nc, nx = int(info[0]), int(info[1])
        return out[:nc].copy(), bool(info[2]), out[nc:nc + nx].copy(), {"fell_back": bool(info[3]), "verified": int(info[4])}

    def lookup_subjects(self, res_type, res_id, perm, subj_type, subj_rel="", include_wildcard=True, **kw):
        """The same by names (write_rels interning) -> (concrete names, wildcard, excluded names, info)."""
        rid = self._id(res_type, res_id, False)
        if rid is None:
            return [], False, [], {}
        sr = self.slot_id(subj_type, subj_rel) if subj_rel else SREL_NONE
        ids, wild, ex, info = self.lookup_subjects_ids(self.type_id(res_type), rid, self.slot_id(res_type, perm),
                                                       self.type_id(subj_type), sr, include_wildcard, **kw)
        names = {i: n for (t, n), i in self._names.items() if t == subj_type}
        return [names[int(i)] for i in ids], wild, [names[int(i)] for i in ex], info

