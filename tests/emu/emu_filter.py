"""ctypes binding of tests/emu/emu_filter.cc: the relationship-filter kernels (csrc/filter.cuh) and their plan run by
the CPU SIMT emulator, beside Store::match over the same store. TEST INFRASTRUCTURE ONLY -- never imported by the
product, never linked into libzgpu.so. The library also carries every entry point of the emulator driver (emu_main.cc
is compiled into it), so EmuEngine below is emu.EmuEngine over this library."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import emu as _emu
from emu import SREL_NONE, SREL_WILDCARD, TUPLE_DTYPE  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None
_DRIVER = ["emu_create", "emu_destroy", "emu_type_id", "emu_slot_id", "emu_load", "emu_publish", "emu_stat", "emu_apply",
           "emu_journal_start", "emu_merge_and_verify"]


class Filter(C.Structure):
    _fields_ = [("res_type", C.c_int32), ("rel", C.c_int32), ("subj_type", C.c_int32), ("has_res", C.c_uint32),
                ("res", C.c_uint32), ("has_subj", C.c_uint32), ("subj", C.c_uint32), ("subj_wildcard", C.c_uint32),
                ("has_srel", C.c_uint32), ("srel", C.c_uint32)]


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_filter.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_filter.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("filter.cuh", "kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_filter.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
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
        L.emu_filter_host.restype = C.c_uint64
        L.emu_filter_host.argtypes = [C.c_void_p, C.POINTER(Filter), C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64]
        L.emu_filter_device.argtypes = [C.c_void_p, C.POINTER(Filter), C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        _LIB = L
    return _LIB


def _canon(t, ex):
    """Records and expirations as a sorted list of tuples: the kernels append in no particular order."""
    return sorted(zip(t["res"].tolist(), t["subj"].tolist(), t["rel"].tolist(), t["stype"].tolist(), t["srel"].tolist(),
                      t["flags"].tolist(), ex.tolist()))


class EmuEngine(_emu.EmuEngine):
    """emu.EmuEngine driven through this library, plus the relationship filters."""

    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = _emu.default_opts()

    def resolve(self, f: dict):
        """A filter of names -> Filter of ids the way capi.cu resolve_filter does it, or None when it names an object or
        subject relation that does not exist (nothing matches)."""
        x = Filter(-1, -1, -1, 0, 0, 0, 0, 0, 0, SREL_NONE)
        if f.get("res_type"):
            x.res_type = self.type_id(f["res_type"])
        if f.get("res_id"):
            i = self._id(f["res_type"], f["res_id"], False)
            if i is None:
                return None
            x.has_res, x.res = 1, i
        if f.get("rel"):
            x.rel = self.slot_id(f["res_type"], f["rel"])
        if f.get("subj_type"):
            x.subj_type = self.type_id(f["subj_type"])
        if f.get("subj_id"):
            if f["subj_id"] == "*":
                x.subj_wildcard = 1
            else:
                i = self._id(f["subj_type"], f["subj_id"], False)
                if i is None:
                    return None
                x.has_subj, x.subj = 1, i
        if f.get("subj_rel"):
            x.has_srel = 1
            if f["subj_rel"] != "...":
                s = self.slot_id(f["subj_type"], f["subj_rel"])
                if s < 0:
                    return None
                x.srel = s
        return x

    def host_match(self, x: Filter, now=0, cap=1 << 16):
        t, ex = np.zeros(cap, dtype=TUPLE_DTYPE), np.zeros(cap, dtype=np.uint32)
        n = int(self._L.emu_filter_host(self._h, C.byref(x), now, t.ctypes.data, ex.ctypes.data, cap))
        assert n <= cap
        return _canon(t[:n], ex[:n])

    def device_match(self, x: Filter, now=0, grid=2, max_sel=64, emit=True, cap=1 << 16):
        """-> (records or None for a count, info dict)."""
        t, ex = np.zeros(cap, dtype=TUPLE_DTYPE), np.zeros(cap, dtype=np.uint32)
        info = np.zeros(4, dtype=np.uint64)
        rc = self._L.emu_filter_device(self._h, C.byref(x), now, grid, max_sel, 1 if emit else 0, t.ctypes.data, ex.ctypes.data,
                                       cap, info.ctypes.data)
        if rc:
            raise RuntimeError(f"emu_filter_device rc={rc}")
        d = {"count": int(info[0]), "emitted": int(info[1]), "shape": int(info[2]), "launches": int(info[3])}
        return (_canon(t[:d["emitted"]], ex[:d["emitted"]]) if emit else None), d
