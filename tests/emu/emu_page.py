"""ctypes binding of tests/emu/emu_page.cc: the page kernels (csrc/filter.cuh page_*) and their host side (page_walk,
page_merge) run by the CPU SIMT emulator, beside Store::page over the same store. TEST INFRASTRUCTURE ONLY -- never
imported by the product, never linked into libzgpu.so. The library carries emu_filter.cc and the emulator driver, so
EmuEngine below is emu_filter.EmuEngine over this library."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import emu as _emu
import emu_filter as _flt
from emu_filter import Filter, SREL_NONE, SREL_WILDCARD, TUPLE_DTYPE  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_page.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_page.cc", "emu_filter.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("filter.cuh", "kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_page.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        base = _flt.lib()  # the driver's and the filter harness's signatures
        for name in _flt._DRIVER + ["emu_filter_host", "emu_filter_device"]:
            fn, ref = getattr(L, name), getattr(base, name)
            fn.argtypes, fn.restype = ref.argtypes, ref.restype
        L.emu_page_host.restype = C.c_uint64
        L.emu_page_host.argtypes = [C.c_void_p, C.POINTER(Filter), C.c_uint32, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p,
                                    C.c_void_p]
        L.emu_page_device.argtypes = [C.c_void_p, C.POINTER(Filter), C.c_uint32, C.c_int, C.c_void_p, C.c_uint64, C.c_uint32,
                                      C.c_void_p, C.c_void_p, C.c_void_p]
        L.emu_page_class_pos.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.emu_page_slot_type.argtypes = [C.c_void_p, C.c_int]
        _LIB = L
    return _LIB


def _rows(t, ex):
    return list(zip(t["res"].tolist(), t["subj"].tolist(), t["rel"].tolist(), t["stype"].tolist(), t["srel"].tolist(),
                    ex.tolist()))


class EmuEngine(_flt.EmuEngine):
    """emu_filter.EmuEngine driven through this library, plus pages."""

    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = _emu.default_opts()

    def key(self, row):
        """K of a row (res, subj, rel, stype, srel, ...), restated: (resource type, resource, class position, subject)."""
        res, subj, rel, stype, srel = row[:5]
        return (self._L.emu_page_slot_type(self._h, rel), res, self._L.emu_page_class_pos(self._h, rel, stype, srel),
                0 if srel == SREL_WILDCARD else subj)

    @staticmethod
    def _after(after):
        return (1, np.array(after, dtype=np.uint32)) if after is not None else (0, np.zeros(4, dtype=np.uint32))

    def host_page(self, x: Filter, want, now=0, after=None):
        """Store::page -> [(res, subj, rel, stype, srel, expires)] in page order."""
        has, a = self._after(after)
        t, ex = np.zeros(max(want, 1), dtype=TUPLE_DTYPE), np.zeros(max(want, 1), dtype=np.uint32)
        n = int(self._L.emu_page_host(self._h, C.byref(x), now, has, a.ctypes.data, want, t.ctypes.data, ex.ctypes.data))
        return _rows(t[:n], ex[:n])

    def device_page(self, x: Filter, want, now=0, after=None, grid=2):
        """-> (rows in the order the kernels wrote them, info dict)."""
        has, a = self._after(after)
        t, ex = np.zeros(max(want, 1), dtype=TUPLE_DTYPE), np.zeros(max(want, 1), dtype=np.uint32)
        info = np.zeros(5, dtype=np.uint64)
        rc = self._L.emu_page_device(self._h, C.byref(x), now, has, a.ctypes.data, want, grid, t.ctypes.data, ex.ctypes.data,
                                     info.ctypes.data)
        if rc:
            raise RuntimeError(f"emu_page_device rc={rc}")
        d = dict(zip(("records", "windows", "launches", "max_tiles", "scanned"), (int(v) for v in info)))
        return _rows(t[:d["records"]], ex[:d["records"]]), d
