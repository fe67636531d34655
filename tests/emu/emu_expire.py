"""ctypes binding of tests/emu/emu_expire.cc: the collection scan (csrc/filter.cuh filter_expired_kernel) and its plan
run by the CPU SIMT emulator, beside Store::expired over the same store. TEST INFRASTRUCTURE ONLY -- never imported by
the product, never linked into libzgpu.so. The library also carries every entry point of the emulator driver
(emu_main.cc is compiled into it), so EmuEngine below is emu.EmuEngine over this library."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import emu as _emu
import emu_filter
from emu import SREL_NONE, SREL_WILDCARD, TUPLE_DTYPE  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_expire.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_expire.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("filter.cuh", "kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_expire.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        base = _emu.lib()  # the driver's signatures, declared once in emu.py
        for name in emu_filter._DRIVER:
            fn, ref = getattr(L, name), getattr(base, name)
            fn.argtypes, fn.restype = ref.argtypes, ref.restype
        L.emu_expired_host.restype = C.c_uint64
        L.emu_expired_host.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64]
        L.emu_expired_device.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_uint64, C.c_void_p]
        _LIB = L
    return _LIB


class EmuEngine(_emu.EmuEngine):
    """emu.EmuEngine driven through this library, plus the collection scan."""

    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = _emu.default_opts()

    def host_expired(self, before, cap=1 << 16):
        t, ex = np.zeros(cap, dtype=TUPLE_DTYPE), np.zeros(cap, dtype=np.uint32)
        n = int(self._L.emu_expired_host(self._h, before, t.ctypes.data, ex.ctypes.data, cap))
        assert n <= cap
        return emu_filter._canon(t[:n], ex[:n])

    def device_expired(self, before, grid=2, max_sel=64, emit=True, poison=True, cap=1 << 16):
        """-> (records or None for a count, info dict)."""
        t, ex = np.zeros(cap, dtype=TUPLE_DTYPE), np.zeros(cap, dtype=np.uint32)
        info = np.zeros(4, dtype=np.uint64)
        rc = self._L.emu_expired_device(self._h, before, grid, max_sel, 1 if emit else 0, 1 if poison else 0,
                                        t.ctypes.data, ex.ctypes.data, cap, info.ctypes.data)
        if rc:
            raise RuntimeError(f"emu_expired_device rc={rc}")
        d = {"count": int(info[0]), "emitted": int(info[1]), "selected": int(info[2]), "launches": int(info[3])}
        return (emu_filter._canon(t[:d["emitted"]], ex[:d["emitted"]]) if emit else None), d
