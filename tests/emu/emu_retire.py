"""ctypes binding of tests/emu/emu_retire.cc: the mention scan (csrc/filter.cuh mention_scan_kernel) and its plan run
by the CPU SIMT emulator, beside Store::mentioned over the same store. TEST INFRASTRUCTURE ONLY -- never imported by
the product, never linked into libzgpu.so. The library also carries every entry point of the emulator driver
(emu_main.cc is compiled into it), so EmuEngine below is emu.EmuEngine over this library."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import emu as _emu
import emu_filter
from emu import SREL_NONE, SREL_WILDCARD, TUPLE_DTYPE, UPDATE_DTYPE  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_retire.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_retire.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("filter.cuh", "kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_retire.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
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
        L.emu_mention_host.restype = C.c_uint64
        L.emu_mention_host.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64]
        L.emu_mention_device.restype = C.c_uint64
        L.emu_mention_device.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                         C.c_uint64, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


class EmuEngine(_emu.EmuEngine):
    """emu.EmuEngine driven through this library, plus the mention scan."""

    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = _emu.default_opts()

    def host_mentions(self, type_id, cap=1 << 16):
        out = np.zeros(cap, dtype=np.uint32)
        n = int(self._L.emu_mention_host(self._h, type_id, out.ctypes.data, cap))
        assert n <= cap
        return out[:n]

    def device_mentions(self, n_types, rank=0, count=1, grid=2, max_types=64, cap=1 << 16):
        """-> ([bitmap words of type t for t < n_types], launches)."""
        out = np.zeros(cap, dtype=np.uint32)
        word0 = np.zeros(n_types + 1, dtype=np.uint64)
        launches = np.zeros(1, dtype=np.uint64)
        n = int(self._L.emu_mention_device(self._h, rank, count, grid, max_types, out.ctypes.data, cap,
                                           word0.ctypes.data, launches.ctypes.data))
        if n == 0:
            raise RuntimeError("emu_mention_device: not published or cap too small")
        assert int(word0[n_types]) == n
        return [out[int(word0[t]):int(word0[t + 1])] for t in range(n_types)], int(launches[0])
