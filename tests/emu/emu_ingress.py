"""ctypes binding of tests/emu/emu_ingress.cc: the device-ingress kernels (csrc/ingress.cuh) run by the CPU SIMT
emulator against a real Store. TEST INFRASTRUCTURE ONLY -- never imported by the product, never linked into
libzgpu.so."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None

CHECK_DTYPE = np.dtype([("res", "<u4"), ("subj", "<u4"), ("perm", "<u2"), ("stype", "<u2"), ("srel", "<u2"),
                        ("flags", "<u2")])
TAG_MASK = 0xFFFFFF0000000000


class Opts(C.Structure):
    _fields_ = [("tag_mask", C.c_uint64), ("min_table", C.c_uint64), ("grid", C.c_uint32), ("threads", C.c_uint32)]


def opts(tag_filter=True, min_table=1024, grid=2, threads=64) -> Opts:
    """The product's settings by default; tag_filter=False / a small min_table are the emulator-only switches."""
    return Opts(TAG_MASK if tag_filter else 0, min_table, grid, threads)


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_ingress.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_ingress.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("ingress.cuh", "hash_bytes.h", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_ingress.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.emu_ing_create.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
        L.emu_ing_create.restype = C.c_void_p
        L.emu_ing_destroy.argtypes = [C.c_void_p]
        L.emu_ing_type_id.argtypes = [C.c_void_p, C.c_char_p]
        L.emu_ing_intern.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.emu_ing_load.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.emu_ing_resolve.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(Opts)]
        L.emu_ing_counters.argtypes = [C.c_void_p, C.c_void_p]
        L.emu_guarded_alloc.argtypes = [C.c_size_t]
        L.emu_guarded_alloc.restype = C.c_void_p
        _LIB = L
    return _LIB


def pack(ids):
    enc = [i.encode() if isinstance(i, str) else bytes(i) for i in ids]
    off = np.zeros(len(enc) + 1, dtype=np.uint32)
    np.cumsum([len(x) for x in enc], out=off[1:])
    return b"".join(enc), off


def guarded(data: bytes):
    """A copy of data whose last byte sits just before a PROT_NONE page -> (address, keep-alive)."""
    p = lib().emu_guarded_alloc(max(len(data), 1))
    assert p, "mmap failed"
    C.memmove(p + max(len(data), 1) - len(data), data, len(data))
    return p + max(len(data), 1) - len(data)


class EmuIngress:
    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_ing_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.emu_ing_destroy(self._h)
            self._h = None

    def type_id(self, name):
        return self._L.emu_ing_type_id(self._h, name.encode())

    def intern_packed(self, type_name, ids) -> np.ndarray:
        blob, off = pack(ids)
        out = np.empty(len(ids), dtype=np.uint32)
        rc = self._L.emu_ing_intern(self._h, self.type_id(type_name), blob or b"\0", off.ctypes.data, len(ids), out.ctypes.data)
        assert rc == 0, rc
        return out

    def load_tuples(self, t: np.ndarray):
        assert self._L.emu_ing_load(self._h, t.ctypes.data, t.size) == 0

    def resolve_ptr(self, res_type, relation, subj_type, subj_rel, res_ids, res_off, subj_ids, subj_off, n, o=None):
        """Raw pointers (ints or bytes) -> (rc, items)."""
        out = np.zeros(n, dtype=CHECK_DTYPE)
        rc = self._L.emu_ing_resolve(self._h, res_type.encode(), relation.encode(), subj_type.encode(),
                                     (subj_rel or "").encode(), res_ids, res_off, subj_ids, subj_off, n, out.ctypes.data,
                                     C.byref(o or opts()))
        return rc, out

    def resolve_packed(self, res_type, relation, subj_type, res_ids, subjects, subj_rel="", o=None) -> np.ndarray:
        """Engine.resolve_checks_packed's arguments: `subjects` is one id (str) or a list of n ids."""
        blob, off = pack(res_ids)
        if isinstance(subjects, (str, bytes)):
            sblob, soff = (subjects.encode() if isinstance(subjects, str) else subjects), None
        else:
            sblob, so = pack(subjects)
            soff, sblob = so.ctypes.data, sblob or b"\0"
        rc, out = self.resolve_ptr(res_type, relation, subj_type, subj_rel, blob or b"\0", off.ctypes.data, sblob, soff,
                                   len(res_ids), o)
        assert rc == 0, rc
        return out

    def counters(self) -> dict:
        c = np.zeros(4, dtype=np.uint64)
        self._L.emu_ing_counters(self._h, c.ctypes.data)
        return {"names": int(c[0]), "sync_uploads": int(c[1]), "rebuilds": int(c[2]), "items_resolved": int(c[3])}
