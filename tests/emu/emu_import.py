"""ctypes binding of tests/emu/emu_import.cc: zg_import_relationships' kernels (csrc/import.cuh) run by the CPU SIMT
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

TUPLE_DTYPE = np.dtype([("res", "<u4"), ("subj", "<u4"), ("rel", "<u2"), ("stype", "<u2"), ("srel", "<u2"),
                        ("flags", "<u2")])
TAG_MASK = 0xFFFFFF0000000000
NONE = (1 << 64) - 1


class Opts(C.Structure):
    _fields_ = [("tag_mask", C.c_uint64), ("grid", C.c_uint32), ("threads", C.c_uint32)]


class Group(C.Structure):
    _fields_ = [("res_type", C.c_char_p), ("relation", C.c_char_p), ("subj_type", C.c_char_p), ("subj_rel", C.c_char_p),
                ("res_ids", C.c_char_p), ("res_off", C.c_void_p), ("subj_ids", C.c_char_p), ("subj_off", C.c_void_p),
                ("n", C.c_uint64)]


def opts(tag_filter=True, grid=2, threads=64) -> Opts:
    """The product's tag filter by default; tag_filter=False makes every probe compare bytes (emulator only)."""
    return Opts(TAG_MASK if tag_filter else 0, grid, threads)


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_import.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_import.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("import.cuh", "ingress.cuh", "hash_bytes.h", "schema.cc", "schema.h",
                                             "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_import.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.emu_imp_create.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
        L.emu_imp_create.restype = C.c_void_p
        L.emu_imp_destroy.argtypes = [C.c_void_p]
        L.emu_imp_type_id.argtypes = [C.c_void_p, C.c_char_p]
        L.emu_imp_slot_id.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
        L.emu_imp_intern.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.emu_imp_load.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.emu_imp_arena.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint64]
        L.emu_imp_arena.restype = C.c_uint64
        L.emu_imp_run.argtypes = [C.c_void_p, C.POINTER(Group), C.c_uint64, C.POINTER(Opts), C.POINTER(C.c_uint64),
                                  C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_void_p]
        _LIB = L
    return _LIB


def pack(ids, pad=0):
    """[str | bytes] -> (blob, offsets): the blob starts with `pad` filler bytes, so the ids sit at other alignments."""
    enc = [i.encode() if isinstance(i, str) else bytes(i) for i in ids]
    off = np.zeros(len(enc) + 1, dtype=np.uint32)
    np.cumsum([len(x) for x in enc], out=off[1:])
    return b"#" * pad + b"".join(enc), off + pad


class EmuImport:
    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_imp_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.emu_imp_destroy(self._h)
            self._h = None

    def type_id(self, name):
        return self._L.emu_imp_type_id(self._h, name.encode())

    def slot_id(self, type_name, rel):
        return self._L.emu_imp_slot_id(self._h, self.type_id(type_name), rel.encode())

    def intern_packed(self, type_name, ids) -> np.ndarray:
        blob, off = pack(ids)
        out = np.empty(len(ids), dtype=np.uint32)
        assert self._L.emu_imp_intern(self._h, self.type_id(type_name), blob or b"\0", off.ctypes.data, len(ids),
                                      out.ctypes.data) == 0
        return out

    def load_tuples(self, t: np.ndarray):
        t = np.ascontiguousarray(t, dtype=TUPLE_DTYPE)
        assert self._L.emu_imp_load(self._h, t.ctypes.data, t.size) == 0

    def arena(self, type_name) -> bytes:
        t = self.type_id(type_name)
        n = self._L.emu_imp_arena(self._h, t, None, 0)
        buf = C.create_string_buffer(max(n, 1))
        self._L.emu_imp_arena(self._h, t, buf, n)
        return buf.raw[:n]

    def run(self, groups, o=None, pads=None):
        """groups as Engine.import_relationships takes them (expirations ignored) -> (bad, dup, n_new, tuples):
        the smallest call positions of a malformed id / a duplicate (None: none), the new names, and on success the
        tuples in call order (committed to the store)."""
        arr = (Group * max(len(groups), 1))()
        keep = []
        n = 0
        for i, (rt, rel, st, srel, res, subj, _ex) in enumerate(groups):
            pr, ps = (pads[i] if pads else (0, 0))
            rb, ro = pack(res, pr)
            sb, so = pack(subj, ps)
            keep.append((rb, ro, sb, so))
            arr[i] = Group(rt.encode(), rel.encode(), st.encode(), (srel or "").encode(), rb or b"\0", ro.ctypes.data,
                           sb or b"\0", so.ctypes.data, len(res))
            n += len(res)
        bad, dup, nn = C.c_uint64(), C.c_uint64(), C.c_uint64()
        out = np.zeros(max(n, 1), dtype=TUPLE_DTYPE)
        rc = self._L.emu_imp_run(self._h, arr, len(groups), C.byref(o or opts()), C.byref(bad), C.byref(dup),
                                 C.byref(nn), out.ctypes.data)
        assert rc == 0, rc
        fix = lambda v: None if v == NONE else int(v)  # noqa: E731
        return fix(bad.value), fix(dup.value), int(nn.value), out[:n]
