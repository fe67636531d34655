"""ctypes binding of tests/emu/emu_expand.cc: ExpandPermissionTree's kernels (csrc/expand.cuh) and Device::expand's level
loop run by the CPU SIMT emulator. TEST INFRASTRUCTURE ONLY -- never imported by the product, never linked into
libzgpu.so. The library also carries every entry point of the emulator driver (emu_main.cc is compiled into it), so
EmuEngine below is emu.EmuEngine over this library."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import emu as _emu
from oracle.mini_oracle import parse_schema

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None
_DRIVER = ["emu_create", "emu_destroy", "emu_type_id", "emu_slot_id", "emu_load", "emu_publish", "emu_stat"]
NO_OBJECT = 0xFFFFFFFF
REQUEST_DTYPE = np.dtype([("perm", "<u2"), ("pad", "<u2"), ("res", "<u4")])
NODE_DTYPE = np.dtype([("request", "<u4"), ("parent", "<u4"), ("rank", "<u4"), ("object", "<u4"), ("slot", "<u2"),
                       ("op", "<u2"), ("n_subjects", "<u4"), ("subjects", "<u8")])
SUBJECT_DTYPE = np.dtype([("id", "<u4"), ("type", "<u2"), ("srel", "<u2")])


class CapError(Exception):
    """The trees pass the cap (ZG_ENOMEM)."""


def build() -> str:
    so = os.path.join(_HERE, "libzgemu_expand.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_expand.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("expand.cuh", "filter.cuh", "kernels.cuh", "delta.cuh", "schema.cc", "schema.h",
                                             "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _HERE,
                        os.path.join(_HERE, "emu_expand.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
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
        L.emu_expand.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p,
                                 C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p, C.c_uint64,
                                 C.POINTER(C.c_uint64), C.c_void_p]
        _LIB = L
    return _LIB


class EmuEngine(_emu.EmuEngine):
    """emu.EmuEngine driven through this library, plus ExpandPermissionTree."""

    def __init__(self, schema: str):
        self._L = lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = _emu.default_opts()
        self._slots = {}  # slot -> (type, name)
        defs = parse_schema(schema)
        self._tnames = {self.type_id(t): t for t in defs}
        for t, d in defs.items():
            for name in list(d["relations"]) + list(d["permissions"]):
                self._slots[self.slot_id(t, name)] = (t, name)

    def expand(self, requests, now=0, cap=1 << 26, threads=64):
        """requests: [(type, name, relation or permission)] (a name never written: a never-written object). Returns
        (one tree per request in the nesting of _lib.parse_expand_lines, or "EDEPTH"; info: levels, warps per job).
        Raises CapError."""
        reqs = np.zeros(len(requests), dtype=REQUEST_DTYPE)
        for i, (t, rid, perm) in enumerate(requests):
            oid = self._id(t, rid, False)
            reqs[i] = (self.slot_id(t, perm), 0, NO_OBJECT if oid is None else oid)
        status = np.zeros(max(len(reqs), 1), dtype=np.int32)
        info = np.zeros(2, dtype=np.uint64)
        ncap, scap = 1 << 12, 1 << 14
        while True:
            nodes, subj = np.zeros(ncap, dtype=NODE_DTYPE), np.zeros(scap, dtype=SUBJECT_DTYPE)
            nn, ns = C.c_uint64(0), C.c_uint64(0)
            rc = self._L.emu_expand(self._h, reqs.ctypes.data, len(reqs), now, cap, threads, status.ctypes.data,
                                    nodes.ctypes.data, ncap, C.byref(nn), subj.ctypes.data, scap, C.byref(ns),
                                    info.ctypes.data)
            if rc == -7:
                ncap, scap = max(ncap, nn.value), max(scap, ns.value)
                continue
            if rc == -8:
                raise CapError()
            assert rc == 0, rc
            break
        names = {(t, i): name for (t, name), i in self._names.items()}
        out = ["EDEPTH" if status[i] else None for i in range(len(requests))]
        built = []
        for nd in nodes[: nn.value]:
            t, rel = self._slots[int(nd["slot"])]
            obj = requests[int(nd["request"])][1] if nd["object"] == NO_OBJECT else names[(t, int(nd["object"]))]
            b = int(nd["subjects"])
            subs = []
            for x in subj[b: b + int(nd["n_subjects"])]:
                st = self._tnames[int(x["type"])]
                if x["srel"] == _emu.SREL_WILDCARD:
                    subs.append(f"{st}:*")
                else:
                    subs.append(f"{st}:{names[(st, int(x['id']))]}" +
                                ("" if x["srel"] == _emu.SREL_NONE else f"#{self._slots[int(x['srel'])][1]}"))
            n = {"op": "?UIXL"[int(nd["op"])], "object": f"{t}:{obj}", "relation": rel, "subjects": subs, "children": []}
            built.append((n, int(nd["rank"])))
            if nd["parent"] == 0xFFFFFFFF:
                out[int(nd["request"])] = n
            else:
                built[int(nd["parent"])][0]["children"].append((int(nd["rank"]), n))
        for n, _ in built:
            ranks = sorted(r for r, _ in n["children"])
            assert ranks == list(range(len(ranks))), f"{n['object']}#{n['relation']}: child ranks {ranks}"
            n["children"] = [c for _, c in sorted(n["children"], key=lambda x: x[0])]
        return out, {"levels": int(info[0]), "warps": int(info[1])}
