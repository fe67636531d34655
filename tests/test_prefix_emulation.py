"""The resource id prefix scan (csrc/ingress.cuh prefix_match_kernel) under the CPU SIMT emulator against a Python
restatement: arenas whose records start at every byte alignment and end at a guard page, prefixes of 1 to 1 024 bytes,
names shorter than, equal to and longer than the prefix, names that differ only in the last byte of a shared 8-byte
word, an arena rewritten by a retirement (ids no longer in order, gaps), ids past the bitmap, and numeric-only ids
(no record: never set). Then the scan over the store's own name arenas followed by the filter and page kernels with
bitmaps, the match lists of a prefix page and page_walk (tests/emu/emu_prefix_filter.cc), against Store::match and
Store::page with the prefix. TEST INFRASTRUCTURE ONLY: tests/emu/emu_prefix.cc and emu_prefix_filter.cc are built into
libraries of their own."""
import ctypes as C
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

import filter_cases as cases
import randgen

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
CSRC = os.path.join(os.path.dirname(HERE), "spicedb-kubeapi-proxy_b200", "csrc")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(EMU, "libzgemu_prefix.so")
        srcs = [os.path.join(EMU, f) for f in ("emu_prefix.cc", "cuda_emu.h")] + \
               [os.path.join(CSRC, f) for f in ("ingress.cuh", "hash_bytes.h")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", EMU,
                            os.path.join(EMU, "emu_prefix.cc"), "-o", so], check=True)
        L = C.CDLL(so)
        L.emu_prefix_scan.restype = C.c_longlong
        L.emu_prefix_scan.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint32, C.c_char_p, C.c_uint64,
                                      C.c_void_p, C.c_uint, C.c_uint]
        _LIB = L
    return _LIB


def arena_of(names, pad=0):
    """(arena, record offsets) for [(id, name bytes)]: `pad` junk bytes first, so that records start at other
    alignments (the arena's end is fixed at the guard page)."""
    out, offs = bytearray(b"\xa5" * pad), []
    for i, n in names:
        offs.append(len(out))
        out += struct.pack("<II", i, len(n)) + n
    return bytes(out), np.asarray(offs, dtype=np.uint64)


def scan(names, prefix: bytes, n_ids, pad=0, grid=2, threads=64):
    arena, offs = arena_of(names, pad)
    bits = np.zeros((n_ids + 31) // 32 or 1, dtype=np.uint32)
    n = lib().emu_prefix_scan(arena, len(arena), offs.ctypes.data, offs.size, n_ids, prefix, len(prefix),
                              bits.ctypes.data, grid, threads)
    assert n >= 0, "no guard page"
    got = {i for i in range(n_ids) if bits[i >> 5] >> (i & 31) & 1}
    return got, n


def restate(names, prefix: bytes, n_ids):
    return {i for i, n in names if i < n_ids and n.startswith(prefix)}


def _check(names, prefix, n_ids, pad=0, **kw):
    got, n = scan(names, prefix, n_ids, pad, **kw)
    want = restate(names, prefix, n_ids)
    assert got == want, (prefix[:40], pad, sorted(got ^ want)[:10])
    assert n == len(want)


LENGTHS = (1, 7, 8, 9, 15, 16, 17, 1024)


@pytest.mark.parametrize("pad", range(8))
def test_every_alignment_and_prefix_length(pad):
    rng = random.Random(100 + pad)
    base = bytes(rng.choice(b"abcdefghij/_-=+|0123456789") for _ in range(1100))
    names = []
    for i in range(300):
        k = rng.choice([0, 1, 3, 7, 8, 9, 15, 16, 17, 24, 1023, 1024, 1025, 1100])
        n = bytearray(base[:k])
        if n and rng.random() < 0.4:  # differ in one byte, often the last of a shared word
            j = rng.choice([len(n) - 1, (len(n) - 1) | 7 if ((len(n) - 1) | 7) < len(n) else len(n) - 1, rng.randrange(len(n))])
            n[j] = ord("Z")
        names.append((i, bytes(n)))
    for L in LENGTHS:
        _check(names, base[:L], 300, pad)
        p = bytearray(base[:L])
        p[-1] = ord("Z")  # the last byte of the prefix differs
        _check(names, bytes(p), 300, pad)


def test_short_equal_and_last_byte_of_word():
    for L in LENGTHS:
        p = bytes((65 + i % 26) for i in range(L))
        names = [(0, p), (1, p[:-1]), (2, p + b"x"), (3, p[:-1] + b"!"), (4, b""), (5, p + p)]
        if L >= 8:  # the byte before the last word's end, and the last byte of the first word
            names.append((6, p[:7] + b"?" + p[8:]))
        for pad in (0, 3, 7):
            _check(names, p, 8, pad)
            assert restate(names, p, 8) == {0, 2, 5}


def test_retired_arena_and_id_bounds():
    # an arena rewritten by a retirement keeps its records' ids with gaps, not in record order; a reused id's new
    # record sits at the end
    rng = random.Random(7)
    names = [(i, f"ns{i % 5:02d}/p{i:05d}".encode()) for i in range(2000)]
    kept = [x for x in names if rng.random() < 0.6]
    rng.shuffle(kept)
    kept = [x for x in kept if x[0] != 3] + [(3, b"ns99/reused")]
    for p in (b"ns0", b"ns01/", b"ns99/", b"ns01/p0001", b"n"):
        _check(kept, p, 2000, pad=5)
    # ids at or past the bitmap's coverage are never set (interned after the snapshot)
    _check(names, b"ns0", 1000)
    got, _ = scan(names, b"ns", 1000)
    assert max(got) < 1000


def test_numeric_only_ids_never_match():
    # a bulk load uses ids 0..99 without names; only the named ids 100.. have records
    names = [(100 + i, str(i).encode()) for i in range(50)]
    got, n = scan(names, b"1", 200)
    assert got == {100 + i for i in range(50) if str(i).startswith("1")} and n == len(got)
    assert not got & set(range(100))


@pytest.mark.parametrize("grid,threads", [(1, 32), (3, 64), (2, 96)])
def test_launch_shapes(grid, threads):
    names = [(i, f"t{i % 3}/{i}".encode()) for i in range(777)]
    _check(names, b"t1/", 777, 1, grid=grid, threads=threads)


# ---- the filter and page kernels with bitmaps (tests/emu/emu_prefix_filter.cc) ----
# The scan runs over the store's own name arenas, and the kPrefix filter and page kernels with the match lists and
# page_walk run against Store::match and Store::page with the same prefix. Every buffer those kernels touch ends at a
# guard page and is sized exactly, so a read past a bitmap, a match list or its sums faults here.

_PF = None


def pf_lib():
    global _PF
    if _PF is None:
        sys.path.insert(0, EMU)
        import emu_page

        so = os.path.join(EMU, "libzgemu_prefix_filter.so")
        srcs = [os.path.join(EMU, f) for f in ("emu_prefix_filter.cc", "emu_page.cc", "emu_filter.cc", "emu_main.cc",
                                               "cuda_emu.h")] + \
               [os.path.join(CSRC, f) for f in ("filter.cuh", "ingress.cuh", "kernels.cuh", "delta.cuh", "schema.cc",
                                                "schema.h", "store.cc", "store.h")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", EMU,
                            os.path.join(EMU, "emu_prefix_filter.cc"), os.path.join(CSRC, "schema.cc"),
                            os.path.join(CSRC, "store.cc"), "-o", so], check=True)
        L = C.CDLL(so)
        base = emu_page.lib()
        import emu_filter
        for name in emu_filter._DRIVER + ["emu_filter_host", "emu_filter_device", "emu_page_host", "emu_page_device",
                                          "emu_page_class_pos", "emu_page_slot_type"]:
            fn, ref = getattr(L, name), getattr(base, name)
            fn.argtypes, fn.restype = ref.argtypes, ref.restype
        F = C.POINTER(emu_filter.Filter)
        for name in ("emu_prefix_intern", "emu_prefix_find"):
            getattr(L, name).argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint64]
            getattr(L, name).restype = C.c_uint32
        L.emu_prefix_bits.restype = C.c_longlong
        L.emu_prefix_bits.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64,
                                      C.c_void_p]
        L.emu_prefix_match_host.restype = C.c_uint64
        L.emu_prefix_match_host.argtypes = [C.c_void_p, F, C.c_char_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p,
                                            C.c_uint64]
        L.emu_prefix_match_device.argtypes = [C.c_void_p, F, C.c_char_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32,
                                              C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.emu_prefix_page_host.restype = C.c_uint64
        L.emu_prefix_page_host.argtypes = [C.c_void_p, F, C.c_char_p, C.c_uint64, C.c_uint32, C.c_int, C.c_void_p,
                                           C.c_uint64, C.c_void_p, C.c_void_p]
        L.emu_prefix_page_device.argtypes = [C.c_void_p, F, C.c_char_p, C.c_uint64, C.c_uint32, C.c_int, C.c_void_p,
                                             C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        _PF = L
    return _PF


def _prefix_engine(schema, rels, expires=None, numeric=()):
    """An emulator engine whose ids are the store's interned names (Store::intern), with `rels` loaded (expires: {rel:
    unix seconds}) and published. numeric: extra (relationship with numeric ids, as a bulk load writes it)."""
    sys.path.insert(0, EMU)
    import emu
    import emu_filter
    import emu_page
    from golden_runner import split_rel

    class Engine(emu_page.EmuEngine):
        def __init__(self, schema):
            self._L = pf_lib()
            err = C.create_string_buffer(512)
            self._h = self._L.emu_create(schema.encode(), err, 512)
            if not self._h:
                raise RuntimeError(err.value.decode())
            self._names = {}
            self.shard_opts = emu.default_opts()

        def _id(self, t, name, create):
            b = name.encode()
            i = self._L.emu_prefix_find(self._h, self.type_id(t), b, len(b))
            if i == 0xFFFFFFFF:
                if not create:
                    return None
                i = self._L.emu_prefix_intern(self._h, self.type_id(t), b, len(b))
            return i

        def _rows(self, t, ex):
            return list(zip(t["res"].tolist(), t["subj"].tolist(), t["rel"].tolist(), t["stype"].tolist(),
                            t["srel"].tolist(), ex.tolist()))

        def host_match_p(self, x, prefix, now):
            t, ex = np.zeros(1 << 16, dtype=emu_filter.TUPLE_DTYPE), np.zeros(1 << 16, dtype=np.uint32)
            p = prefix.encode()
            n = int(self._L.emu_prefix_match_host(self._h, C.byref(x), p, len(p), now, t.ctypes.data, ex.ctypes.data,
                                                  1 << 16))
            return sorted(self._rows(t[:n], ex[:n]))

        def device_match_p(self, x, prefix, now, grid=2, max_sel=64):
            t, ex = np.zeros(1 << 16, dtype=emu_filter.TUPLE_DTYPE), np.zeros(1 << 16, dtype=np.uint32)
            info = np.zeros(5, dtype=np.uint64)
            p = prefix.encode()
            rc = self._L.emu_prefix_match_device(self._h, C.byref(x), p, len(p), now, grid, max_sel, t.ctypes.data,
                                                 ex.ctypes.data, 1 << 16, info.ctypes.data)
            assert rc == 0, rc
            d = dict(zip(("count", "emitted", "shape", "launches", "matched"), (int(v) for v in info)))
            return sorted(self._rows(t[:d["emitted"]], ex[:d["emitted"]])), d

        def _after(self, after):
            return (1, np.array(after, dtype=np.uint32)) if after is not None else (0, np.zeros(4, dtype=np.uint32))

        def host_page_p(self, x, prefix, want, now=0, after=None):
            has, a = self._after(after)
            t, ex = np.zeros(max(want, 1), dtype=emu_filter.TUPLE_DTYPE), np.zeros(max(want, 1), dtype=np.uint32)
            p = prefix.encode()
            n = int(self._L.emu_prefix_page_host(self._h, C.byref(x), p, len(p), now, has, a.ctypes.data, want,
                                                 t.ctypes.data, ex.ctypes.data))
            return self._rows(t[:n], ex[:n])

        def device_page_p(self, x, prefix, want, now=0, after=None, grid=2):
            has, a = self._after(after)
            t, ex = np.zeros(max(want, 1), dtype=emu_filter.TUPLE_DTYPE), np.zeros(max(want, 1), dtype=np.uint32)
            info = np.zeros(6, dtype=np.uint64)
            p = prefix.encode()
            rc = self._L.emu_prefix_page_device(self._h, C.byref(x), p, len(p), now, has, a.ctypes.data, want, grid,
                                                t.ctypes.data, ex.ctypes.data, info.ctypes.data)
            assert rc == 0, rc
            d = dict(zip(("records", "windows", "launches", "max_tiles", "scanned", "list_launches"),
                         (int(v) for v in info)))
            return self._rows(t[:d["records"]], ex[:d["records"]]), d

    e = Engine(schema)
    t = np.zeros(len(rels), dtype=emu_filter.TUPLE_DTYPE)
    for i, r in enumerate(rels):
        rt, rid, rel, st, sid, srel = split_rel(r)
        t["rel"][i], t["stype"][i], t["res"][i] = e.slot_id(rt, rel), e.type_id(st), e._id(rt, rid, True)
        if sid == "*":
            t["srel"][i] = emu_filter.SREL_WILDCARD
        else:
            t["srel"][i] = e.slot_id(st, srel) if srel else emu_filter.SREL_NONE
            t["subj"][i] = e._id(st, sid, True)
    ex = np.array([(expires or {}).get(r, 0) for r in rels], dtype=np.uint32)
    e.load_tuples(t, ex)
    if numeric:
        n = np.zeros(len(numeric), dtype=emu_filter.TUPLE_DTYPE)
        for i, (rt, res, rel, st, subj) in enumerate(numeric):
            n["rel"][i], n["stype"][i], n["res"][i], n["subj"][i] = e.slot_id(rt, rel), e.type_id(st), res, subj
            n["srel"][i] = emu_filter.SREL_NONE
        e.load_tuples(n)
    e.publish()
    return e, split_rel


def _pf_filters(e, rels, split_rel, rng, samples=2):
    out = []
    for f in cases.filters_for(rels, split_rel, rng, samples=samples):
        if f.get("res_id"):
            continue
        x = e.resolve(f)
        if x is not None:
            out.append(x)
    return out


def _pf_prefixes(rels, split_rel, rng):
    names = sorted({split_rel(r)[1] for r in rels})
    out = {"zz-nobody-"}
    for name in rng.sample(names, min(2, len(names))):
        out.update(name[:k] for k in range(1, len(name) + 1))
    return sorted(out)


def _pf_restated(e, x, prefix, now, after, want):
    rows = sorted(e.host_match_p(x, prefix, now), key=e.key)
    return [r for r in rows if after is None or e.key(r) > tuple(after)][:want]


def _pf_drain(e, x, prefix, limit, now=0, after=None):
    """Pages from `after` to the end on both paths and the restatement; -> (rows, infos)."""
    rows, infos = [], []
    while True:
        want = limit + 1
        got, info = e.device_page_p(x, prefix, want, now, after)
        assert got == e.host_page_p(x, prefix, want, now, after) == _pf_restated(e, x, prefix, now, after, want), \
            (prefix, limit, after)
        rows += got[:limit]
        infos.append(info)
        if len(got) <= limit:
            return rows, infos
        after = e.key(got[limit - 1])


def _ns_names(n_ns, n_per):
    return [f"ns{i:02d}/d{j:03d}" for i in range(n_ns) for j in range(n_per)]


@pytest.mark.parametrize("name", ["docs", "exp"])
@pytest.mark.parametrize("now", [100, 200])
def test_filter_and_page_kernels_with_bitmaps(name, now):
    """Every filter shape the prefix allows (scan and subject), with every proper prefix of sampled names, a prefix
    nobody has and one without a type, at two clocks: the emitted records == Store::match, the count launch == the emit
    launch, and pages at limits 1, 2, 7, 33 and 1000 == Store::page == the restatement."""
    rng = random.Random(6100 + now)
    schema = cases.EXP_SCHEMA if name == "exp" else randgen.FIXED_SCHEMAS["docs"]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=12, n_user=6, density=0.3)
    expires = {r: rng.choice([50, 150, 250]) for r in rels if rng.random() < 0.5} if name == "exp" else None
    e, split_rel = _prefix_engine(schema, rels, expires)
    prefixes = _pf_prefixes(rels, split_rel, rng)
    shapes = set()
    for i, x in enumerate(_pf_filters(e, rels, split_rel, rng)):
        for p in rng.sample(prefixes, min(3, len(prefixes))):
            for clock in (now, 0):
                want = e.host_match_p(x, p, clock)
                got, info = e.device_match_p(x, p, clock, max_sel=1 + i % 3)
                assert got == want, (p, clock)
                assert info["count"] == info["emitted"] == len(want)
                if info["shape"]:  # 0: nothing selected, no launch
                    shapes.add(info["shape"])
            for limit in ((1, 2, 7, 33, 1000) if i % 6 == 0 else (2,)):
                _pf_drain(e, x, p, limit, now)
    assert shapes == {1, 2}
    every = e.resolve({})
    for p in prefixes:
        _pf_drain(e, every, p, 3, now)


def test_windows_skip_unmatched_objects():
    """A prefix that matches one object in 200: the page's windows are sized over the list of matched ids, so the
    windows and launches of a page do not grow with the unmatched objects between matches; limits that make the
    windows come up short and grow; cursors inside the type, between types and past the end."""
    schema = randgen.FIXED_SCHEMAS["docs"]
    counts = []
    for gap in (200, 2000):
        names = [f"a{i:05d}" if i % gap else f"m{i:05d}" for i in range(20 * gap)]
        rels = [f"document:{n}#viewer@user:u{i % 5}" for i, n in enumerate(names)]
        rels += [f"document:{n}#owner@user:u{i % 3}" for i, n in enumerate(names) if i % 3 == 0]
        rels += [f"org:m{i}#member@user:u{i % 5}" for i in range(7)]
        e, split_rel = _prefix_engine(schema, rels)
        scan = e.resolve({"res_type": "document", "rel": "viewer"})
        rows, infos = _pf_drain(e, scan, "m", 3)
        assert len(rows) == 20
        counts.append([(i["windows"], i["launches"]) for i in infos])
        assert max(i["max_tiles"] for i in infos) > 0
        everything = e.resolve({})
        all_rows, _ = _pf_drain(e, everything, "m", 1000)
        keys = [e.key(r) for r in all_rows]
        doc, user = e.type_id("document"), e.type_id("user")
        for after in keys[::5] + [keys[-1], (doc, 1, 0, 0), (doc, 0xFFFFFFF0, 0, 0), (user, 0, 0, 0), (0xFFFF, 0, 0, 0)]:
            for limit in (1, 7):
                _pf_drain(e, everything, "m", limit, after=after)
    assert counts[0] == counts[1], counts


def test_numeric_ids_and_bitmaps():
    """Ids a bulk load uses without a name never match, even past the names; the bitmaps the scan builds from the
    store's arenas hold exactly the named ids with the prefix."""
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = [f"document:p{i}#viewer@user:u0" for i in range(40)]
    e, split_rel = _prefix_engine(schema, rels, numeric=[("document", 100 + i, "viewer", "user", 0) for i in range(30)])
    x = e.resolve({"res_type": "document"})
    for p in ("p", "p1", "1", "p39", "p399"):
        got, info = e.device_match_p(x, p, 0)
        assert got == e.host_match_p(x, p, 0)
        assert all(r[0] < 40 for r in got)
        _pf_drain(e, x, p, 4)
    bits = np.zeros(1 << 12, dtype=np.uint32)
    info = np.zeros(3, dtype=np.uint64)
    doc = e.type_id("document")
    w = e._L.emu_prefix_bits(e._h, doc, b"p1", 2, 2, bits.ctypes.data, bits.size, info.ctypes.data)
    assert w > 0
    got = {i for i in range(w * 32) if bits[i >> 5] >> (i & 31) & 1}
    assert got == {e._id("document", f"p{i}", False) for i in range(40) if str(i).startswith("1")}
    assert int(info[1]) == len(got)
