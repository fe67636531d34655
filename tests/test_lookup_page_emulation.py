"""The kernels of a LookupResources page (kernels.cuh lookup_select_kernel, lookup_bound_kernel, lookup_window_kernel)
under the CPU SIMT emulator, driven by tests/emu/emu_lookup_page.cc, a restatement of Device::lookup_page's loop. Every
page is compared with the C oracle's LookupResources sliced after the cursor, and with a model of the windows: which
candidates they verify, where the page is decided, and whether an undecidable candidate fails it."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np

_EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
sys.path.insert(0, _EMU)

import emu  # noqa: E402
from golden_runner import split_rel  # noqa: E402

LIMITS = (1, 2, 31, 32, 33, 1000)
NO_OBJECT, HAS, ERR = 0xFFFFFFFF, 2, 255
_LIB = None

SPARSE = ("definition user {}\ndefinition doc {\n  relation viewer: user\n  relation banned: user\n"
          "  relation editor: user\n  permission view = viewer - banned\n  permission both = viewer & editor\n}\n")


def _lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_EMU, "libzgemu_lookup_page.so")
        csrc = os.path.join(os.path.dirname(_EMU), "..", "spicedb-kubeapi-proxy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_lookup_page.cc", "emu_main.cc", "cuda_emu.h")] + \
               [os.path.join(csrc, f) for f in ("kernels.cuh", "delta.cuh", "schema.cc", "store.cc", "store.h")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                            os.path.join(_EMU, "emu_lookup_page.cc"), os.path.join(csrc, "schema.cc"),
                            os.path.join(csrc, "store.cc"), "-o", tmp], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        base = emu.lib()
        for name in ("emu_create", "emu_destroy", "emu_type_id", "emu_slot_id", "emu_load", "emu_publish", "emu_check",
                     "emu_journal_start"):
            getattr(L, name).argtypes, getattr(L, name).restype = getattr(base, name).argtypes, getattr(base, name).restype
        L.emu_lookup_page.argtypes = [C.c_void_p, C.c_uint16, C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32,
                                      C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.POINTER(emu.Opts),
                                      C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


class Engine(emu.EmuEngine):
    def __init__(self, schema):
        self._L = _lib()
        err = C.create_string_buffer(512)
        self._h = self._L.emu_create(schema.encode(), err, 512)
        if not self._h:
            raise RuntimeError(err.value.decode())
        self._names = {}
        self.shard_opts = emu.default_opts()

    def page(self, rt, proto, after, want, self_id=NO_OBJECT, cand=(), sorted_=False, flat=False, first_w=4, growth=4):
        c = np.ascontiguousarray(cand, dtype=np.uint32)
        out = np.zeros(max(int(want), 1), dtype=np.uint32)
        info = np.zeros(5, dtype=np.uint64)
        p = np.array([proto], dtype=emu.CHECK_DTYPE)
        rc = self._L.emu_lookup_page(self._h, self.type_id(rt), p.ctypes.data, after is not None, after or 0, int(want), self_id,
                                     first_w, growth, c.ctypes.data, c.size, int(sorted_), int(flat), C.byref(emu.default_opts()),
                                     out.ctypes.data, info.ctypes.data)
        d = dict(zip(("found", "after", "verified", "windows", "launches"), (int(x) for x in info)))
        return rc, [int(x) for x in out[:d["found"]]], d


def _model(cand, codes, after, want, quiet=NO_OBJECT, first_w=4, growth=4):
    """The page the windows must give: (rc, ids, candidates after the cursor, verified, windows)."""
    sel = sorted(int(x) for x in cand if after is None or x > after)  # a repeated id is verified again, counted once
    m, pos, w, found, windows = len(sel), 0, max(first_w, 2 * want), [], 0
    while pos < m:
        w = min(w, m - pos)
        windows += 1
        for i in range(pos, pos + w):
            if i and sel[i] == sel[i - 1]:
                continue
            if len(found) < want and codes[sel[i]] == ERR and sel[i] != quiet:
                return -3, None, m, pos + w, windows
            if codes[sel[i]] == HAS:
                found.append(sel[i])
                if len(found) == want:
                    return 0, found, m, pos + w, windows
        pos += w
        left = m - pos
        nxt = min(left, w * growth)
        if found:
            est = (want - len(found)) * pos / len(found) * 1.25
            nxt = left if est >= left else max(nxt, int(est) + 1)
        w = nxt
    return 0, found, m, pos, windows


def _setup(schema, rels):
    from oracle.pyoracle import Oracle

    e, o = Engine(schema), Oracle(schema)
    e.write_rels(rels, split_rel)
    e.publish()
    for r in rels:
        o.touch(r, 0)
    return e, o


def _proto(e, rt, perm, st, subj, srel=None):
    p = np.zeros(1, dtype=emu.CHECK_DTYPE)[0]
    p["perm"], p["stype"], p["subj"] = e.slot_id(rt, perm), e.type_id(st), subj
    p["srel"] = emu.SREL_NONE if srel is None else e.slot_id(st, srel)
    return p


def _codes(e, rt, proto, ids):
    items = np.zeros(len(ids), dtype=emu.CHECK_DTYPE)
    for f in ("perm", "stype", "subj", "srel"):
        items[f] = proto[f]
    items["res"] = ids
    return dict(zip((int(i) for i in ids), e.check_bulk(items).tolist()))


def _all_ids(e, t):
    return sorted(i for (tt, _), i in e._names.items() if tt == t)


def _check_pages(e, o, q, cursors, limits=LIMITS, self_id=NO_OBJECT, shuffle=True):
    rt, perm, st, sid, srel = q
    proto = _proto(e, rt, perm, st, e._names[(st, sid)], srel)
    cand = _all_ids(e, rt)
    codes = _codes(e, rt, proto, cand + ([self_id] if self_id != NO_OBJECT else []))
    whole = sorted(e._names[(rt, n)] for n in o.lookup_resources(rt, perm, st, sid, srel or ""))
    rng = random.Random(7)
    for after in cursors:
        for limit in limits:
            want = limit + 1
            for sorted_ in ((True, False) if self_id == NO_OBJECT else (False,)):
                c = list(cand)
                if not sorted_ and shuffle:
                    rng.shuffle(c)
                rc, ids, info = e.page(rt, proto, after, want, self_id, c, sorted_)
                m_rc, m_ids, m_after, m_ver, m_win = _model(cand + ([self_id] if self_id != NO_OBJECT else []), codes, after,
                                                             want, self_id if self_id not in cand else NO_OBJECT)
                assert rc == m_rc, (q, after, limit, sorted_)
                assert (info["after"], info["verified"], info["windows"]) == (m_after, m_ver, m_win), (q, after, limit)
                if rc == 0:
                    assert ids == m_ids, (q, after, limit)
                    assert ids == [i for i in whole if after is None or i > after][:want], (q, after, limit)


def test_limits_and_cursors_with_sparse_answers():
    rng = random.Random(1)
    rels = [f"doc:d{i}#viewer@user:a" for i in range(700)]
    rels += [f"doc:d{i}#banned@user:a" for i in range(700) if i % 23]  # 1 in 23 is an answer
    rels += [f"doc:d{i}#editor@user:a" for i in rng.sample(range(700), 40)]
    e, o = _setup(SPARSE, rels)
    ids = _all_ids(e, "doc")
    answers = sorted(e._names[("doc", n)] for n in o.lookup_resources("doc", "view", "user", "a", ""))
    not_answer = next(i for i in ids if i not in answers and i > answers[0])
    for perm in ("view", "both"):
        _check_pages(e, o, ("doc", perm, "user", "a", None), [None, not_answer, answers[-1], 10 ** 6])
    # the windows grew several times: 1 in 23 answers, the first window of 4
    _, _, info = e.page("doc", _proto(e, "doc", "view", "user", e._names[("user", "a")]), None, 3, cand=ids, sorted_=True)
    assert info["windows"] >= 3 and info["verified"] < len(ids)


def test_flat_union_with_repeated_ids():
    e, _ = _setup(SPARSE, ["doc:d0#viewer@user:a"])
    cand = [9, 3, 3, 7, 1, 9, 9, 2, 5, 7] * 3 + list(range(100, 2200))
    rng = random.Random(3)
    rng.shuffle(cand)
    uniq = sorted(set(cand))
    proto = _proto(e, "doc", "viewer", "user", 0)
    for after in (None, 3, 99, 2199):
        for limit in LIMITS:
            rc, ids, info = e.page("doc", proto, after, limit + 1, cand=cand, flat=True)
            assert rc == 0 and ids == [i for i in uniq if after is None or i > after][:limit + 1], (after, limit)
            assert info["verified"] == 0 and info["windows"] == 0


def test_self_candidate():
    from test_oracle_random import SELF_RELS, SELF_SCHEMA

    e, o = _setup(SELF_SCHEMA, SELF_RELS)
    five = e._names[("doc", "5")]
    for q in (("doc", "view", "doc", "5", "viewer"), ("doc", "safe", "doc", "5", "viewer"), ("doc", "view", "doc", "5", "editor")):
        _check_pages(e, o, q, [None, five - 1 if five else None, five], limits=(1, 2, 33), self_id=five)


def test_undecidable_candidate_before_and_after_the_deciding_answer():
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i + 1}#member" for i in range(5, 55)] + ["group:g55#member@user:deep"]
    rels += [f"group:g{i}#member@group:g{i + 1}#member" for i in range(0, 5)]
    e, o = _setup(CHAIN, rels)
    proto = _proto(e, "group", "member", "user", e._names[("user", "deep")])
    ids = _all_ids(e, "group")
    codes = _codes(e, "group", proto, ids)
    bad = [i for i in ids if codes[i] == ERR]
    good = [i for i in ids if codes[i] == HAS]
    assert bad and good and max(good) < min(bad)
    # the deciding answer comes before the undecidable ones: the page succeeds
    rc, got, _ = e.page("group", proto, None, 11, cand=ids, sorted_=True)
    assert rc == 0 and got == good[:11]
    # the page reaches past the last answer: it fails, as the unpaged call does
    rc, _, _ = e.page("group", proto, None, len(good) + 1, cand=ids, sorted_=True)
    assert rc == -3
    rc, _, _ = e.page("group", proto, good[-2], 2, cand=ids, sorted_=False)
    assert rc == -3
    _check_pages(e, o, ("group", "member", "user", "deep", None), [None, good[5]], limits=(1, 2, 31, 1000))
