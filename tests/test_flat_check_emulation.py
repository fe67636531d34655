"""The lean check kernel (csrc/kernels.cuh flat_check_kernel) and the residual pass behind it under the SIMT emulator
(tests/emu/): checks of an SF_FLAT slot are answered one per thread, and every other item goes to check_kernel<kMeetSet16>
through the residual list (KParams::idx / nq_dev). The driver (tests/emu/emu_flat.cc) reuses emu_set.cc's host-built
closure indexes, signatures and set tables. Answers must equal the oracle's, the generic kernel's (emu_set_check, or
the plain check_kernel<kMeetSet16> with the clock and no_wildcards set) and a run with no slot marked (every item
residual); the COUNT bytes must equal the generic kernel's. A second store puts direct (expiring) and wildcard probes
in front of the meet in flat slots."""
import ctypes as C
import os

import numpy as np
import pytest

from test_closure_set_emulation import SetStore
from test_rsetless_emulation import CFG3, ZG_MAX_DEPTH, cfg3_groups

_TESTS = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_TESTS, "emu")
_CSRC = os.path.join(os.path.dirname(_TESTS), "spicedb-kubeapi-proxy_b200", "csrc")
SF_FLAT = 2
K_VAL_T = 1
HAS = 2  # ZG_HAS_PERMISSION


@pytest.fixture(scope="module")
def emu():
    import emu as E

    so = os.path.join(_EMU, "libzgemu_flat.so")
    srcs = [os.path.join(_EMU, f) for f in ("emu_flat.cc", "emu_set.cc", "emu_sig.cc", "emu_rset.cc", "emu_main.cc",
                                             "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "closure_sig.cuh", "delta.cuh", "schema.cc", "schema.h",
                                             "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        import subprocess

        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                        os.path.join(_EMU, "emu_flat.cc"), os.path.join(_CSRC, "schema.cc"),
                        os.path.join(_CSRC, "store.cc"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_create.restype = C.c_void_p
    L.emu_create.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    L.emu_destroy.argtypes = [C.c_void_p]
    L.emu_type_id.argtypes = [C.c_void_p, C.c_char_p]
    L.emu_slot_id.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    L.emu_load.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_size_t]
    L.emu_publish.argtypes = [C.c_void_p]
    L.emu_index_create.restype = C.c_void_p
    L.emu_index_create.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    L.emu_index_destroy.argtypes = [C.c_void_p]
    L.emu_index_slot_flags.restype = C.c_uint32
    L.emu_index_slot_flags.argtypes = [C.c_void_p, C.c_int]
    L.emu_sig_create.restype = C.c_void_p
    L.emu_sig_create.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    L.emu_sig_destroy.argtypes = [C.c_void_p]
    L.emu_set_create.restype = C.c_void_p
    L.emu_set_create.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    L.emu_set_destroy.argtypes = [C.c_void_p]
    L.emu_set_meet.argtypes = [C.c_void_p]
    L.emu_set_check.restype = C.c_uint32
    L.emu_set_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    L.emu_flat_mark.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.emu_flat_check.restype = C.c_uint32
    L.emu_flat_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                 C.c_uint32, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    return E, L


class FlatStore(SetStore):
    def flat_flags(self):
        flags = np.zeros(64, dtype=np.uint16)
        n = self.L.emu_flat_mark(self.set(), flags.ctypes.data, flags.size)
        return n, flags

    def run_flat(self, items, lean=1, count=False, val=False, now=0, no_wildcards=False):
        """lean 1: the lean kernel and the residual pass; 0: every item through the residual pass; -1: the plain
        check_kernel<kMeetSet16> (the reference)."""
        out = np.zeros(items.size, dtype=np.uint8)
        v = np.zeros(max(items.size, 1), dtype=np.uint8) if val else None
        nb, nr = C.c_uint64(0), C.c_uint64(0)
        raw = int(not items["flags"].any())
        fl = self.L.emu_flat_check(self.set(), items.ctypes.data, items.size, out.ctypes.data,
                                   None if v is None else v.ctypes.data, raw, int(count), int(lean), now,
                                   int(no_wildcards), C.byref(nb), C.byref(nr))
        assert fl & 3 == 0, fl  # no spill or sub-query overflow (~0: the residual counts disagree)
        return out, nb.value, nr.value, v


@pytest.fixture(scope="module")
def cfg3(emu):
    rng = np.random.default_rng(7)
    groups, n_users, n_ns = cfg3_groups(rng)
    groups = [g for g in groups if not (g[0] == "namespace" and g[2] == "user")]  # no direct viewers: SF_NO_RSET
    s = FlatStore(emu, CFG3, groups)
    s.groups, s.n_users, s.n_ns = groups, n_users, n_ns
    yield s
    s.close()


def mixed(s, rng, n):
    """namespace#view@user checks interleaved with every kind of item the lean kernel must leave: userset subjects,
    invalid items, the wrong subject type, subjects past the closure rows, and a slot that is not flat."""
    res = rng.integers(0, s.n_ns, n).astype(np.uint32)
    subj = rng.integers(0, s.n_users, n).astype(np.uint32)
    it = s.items("namespace", "view", "user", res, subj)
    kind = rng.integers(0, 8, n)
    team, grp = s.type("team"), s.type("group")
    it["srel"][kind == 1] = s.slot("team", "member")  # team:t#member
    it["stype"][kind == 1] = team
    it["subj"][kind == 1] %= 20
    it["perm"][kind == 2] = 0xFFF0  # invalid permission
    it["stype"][kind == 3] = grp  # a group as a direct subject: no closure row of its type
    it["subj"][kind == 3] %= 60
    it["subj"][kind == 4] = s.n_users + rng.integers(0, 50, (kind == 4).sum())  # past the rows
    tm = kind == 5  # team#member@user: a one-level slot, not flat
    it["perm"][tm] = s.slot("team", "member")
    it["res"][tm] %= 20
    return it, kind


def test_cfg3_slot_is_flat_and_others_are_not(cfg3):
    n, flags = cfg3.flat_flags()
    assert flags[cfg3.slot("namespace", "view")] & SF_FLAT
    assert not flags[cfg3.slot("team", "member")] & SF_FLAT and not flags[cfg3.slot("group", "member")] & SF_FLAT
    assert n >= 1


@pytest.mark.parametrize("n", [1, 31, 257, 1000])
def test_cfg3_checks_match_the_oracle_with_no_residual(cfg3, n):
    rng = np.random.default_rng(100 + n)
    res = rng.integers(0, cfg3.n_ns, n).astype(np.uint32)
    subj = rng.integers(0, cfg3.n_users, n).astype(np.uint32)
    items = cfg3.items("namespace", "view", "user", res, subj)
    got, _, resid, _ = cfg3.run_flat(items)
    assert resid == 0
    assert np.array_equal(got, cfg3.oracle_answers("namespace", "view", "user", res, subj))
    assert np.array_equal(got, cfg3.run_set(items)[0])


@pytest.mark.parametrize("n", [77, 600])
def test_mixed_batches_take_the_residual_pass(cfg3, n):
    rng = np.random.default_rng(200 + n)
    items, kind = mixed(cfg3, rng, n)
    got, _, resid, val = cfg3.run_flat(items, val=True)
    # (a subject id past the users may still have a row: the index covers the inner class's capacity)
    assert int(np.isin(kind, [1, 2, 3, 5]).sum()) <= resid <= int(((kind >= 1) & (kind <= 5)).sum())
    want = cfg3.run_set(items)[0]
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    assert np.array_equal(got, cfg3.run_flat(items, lean=0)[0])  # every item through idx
    flat = kind == 0
    assert np.array_equal(got[flat], cfg3.oracle_answers("namespace", "view", "user", items["res"][flat],
                                                         items["subj"][flat]))
    assert np.array_equal(val[:n] == K_VAL_T, got == HAS)


@pytest.mark.parametrize("depth", [ZG_MAX_DEPTH - 3, ZG_MAX_DEPTH - 2, ZG_MAX_DEPTH - 1, ZG_MAX_DEPTH])
def test_items_at_the_depth_limit(cfg3, depth):
    """Items whose hop depth leaves no room for the two-level meet go to check_kernel, which walks their ranges."""
    rng = np.random.default_rng(300 + depth)
    res = rng.integers(0, cfg3.n_ns, 300).astype(np.uint32)
    subj = rng.integers(0, cfg3.n_users, 300).astype(np.uint32)
    items = cfg3.items("namespace", "view", "user", res, subj, depth=depth)
    items["flags"][::3] = 1  # and shallow ones among them
    got, _, resid, _ = cfg3.run_flat(items)
    assert resid == (0 if depth + 2 <= ZG_MAX_DEPTH else int((items["flags"] == depth).sum()))
    assert np.array_equal(got, cfg3.run_set(items)[0])


@pytest.mark.parametrize("past_rows", [False, True])
def test_count_bytes_equal_the_generic_kernel(cfg3, past_rows):
    """On batches the lean kernel answers, and with subjects past the rows among them (residual items that walk nothing:
    the bytes of items that traverse depend on which checks share their warp in check_kernel)."""
    rng = np.random.default_rng(400)
    subj = rng.integers(0, cfg3.n_users, 500).astype(np.uint32)
    if past_rows:
        subj[::5] += np.uint32(1 << 20)
    items = cfg3.items("namespace", "view", "user", rng.integers(0, cfg3.n_ns, 500).astype(np.uint32), subj)
    got, nb, resid, _ = cfg3.run_flat(items, count=True)
    assert resid == (100 if past_rows else 0)
    want, wb = cfg3.run_set(items, count=True)
    assert np.array_equal(got, want)
    assert nb == wb, (nb, wb)


PROBES = """use expiration
definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member | user with expiration | user:*
  relation reader: team#member | user:* with expiration
  permission view = viewer
  permission read = reader
}
"""
T0 = 1_000_000  # the first clock; the second is T0 + 1000


class ProbeStore(FlatStore):
    """A FlatStore whose relationships may expire (groups' 7th field) or be wildcards (subject relation "*"), with a
    second oracle that has no wildcard relationship (what a check with no_wildcards sees)."""

    def __init__(self, emu, schema, groups):
        from oracle.pyoracle import Oracle

        self.E, self.L = emu
        err = C.create_string_buffer(512)
        self.h = self.L.emu_create(schema.encode(), err, 512)
        assert self.h, err.value
        self.oracle, self.oracle_nowild = Oracle(schema), Oracle(schema)
        for rt, rel, st, res, subj, srel, exp in groups:
            t = np.zeros(len(res), dtype=self.E.TUPLE_DTYPE)
            t["res"], t["subj"] = res, subj
            t["rel"], t["stype"] = self.slot(rt, rel), self.type(st)
            t["srel"] = self.E.SREL_WILDCARD if srel == "*" else (self.E.SREL_NONE if srel is None else self.slot(st, srel))
            ex = np.zeros(len(res), dtype=np.uint32) if exp is None else np.ascontiguousarray(exp, dtype=np.uint32)
            assert self.L.emu_load(self.h, t.ctypes.data, ex.ctypes.data, t.size, err, 512) == 0, err.value
            for o in (self.oracle,) if srel == "*" else (self.oracle, self.oracle_nowild):
                sr = 0xFFFE if srel == "*" else (0xFFFF if srel is None else o.slot_id(st, srel))
                for r, u, x in zip(t["res"].tolist(), t["subj"].tolist(), ex.tolist()):
                    o.write_ids(0, o.slot_id(rt, rel), r, o.type_id(st), u, sr, x)  # ZG_OP_TOUCH
        assert self.L.emu_publish(self.h) == 0
        self.marked, self.idx = {}, {}
        for mark in (0, 1):
            n = C.c_int(0)
            self.idx[mark] = self.L.emu_index_create(self.h, mark, C.byref(n))
            self.marked[mark] = n.value
        self.sigs, self.sets = {}, {}


@pytest.fixture(scope="module")
def probes(emu):
    """cfg3's meets plus, on the flat slots, expiring direct viewers (never, before and after the second clock, and
    already expired at the first) and wildcards on a few namespaces (one of them expiring between the clocks)."""
    rng = np.random.default_rng(31)
    groups, n_users, n_ns = cfg3_groups(rng)
    groups = [g + (None,) for g in groups if not (g[0] == "namespace" and g[2] == "user")]
    dv_n, dv_u = rng.integers(0, n_ns, 400), rng.integers(0, n_users, 400)
    dv_x = np.array([0, T0 - 10, T0 + 500, T0 + 5000], dtype=np.uint32)[rng.integers(0, 4, 400)]
    pairs = {}
    for n_, u, x in zip(dv_n.tolist(), dv_u.tolist(), dv_x.tolist()):
        pairs[n_, u] = x
    dv = np.array([(n_, u, x) for (n_, u), x in sorted(pairs.items())], dtype=np.int64)
    groups.append(("namespace", "viewer", "user", dv[:, 0], dv[:, 1], None, dv[:, 2]))
    groups.append(("namespace", "viewer", "user", [3, 7], [0, 0], "*", None))
    groups.append(("namespace", "reader", "team", rng.integers(0, n_ns, 100), rng.integers(0, 20, 100), "member", None))
    groups.append(("namespace", "reader", "user", [2, 5, 11], [0, 0, 0], "*", [0, T0 + 500, T0 - 10]))
    s = ProbeStore(emu, PROBES, groups)
    s.groups, s.n_users, s.n_ns = groups, n_users, n_ns
    yield s
    s.close()


def probe_items(s, rng, n):
    """view and read checks of users that have rows, a third of them on a direct viewer's own namespace."""
    res = rng.integers(0, s.n_ns, n).astype(np.uint32)
    subj = rng.integers(0, s.n_users, n).astype(np.uint32)
    dv = s.groups[3]
    pick = rng.integers(0, len(dv[3]), n)
    own = rng.random(n) < 0.34
    res[own], subj[own] = np.asarray(dv[3])[pick[own]], np.asarray(dv[4])[pick[own]]
    it = s.items("namespace", "view", "user", res, subj)
    it["perm"][rng.random(n) < 0.5] = s.slot("namespace", "read")
    return it


def oracle_of(s, o, items, now):
    it = items.copy()
    it["perm"] = [o.slot_id("namespace", "view" if p == s.slot("namespace", "view") else "read") for p in items["perm"]]
    it["stype"] = o.type_id("user")
    return np.asarray(o.check_bulk(it, now=now), dtype=np.uint8)


def test_probe_slots_are_flat(probes):
    _, flags = probes.flat_flags()
    assert flags[probes.slot("namespace", "view")] & SF_FLAT and flags[probes.slot("namespace", "read")] & SF_FLAT


@pytest.mark.parametrize("now", [T0, T0 + 1000])
@pytest.mark.parametrize("no_wildcards", [False, True])
def test_direct_and_wildcard_probes(probes, now, no_wildcards):
    """Expiring direct viewers and wildcards (with and without expiry) at two clocks, with wildcards visible and
    hidden: the lean kernel answers every check and agrees with the oracle and the plain check_kernel<kMeetSet16>."""
    rng = np.random.default_rng(500 + now % 7 + no_wildcards)
    items = probe_items(probes, rng, 700)
    got, _, resid, _ = probes.run_flat(items, now=now, no_wildcards=no_wildcards)
    assert resid == 0
    want = probes.run_flat(items, lean=-1, now=now, no_wildcards=no_wildcards)[0]
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    o = probes.oracle_nowild if no_wildcards else probes.oracle
    assert np.array_equal(got, oracle_of(probes, o, items, now))
    granted = got == HAS
    assert granted.any() and (~granted).any()


def test_probes_decide_checks(probes):
    """The probes matter here: hiding the wildcards or moving the clock changes answers."""
    items = probe_items(probes, np.random.default_rng(600), 700)
    a = probes.run_flat(items, now=T0)[0]
    assert not np.array_equal(a, probes.run_flat(items, now=T0 + 1000)[0])
    assert not np.array_equal(a, probes.run_flat(items, now=T0, no_wildcards=True)[0])


@pytest.mark.parametrize("now", [T0, T0 + 1000])
@pytest.mark.parametrize("no_wildcards", [False, True])
def test_probe_count_bytes_equal_the_generic_kernel(probes, now, no_wildcards):
    items = probe_items(probes, np.random.default_rng(700), 500)
    got, nb, _, _ = probes.run_flat(items, count=True, now=now, no_wildcards=no_wildcards)
    want, wb, _, _ = probes.run_flat(items, lean=-1, count=True, now=now, no_wildcards=no_wildcards)
    assert np.array_equal(got, want)
    assert nb == wb, (nb, wb)
