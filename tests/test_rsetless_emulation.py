"""Admission without the per-check membership set (SF_NO_RSET, csrc/kernels.cuh) under the SIMT emulator (tests/emu/):
a permission whose root units have no invertible probe and meet only over closure indexes loads none of the subject's
memberships, and its checks take the paths of a subject whose memberships overflow the set. The answers with the flag
on must equal the oracle's and the flag-off run's; the COUNT variant's bytes must fall by exactly the membership reads.
The driver (tests/emu/emu_rset.cc) builds the 16-bit closure index of every two-level pair on the host."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

_TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(_TESTS, "emu"))
sys.path.insert(0, os.path.dirname(_TESTS))

_EMU = os.path.join(_TESTS, "emu")
_CSRC = os.path.join(os.path.dirname(_TESTS), "spicedb-kubeapi-proxy_b200", "csrc")
RSET_CAP = 16  # kernels.cuh kRsetCap
FCAP = 64      # kernels.cuh kFCap
SF_NO_RSET = 1
ZG_MAX_DEPTH = 50
GRANTED = 1  # the answer code of a check that holds


@pytest.fixture(scope="module")
def emu():
    import emu as E

    so = os.path.join(_EMU, "libzgemu_rset.so")
    srcs = [os.path.join(_EMU, f) for f in ("emu_rset.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "delta.cuh", "schema.cc", "schema.h", "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        import subprocess

        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                        os.path.join(_EMU, "emu_rset.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
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
    L.emu_index_check.restype = C.c_uint32
    L.emu_index_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    return E, L


class Store:
    """One schema and its relationships in the emulator and in the oracle; flag-on and flag-off indexed engines."""

    def __init__(self, emu, schema, groups):
        from oracle.pyoracle import Oracle

        self.E, self.L = emu
        err = C.create_string_buffer(512)
        self.h = self.L.emu_create(schema.encode(), err, 512)
        assert self.h, err.value
        self.oracle = Oracle(schema)
        for rt, rel, st, res, subj, srel in groups:
            t = np.zeros(len(res), dtype=self.E.TUPLE_DTYPE)
            t["res"], t["subj"] = res, subj
            t["rel"], t["stype"] = self.slot(rt, rel), self.type(st)
            t["srel"] = self.E.SREL_NONE if srel is None else self.slot(st, srel)
            assert self.L.emu_load(self.h, t.ctypes.data, None, t.size, err, 512) == 0, err.value
            self.oracle.add_bulk(rt, rel, st, np.asarray(res, dtype=np.uint32), np.asarray(subj, dtype=np.uint32), srel=srel)
        assert self.L.emu_publish(self.h) == 0
        self.marked = {}
        self.idx = {}
        for mark in (0, 1):
            n = C.c_int(0)
            self.idx[mark] = self.L.emu_index_create(self.h, mark, C.byref(n))
            self.marked[mark] = n.value

    def close(self):
        for x in self.idx.values():
            self.L.emu_index_destroy(x)
        self.L.emu_destroy(self.h)

    def type(self, name):
        return self.L.emu_type_id(self.h, name.encode())

    def slot(self, t, rel):
        return self.L.emu_slot_id(self.h, self.type(t), rel.encode())

    def flag(self, t, perm):
        return self.L.emu_index_slot_flags(self.idx[1], self.slot(t, perm)) & SF_NO_RSET

    def items(self, rt, perm, st, res, subj, depth=None):
        it = np.zeros(len(res), dtype=self.E.CHECK_DTYPE)
        it["res"], it["subj"] = res, subj
        it["perm"], it["stype"], it["srel"] = self.slot(rt, perm), self.type(st), self.E.SREL_NONE
        if depth is not None:
            it["flags"] = depth
        return it

    def run(self, items, mark, count=False):
        out = np.zeros(items.size, dtype=np.uint8)
        nb = C.c_uint64(0)
        raw = int(not items["flags"].any())
        fl = self.L.emu_index_check(self.idx[mark], items.ctypes.data, items.size, out.ctypes.data, raw, int(count), C.byref(nb))
        assert fl & 3 == 0, fl  # no spill or sub-query overflow
        return out, nb.value

    def oracle_answers(self, rt, perm, st, res, subj):
        it = np.zeros(len(res), dtype=self.E.CHECK_DTYPE)
        it["res"], it["subj"] = res, subj
        it["perm"], it["stype"] = self.oracle.slot_id(rt, perm), self.oracle.type_id(st)
        it["srel"] = self.E.SREL_NONE
        return np.asarray(self.oracle.check_bulk(it), dtype=np.uint8)


CFG3 = """definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member | user }
definition namespace {
  relation viewer: team#member | user
  permission view = viewer
}
"""


def cfg3_groups(rng, n_users=300, n_groups=60, n_teams=20, n_ns=40):
    """cfg3's shape (namespace -> team -> group -> user), plus: user 0 in more groups than the set holds, user 1 in
    exactly kRsetCap, namespace n_ns - 1 viewed by 100 teams (a range over kFCap), and a few direct viewers."""
    big_teams = 100
    gm_g = list(rng.integers(0, n_groups, 1500)) + list(range(RSET_CAP + 4)) + list(range(20, 20 + RSET_CAP))
    gm_u = list(rng.integers(2, n_users, 1500)) + [0] * (RSET_CAP + 4) + [1] * RSET_CAP
    tm_t = list(rng.integers(0, n_teams, 120)) + list(range(n_teams, n_teams + big_teams))
    tm_g = list(rng.integers(0, n_groups, 120)) + list(rng.integers(0, n_groups, big_teams))
    nv_n = list(rng.integers(0, n_ns - 1, 100)) + [n_ns - 1] * big_teams
    nv_t = list(rng.integers(0, n_teams, 100)) + list(range(n_teams, n_teams + big_teams))
    dv_n, dv_u = list(rng.integers(0, n_ns, 30)), list(rng.integers(0, n_users, 30))
    pair = {(int(g), int(u)) for g, u in zip(gm_g, gm_u)}
    gm = sorted(pair)
    return [("group", "member", "user", [g for g, _ in gm], [u for _, u in gm], None),
            ("team", "member", "group", tm_t, tm_g, "member"),
            ("namespace", "viewer", "team", nv_n, nv_t, "member"),
            ("namespace", "viewer", "user", dv_n, dv_u, None)], n_users, n_ns


@pytest.fixture(scope="module")
def cfg3(emu):
    rng = np.random.default_rng(7)
    groups, n_users, n_ns = cfg3_groups(rng)
    s = Store(emu, CFG3, groups)
    s.n_users, s.n_ns = n_users, n_ns
    yield s
    s.close()


def test_cfg3_shape_sets_the_flag_and_answers_match_the_oracle(cfg3):
    assert cfg3.flag("namespace", "view") and cfg3.flag("namespace", "viewer")
    assert not cfg3.flag("team", "member") and not cfg3.flag("group", "member")  # invertible probes at the root
    rng = np.random.default_rng(8)
    res = np.concatenate([rng.integers(0, cfg3.n_ns, 600), np.full(64, cfg3.n_ns - 1)]).astype(np.uint32)
    subj = np.concatenate([rng.integers(0, cfg3.n_users, 600), np.arange(64) % 8]).astype(np.uint32)
    want = cfg3.oracle_answers("namespace", "view", "user", res, subj)
    assert (want == GRANTED).any() and (want != GRANTED).any()
    items = cfg3.items("namespace", "view", "user", res, subj)
    for mark in (1, 0):
        got, _ = cfg3.run(items, mark)
        assert np.array_equal(got, want), (mark, np.flatnonzero(got != want)[:8])


def test_subjects_over_and_at_the_set_cap(cfg3):
    """User 0 has more memberships than the set holds, user 1 exactly kRsetCap: both answered, flag on and off."""
    res = np.tile(np.arange(cfg3.n_ns, dtype=np.uint32), 2)
    subj = np.repeat(np.array([0, 1], dtype=np.uint32), cfg3.n_ns)
    want = cfg3.oracle_answers("namespace", "view", "user", res, subj)
    assert (want == GRANTED).any()
    items = cfg3.items("namespace", "view", "user", res, subj)
    for mark in (1, 0):
        assert np.array_equal(cfg3.run(items, mark)[0], want)


def test_range_over_fcap_meets_over_the_index(cfg3):
    """Namespace n_ns - 1 lists 100 teams. Checked by a subject that reaches none of them, the meet over the closure
    row reads at most 4 bytes per child; walking the range would read two row offsets per child (8 bytes) and more."""
    reach = set()
    for u in range(2, cfg3.n_users):
        if cfg3.oracle_answers("namespace", "view", "user", [cfg3.n_ns - 1], [u])[0] != GRANTED:
            reach.add(u)
        if len(reach) == 3:
            break
    for u in sorted(reach) + [0]:  # user 0: over the cap, the path the flag gives every check
        items = cfg3.items("namespace", "view", "user", [cfg3.n_ns - 1], [u])
        want = cfg3.oracle_answers("namespace", "view", "user", [cfg3.n_ns - 1], [u])
        for mark in (1, 0):
            got, nb = cfg3.run(items, mark, count=True)
            assert got[0] == want[0]
            if want[0] != GRANTED:
                assert nb < 8 * 100, (u, mark, nb)


@pytest.mark.parametrize("depth", [ZG_MAX_DEPTH - 3, ZG_MAX_DEPTH - 2, ZG_MAX_DEPTH - 1, ZG_MAX_DEPTH])
def test_checks_at_the_depth_limit(cfg3, depth):
    """Raised at a depth where the two-level step may no longer meet: its children are pushed and visited without
    the set. Answers (including the depth errors) equal the flag-off run's, and the oracle's where it has room."""
    rng = np.random.default_rng(9 + depth)
    res = rng.integers(0, cfg3.n_ns, 200).astype(np.uint32)
    subj = rng.integers(0, cfg3.n_users, 200).astype(np.uint32)
    items = cfg3.items("namespace", "view", "user", res, subj, depth=depth)
    on, off = cfg3.run(items, 1)[0], cfg3.run(items, 0)[0]
    assert np.array_equal(on, off)
    if depth <= ZG_MAX_DEPTH - 3:
        assert np.array_equal(on, cfg3.oracle_answers("namespace", "view", "user", res, subj))


def test_count_bytes_fall_by_the_membership_reads(cfg3):
    """Flag off, a cfg3 check reads its subject's row offsets of the one non-empty invertible class (8 bytes) and,
    when they fit the set, its memberships (4 bytes each); flag on, neither. Nothing else differs."""
    rng = np.random.default_rng(11)
    res = rng.integers(0, cfg3.n_ns - 1, 512).astype(np.uint32)
    subj = rng.integers(0, cfg3.n_users, 512).astype(np.uint32)
    items = cfg3.items("namespace", "view", "user", res, subj)
    a_off, b_off = cfg3.run(items, 0, count=True)
    a_on, b_on = cfg3.run(items, 1, count=True)
    assert np.array_equal(a_on, a_off)
    g = np.zeros(cfg3.n_users, dtype=np.int64)
    for rt, rel, st, _res, sub, srel in cfg3_groups(np.random.default_rng(7))[0]:
        if (rt, rel, st, srel) == ("group", "member", "user", None):
            np.add.at(g, np.asarray(sub), 1)
    m = g[subj]
    adm = int(np.sum(8 + np.where(m <= RSET_CAP, 4 * m, 0)))
    assert b_off - b_on == adm, (b_off, b_on, adm)
    print(f"COUNT bytes per check: flag off {b_off / subj.size:.1f}, flag on {b_on / subj.size:.1f}")


def test_invertible_probe_at_the_root_keeps_the_flag_off(emu):
    """doc#view pushes namespace#view through an arrow, so namespace#viewer@user becomes an invertible class:
    namespace#view's root unit now probes it from the set, and neither permission may skip the set."""
    schema = CFG3 + """definition doc {
  relation ns: namespace
  relation viewer: user
  permission view = viewer + ns->view
}
"""
    rng = np.random.default_rng(12)
    groups, n_users, n_ns = cfg3_groups(rng)
    groups.append(("doc", "ns", "namespace", list(range(30)), list(rng.integers(0, n_ns, 30)), None))
    groups.append(("doc", "viewer", "user", list(range(0, 30, 3)), list(rng.integers(0, n_users, 10)), None))
    s = Store(emu, schema, groups)
    try:
        assert s.marked[1] > 0  # some slot still qualifies (namespace#viewer's relation slot is not pushed)
        assert not s.flag("namespace", "view") and not s.flag("doc", "view")
        for rt, n_res in (("namespace", n_ns), ("doc", 30)):
            res = rng.integers(0, n_res, 300).astype(np.uint32)
            subj = rng.integers(0, n_users, 300).astype(np.uint32)
            want = s.oracle_answers(rt, "view", "user", res, subj)
            for mark in (1, 0):
                assert np.array_equal(s.run(s.items(rt, "view", "user", res, subj), mark)[0], want)
    finally:
        s.close()
