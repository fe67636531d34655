"""Device ingress under the CPU SIMT emulator: the insert and resolve kernels of csrc/ingress.cuh, run unchanged
against a real Store (tests/emu/emu_ingress.cc), must give byte-identical items to the host resolver
zg_resolve_checks_packed of a host-only engine holding the same names. Also: the table synced incrementally while it
grows, the tag filter off, a blob that ends just before a PROT_NONE page, and zg_intern_objects_packed."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import emu_ingress as ei  # noqa: E402
import zgpu  # noqa: E402

SCHEMA = """
definition user {}
definition group {
  relation member: user | group#member
}
definition doc {
  relation viewer: user | group#member
  relation owner: user
  relation parent: doc
  permission view = viewer + owner + parent->view
}
"""


def _pair(names):
    """A host-only engine and an emulator store holding the same names (same ids)."""
    e, m = zgpu.Engine(SCHEMA, host_only=True), ei.EmuIngress(SCHEMA)
    for t, ids in names.items():
        a, b = e.intern_packed(t, ids), m.intern_packed(t, ids)
        assert np.array_equal(a, b)
    return e, m


def _same(e, m, res_type, rel, subj_type, res_ids, subjects, subj_rel="", o=None):
    want = e.resolve_checks_packed(res_type, rel, subj_type, res_ids, subjects, subj_rel=subj_rel)
    got = m.resolve_packed(res_type, rel, subj_type, res_ids, subjects, subj_rel=subj_rel, o=o)
    assert got.tobytes() == want.tobytes(), (res_type, rel, subj_type, subj_rel, np.flatnonzero(got != want)[:8])
    return got


def _random_ids(rng, n, max_len=1100):
    """Byte strings of length 0..max_len over every byte value, many sharing long prefixes."""
    prefixes = [bytes(rng.getrandbits(8) for _ in range(rng.choice([8, 63, 200, 1024]))) for _ in range(4)]
    out = set()
    while len(out) < n:
        k = rng.random()
        if k < 0.4:
            p = rng.choice(prefixes)
            s = p[:rng.randint(0, len(p))] + bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 12)))
        elif k < 0.8:
            s = bytes(rng.getrandbits(8) for _ in range(rng.randint(0, 48)))
        else:
            s = bytes(rng.getrandbits(8) for _ in range(rng.randint(0, max_len)))
        out.add(s[:max_len])
    return sorted(out)


@pytest.mark.parametrize("seed", [1, 2])
def test_random_bytes_match_host_resolver(seed):
    rng = random.Random(seed)
    ids = _random_ids(rng, 600)
    known = [i for i in ids if i and rng.random() < 0.6]
    e, m = _pair({"user": known, "group": known[: len(known) // 2], "doc": known[::3]})
    for n in (0, 1, 31, 33, 2000):
        res = [rng.choice(ids) for _ in range(n)]
        subj = [rng.choice(ids) if rng.random() < 0.7 else res[i] for i in range(n)]
        _same(e, m, "doc", "view", "user", res, subj)
        _same(e, m, "group", "member", "group", res, subj, subj_rel="member")  # self-membership on every unknown pair
        for one in (known[0], b"never-written", b""):
            _same(e, m, "group", "member", "group", res, one)
            _same(e, m, "doc", "viewer", "group", res, one, subj_rel="member")


def test_every_alignment_and_length():
    """Ids of every length 0..70 and 1 020..1 030 starting at every byte offset mod 8 of the blob."""
    lens = list(range(0, 71)) + list(range(1020, 1031))
    names = [bytes((7 * i + j) % 256 for j in range(L)) for i, L in enumerate(lens)]
    e, m = _pair({"user": [x for x in names if x], "doc": [x for x in names if x][::2]})
    for pad in range(8):
        res = [b"\x01" * pad] + names + [x + b"\x00" for x in names]  # the pad shifts every later id's alignment
        _same(e, m, "doc", "view", "user", res, list(reversed(res)))
        _same(e, m, "doc", "view", "user", res, names[9])


def test_punctuation_ids():
    ids = ["a/b", "a_b", "a|b", "a-b", "a=b", "a+b", "/", "_", "|", "-", "=", "+", "ns/p_1|x-y=z+w", "a/b/", "/a/b"]
    e, m = _pair({"user": ids[::2], "doc": ids[1::2], "group": ids})
    _same(e, m, "doc", "view", "user", ids, ids[::-1])
    _same(e, m, "group", "member", "group", ids + ["zz/never"], ids[::-1] + ["zz/never"], subj_rel="member")
    _same(e, m, "doc", "owner", "user", ids, "a/b")


def test_unknown_literals_give_error_items():
    e, m = _pair({"user": ["alice", "bob"], "doc": ["d1", "d2"], "group": ["g"]})
    res, subj = ["d1", "d2", "nope", ""], ["alice", "zed", "", "bob"]
    for args in (("nodoc", "view", "user", ""), ("doc", "nosuch", "user", ""), ("doc", "view", "nouser", ""),
                 ("doc", "viewer", "group", "nosuch"), ("doc", "viewer", "group", "..."), ("doc", "view", "user", "member")):
        got = _same(e, m, args[0], args[1], args[2], res, subj, subj_rel=args[3])
        _same(e, m, args[0], args[1], args[2], res, "alice", subj_rel=args[3])
        if args[1] != "viewer" or args[3] != "...":
            assert (got["perm"] == 0xFFFF).all() or args[3] == "..."


def test_never_written_and_self_membership():
    e, m = _pair({"group": ["g1", "g2"], "user": ["u1"]})
    got = _same(e, m, "group", "member", "group", ["g1", "x", "x", "x", "", ""], ["g1", "x", "y", "g2", "", "x"],
                subj_rel="member")
    assert list(got["res"][1:4]) == [0xFFFFFFFF] * 3
    assert list(got["subj"][1:4]) == [0xFFFFFFFF, 0xFFFFFFFE, 1]  # same bytes, same type: one never-written object
    got = _same(e, m, "group", "member", "group", ["x", "g1", "xy"], "x", subj_rel="member")
    assert list(got["subj"]) == [0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFE]
    # different types never compare equal
    got = _same(e, m, "doc", "viewer", "user", ["x"], ["x"])
    assert got["subj"][0] == 0xFFFFFFFE


@pytest.mark.parametrize("tag_filter,min_table", [(True, 1024), (True, 2), (False, 2), (False, 64)])
def test_table_grows_while_synced_incrementally(tag_filter, min_table):
    rng = random.Random(7)
    e, m = zgpu.Engine(SCHEMA, host_only=True), ei.EmuIngress(SCHEMA)
    o = ei.opts(tag_filter=tag_filter, min_table=min_table)
    all_names = []
    before = m.counters()
    for step, k in enumerate((1, 3, 10, 40, 150, 600, 2000)):
        new = ["s%d-%d-%s" % (step, i, "x" * rng.randint(0, 30)) for i in range(k)]
        assert np.array_equal(e.intern_packed("user", new), m.intern_packed("user", new))
        all_names += new
        q = [rng.choice(all_names) for _ in range(500)] + ["missing-%d" % i for i in range(20)]
        _same(e, m, "doc", "owner", "user", ["d"] * len(q), q, o=o)
        _same(e, m, "group", "member", "user", q[:50], q[50:100], o=o)
    c = m.counters()
    assert c["names"] == len(all_names)
    assert c["sync_uploads"] - before["sync_uploads"] == 7
    assert c["rebuilds"] >= (6 if min_table == 2 else 2)  # a 2-slot table is rebuilt by every sync after the first
    # a call with nothing new uploads nothing
    _same(e, m, "doc", "owner", "user", ["d"], [all_names[0]], o=o)
    assert m.counters()["sync_uploads"] == c["sync_uploads"]


def test_ids_after_numeric_bulk_load():
    e, m = zgpu.Engine(SCHEMA, host_only=True), ei.EmuIngress(SCHEMA)
    t = np.zeros(3, dtype=zgpu.TUPLE_DTYPE)
    t["res"], t["subj"] = [5, 9, 100], [7, 0, 42]
    t["rel"], t["stype"], t["srel"] = e.slot_id("doc", "viewer"), e.type_id("user"), zgpu.SREL_NONE
    e.load_tuples(t)
    m.load_tuples(t)
    names = ["after-%d" % i for i in range(10)]
    a, b = e.intern_packed("user", names), m.intern_packed("user", names)
    assert np.array_equal(a, b) and int(a[0]) == 43
    _same(e, m, "doc", "viewer", "user", ["x"] * 10, names)


_GUARD_SCRIPT = r"""
import sys
sys.path.insert(0, sys.argv[1])
import emu_ingress as ei, numpy as np
m = ei.EmuIngress(sys.argv[2])
names = ["g%d" % i + "y" * (i % 37) for i in range(300)]
m.intern_packed("user", names)
m.intern_packed("doc", names[::2])
ids = [n.encode() for n in names] + [b"never" * 51, b"z"]
for cut in range(len(ids) - 5, len(ids) + 1):
    part = ids[:cut]
    blob, off = ei.pack(part)
    rid = ei.guarded(blob)
    roff = ei.guarded(off.tobytes())
    sblob, soff = ei.pack(list(reversed(part)))
    sid = ei.guarded(sblob)
    so = ei.guarded(soff.tobytes())
    for o in (ei.opts(), ei.opts(tag_filter=False, min_table=2)):
        rc, a = m.resolve_ptr("doc", "view", "user", "", rid, roff, sid, so, len(part), o)
        assert rc == 0
        rc, b = m.resolve_ptr("doc", "view", "user", "", rid, roff, ei.guarded(part[-1] + b"\0"), None, len(part), o)
        assert rc == 0
print("ok")
"""


def test_no_read_past_the_blob():
    """Blobs, offsets and the one subject each end just before a PROT_NONE page: a read past the end of any of them
    faults the child process, which this test reports."""
    r = subprocess.run([sys.executable, "-c", _GUARD_SCRIPT, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"),
                        SCHEMA], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stderr[-2000:])


def test_decreasing_offset_is_refused():
    m = ei.EmuIngress(SCHEMA)
    m.intern_packed("user", ["a", "b"])
    off = np.array([0, 2, 1, 3], dtype=np.uint32)
    rc, _ = m.resolve_ptr("doc", "view", "user", "", b"abc\0", off.ctypes.data, b"a\0", None, 3)
    assert rc == -1
    e = zgpu.Engine(SCHEMA, host_only=True)
    with pytest.raises(zgpu.ZgpuError):
        e._ck(e._L.zg_intern_objects_packed(e._h, e.type_id("user"), b"abc", off.ctypes.data, 3,
                                            np.zeros(3, dtype=np.uint32).ctypes.data))


def test_bulk_intern_equals_one_by_one():
    rng = random.Random(3)
    names = ["n%d" % rng.randint(0, 400) for _ in range(1000)] + ["", "a/b", "x" * 1024]
    a, b = zgpu.Engine(SCHEMA, host_only=True), zgpu.Engine(SCHEMA, host_only=True)
    for _round in range(2):  # the second round re-interns every name
        bulk = a.intern_packed("user", names)
        one = np.array([b.intern("user", n) for n in names], dtype=np.uint32)
        assert np.array_equal(bulk, one)
    assert bulk[names.index("")] == 0xFFFFFFFF
    assert all(a.find("user", n) == i for n, i in zip(names, bulk) if n)
    with pytest.raises(zgpu.ZgpuError):
        a._ck(a._L.zg_intern_objects_packed(a._h, 99, b"x", np.array([0, 1], dtype=np.uint32).ctypes.data, 1,
                                            np.zeros(1, dtype=np.uint32).ctypes.data))


def test_device_calls_refused_on_host_only_engine():
    e = zgpu.Engine(SCHEMA, host_only=True)
    e.intern("user", "u")
    with pytest.raises(zgpu.ZgpuError) as ex:
        e.check_bulk_packed_ingress("doc", "view", "user", ["d"], "u")
    assert ex.value.code == -4
    with pytest.raises(zgpu.ZgpuError) as ex:
        e.resolve_checks_packed_device("doc", "view", "user", 1, 1, 1, 1, subjects="u")
    assert ex.value.code == -4
    assert e.ingress_counters() == {"names": 0, "device_bytes": 0, "sync_uploads": 0, "rebuilds": 0, "items_resolved": 0}
