"""zg_import_relationships' kernels (csrc/import.cuh) under the CPU SIMT emulator (tests/emu/emu_import.cc), against
the host path of a host-only engine holding the same names and relationships: the tuples in call order, the new names'
ids and arena records, and the first malformed id or duplicate must be identical. Covered: ids at every byte alignment
and up to 1 024 bytes, names repeated across groups and across the subject and resource columns, every probe comparing
bytes (tag filter off), duplicates within the call and against the store, at the start, middle and end of a call."""
import os
import random
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import emu_import as em  # noqa: E402
import zgpu  # noqa: E402

SCHEMA = """
definition user {}
definition group { relation member: user | user:* | group#member }
definition doc {
  relation viewer: user | user:* | group#member
  relation owner: user
  permission view = viewer + owner
}
"""
WILD, NONE = 0xFFFE, 0xFFFF
CHARS = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789/_|-=+"


def _name(rng, lo=1, hi=40):
    return "".join(rng.choice(CHARS) for _ in range(rng.randint(lo, hi)))


def _pair(prior_names=None, prior_rels=()):
    """A host-only engine and an emulator store with the same names (same ids) and relationships."""
    e, m = zgpu.Engine(SCHEMA, host_only=True), em.EmuImport(SCHEMA)
    for t, ids in (prior_names or {}).items():
        assert np.array_equal(e.intern_packed(t, ids), m.intern_packed(t, ids))
    if prior_rels:
        e.write_relationships([(1, r, 0) for r in prior_rels])
        t = np.zeros(len(prior_rels), dtype=em.TUPLE_DTYPE)
        for i, r in enumerate(prior_rels):
            rt, rid, rel, st, sid, srel = zgpu._lib.split_rel(r)
            if sid != "*":  # the write path interns the subject's name, then the resource's
                assert m.intern_packed(st, [sid])[0] == e.find(st, sid)
            assert m.intern_packed(rt, [rid])[0] == e.find(rt, rid)
            t[i] = (e.find(rt, rid), 0 if sid == "*" else e.find(st, sid), e.slot_id(rt, rel), e.type_id(st),
                    WILD if sid == "*" else (NONE if not srel else e.slot_id(st, srel)), 0)
        m.load_tuples(t)
    return e, m


def _expected(e, groups, before):
    """The host path's tuples in call order and the records its new names appended, per type."""
    tuples, recs, seen = [], {}, set(before)
    for rt, rel, st, srel, res, subj, _ in groups:
        for rid, sid in zip(res, subj):
            for t, x in ((st, sid), (rt, rid)):
                if (t, x) not in seen and not (t == st and x == sid and sid == "*"):
                    seen.add((t, x))
                    b = x.encode()
                    recs[t] = recs.get(t, b"") + struct.pack("<II", e.find(t, x), len(b)) + b
            tuples.append((e.find(rt, rid), 0 if sid == "*" else e.find(st, sid), e.slot_id(rt, rel), e.type_id(st),
                           WILD if sid == "*" else (NONE if not srel else e.slot_id(st, srel)), 0))
    return np.array(tuples, dtype=em.TUPLE_DTYPE), recs


def _names(e):
    out = set()
    for t in ("user", "group", "doc"):
        for i in range(e.name_counters()["id_extent"] + 1):
            try:
                out.add((t, e.object_name(t, i)))
            except zgpu.ZgpuError:
                pass
    return out


def _same(e, m, groups, o=None, pads=None):
    before = _names(e)
    arenas = {t: m.arena(t) for t in ("user", "group", "doc")}
    try:
        e.import_relationships(groups)
        want_err = None
    except zgpu.ZgpuError as ex:
        want_err = (ex.code, int(str(ex).split("relationship ")[1].split()[0].rstrip(":")))
    bad, dup, _, got = m.run(groups, o, pads)
    if want_err is not None:
        first = min(x for x in (bad, dup) if x is not None)
        assert (want_err[1], want_err[0]) == (first, -1 if first == bad else -2)
        assert {t: m.arena(t) for t in arenas} == arenas  # nothing interned
        return want_err
    assert bad is None and dup is None
    want, recs = _expected(e, groups, before)
    assert got.tobytes() == want.tobytes()
    for t in arenas:
        assert m.arena(t) == arenas[t] + recs.get(t, b"")
    return None


def _groups(rng, n_items, names, wild=0.1):
    """Groups over a pool of names: doc#viewer@user, group#member@group#member (one pool both columns),
    doc#viewer@group#member, doc#owner@user, with wildcard subjects; pairs unique."""
    gs, used = [], set()
    for rt, rel, st, srel in (("doc", "viewer", "user", ""), ("group", "member", "group", "member"),
                              ("doc", "viewer", "group", "member"), ("doc", "owner", "user", ""),
                              ("group", "member", "user", "")):
        res, subj = [], []
        for _ in range(n_items):
            r = rng.choice(names[rt])
            s = "*" if st == "user" and rel != "owner" and rng.random() < wild else rng.choice(names[st])
            if (rt, rel, st, srel, r, s) in used:
                continue
            used.add((rt, rel, st, srel, r, s))
            res.append(r)
            subj.append(s)
        gs.append((rt, rel, st, srel, res, subj, None))
    return gs


def _pool(rng, k, lo=1, hi=40):
    return {t: list({_name(rng, lo, hi) for _ in range(k)}) for t in ("user", "group", "doc")}


@pytest.mark.parametrize("tag_filter", [True, False])
def test_random_calls_equal_the_host_path(tag_filter):
    rng = random.Random(1 + tag_filter)
    names = _pool(rng, 30)
    prior = {t: v[:10] for t, v in names.items()}
    e, m = _pair(prior, ["doc:%s#viewer@user:%s" % (names["doc"][0], names["user"][0])])
    stored = {("doc", "viewer", "user", "", names["doc"][0], names["user"][0])}
    for k in range(3):
        gs = _groups(rng, 25, {t: v + [_name(rng) for _ in range(5)] for t, v in names.items()})
        keep = [[(r, s) for r, s in zip(res, subj) if (rt, rel, st, srel, r, s) not in stored]
                for rt, rel, st, srel, res, subj, _ in gs]
        gs = [(rt, rel, st, srel, [r for r, _ in kp], [s for _, s in kp], None)
              for (rt, rel, st, srel, _, _, _), kp in zip(gs, keep)]
        assert _same(e, m, gs, em.opts(tag_filter)) is None
        stored |= {(rt, rel, st, srel, r, s) for rt, rel, st, srel, res, subj, _ in gs for r, s in zip(res, subj)}


def test_ids_at_every_alignment_and_length():
    rng = random.Random(5)
    lengths = list(range(1, 18)) + [63, 64, 65, 255, 256, 1023, 1024]
    res = [_name(rng, n, n) for n in lengths]
    subj = [_name(rng, n, n) for n in reversed(lengths)]
    for pad in range(8):
        e, m = _pair()
        gs = [("doc", "viewer", "user", "", res, subj, None), ("doc", "owner", "user", "", subj[:5], res[:5], None)]
        assert _same(e, m, gs, pads=[(pad, 7 - pad), ((pad * 3) % 8, pad)]) is None


def test_name_in_both_columns_and_across_groups():
    e, m = _pair({"group": ["old"]})
    gs = [("group", "member", "group", "member", ["a", "b", "old"], ["b", "c", "a"], None),
          ("doc", "viewer", "group", "member", ["d1", "d1"], ["c", "old"], None),
          ("group", "member", "user", "", ["c", "a"], ["u", "*"], None)]
    assert _same(e, m, gs, em.opts(False)) is None


@pytest.mark.parametrize("where", ["start", "middle", "end"])
@pytest.mark.parametrize("kind", ["bad_res", "bad_subj", "wild_res", "too_long", "dup_call", "dup_store"])
def test_first_offender(where, kind):
    rng = random.Random(hash((where, kind)) & 0xFFFF)
    n = 40
    res = ["r%d" % i for i in range(n)]
    subj = ["s%d" % (i % 7) for i in range(n)]
    at = {"start": 0, "middle": n // 2, "end": n - 1}[where]
    e, m = _pair({"user": ["s0", "s1"], "doc": ["r0", "r%d" % (n // 2), "r%d" % (n - 1)]},
                 ["doc:r%d#viewer@user:s%d" % (at, at % 7)] if kind == "dup_store" else [])
    if kind == "bad_res":
        res[at] = "bad!"
    elif kind == "bad_subj":
        subj[at] = "no space"
    elif kind == "wild_res":
        res[at] = "*"
    elif kind == "too_long":
        res[at] = "x" * 1025
    elif kind == "dup_call":
        if at == 0:
            at = 1
        res[at], subj[at] = res[at - 1 - rng.randrange(at)], None
        j = res.index(res[at])
        subj[at] = subj[j]
    # a later duplicate and a later bad id must not be the ones reported
    res.append(res[0])
    subj.append(subj[0])
    res.append("later!")
    subj.append("s1")
    err = _same(e, m, [("doc", "viewer", "user", "", res, subj, None)])
    assert err is not None and err[1] == at
