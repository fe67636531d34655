"""The check kernel's specialised paths (csrc/kernels.cuh) on generated schemas whose stores reach them, under the SIMT
emulator (tests/emu/), against the oracle: tests/randgen.py shaped_schema composes a schema from units that compile
into each step kind, and shaped_relationships fills it with rows at the kernel's thresholds -- ranges around kFCap,
subjects around kRsetCap memberships split over classes, closure rows of 1 .. 33 entries, a two-level pair past
kMaxClosure, expiring classes, a leaf meet two subject types reach. Three drivers: emu.EmuEngine (no closure index:
every two-level step meets through batch_l2 or walks its range), the 16-bit index driver of test_rsetless_emulation.py
(indexed meets and SF_NO_RSET slots), and the closure_meet driver of test_closure_emulation.py (32-bit rows). GPU twin:
tests/test_gpu_step_shapes.py."""
import os
import random
import sys

import numpy as np
import pytest

_TESTS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, _TESTS)
sys.path.insert(0, os.path.join(_TESTS, "emu"))
sys.path.insert(0, os.path.dirname(_TESTS))

import randgen as R  # noqa: E402
from test_closure_emulation import build_index, meet, run  # noqa: E402,F401  (meet: the closure_meet driver fixture)
from test_rsetless_emulation import Store, emu  # noqa: E402,F401  (emu: the 16-bit index driver fixture)

SEEDS = list(range(5))
SMALL = dict(n_user=500, n_bot=80, n_group=260, n_crew=60, n_pair=70, n_folder=24, n_doc=110)
N_CHECKS = 800
HAS = 2


def _case(seed, **kw):
    rng = random.Random(seed)
    text, plan = R.shaped_schema(rng, **{k: kw.pop(k) for k in ("n_pairs", "expiry", "wildcard") if k in kw})
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan, **{**SMALL, **kw})
    return rng, text, plan, store


def _seed_plan(seed):
    """Seeds 0 .. 4 take 1 .. 5 pairs; the rest draw."""
    return {"n_pairs": seed + 1} if seed < 5 else {}


def _fail(seed, text, got, want, queries, res, subj, label):
    bad = np.flatnonzero(got != want)
    first = [(queries[i], int(res[i]), int(subj[i]), int(got[i]), int(want[i])) for i in bad[:6]]
    return f"seed {seed} [{label}]: {bad.size} mismatches, first {first}\n{text}"


def assert_buckets(store):
    """The buckets the checks are drawn from exist in the data (computed from the generated rows)."""
    g = {(rt, rel, st): (res, subj) for rt, rel, st, res, subj, srel, ex in store["groups"] if ex is None}
    cnt = np.zeros((3, store["n"]["user"]), dtype=np.int64)
    for k, key in enumerate((("group", "member", "user"), ("role", "member", "user"), ("folder", "viewer", "user"))):
        np.add.at(cnt[k], g[key][1], 1)
    tot = cnt.sum(axis=0)
    for m in (R.RSET_CAP - 1, R.RSET_CAP, R.RSET_CAP + 1):
        assert ((tot == m) & (cnt.max(axis=0) == m)).any(), f"no user with {m} memberships in one class"
    for m in (R.RSET_CAP, R.RSET_CAP + 1):
        assert ((tot == m) & ((cnt > 0).sum(axis=0) == 2)).any(), f"no user with {m} memberships over two classes"
        assert ((tot == m) & ((cnt > 0).sum(axis=0) == 3)).any(), f"no user with {m} memberships over three classes"
    # the cap falls inside the second class: fewer than kRsetCap in the first, more than kRsetCap in the first two
    assert ((cnt[0] < R.RSET_CAP) & (cnt[0] + cnt[1] > R.RSET_CAP)).any()
    # leaf-meet ranges (doc#reader's groups) on both sides of the membership counts the meet compares them with
    reader = np.bincount(g[("doc", "reader", "group")][0])
    for s in (1, R.RSET_CAP - 1, R.RSET_CAP, R.RSET_CAP + 1):
        assert (reader == s).any(), f"no reader range of {s} children"
    # two-level ranges (doc#l2's objects of the first pair) around kFCap, which picks batch_l2 / closure_meet or the
    # per-lane intersection
    crow, rows, _col, ptr = R.closure_rows(store, store["pairs"][0])
    l2 = np.diff(ptr)
    for s in (R.FCAP - 1, R.FCAP, R.FCAP + 1):
        assert (l2 == s).any(), f"no two-level range of {s} children"
    assert l2.max() > R.FCAP + 1
    # closure rows of every size in CLOSURE_SIZES, each starting at every offset mod 16 (so mod 4 too)
    lens = np.diff(crow)
    for k in R.CLOSURE_SIZES:
        starts = {int(b) % 16 for b in crow[:-1][lens == k]}
        assert starts == set(range(16)), f"closure rows of {k} entries start at offsets {sorted(starts)} mod 16"


@pytest.mark.parametrize("seed", [0, 2, 4])
def test_shaped_schemas_without_index(seed):
    """EmuEngine: leaf meets, batch_l2 over ranges up to kFCap and walks past it, admission around the cap, the bot
    subject on a step built for users, userset subjects, sub-query passes, the path memo, forward only, two clocks."""
    import emu as E
    from oracle.pyoracle import Oracle

    rng, text, plan, store = _case(seed, **_seed_plan(seed))
    assert_buckets(store)
    e, o = E.EmuEngine(text), Oracle(text)
    R.load_shaped(e, store), R.load_shaped(o, store)
    e.publish()
    queries, res, subj = R.shaped_checks(rng, store, plan, N_CHECKS)
    items = R.shaped_items(e, E.CHECK_DTYPE, queries, res, subj)
    assert np.array_equal(items, R.shaped_items(o, E.CHECK_DTYPE, queries, res, subj))
    clocks = (store["now"], store["now"] + 1000) if plan["expiry"] else (store["now"],)
    passes = memo = 0
    for now in clocks:
        want = o.check_bulk(items, now=now)
        assert 0.05 < (want == HAS).mean() < 0.95
        for label, opts in (("default", E.default_opts(now=now)), ("forward", E.default_opts(now=now, invert=0)),
                            ("memo", E.default_opts(now=now, memo_after=0))):
            got = e.check_bulk(items, opts)
            assert np.array_equal(got, want), _fail(seed, text, got, want, queries, res, subj, f"{label} now={now}")
            passes += e.stat("passes")
            memo += e.stat("memo_batches") if label == "memo" else 0
    assert passes > 0 and memo > 0, (passes, memo)


@pytest.mark.parametrize("seed", SEEDS)
def test_shaped_schemas_over_the_closure_index(emu, seed):
    """The 16-bit index driver: the first kMaxClosure pairs indexed, the SF_NO_RSET slots built to qualify marked, and
    every pure permission's answers equal to the oracle's with the flags on and off."""
    rng, text, plan, store = _case(seed, **_seed_plan(seed), expiry=False, wildcard=False)
    s = Store(emu, text, [g[:6] for g in store["groups"]])
    try:
        assert s.L.emu_index_pairs(s.idx[1]) == min(len(plan["pairs"]), R.MAX_CLOSURE)
        for p in plan["rsetless"]:
            assert s.flag("doc", p), (seed, p)
        if "with5" in plan["perms"]:
            assert not s.flag("doc", "with5")  # its fifth pair has no index: it keeps the set
        queries, res, subj = R.shaped_checks(rng, store, plan, N_CHECKS)
        keep = [i for i, q in enumerate(queries) if q[3] is None and (q[0] == "folder" or q[1] in plan["pure"] + ["l2"])]
        queries, res, subj = [queries[i] for i in keep], res[keep], subj[keep]
        ids = type("Ids", (), {"slot_id": lambda _, t, r: s.slot(t, r), "type_id": lambda _, t: s.type(t)})()
        items = R.shaped_items(ids, s.E.CHECK_DTYPE, queries, res, subj)
        want = s.oracle.check_bulk(items)
        for mark in (1, 0):
            got, _ = s.run(items, mark)
            assert np.array_equal(got, want), _fail(seed, text, got, want, queries, res, subj, f"index, flags {mark}")
    finally:
        s.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_shaped_closure_rows_with_32_bit_entries(meet, seed):
    """closure_meet over 32-bit rows (pair-type ids past 65 536) of 1 .. 33 entries starting at every offset mod 4,
    whose neighbours hold children of the ranges: one entry read past a row's end turns a NO into HAS."""
    _rng, _text, _plan, store = _case(seed, n_pairs=2, wide=True)
    crow_data, rows, col, ptr = R.closure_rows(store, "team")
    assert int(col.max()) > 65536
    crow, ccol = build_index(rows)
    assert np.array_equal(crow, crow_data)  # rows of every CLOSURE_SIZES length at every offset (assert_buckets)
    assert_buckets(store)
    rng = np.random.default_rng(seed)
    users = np.array(sorted(store["closure"]) + list(rng.integers(0, len(rows), 200)), dtype=np.uint32)
    docs = np.flatnonzero(np.diff(ptr) > 0)
    n = 32 * ((users.size * 6 + 31) // 32)
    u = np.resize(np.repeat(users, 6), n)
    d = rng.choice(docs, n)
    lanes = np.stack([np.ones(n, np.uint32), ptr[d], ptr[d + 1], u, np.tile(np.arange(32, dtype=np.uint32), n // 32)],
                     axis=1).reshape(-1, 32, 5).astype(np.uint32)
    hits, _ = run(meet, col, crow, ccol, len(rows), lanes)
    want = np.array([np.intersect1d(col[ptr[a]:ptr[a + 1]], rows[b]).size > 0 for a, b in zip(d, u)]).reshape(-1, 32)
    got = ((hits[:, None] >> np.arange(32)) & 1).astype(bool)
    assert 0.05 < want.mean() < 0.95
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"seed {seed}: {len(bad)} lanes differ, first (warp, lane) {bad[:6].tolist()}"


CHAIN = """definition user {}
definition group { relation member: user }
definition team { relation member: group#member }
definition folder {
  relation parent: folder
  relation viewer: group#member
  relation lead: team#member
  permission view = viewer + lead + parent->view
}
"""
CHAIN_LEN = 60


def chain_store():
    """folder i's parent is folder i + 1; the last folder's viewer is group 0 (user 0) and its lead team 0 (group 1,
    user 1): a check of folder last - h reaches user 0 in h hops and a leaf meet, user 1 in h hops and a two-level
    meet."""
    last = CHAIN_LEN - 1
    return [("folder", "parent", "folder", np.arange(last), np.arange(1, CHAIN_LEN), None),
            ("folder", "viewer", "group", [last], [0], "member"), ("folder", "lead", "team", [last], [0], "member"),
            ("team", "member", "group", [0], [1], "member"), ("group", "member", "user", [0, 1], [0, 1], None)]


def chain_items(t, dtype):
    hops = np.arange(40, CHAIN_LEN)
    res = np.repeat(CHAIN_LEN - 1 - hops, 3).astype(np.uint32)
    subj = np.tile(np.array([0, 1, 2], dtype=np.uint32), hops.size)
    items = np.zeros(res.size, dtype=dtype)
    items["res"], items["subj"] = res, subj
    items["perm"], items["stype"], items["srel"] = t.slot_id("folder", "view"), t.type_id("user"), 0xFFFF
    return items


def test_depth_cap_through_each_meet(emu):
    """Leaf meets at depth 49 and 50 and two-level meets at 48 and 49, with and without the index: HAS where the
    path fits ZG_MAX_DEPTH, the oracle's answer (ERROR) one hop further."""
    import emu as E
    from oracle.pyoracle import Oracle

    groups = chain_store()
    o = Oracle(CHAIN)
    for rt, rel, st, res, subj, srel in groups:
        o.add_bulk(rt, rel, st, np.asarray(res), np.asarray(subj), srel=srel)
    items = chain_items(o, E.CHECK_DTYPE)
    want = o.check_bulk(items)
    for k in (0, 1):  # user 0 (leaf) and user 1 (two levels): HAS at the deepest path that fits, ERROR past it
        w = want[k::3]
        assert (w == HAS).any() and (w == 255).any() and np.all(np.diff((w == 255).astype(int)) >= 0), w
    e = E.EmuEngine(CHAIN)
    for rt, rel, st, res, subj, srel in groups:
        e.add_bulk(rt, rel, st, res, subj, srel=srel)
    e.publish()
    for opts in (E.default_opts(), E.default_opts(invert=0)):
        assert np.array_equal(e.check_bulk(items, opts), want), (e.check_bulk(items, opts), want)
    s = Store(emu, CHAIN, groups)
    try:
        assert s.L.emu_index_pairs(s.idx[1]) == 1
        for mark in (1, 0):
            got, _ = s.run(items, mark)
            assert np.array_equal(got, want), (mark, got, want)
    finally:
        s.close()


def hub_schema(k):
    """user is the subject of k invertible classes (hub#h0 .. hub#h{k-1}, each pushed by doc#v0 or doc#v1: a relation
    allows at most 8 subject kinds)."""
    rels = "".join(f"  relation h{i}: user\n" for i in range(k))
    half = (k + 1) // 2
    return ("definition user {}\ndefinition hub {\n" + rels + "}\ndefinition doc {\n" +
            "".join(f"  relation v{j}: " + " | ".join(f"hub#h{i}" for i in r) + "\n"
                    for j, r in enumerate((range(half), range(half, k)))) + "  permission view = v0 + v1\n}\n")


def hub_store(k, seed, n_user=64, n_hub=40, n_doc=40):
    """User u holds min(u // 2, 24) memberships, dealt round-robin over the k classes to distinct hub objects of each
    class (so 16 and 17 cross the cap inside a class past the first); docs list hub objects of every class."""
    rng = np.random.default_rng(seed)
    groups = []
    mem = {i: [] for i in range(k)}
    for u in range(n_user):
        m = min(u // 2, 24)
        for i in range(k):
            mem[i] += [(int(h), u) for h in rng.choice(n_hub, len(range(i, m, k)), replace=False)]
    for i in range(k):
        rows = sorted(mem[i])
        groups.append(("hub", f"h{i}", "user", [a for a, _ in rows], [b for _, b in rows], None))
        d = sorted({(int(rng.integers(0, n_doc)), int(rng.integers(0, n_hub))) for _ in range(3 * n_doc)})
        groups.append(("doc", f"v{int(i >= (k + 1) // 2)}", "hub", [a for a, _ in d], [b for _, b in d], f"h{i}"))
    return groups, n_user, n_doc


def assert_hub_buckets(groups, k, n_user):
    """From the data: users with exactly kRsetCap and kRsetCap + 1 memberships, and one of the latter whose
    memberships cross the cap in a class past the first: part-way through that class where classes hold two or more
    of a user's memberships (k = 2, 3), at its first membership where they hold one or two (k = 11, 12)."""
    cnt = np.zeros((k, n_user), dtype=np.int64)
    for rt, rel, st, res, subj, srel in groups:
        if rt == "hub":
            np.add.at(cnt[int(rel[1:])], np.asarray(subj), 1)
    cum = np.cumsum(cnt, axis=0)
    tot = cum[-1]
    assert (tot == R.RSET_CAP).any() and (tot == R.RSET_CAP + 1).any(), tot
    before = cum[:-1] < R.RSET_CAP if k <= 3 else cum[:-1] <= R.RSET_CAP
    inside = before & (cum[1:] > R.RSET_CAP)  # class j + 1 holds the crossing
    assert (inside[:, tot == R.RSET_CAP + 1]).any(), cnt[:, tot == R.RSET_CAP + 1]


@pytest.mark.parametrize("k", [2, 3, R.MAX_INV_CLASSES, R.MAX_INV_CLASSES + 1])
def test_admission_at_the_set_cap_split_over_classes(k):
    """Memberships 0 .. 24 spread over k classes (16 and 17 with the cap inside a later class); k = 12 is one class
    past kMaxInvClasses, where the check does not meet at all."""
    import emu as E
    from oracle.pyoracle import Oracle

    text = hub_schema(k)
    groups, n_user, n_doc = hub_store(k, seed=k)
    assert_hub_buckets(groups, k, n_user)
    e, o = E.EmuEngine(text), Oracle(text)
    for t in (e, o):
        for rt, rel, st, res, subj, srel in groups:
            t.add_bulk(rt, rel, st, np.asarray(res), np.asarray(subj), srel=srel)
    e.publish()
    items = np.zeros(n_doc * n_user, dtype=E.CHECK_DTYPE)
    items["res"], items["subj"] = np.repeat(np.arange(n_doc), n_user), np.tile(np.arange(n_user), n_doc)
    items["perm"], items["stype"], items["srel"] = e.slot_id("doc", "view"), e.type_id("user"), 0xFFFF
    want = o.check_bulk(items)
    assert 0.05 < (want == HAS).mean() < 0.95
    for opts in (E.default_opts(), E.default_opts(invert=0)):
        got = e.check_bulk(items, opts)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"k={k}: first (doc, user) {[(int(items['res'][i]), int(items['subj'][i])) for i in bad[:6]]}"
