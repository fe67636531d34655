"""The closure index of the two-level meet (csrc/build.cu gpu_build_closure, csrc/kernels.cuh closure_meet) on the GPU:
its size against a numpy construction from the same relationships, answers against the oracle and against the same
engine without the index (ZGPU_CLOSURE_CAP=0: every two-level step meets through batch_l2), after writes too."""
import numpy as np
import pytest

import l2_batch_cases as B

pytestmark = pytest.mark.gpu


def _closure_index(n_users, gm_group, gm_user, tm_team, tm_group):
    """(row_ptr, col) of the closure index built in numpy: row u = the teams user u reaches through a group,
    ascending and distinct."""
    g2t = {}
    for t, g in zip(np.asarray(tm_team).tolist(), np.asarray(tm_group).tolist()):
        g2t.setdefault(g, set()).add(t)
    rows = [set() for _ in range(n_users)]
    for g, u in set(zip(np.asarray(gm_group).tolist(), np.asarray(gm_user).tolist())):
        rows[u].update(g2t.get(g, ()))
    row_ptr = np.zeros(n_users + 1, dtype=np.uint32)
    row_ptr[1:] = np.cumsum([len(r) for r in rows])
    col = np.array([t for r in rows for t in sorted(r)], dtype=np.uint32)
    return row_ptr, col


def _assert_index_equals(e, pair, gm_group, gm_user, tm_team, tm_group):
    row_ptr, col = e.closure_index(pair)
    want_ptr, want_col = _closure_index(row_ptr.size - 1, gm_group, gm_user, tm_team, tm_group)
    assert int(np.asarray(gm_user).max()) < row_ptr.size
    assert np.array_equal(row_ptr, want_ptr)
    assert np.array_equal(col, want_col)


def _engines(schema, load, monkeypatch):
    import zgpu

    e = zgpu.Engine(schema, device=0)
    load(e), e.publish()
    monkeypatch.setenv("ZGPU_CLOSURE_CAP", "0")
    f = zgpu.Engine(schema, device=0)
    load(f), f.publish()
    monkeypatch.delenv("ZGPU_CLOSURE_CAP")
    return e, f


def test_cfg3_index_size_and_answers(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.1)
    e, f = _engines(w.schema, w.load_into, monkeypatch)
    gm, tm = w.groups[0], w.groups[1]
    ce, cf = e.closure_index_counters(), f.closure_index_counters()
    assert ce["indexed"] == 1 and ce["over_budget"] == 0, ce
    _assert_index_equals(e, 0, gm.res, gm.subj, tm.res, tm.subj)
    assert ce["entries"] == e.closure_index(0)[1].size, ce
    assert cf["indexed"] == 0 and cf["over_budget"] == 1 and cf["entries"] == 0, cf
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    want = o.check_bulk(items)
    assert np.array_equal(e.check_bulk(items), want)
    assert np.array_equal(f.check_bulk(items), want)
    # the byte model: the index streams far fewer bytes than the memberships' rows
    assert e.count_alg_bytes(items[:20000]) < f.count_alg_bytes(items[:20000])
    for rt, perm, st, u in w.lookups[:4]:
        assert np.array_equal(e.lookup_resources_ids(rt, perm, st, u), o.lookup_resources_ids(rt, perm, st, u))
    # LookupSubjects: exactly the users the oracle grants among every user id (cfg3 has no wildcard)
    c = w.checks[0]
    n_users = int(gm.subj.max()) + 1
    for res in c.res[:3]:
        ids, wild, ex = e.lookup_subjects_ids(c.res_type, int(res), c.perm, c.subj_type)
        q = np.zeros(n_users, dtype=zgpu.CHECK_DTYPE)
        q["res"], q["subj"] = int(res), np.arange(n_users)
        q["perm"], q["stype"], q["srel"] = o.slot_id(c.res_type, c.perm), o.type_id(c.subj_type), zgpu.SREL_NONE
        assert np.array_equal(ids, np.flatnonzero(o.check_bulk(q) == 2)) and not wild and ex.size == 0


def test_cfg3_full_size_equals_the_meet_without_index(monkeypatch):
    import zgpu
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3()
    e, f = _engines(w.schema, w.load_into, monkeypatch)
    c = e.closure_index_counters()
    assert c["indexed"] == 1, c
    print(f"cfg3 full-size closure index: {c}")
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    assert np.array_equal(e.check_bulk(items), f.check_bulk(items))


@pytest.mark.parametrize("case", ["mixed", "collisions"])
def test_two_level_meet_sweeps_with_the_index(case, monkeypatch):
    """The shapes of the batched meet's sweeps (tests/l2_batch_cases.py): range sizes around kFCap, 1 .. 24
    memberships, filter collisions."""
    import zgpu
    from oracle.pyoracle import Oracle

    if case == "mixed":
        groups, checks = B.mixed_case()
    else:
        groups, cases = B.collision_cases(4000)
        checks = [q for q, _ in cases]
    e, f = _engines(B.SCHEMA, lambda x: B.load(x, groups), monkeypatch)
    assert e.closure_index_counters()["indexed"] == 1
    o = Oracle(B.SCHEMA)
    B.load(o, groups)
    want = o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE))
    assert np.array_equal(e.check_bulk(B.items(e, checks, zgpu.CHECK_DTYPE)), want)
    assert np.array_equal(f.check_bulk(B.items(f, checks, zgpu.CHECK_DTYPE)), want)
    if case == "collisions":
        assert [int(x) for x in want] == [v for _, v in cases]


RANDOM_SCHEMA = """definition user {}
definition group { relation member: user | group#member }
definition team {
  relation member: group#member
  relation lead: user
}
definition org { relation member: group#member }
definition namespace {
  relation viewer: team#member
  relation admin: org#member
  relation owner: user
  permission view = viewer + admin + owner
  permission manage = admin + owner
}"""


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_two_level_schemas(seed, monkeypatch):
    """Two pairs (team#member, org#member over group#member) with random fan-outs; nested groups make group#member
    not a leaf for some seeds' data, which leaves the steps without a two-level meet."""
    import zgpu
    from oracle.pyoracle import Oracle

    rng = np.random.default_rng(seed)
    nu, ng, nt, no, nn = 300, 120, 60, 30, 200
    nested = seed == 3
    r = lambda hi, n: rng.integers(0, hi, n, dtype=np.uint32)  # noqa: E731
    rels = [("group", "member", "user", r(ng, 900), r(nu, 900), None),
            ("team", "member", "group", r(nt, 400), r(ng, 400), "member"),
            ("team", "lead", "user", r(nt, 50), r(nu, 50), None),
            ("org", "member", "group", r(no, 150), r(ng, 150), "member"),
            ("namespace", "viewer", "team", r(nn, 1500), r(nt, 1500), "member"),
            ("namespace", "admin", "org", r(nn, 300), r(no, 300), "member"),
            ("namespace", "owner", "user", r(nn, 100), r(nu, 100), None)]
    if nested:  # acyclic: a group nests only groups of lower ids
        sub = rng.integers(1, ng, 40, dtype=np.uint32)
        rels.append(("group", "member", "group", sub, sub // 2, "member"))

    def load(x):
        for rt, rel, st, res, subj, srel in rels:
            x.add_bulk(rt, rel, st, res, subj, srel=srel)

    e, f = _engines(RANDOM_SCHEMA, load, monkeypatch)
    assert e.closure_index_counters()["indexed"] == (0 if nested else 2), e.closure_index_counters()
    if not nested:  # one pair through team#member, one through org#member, in the program's step order
        gm, tm, om = rels[0], rels[1], rels[3]
        got = [e.closure_index(k) for k in range(2)]
        want = [_closure_index(got[0][0].size - 1, gm[3], gm[4], x[3], x[4]) for x in (tm, om)]
        same = lambda a, b: np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])  # noqa: E731
        assert (same(got[0], want[0]) and same(got[1], want[1])) or (same(got[0], want[1]) and same(got[1], want[0]))
    o = Oracle(RANDOM_SCHEMA)
    load(o)
    n = 20000
    items = np.zeros(n, dtype=zgpu.CHECK_DTYPE)
    items["res"] = rng.integers(0, nn + 5, n)
    items["subj"] = rng.integers(0, nu + 5, n)  # ids past every class's subjects too
    items["perm"] = np.where(rng.random(n) < 0.7, e.slot_id("namespace", "view"), e.slot_id("namespace", "manage"))
    items["stype"], items["srel"] = e.type_id("user"), zgpu.SREL_NONE
    want = o.check_bulk(items)
    assert np.array_equal(e.check_bulk(items), want)
    assert np.array_equal(f.check_bulk(items), want)
    assert 0.05 < (want == 2).mean() < 0.95


def test_writes_rebuild_the_index(monkeypatch):
    """5 x 1000 writes touching group#member and team#member (inserts and deletes): each publish merges them and
    rebuilds the index from the merged rows; answers equal the oracle's after every publish."""
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.02)
    e, o = zgpu.Engine(w.schema, device=0), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    rng = np.random.default_rng(11)
    builds = e.closure_index_counters()["builds"]
    for step in range(5):
        ups = np.zeros(1000, dtype=zgpu.UPDATE_DTYPE)
        for i in range(ups.size):
            g = w.groups[int(rng.integers(0, 2))]  # group#member@user, team#member@group#member
            ups["rel"][i], ups["stype"][i] = e.slot_id(g.res_type, g.rel), e.type_id(g.subj_type)
            ups["srel"][i] = zgpu.SREL_NONE if g.srel is None else e.slot_id(g.subj_type, g.srel)
            k = int(rng.integers(0, g.res.size))
            if rng.random() < 0.5:
                ups["res"][i], ups["subj"][i], ups["op"][i] = g.res[k], g.subj[k], 2  # DELETE
            else:
                ups["res"][i] = g.res[int(rng.integers(0, g.res.size))]
                ups["subj"][i], ups["op"][i] = g.subj[k], 0  # TOUCH of a new pairing: an insert
        key = np.stack([ups["rel"], ups["res"], ups["stype"], ups["srel"], ups["subj"]], axis=1)
        ups = ups[np.sort(np.unique(key, axis=0, return_index=True)[1])]
        e.apply_updates(ups), o.apply_updates(ups)
        e.publish()
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items)), f"step {step}"
    st, c = e.stats(), e.closure_index_counters()
    assert st["delta_publishes"] >= 4, st
    assert c["builds"] >= builds + 4 and c["indexed"] == 1, c


def test_over_budget_pair_is_reported_and_meets_without_index(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle

    groups, checks = B.mixed_case()
    monkeypatch.setenv("ZGPU_CLOSURE_CAP", "100")  # far fewer entries than the pair needs
    e = zgpu.Engine(B.SCHEMA, device=0)
    B.load(e, groups), e.publish()
    c = e.closure_index_counters()
    assert c["indexed"] == 0 and c["over_budget"] == 1 and c["entries"] == 0 and c["device_bytes"] == 0, c
    with pytest.raises(zgpu.ZgpuError):
        e.closure_index(0)
    o = Oracle(B.SCHEMA)
    B.load(o, groups)
    assert np.array_equal(e.check_bulk(B.items(e, checks, zgpu.CHECK_DTYPE)), o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE)))
