"""The width of the closure index (csrc/build.cu gpu_build_closure, csrc/kernels.cuh closure_meet) on the GPU: 16-bit
entries when every object id of the target type fits (cfg3's teams), 32-bit past 65 536 target objects, decided again
when a write lays the store out anew. Answers against the oracle and against the same engine without the index."""
import numpy as np
import pytest

import l2_batch_cases as B

pytestmark = pytest.mark.gpu


def _closure_index_np(n_users, gm_group, gm_user, tm_team, tm_group):
    """(row_ptr, col) of the closure index built with vectorised numpy: row u = the teams user u reaches through a
    group, ascending and distinct (full-size cfg3 has about 80 M entries)."""
    gm_group, gm_user = (np.asarray(x, dtype=np.uint64) for x in (gm_group, gm_user))
    tm_team, tm_group = (np.asarray(x, dtype=np.uint64) for x in (tm_team, tm_group))
    order = np.argsort(tm_group, kind="stable")
    tg, tt = tm_group[order], tm_team[order]
    lo, hi = np.searchsorted(tg, gm_group, "left"), np.searchsorted(tg, gm_group, "right")
    cnt = hi - lo
    users = np.repeat(gm_user, cnt)
    first = np.repeat(lo - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
    teams = tt[first + np.arange(users.size)]
    key = np.unique((users << np.uint64(32)) | teams)
    u, t = (key >> np.uint64(32)).astype(np.int64), (key & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    row_ptr = np.zeros(n_users + 1, dtype=np.uint32)
    row_ptr[1:] = np.cumsum(np.bincount(u, minlength=n_users))
    return row_ptr, t


def _assert_index_equals(e, gm, tm):
    row_ptr, col = e.closure_index(0)
    want_ptr, want_col = _closure_index_np(row_ptr.size - 1, gm.res, gm.subj, tm.res, tm.subj)
    assert np.array_equal(row_ptr, want_ptr)
    assert np.array_equal(col, want_col)


def _without_index(schema, load, monkeypatch):
    import zgpu

    monkeypatch.setenv("ZGPU_CLOSURE_CAP", "0")
    f = zgpu.Engine(schema, device=0)
    load(f), f.publish()
    monkeypatch.delenv("ZGPU_CLOSURE_CAP")
    return f


def test_cfg3_narrow_index_answers_and_lookups(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.1)
    e = zgpu.Engine(w.schema, device=0)
    w.load_into(e), e.publish()
    info = e.closure_index_info(0)
    assert info["built"] == 1 and info["width"] == 2, info
    gm, tm = w.groups[0], w.groups[1]
    _assert_index_equals(e, gm, tm)
    # 2 bytes per entry (plus the 16-entry padding) and 4 per row offset
    assert info["device_bytes"] >= 2 * info["entries"] + 4 * (int(gm.subj.max()) + 2)
    assert info["device_bytes"] == e.closure_index_counters()["device_bytes"]
    f = _without_index(w.schema, w.load_into, monkeypatch)
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    want = o.check_bulk(items)
    assert np.array_equal(e.check_bulk(items), want)
    assert np.array_equal(f.check_bulk(items), want)
    for rt, perm, st, u in w.lookups[:4]:
        assert np.array_equal(e.lookup_resources_ids(rt, perm, st, u), o.lookup_resources_ids(rt, perm, st, u))
    c = w.checks[0]
    n_users = int(gm.subj.max()) + 1
    for res in c.res[:3]:
        ids, wild, ex = e.lookup_subjects_ids(c.res_type, int(res), c.perm, c.subj_type)
        q = np.zeros(n_users, dtype=zgpu.CHECK_DTYPE)
        q["res"], q["subj"] = int(res), np.arange(n_users)
        q["perm"], q["stype"], q["srel"] = o.slot_id(c.res_type, c.perm), o.type_id(c.subj_type), zgpu.SREL_NONE
        assert np.array_equal(ids, np.flatnonzero(o.check_bulk(q) == 2)) and not wild and ex.size == 0


def test_cfg3_full_size_narrow_index_equals_numpy():
    import zgpu
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3()
    e = zgpu.Engine(w.schema, device=0)
    w.load_into(e), e.publish()
    info = e.closure_index_info(0)
    assert info["built"] == 1 and info["width"] == 2, info
    print(f"cfg3 full-size closure index: {info} {e.closure_index_counters()}")
    _assert_index_equals(e, w.groups[0], w.groups[1])


TEAM_OFFSET = 66000  # team ids past 16 bits: the index of (group#member, team#member) must keep 32-bit entries


def _wide_case():
    groups, checks = B.mixed_case()
    out = []
    for rt, rel, st, res, subj, srel in groups:
        res = [x + TEAM_OFFSET for x in res] if rt == "team" else res
        subj = [x + TEAM_OFFSET for x in subj] if st == "team" else subj
        out.append((rt, rel, st, res, subj, srel))
    return out, [(rt, perm, r + TEAM_OFFSET if rt == "team" else r, u) for rt, perm, r, u in checks]


def test_target_ids_past_16_bits_keep_a_32_bit_index(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle

    groups, checks = _wide_case()
    e = zgpu.Engine(B.SCHEMA, device=0)
    B.load(e, groups), e.publish()
    info = e.closure_index_info(0)
    assert info["built"] == 1 and info["width"] == 4, info
    o = Oracle(B.SCHEMA)
    B.load(o, groups)
    want = o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE))
    assert np.array_equal(e.check_bulk(B.items(e, checks, zgpu.CHECK_DTYPE)), want)
    f = _without_index(B.SCHEMA, lambda x: B.load(x, groups), monkeypatch)
    assert np.array_equal(f.check_bulk(B.items(f, checks, zgpu.CHECK_DTYPE)), want)
    assert 0.05 < (want == 2).mean() < 0.95


def test_write_past_16_bit_team_ids_rebuilds_a_32_bit_index():
    """A write that adds a team with an id past 65 536 (and namespaces that list it) lays the store out again: the
    rebuilt index has 32-bit entries, never truncated 16-bit ones, and the answers stay the oracle's."""
    import zgpu
    from oracle.pyoracle import Oracle

    groups, checks = B.mixed_case()
    e, o = zgpu.Engine(B.SCHEMA, device=0), Oracle(B.SCHEMA)
    B.load(e, groups), B.load(o, groups)
    e.publish()
    assert e.closure_index_info(0)["width"] == 2
    before = int((o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE)) == 2).sum())
    big = 70000  # truncated to 16 bits it would read as team 4464 (0x1170), a team no range lists
    ups = np.zeros(2 * 20 + len(B.SIZES), dtype=zgpu.UPDATE_DTYPE)
    k = 0
    for g in range(20):  # team `big` holds groups 0 .. 19 (members of their users); team big + 1 holds the same
        for t in (big, big + 1):
            ups["rel"][k], ups["res"][k], ups["stype"][k] = e.slot_id("team", "member"), t, e.type_id("group")
            ups["srel"][k], ups["subj"][k], ups["op"][k] = e.slot_id("group", "member"), g, 0
            k += 1
    for i in range(len(B.SIZES)):  # every namespace lists team `big` as a viewer
        ups["rel"][k], ups["res"][k], ups["stype"][k] = e.slot_id("namespace", "viewer"), i, e.type_id("team")
        ups["srel"][k], ups["subj"][k], ups["op"][k] = e.slot_id("team", "member"), big, 0
        k += 1
    e.apply_updates(ups), o.apply_updates(ups)
    e.publish()
    info = e.closure_index_info(0)
    assert info["built"] == 1 and info["width"] == 4, info
    row_ptr, col = e.closure_index(0)
    assert big in col and big + 1 in col
    items_e, items_o = B.items(e, checks, zgpu.CHECK_DTYPE), B.items(o, checks, zgpu.CHECK_DTYPE)
    want = o.check_bulk(items_o)
    assert np.array_equal(e.check_bulk(items_e), want)
    # members of groups 0 .. 19 now view every namespace through team `big`
    assert int((want == 2).sum()) > before


def test_writes_keep_the_narrow_index():
    """5 x 1000 writes touching group#member and team#member on cfg3: every rebuild keeps 16-bit entries and the
    answers stay the oracle's."""
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.02)
    e, o = zgpu.Engine(w.schema, device=0), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    rng = np.random.default_rng(12)
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
        assert e.closure_index_info(0)["width"] == 2, f"step {step}"
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items)), f"step {step}"
    assert e.closure_index_counters()["builds"] >= builds + 4
