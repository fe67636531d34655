"""zg_retire_unused_names on host-only engines (the host scan of the store): which names are retired and which stay,
ids of kept names, lowest-first reuse of freed ids, raw-id loads taking a free id, the arena rewrite, the refusals,
the counters, and the proxy's churn shape keeping the id extent and the capacities flat."""
import numpy as np
import pytest

import filter_cases as cases

EINVAL, ENOSCHEMA = -1, -3  # include/zgpu.h
NO_OBJECT = 0xFFFFFFFF
TOUCH, CREATE, DELETE = 0, 1, 2


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _host(zg, schema=cases.EXP_SCHEMA, clock=100):
    e = zg.Engine(schema, host_only=True)
    e.set_clock(clock)
    return e


def _gone(zg, e, t, name, old_id):
    assert e.find(t, name) == NO_OBJECT
    with pytest.raises(zg.ZgpuError) as ex:
        e.object_name(t, old_id)
    assert ex.value.code == EINVAL


def _ups(zg, e, rows):
    """Interned updates (zg_apply_updates, which records nothing in the watch feed): rows of
    (op, resource type, resource, relation, subject type, subject, expires_at)."""
    u = np.zeros(len(rows), dtype=zg.UPDATE_DTYPE)
    for i, (op, rt, r, rel, st, sj, exp) in enumerate(rows):
        u[i]["res"], u[i]["subj"], u[i]["rel"] = e.intern(rt, r), e.intern(st, sj), e.slot_id(rt, rel)
        u[i]["stype"], u[i]["srel"], u[i]["expires_at"], u[i]["op"] = e.type_id(st), 0xFFFF, exp, op
    e.apply_updates(u)
    e.publish()


def test_unused_deleted_collected_and_cleared(zg):
    e = _host(zg)
    never = e.intern("user", "never")
    _ups(zg, e, [(TOUCH, "doc", "d", "viewer", "user", "del", 0), (TOUCH, "doc", "x", "viewer", "user", "exp", 50),
                 (TOUCH, "doc", "k", "viewer", "user", "keep", 0)])
    ids = {n: e.find("user", n) for n in ("del", "exp", "keep")}
    _ups(zg, e, [(DELETE, "doc", "d", "viewer", "user", "del", 0)])
    assert e.collect_expired(100) == 1
    assert e.retire_unused_names() == 5  # user:never, doc:d, user:del, doc:x, user:exp
    _gone(zg, e, "user", "never", never)
    _gone(zg, e, "user", "del", ids["del"])
    _gone(zg, e, "user", "exp", ids["exp"])
    assert e.find("doc", "d") == NO_OBJECT and e.find("doc", "x") == NO_OBJECT
    assert e.find("user", "keep") == ids["keep"] and e.object_name("user", ids["keep"]) == "keep"
    assert e.read_relationships() == ["doc:k#viewer@user:keep"]
    assert e.retire_unused_names() == 0
    # the string write calls record their changes in the watch feed, which keeps their names
    e.write_relationships([(TOUCH, "doc:s#viewer@user:s", 0)])
    e.write_relationships([(DELETE, "doc:s#viewer@user:s", 0)])
    assert e.retire_unused_names() == 0 and e.find("user", "s") != NO_OBJECT
    # a clear restarts the feed: nothing mentions any name afterwards
    e._ck(e._L.zg_clear_relationships(e._h))
    assert e.retire_unused_names() == 4  # doc:k, user:keep, doc:s, user:s
    assert e.name_counters()["named"] == 0


def test_what_stays(zg):
    e = _host(zg, clock=100)
    e.write_relationships([(TOUCH, "doc:live#viewer@user:a", 0), (TOUCH, "doc:old#viewer@user:b", 60),
                           (TOUCH, "group:g#member@user:c", 0), (TOUCH, "doc:live#viewer@group:g#member", 0),
                           (TOUCH, "doc:w#viewer@user:*", 0)])
    feed_before = e.watch_read(0)
    # an unpublished bulk load names user:d and doc:u
    d, u = e.intern("user", "d"), e.intern("doc", "u")
    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = u, d, e.slot_id("doc", "viewer"), e.type_id("user"), 0xFFFF
    e.load_tuples(t)
    # a numeric-only id beyond every name
    t2 = t.copy()
    t2["res"], t2["subj"] = 500, 501
    e.load_tuples(t2)
    before = {(ty, n): e.find(ty, n) for ty, n in [("doc", "live"), ("doc", "old"), ("doc", "w"), ("doc", "u"),
                                                      ("user", "a"), ("user", "b"), ("user", "c"), ("user", "d"),
                                                      ("group", "g")]}
    assert e.retire_unused_names() == 0
    assert {k: e.find(*k) for k in before} == before
    assert e.watch_read(0) == feed_before
    e.publish()
    assert e.name_counters()["id_extent"] >= 502 + 502


def test_watch_feed_text_identical(zg):
    e = _host(zg)
    e.write_relationships([(TOUCH, "doc:a#viewer@user:u0", 0), (TOUCH, "group:g#member@user:u1", 0)])
    e.write_relationships([(DELETE, "doc:a#viewer@user:u0", 0), (DELETE, "group:g#member@user:u1", 0)])
    feed = e.watch_read(0)
    e.intern("user", "nobody")
    assert e.retire_unused_names() == 1
    assert e.watch_read(0) == feed
    assert e.watch_read(0, "doc") == ([f for f in feed[0] if f[2].startswith("doc:")], feed[1])


def test_lowest_first_reuse_and_raw_ids(zg):
    e = _host(zg)
    ids = [e.intern("user", f"u{i}") for i in range(10)]
    assert ids == list(range(10))
    e.write_relationships([(TOUCH, f"doc:d#viewer@user:u{i}", 0) for i in (0, 4, 9)])
    assert e.retire_unused_names() == 7  # u1 u2 u3 u5 u6 u7 u8
    c = e.name_counters()
    assert c["free_ids"] == 7 and c["retired"] == 7
    # a raw update names free id 2 directly: it is no longer free, and has no name
    up = np.zeros(1, dtype=zg.UPDATE_DTYPE)
    up["res"], up["subj"] = e.find("doc", "d"), 2
    up["rel"], up["stype"], up["srel"], up["op"] = e.slot_id("doc", "viewer"), e.type_id("user"), 0xFFFF, TOUCH
    e.apply_updates(up)
    # a raw bulk load names free id 6
    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = e.find("doc", "d"), 6, e.slot_id("doc", "viewer"), e.type_id("user"), 0xFFFF
    e.load_tuples(t)
    assert e.name_counters()["free_ids"] == 5
    assert [e.intern("user", f"n{i}") for i in range(7)] == [1, 3, 5, 7, 8, 10, 11]
    assert e.intern("user", "n0") == 1 and e.object_name("user", 1) == "n0"
    # the write path takes freed ids too
    e.write_relationships([(TOUCH, f"doc:d#viewer@user:n{i}", 0) for i in range(7)])
    assert e.retire_unused_names() == 0
    e.write_relationships([(DELETE, "doc:d#viewer@user:n2", 0)])
    e.intern("user", "m")
    assert e.retire_unused_names() == 1  # only m: n2 is in the watch feed
    assert e.find("user", "n2") == 5 and e.intern("user", "m2") == 12


def test_packed_intern_takes_freed_ids(zg):
    e = _host(zg)
    for i in range(6):
        e.intern("user", f"x{i}")
    assert e.retire_unused_names() == 6
    got = e.intern_packed("user", ["p", "q", "", "r"])
    assert list(got) == [0, 1, NO_OBJECT, 2]


def test_arena_rewrite_keeps_every_pair(zg):
    e = _host(zg)
    rng = np.random.default_rng(7)
    names = [f"obj-{i}-" + "z" * int(rng.integers(0, 40)) for i in range(3000)]
    ids = {n: e.intern("user", n) for n in names}
    keep = [n for i, n in enumerate(names) if i % 3 == 0]
    for i in range(0, len(keep), 500):
        e.write_relationships([(TOUCH, f"doc:d#viewer@user:{n}", 0) for n in keep[i:i + 500]])
    arena = e.name_counters()["arena_bytes"]
    assert e.retire_unused_names() == len(names) - len(keep)
    assert e.name_counters()["arena_bytes"] < arena
    for n in names:
        if n in keep:
            assert e.find("user", n) == ids[n] and e.object_name("user", ids[n]) == n
        else:
            _gone(zg, e, "user", n, ids[n])
    # the rebuilt table takes new names and finds old ones
    fresh = [e.intern("user", f"new{i}") for i in range(2500)]
    assert sorted(fresh) == sorted(ids[n] for n in names if n not in keep)[:2000] + list(range(3000, 3500))
    assert all(e.find("user", f"new{i}") == fresh[i] for i in range(2500))
    assert all(e.find("user", n) == ids[n] for n in keep)


def test_refusals(zg):
    e = zg.Engine(None, host_only=True)
    with pytest.raises(zg.ZgpuError) as ex:
        e.retire_unused_names()
    assert ex.value.code == ENOSCHEMA


def test_counters(zg):
    e = _host(zg)
    c0 = e.name_counters()
    assert c0 == {k: 0 for k in c0}
    e.intern("user", "abc")
    e.intern("doc", "de")
    e.write_relationships([(TOUCH, "doc:de#viewer@user:keep", 0)])
    c = e.name_counters()
    assert c["named"] == 3 and c["id_extent"] == 3 and c["arena_bytes"] == 3 * 8 + 3 + 2 + 4
    assert e.retire_unused_names() == 1
    c = e.name_counters()
    assert (c["named"], c["retired"], c["free_ids"], c["id_extent"], c["retired_host"], c["retired_device"]) == (2, 1, 1, 3, 1, 0)
    assert c["arena_bytes"] == 2 * 8 + 2 + 4
    e.intern("user", "x")
    assert e.name_counters()["free_ids"] == 0 and e.name_counters()["id_extent"] == 3


def _churn(e, cycle, k, clock0, retire):
    """One round of the proxy's dual writes over interned ids (zg_apply_updates): k workflows, each taking a lock and
    writing an idempotency key that expires in 24 h, then releasing the lock; a day later the keys are collected and,
    with `retire`, the names retired. The string write calls record every change in the watch feed, which keeps its
    names until the feed drops it (2^20 changes); interned updates write no feed, so the reuse shows from cycle one."""
    now = clock0 + cycle * 86400 * 2
    e.set_clock(now)
    wf = e.intern_packed("workflow", [f"wf-{cycle}-{i}" for i in range(k)])
    act = e.intern_packed("activity", [f"a{cycle:04d}{i:08x}" for i in range(k)])
    lock = e.intern_packed("lock", [f"l{cycle:04d}{i:08x}" for i in range(k)])
    locks = np.zeros(k, dtype=zg_mod().UPDATE_DTYPE)
    locks["res"], locks["subj"], locks["rel"], locks["stype"], locks["srel"] = lock, wf, e.slot_id("lock", "workflow"), e.type_id("workflow"), 0xFFFF
    locks["op"] = TOUCH
    keys = np.zeros(k, dtype=zg_mod().UPDATE_DTYPE)
    keys["res"], keys["subj"], keys["rel"], keys["stype"], keys["srel"] = wf, act, e.slot_id("workflow", "idempotency_key"), e.type_id("activity"), 0xFFFF
    keys["op"], keys["expires_at"] = TOUCH, now + 86400
    e.apply_updates(np.concatenate([locks, keys]))
    e.publish()
    locks["op"] = DELETE
    e.apply_updates(locks)
    e.publish()
    e.set_clock(now + 86400 + 1)
    assert e.collect_expired(now + 86400) == k
    if retire:
        assert e.retire_unused_names() == 3 * k


def zg_mod():
    import zgpu

    return zgpu


@pytest.mark.parametrize("retire", [True, False])
def test_proxy_churn_keeps_the_id_space_flat(zg, retire):
    from spicedb_kubeapi_proxy_b200 import workloads

    e = zg.Engine(workloads.BOOTSTRAP_SCHEMA, host_only=True)
    k = 1000
    ext, caps = [], []
    for cycle in range(20):
        _churn(e, cycle, k, 1_700_000_000, retire)
        ext.append(e.name_counters()["id_extent"])
        caps.append(tuple(e.object_capacity(t) for t in ("workflow", "activity", "lock")))
    assert e.num_tuples() == 0
    if retire:
        assert len(set(ext)) == 1 and len(set(caps)) == 1, (ext, caps)
        assert ext[0] == 3 * k and e.name_counters()["retired"] == 20 * 3 * k
    else:
        assert all(b == a + 3 * k for a, b in zip(ext, ext[1:]))
        assert all(a <= b for a, b in zip(caps, caps[1:]))
        assert all(c > caps[0][j] for j, c in enumerate(caps[-1]))


def test_string_writes_free_names_once_the_feed_drops_them(zg):
    """The same churn through the string write call: the watch feed keeps this run's changes, so nothing is retired
    while it holds them; clearing the store restarts the feed and frees them all."""
    from spicedb_kubeapi_proxy_b200 import workloads

    e = zg.Engine(workloads.BOOTSTRAP_SCHEMA, host_only=True)
    e.set_clock(1_700_000_000)
    e.write_relationships([(TOUCH, "lock:l1#workflow@workflow:w1", 0),
                           (TOUCH, "workflow:w1#idempotency_key@activity:a1", 1_700_086_400)])
    e.write_relationships([(DELETE, "lock:l1#workflow@workflow:w1", 0)])
    e.set_clock(1_700_100_000)
    assert e.collect_expired(1_700_086_400) == 1
    assert e.retire_unused_names() == 0
    e._ck(e._L.zg_clear_relationships(e._h))
    assert e.retire_unused_names() == 3
