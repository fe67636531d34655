"""zg_retire_unused_names on the GPU: the mention scan of the resident snapshot (csrc/filter.cuh mention_scan_kernel)
and the host's retirement. The property: every check, LookupResources, LookupSubjects, ReadRelationships and
zg_watch_read answers the same before and after retire_unused_names, and the checks and lookups equal the oracle's.
Also: the retired set and counts against a host-only engine fed the same operations, the device and host paths, new
names taking freed ids, device ingress on retired and reused names, sharded handles against a replica, a standalone
shard, two devices, and concurrent callers."""
import random
import re
import threading

import numpy as np
import pytest

import randgen
import test_gpu_expire as ge
from golden_runner import split_rel

pytestmark = pytest.mark.gpu

TOUCH, DELETE = 0, 2
T = ge.T
SCHEMA = ge.SCHEMA


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _apply(e, rels, op, expires=None):
    """Interned updates (zg_apply_updates + publish): the path that records nothing in the watch feed."""
    import zgpu

    u = np.zeros(len(rels), dtype=zgpu.UPDATE_DTYPE)
    for i, r in enumerate(rels):
        rt, rid, rel, st, sid, srel = split_rel(r)
        u[i]["res"], u[i]["rel"], u[i]["stype"] = e.intern(rt, rid), e.slot_id(rt, rel), e.type_id(st)
        if sid == "*":
            u[i]["subj"], u[i]["srel"] = 0, 0xFFFE
        else:
            u[i]["subj"], u[i]["srel"] = e.intern(st, sid), (e.slot_id(st, srel) if srel else 0xFFFF)
        u[i]["op"], u[i]["expires_at"] = op, (expires or {}).get(r, 0)
    e.apply_updates(u)
    e.publish()


def _renamed(rels, tag):
    return [re.sub(r":(o|u)(\d+)", lambda m: f":{tag}{m.group(1)}{m.group(2)}", r) for r in rels]


def _names(rels):
    out = set()
    for r in rels:
        rt, rid, _, st, sid, _ = split_rel(r)
        out.add((rt, rid))
        if sid != "*":
            out.add((st, sid))
    return out


def _feed(e):
    return e.watch_read(0)


def _setup(zg, schema, model, rng, n_obj, n_user, **kw):
    """A device engine (kw) and a host-only one fed the same: string writes (kept by the watch feed), interned writes
    that are then deleted or collected, and names interned and never used."""
    rels = randgen.random_relationships(rng, model, n_obj=n_obj, n_user=n_user, density=0.4)
    gone = _renamed(randgen.random_relationships(rng, model, n_obj=n_obj, n_user=n_user, density=0.3), "x")
    exp = _renamed(randgen.random_relationships(rng, model, n_obj=n_obj, n_user=n_user, density=0.3), "y")
    ex = ge._expirations(rng, schema, exp)
    exp = [r for r in exp if r in ex and ex[r] <= T]
    tnames = model.get("tnames", list(model["types"]))
    d, h = zg.Engine(schema, **kw), zg.Engine(schema, host_only=True)
    for e in (d, h):
        e.set_clock(T - 10)
        ge._write(e, rels, {})
        _apply(e, gone, TOUCH)
        _apply(e, gone, DELETE)
        if exp:
            _apply(e, exp, TOUCH, ex)
        for t in tnames:
            e.intern(t, "ghost")
        e.set_clock(T)
        e.collect_expired(T)
    return d, h, rels, (_names(gone) | _names(exp) | {(t, "ghost") for t in tnames}) - _names(rels)


def _invariance(zg, schema, model, seed, n_obj=5, n_user=5, **kw):
    rng = random.Random(seed)
    d, h, rels, want_gone = _setup(zg, schema, model, rng, n_obj, n_user, **kw)
    q = ge._queries(model, n_obj, n_user)
    subjects_too = "n_shards" not in kw or kw.get("handle_subjects", False)
    before = ge._answers(d, q, T, subjects_too)
    feed = _feed(d)
    o = ge._oracle(schema, rels, {})
    assert before["checks"] == [o.check(*split_rel(x), T) for x in q[0]]
    for lk, got in zip(q[1], before["lookups"]):
        assert got == sorted(o.lookup_resources(*lk, T)), lk
    rev, c0 = d.stats()["revision"], d.name_counters()
    n = d.retire_unused_names()
    assert n == h.retire_unused_names() == len(want_gone)
    c = d.name_counters()
    assert c["retired_device"] - c0["retired_device"] == n and c["retired_host"] == c0["retired_host"]
    assert d.stats()["revision"] == rev
    for t, name in want_gone:
        assert d.find(t, name) == h.find(t, name) == 0xFFFFFFFF
    for t, name in _names(rels):
        assert d.find(t, name) == h.find(t, name) != 0xFFFFFFFF
    assert ge._answers(d, q, T, subjects_too) == before
    assert _feed(d) == feed == _feed(h)
    d.set_clock(1)
    h.set_clock(1)
    assert d.read_relationships() == h.read_relationships()
    d.set_clock(T)
    return d, h, rels, q, n


@pytest.mark.parametrize("seed", range(3))
def test_invariance_fixed_schema(zg, seed):
    _, _, _, _, n = _invariance(zg, SCHEMA, randgen.model_from_schema(SCHEMA), 30000 + seed)
    assert n > 0


@pytest.mark.parametrize("seed", range(3))
def test_invariance_random_schemas(zg, seed):
    rng = random.Random(30100 + seed)
    schema, model = randgen.random_schema(rng)
    _invariance(zg, ge._with_expiration(schema, rng), model, 30100 + seed, 4, 4)


def test_host_path_with_unpublished_changes(zg):
    """An unpublished load sends the call to the host scan; its names are kept."""
    model = randgen.model_from_schema(SCHEMA)
    d, h, rels, want_gone = _setup(zg, SCHEMA, model, random.Random(30200), 5, 5)
    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    for e in (d, h):
        t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = e.intern("doc", "pending"), e.intern("user", "pending"), \
            e.slot_id("doc", "owner"), e.type_id("user"), 0xFFFF
        e.load_tuples(t)
    c0 = d.name_counters()
    assert d.retire_unused_names() == h.retire_unused_names() == len(want_gone)
    c = d.name_counters()
    assert c["retired_host"] - c0["retired_host"] == len(want_gone) and c["retired_device"] == c0["retired_device"]
    assert d.find("doc", "pending") != 0xFFFFFFFF and d.find("user", "pending") != 0xFFFFFFFF
    d.publish()
    h.publish()
    d.set_clock(1)
    h.set_clock(1)
    assert d.read_relationships() == h.read_relationships()


def test_reuse_then_write_check_and_look_up(zg):
    model = randgen.model_from_schema(SCHEMA)
    d, h, rels, q, n = _invariance(zg, SCHEMA, model, 30300)
    freed = d.name_counters()["free_ids"]
    assert freed == n > 0
    new = [f"doc:new{i}#viewer@user:newu{i % 3}" for i in range(6)] + ["group:newg#member@user:newu0",
                                                                       "doc:new0#owner@group:newg#member"]
    for e in (d, h):
        ge._write(e, new, {})
    # the same ids as on the host-only engine, freed ids first
    assert all(d.find(t, name) == h.find(t, name) for t, name in _names(new))
    c, ch = d.name_counters(), h.name_counters()
    assert (c["id_extent"], c["free_ids"]) == (ch["id_extent"], ch["free_ids"]) and c["free_ids"] < freed
    o = ge._oracle(SCHEMA, rels + new, {})
    checks = q[0] + [f"doc:new{i}#view@user:newu{j}" for i in range(6) for j in range(3)]
    got = [int(x) for x in d.check_bulk_str([split_rel(c) for c in checks])]
    assert got == [o.check(*split_rel(c), T) for c in checks]
    for u in ("newu0", "newu1", "newu2"):
        assert sorted(d.lookup_resources_str("doc", "view", "user", u, "")) == sorted(o.lookup_resources("doc", "view", "user", u, "", T))


def test_device_ingress_on_retired_and_reused_names(zg):
    e = zg.Engine(SCHEMA)
    e.set_clock(T)
    ge._write(e, ["doc:keep#viewer@user:a", "doc:keep#viewer@user:b"], {})
    for i in range(40):
        e.intern("user", f"ghost{i}")
        e.intern("doc", f"gdoc{i}")
    subjects = ["a", "b"] + [f"ghost{i}" for i in range(40)]
    docs = ["keep"] * 2 + [f"gdoc{i}" for i in range(40)]

    def both():
        ing = e.check_bulk_packed_ingress("doc", "view", "user", docs, subjects)
        ref = e.check_bulk_str([("doc", d, "view", "user", s, "") for d, s in zip(docs, subjects)])
        assert list(ing) == list(ref)
        return list(ref)

    first = both()  # builds the device mirror
    assert e.retire_unused_names() == 80
    assert both() == first  # the mirror was dropped and rebuilt without the retired names
    ge._write(e, [f"doc:gdoc{i}#viewer@user:ghost{i}" for i in range(0, 40, 2)], {})  # names back, on freed ids
    assert e.name_counters()["free_ids"] == 40
    after = both()
    assert after[2:] == [first[0] if i % 2 == 0 else first[2] for i in range(40)]


@pytest.mark.parametrize("S", [2, 3, 4])
def test_sharded_handle_against_a_replica(zg, S):
    model = randgen.model_from_schema(SCHEMA)
    dh, _, _, _, nh = _invariance(zg, SCHEMA, model, 30400 + S, 8, 6, n_shards=S, handle_lookups=True, handle_subjects=True)
    dr, _, _, _, nr = _invariance(zg, SCHEMA, model, 30400 + S, 8, 6)
    assert nh == nr > 0 and dh.name_counters() == dr.name_counters()


def test_standalone_shard_is_refused(zg):
    e = zg.Engine(SCHEMA, shard_rank=0, shard_count=2)
    with pytest.raises(zg.ZgpuError) as ex:
        e.retire_unused_names()
    assert ex.value.code == -1 and "shard" in str(ex.value)


def test_two_devices(zg):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    model = randgen.model_from_schema(SCHEMA)
    _invariance(zg, SCHEMA, model, 30500, n_devices=2)
    _invariance(zg, SCHEMA, model, 30501, n_shards=2, n_devices=2, handle_lookups=True, handle_subjects=True)


def test_interleaved_writes_against_a_host_engine(zg):
    """5 rounds of 1 000 writes on churned names (interned, then deleted) beside stable ones, a retirement each round."""
    rng = random.Random(30600)
    d, h = zg.Engine(SCHEMA), zg.Engine(SCHEMA, host_only=True)
    stable = [f"doc:s{i}#viewer@user:su{i % 7}" for i in range(50)]
    for e in (d, h):
        e.set_clock(T)
        ge._write(e, stable, {})
    for rnd in range(5):
        churn = [f"doc:c{rnd}_{i}#viewer@user:cu{rnd}_{rng.randrange(300)}" for i in range(1000)]
        churn = list(dict.fromkeys(churn))
        for e in (d, h):
            for i in range(0, len(churn), 250):
                _apply(e, churn[i:i + 250], TOUCH)
            _apply(e, churn[: len(churn) // 2], DELETE)
        assert d.retire_unused_names() == h.retire_unused_names()
        assert d.name_counters() == {**h.name_counters(), "retired_device": d.name_counters()["retired_device"],
                                     "retired_host": d.name_counters()["retired_host"]}
        d.set_clock(1)
        h.set_clock(1)
        assert d.read_relationships() == h.read_relationships()
        d.set_clock(T)
        h.set_clock(T)


def test_concurrent_callers(zg):
    """Checkers of untouched names beside a writer, a collector and a retirer on 16 threads: no error, and the
    checkers' answers never change."""
    e = zg.Engine(SCHEMA)
    e.set_clock(T)
    stable = [f"doc:s{i}#viewer@user:su{i % 5}" for i in range(40)]
    ge._write(e, stable, {})
    probes = [("doc", f"s{i}", "view", "user", f"su{j}", "") for i in range(40) for j in range(5)]
    want = list(e.check_bulk_str(probes))
    stop, errors = threading.Event(), []

    def run(fn):
        try:
            while not stop.is_set():
                fn()
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))
            stop.set()

    def checker():
        assert list(e.check_bulk_str(probes)) == want

    k = [0]

    def writer():
        k[0] += 1
        r = f"doc:w{k[0]}#viewer@user:wu{k[0]}"
        e.write_relationships([(TOUCH, r, T + 5)])
        e.write_relationships([(DELETE, r, 0)])
        e.intern("user", f"tmp{k[0]}")

    def collector():
        e.collect_expired(T)

    def retirer():
        e.retire_unused_names()

    threads = [threading.Thread(target=run, args=(f,)) for f in [checker] * 13 + [writer, collector, retirer]]
    for t in threads:
        t.start()
    import time

    time.sleep(4)
    stop.set()
    for t in threads:
        t.join()
    assert not errors, errors[:3]
    assert list(e.check_bulk_str(probes)) == want
    assert e.name_counters()["retired"] > 0


def _hook_once(e, action):
    """A resolve hook that runs `action` on its first call only; returns the list of calls."""
    calls = []

    def hook():
        calls.append(len(calls))
        if len(calls) == 1:
            action()

    e.set_resolve_hook(hook)
    return calls


def _retire_and_reuse(e, old, new):
    """Retires the name `old` (type, id) -- nothing mentions it -- and interns `new` of the same type on its id."""
    oid = e.find(*old)
    assert e.retire_unused_names() >= 1 and e.find(*old) == 0xFFFFFFFF
    assert e.intern(*new) == oid


def test_checks_resolved_before_a_retirement_answer_for_their_own_names(zg):
    """Resolve doc:old, then (in the gap before the answer) retire it, give its id to doc:new and grant on doc:new:
    the check of doc:old must still answer NO, as for a never-written name. The same through the packed call."""
    for packed in (False, True):
        e = zg.Engine(SCHEMA)
        e.set_clock(T)
        ge._write(e, ["doc:keep#viewer@user:a"], {})
        _apply(e, ["doc:old#viewer@user:a"], TOUCH)
        _apply(e, ["doc:old#viewer@user:a"], DELETE)

        def action():
            _retire_and_reuse(e, ("doc", "old"), ("doc", "new"))
            e.write_relationships([(TOUCH, "doc:new#viewer@user:a", 0)])

        calls = _hook_once(e, action)
        if packed:
            got = list(e.check_bulk_packed("doc", "view", "user", ["old", "new", "keep"], "a"))
        else:
            got = list(e.check_bulk_str([("doc", "old", "view", "user", "a", ""), ("doc", "new", "view", "user", "a", ""),
                                         ("doc", "keep", "view", "user", "a", "")]))
        assert len(calls) == 2  # the retirement made the call resolve and answer again
        assert got == [1, 2, 2], packed
        e.set_resolve_hook(None)


def test_lookups_resolved_before_a_retirement_never_print_the_new_name(zg):
    e = zg.Engine(SCHEMA)
    e.set_clock(T)
    ge._write(e, ["doc:keep#viewer@user:a", "doc:keep#viewer@user:c"], {})
    _apply(e, ["doc:d1#viewer@user:a", "doc:keep#viewer@user:b"], TOUCH)

    def drop_d1():
        _apply(e, ["doc:d1#viewer@user:a"], DELETE)
        _retire_and_reuse(e, ("doc", "d1"), ("doc", "z"))

    calls = _hook_once(e, drop_d1)
    assert sorted(e.lookup_resources_str("doc", "view", "user", "a", "")) == ["keep"]
    assert len(calls) == 2

    def drop_b():
        _apply(e, ["doc:keep#viewer@user:b"], DELETE)
        _retire_and_reuse(e, ("user", "b"), ("user", "zz"))

    calls = _hook_once(e, drop_b)
    assert e.lookup_subjects_str("doc", "keep", "view", "user") == (["a", "c"], False, [])
    assert len(calls) == 2
    e.set_resolve_hook(None)


def test_cfg3_closure_index_stays_16_bit_under_churn(zg):
    """cfg3's shape (namespace -> team#member -> group#member -> user): 40 000 named teams, then rounds of 8 000
    teams created in groups, checked through a namespace, and deleted. With retirement the teams' capacity stays at
    49 096 and the closure index keeps 16-bit entries; without it the third round passes 65 536 and rebuilds at 32."""
    import l2_batch_cases as B
    from oracle.pyoracle import Oracle  # noqa: F401

    def run(retire):
        e = zg.Engine(B.SCHEMA)
        teams = e.intern_packed("team", [f"t{i}" for i in range(40000)])
        groups = e.intern_packed("group", [f"g{i}" for i in range(100)])
        users = e.intern_packed("user", [f"u{i}" for i in range(200)])
        ups = np.zeros(40000 + 200 + 4, dtype=zg.UPDATE_DTYPE)
        ups["res"][:40000], ups["subj"][:40000] = teams, groups[np.arange(40000) % 100]
        ups["rel"][:40000], ups["stype"][:40000], ups["srel"][:40000] = e.slot_id("team", "member"), e.type_id("group"), \
            e.slot_id("group", "member")
        ups["res"][40000:40200], ups["subj"][40000:40200] = groups[np.arange(200) % 100], users
        ups["rel"][40000:40200], ups["stype"][40000:40200], ups["srel"][40000:40200] = e.slot_id("group", "member"), \
            e.type_id("user"), 0xFFFF
        ns = e.intern("namespace", "n0")
        ups["res"][40200:], ups["subj"][40200:] = ns, teams[:4]
        ups["rel"][40200:], ups["stype"][40200:], ups["srel"][40200:] = e.slot_id("namespace", "viewer"), \
            e.type_id("team"), e.slot_id("team", "member")
        e.apply_updates(ups)
        e.publish()
        widths, caps = [], []
        for c in range(4):
            new = [f"c{c}_{i}" for i in range(8000)]
            churn = [f"team:{t}#member@group:g{i % 100}#member" for i, t in enumerate(new)]
            _apply(e, churn, TOUCH)
            grant = [f"namespace:m{c}#viewer@team:{new[0]}#member"]
            _apply(e, grant, TOUCH)
            # u0 is in g0, g0 in team new[0], new[0] a viewer team of m{c}; u150 is in g50, which new[0] does not hold
            got = list(e.check_bulk_str([("namespace", f"m{c}", "view", "user", "u0", ""),
                                         ("namespace", f"m{c}", "view", "user", "u150", "")]))
            assert got == [2, 1], c
            _apply(e, churn + grant, DELETE)
            if retire:
                assert e.retire_unused_names() == 8001  # the teams and the namespace
            info = e.closure_index_info(0)
            assert info["built"] == 1
            widths.append(info["width"])
            caps.append(e.object_capacity("team"))
        return widths, caps

    widths, caps = run(True)
    assert widths == [2, 2, 2, 2] and caps == [49096] * 4, (widths, caps)
    widths, caps = run(False)
    assert widths[0] == 2 and widths[-1] == 4 and max(caps) > 65536, (widths, caps)
