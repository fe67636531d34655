"""Relationship filters answered on the GPU from the resident CSR (csrc/filter.cuh): zg_read_relationships,
zg_delete_relationships and the preconditions of both write calls, against a host-only engine holding the same
relationships (Store::match): lines, counts, ZG_EPRECOND texts and the watch feed; zg_filter_counters says which path
answered."""
import random
import threading

import numpy as np
import pytest

import filter_cases as cases
import randgen
from golden_runner import run_case, split_rel

pytestmark = pytest.mark.gpu

EPRECOND, E2BIG = -5, -7  # include/zgpu.h
MUST_MATCH, MUST_NOT_MATCH = 1, 2
TOUCH, DELETE = 0, 2


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _load(e, rels, expires=None):
    ups = [(TOUCH, r, (expires or {}).get(r, 0)) for r in rels]
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])


def _pair(zg, schema, rels, expires=None, now=0, **kw):
    """A device engine (kw: n_shards, or shard_rank / shard_count) and a host-only engine with the same relationships,
    written in the same order. One shard of a sharded store keeps the relationships whose resource it owns; the
    host-only engine, which is never sharded, is given exactly those."""
    d, h = zg.Engine(schema, **kw), zg.Engine(schema, host_only=True)
    for e in (d, h):
        if now:
            e.set_clock(now)
    _load(d, rels, expires)
    if "shard_count" in kw:
        rels = [r for r in rels if d.find(*split_rel(r)[:2]) % kw["shard_count"] == kw["shard_rank"]]
        assert rels
    _load(h, rels, expires)
    return d, h


def _outcome(e, fn):
    try:
        return ("ok", fn(e))
    except Exception as ex:  # ZgpuError: code and text must agree too
        return ("error", getattr(ex, "code", None), str(ex))


def _same_reads(d, h, filters):
    before = d.filter_counters()
    n = 0
    for f in filters:
        got, want = _outcome(d, lambda e: e.read_relationships(**f)), _outcome(h, lambda e: e.read_relationships(**f))
        assert got == want, f
        n += got[0] == "ok"
    after = d.filter_counters()
    assert after["host_filters"] == before["host_filters"], "a read on a current snapshot ran the host scan"
    assert after["device_filters"] - before["device_filters"] == n
    assert h.filter_counters()["device_filters"] == 0
    return after


def _same_preconditions(d, h, filters, probe):
    """Both operations of every filter as the precondition of a TOUCH that changes nothing."""
    for f in filters:
        for op in (MUST_MATCH, MUST_NOT_MATCH):
            w = lambda e: e.write_relationships([(TOUCH, probe, 0)], [(op, f)])  # noqa: E731
            assert _outcome(d, w) == _outcome(h, w), (f, op)
    assert d.filter_counters()["host_filters"] == 0


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas_matrix(zg, name):
    rng = random.Random(9400)
    schema = randgen.FIXED_SCHEMAS[name]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=6, n_user=6, density=0.4)
    d, h = _pair(zg, schema, rels)
    filters = cases.filters_for(rels, split_rel, rng, samples=8)
    c = _same_reads(d, h, filters)
    assert c["by_resource"] and c["by_subject"] and c["by_scan"] and c["device_relationships"]
    _same_preconditions(d, h, filters[::3], rels[0])
    parts = [split_rel(r) for r in rels]
    for f in filters[:60]:
        assert d.read_relationships(**f) == sorted(r for r, p in zip(rels, parts) if cases.matches(f, p)), f


@pytest.mark.parametrize("seed", range(6))
def test_random_schemas_matrix(zg, seed):
    rng = random.Random(9500 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5, density=0.4)
    d, h = _pair(zg, schema, rels)
    filters = cases.filters_for(rels, split_rel, rng, samples=6)
    _same_reads(d, h, filters)
    _same_preconditions(d, h, filters[::4], rels[0])


@pytest.mark.parametrize("now", [100, 200])
def test_expirations(zg, now):
    rng = random.Random(9600)
    rels = randgen.random_relationships(rng, randgen.model_from_schema(cases.EXP_SCHEMA), n_obj=6, n_user=6, density=0.4)
    rels += ["doc:o0#viewer@user:*", "doc:o1#viewer@user:*"]
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    d, h = _pair(zg, cases.EXP_SCHEMA, rels, expires, now=now)
    filters = cases.filters_for(rels, split_rel, rng, samples=8)
    _same_reads(d, h, filters)
    _same_preconditions(d, h, filters[::3], "doc:o0#banned@user:u0")
    # a delete by filter matches expired relationships too (clock 0)
    f = {"res_type": "doc", "rel": "viewer"}
    assert d.delete_relationships(f) == h.delete_relationships(f) == sum(r.startswith("doc:") and "#viewer@" in r for r in rels)
    assert d.watch_read(0) == h.watch_read(0)


@pytest.mark.parametrize("kw", [{}, {"n_shards": 2}, {"n_shards": 3}, {"n_shards": 4}, {"shard_rank": 1, "shard_count": 3}],
                         ids=["single", "S2", "S3", "S4", "standalone-shard"])
def test_delete_by_filter_and_feed(zg, kw):
    """Deletes by every shape (with a failing and a holding precondition) leave the same store, the same counts and the
    same watch feed, in the same order, as the host scan; on a sharded handle and on one shard of a sharded store."""
    rng = random.Random(9700)
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=8, n_user=8, density=0.4)
    d, h = _pair(zg, schema, rels, **kw)
    filters = cases.filters_for(rels, split_rel, rng, samples=6)
    _same_reads(d, h, filters)
    some = split_rel(h.read_relationships()[0])
    exists = {"res_type": some[0], "res_id": some[1]}
    deletes = [{"res_type": "document", "res_id": "o3"}, {"subj_type": "user", "subj_id": "u2"}, {"res_type": "folder", "rel": "viewer"},
               {"res_type": "document", "subj_type": "user", "subj_id": "*"}, {"res_type": "group"}]
    for f in deletes:
        bad = lambda e: e.delete_relationships(f, [(MUST_NOT_MATCH, exists)])  # noqa: E731
        assert _outcome(d, bad) == _outcome(h, bad) and _outcome(d, bad)[1] == EPRECOND
        ok = lambda e: e.delete_relationships(f, [(MUST_MATCH, exists)])  # noqa: E731
        assert _outcome(d, ok) == _outcome(h, ok), f
        assert d.read_relationships() == h.read_relationships()
        assert d.num_tuples() == h.num_tuples()
    # a shard publishes on writes that hold nothing it owns, so only there the revisions differ
    feed = (lambda e: [c[1:] for c in e.watch_read(0)[0]]) if "shard_count" in kw else (lambda e: e.watch_read(0))
    assert feed(d) == feed(h)
    c = d.filter_counters()
    assert c["host_filters"] == 0 and c["device_filters"] > len(filters)


def test_after_incremental_writes(zg):
    """5 x 1 000 incremental writes (inserts, touches, deletes merged into the resident snapshot), then the matrix."""
    rng = random.Random(9800)
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=40, n_user=40, density=0.2)
    rng.shuffle(rels)
    base, rest = rels[:len(rels) // 2], rels[len(rels) // 2:]
    d, h = _pair(zg, schema, base)
    live = list(base)
    for r in range(5):
        ups = [(TOUCH, x, 0) for x in rest[r * 600:(r + 1) * 600]] + [(DELETE, x, 0) for x in live[r * 400:(r + 1) * 400]]
        assert 0 < len(ups) <= 1000
        pre = [(MUST_MATCH, dict(zip(("res_type", "res_id", "rel", "subj_type", "subj_id"), split_rel(live[-1])[:5])))]
        for e in (d, h):
            e.write_relationships(ups, pre)
    assert d.stats()["delta_publishes"] >= 5
    final = sorted(set(base[2000:]) | set(rest[:3000]))
    assert d.read_relationships() == h.read_relationships() == final
    _same_reads(d, h, cases.filters_for(final, split_rel, rng, samples=8))
    assert d.filter_counters()["host_filters"] == 0


def test_unpublished_relationships_take_the_host_scan(zg):
    """Relationships loaded and not yet published: the read sees them through Store::match (as before), the counters
    say so, and the read does not publish."""
    schema = randgen.FIXED_SCHEMAS["nesting"]
    d = zg.Engine(schema)
    d.write_relationships([(TOUCH, "group:g#member@user:a", 0)])
    rev = d.stats()["revision"]
    assert d.read_relationships(res_type="group") == ["group:g#member@user:a"]
    assert d.filter_counters()["device_filters"] == 1
    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = 0, 0, d.slot_id("group", "member"), d.type_id("group"), d.slot_id("group", "member")
    d.load_tuples(t)
    assert d.read_relationships(res_type="group") == ["group:g#member@group:g#member", "group:g#member@user:a"]
    c = d.filter_counters()
    assert (c["device_filters"], c["host_filters"]) == (1, 1) and d.stats()["revision"] == rev
    d.publish()
    assert d.read_relationships(res_type="group") == ["group:g#member@group:g#member", "group:g#member@user:a"]
    assert d.filter_counters()["device_filters"] == 2


def test_e2big_and_retry(zg):
    import ctypes as C

    from spicedb_kubeapi_proxy_b200 import _lib

    schema = randgen.FIXED_SCHEMAS["nesting"]
    rels = [f"group:g#member@user:u{i}" for i in range(300)]
    d, h = _pair(zg, schema, rels)
    f = d._filter({"res_type": "group", "res_id": "g"})
    for e in (d, h):
        need, n = C.c_size_t(0), C.c_uint64(0)
        buf = C.create_string_buffer(16)
        assert e._L.zg_read_relationships(e._h, C.byref(f), buf, 16, C.byref(need), C.byref(n)) == E2BIG
        assert n.value == 300 and need.value == sum(len(r) + 1 for r in rels) + 1
        buf = C.create_string_buffer(need.value)
        assert e._L.zg_read_relationships(e._h, C.byref(f), buf, need.value, C.byref(need), C.byref(n)) == 0
        assert buf.value.decode().split("\n")[:-1] == sorted(rels)
    assert _lib is not None


def test_readers_beside_a_writer_and_checkers(zg):
    """16 threads read by resource and by subject while one writes and two check: every read is a consistent answer
    (the fixed relationships are always all there), nothing fails, and no read ran the host scan."""
    schema = randgen.FIXED_SCHEMAS["docs"]
    fixed = [f"org:acme#member@user:u{i}" for i in range(200)]
    d = zg.Engine(schema)
    _load(d, fixed)
    stop, errors = threading.Event(), []

    def reader(k):
        try:
            while not stop.is_set():
                got = d.read_relationships(res_type="org", res_id="acme")
                assert [g for g in got if g in set(fixed)] == sorted(fixed)
                assert d.read_relationships(subj_type="user", subj_id=f"u{k}")[:1] == [f"org:acme#member@user:u{k}"]
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    def checker():
        try:
            while not stop.is_set():
                assert list(d.check_bulk_str([("org", "acme", "member", "user", "u1", "")])) == [2]
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    ths = [threading.Thread(target=reader, args=(k,)) for k in range(16)] + [threading.Thread(target=checker) for _ in range(2)]
    for t in ths:
        t.start()
    for i in range(60):
        d.write_relationships([(TOUCH, f"org:acme#member@user:w{i}", 0)],
                              [(MUST_NOT_MATCH, {"res_type": "org", "res_id": "acme", "rel": "member", "subj_type": "user", "subj_id": f"w{i}"})])
    stop.set()
    for t in ths:
        t.join()
    assert not errors, errors[0]
    c = d.filter_counters()
    assert c["host_filters"] == 0 and c["device_filters"] >= 60


def test_cfg4_against_numpy(zg):
    """cfg4 (2 M relationships): reads by resource, by subject and by (type, relation) against numpy over the
    generated tuples, right after a bulk load + publish."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.02)
    e = zg.Engine(w.schema)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()

    def lines(g, mask):
        sub = (lambda i: "*") if g.wildcard else (lambda i: workloads.object_name(g.subj_type, int(g.subj[i])) + (f"#{g.srel}" if g.srel else ""))
        return {f"{g.res_type}:{workloads.object_name(g.res_type, int(g.res[i]))}#{g.rel}@{g.subj_type}:{sub(i)}"
                for i in np.flatnonzero(mask)}

    rng = random.Random(9900)
    for g in rng.sample(w.groups, min(6, len(w.groups))):
        i = rng.randrange(g.res.size)
        rid = workloads.object_name(g.res_type, int(g.res[i]))
        want = set()
        for q in w.groups:
            if q.res_type == g.res_type:
                want |= lines(q, q.res == g.res[i])
        assert e.read_relationships(res_type=g.res_type, res_id=rid) == sorted(want)
        if not g.wildcard:
            sid = workloads.object_name(g.subj_type, int(g.subj[i]))
            want = set()
            for q in w.groups:
                if q.subj_type == g.subj_type and not q.wildcard:
                    want |= lines(q, q.subj == g.subj[i])
            assert e.read_relationships(subj_type=g.subj_type, subj_id=sid) == sorted(want)
    small = min(w.groups, key=lambda q: q.res.size)
    want = set()
    for q in w.groups:
        if (q.res_type, q.rel) == (small.res_type, small.rel):
            want |= lines(q, np.ones(q.res.size, dtype=bool))
    assert e.read_relationships(res_type=small.res_type, rel=small.rel) == sorted(want)
    c = e.filter_counters()
    assert c["host_filters"] == 0 and c["by_resource"] and c["by_subject"] and c["by_scan"]


def test_golden_cases_read_on_the_device(zg, golden):
    from test_gpu_parity import EngineBackend

    reads = 0
    for case in golden["cases"]:
        b = EngineBackend(zg, golden["schemas"][case["schema"]])
        run_case(b, case)
        c = b.cl.engine.filter_counters()
        assert c["host_filters"] == 0
        reads += c["device_filters"]
    assert reads > 0
