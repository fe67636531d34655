"""Pages of relationship reads answered on the GPU (csrc/filter.cuh page_*): zg_read_relationships_page and
zg_delete_relationships_limited against a host-only engine holding the same relationships (Store::page), page for page
and byte for byte: lines, expirations, cursors, the next cursor and `more`; the order is the key K restated in Python
(page_keys.py) from find() ids; sharded handles give a replica's pages; pages stay exact across interleaved writes,
collections and retirements; zg_page_counters says which path answered."""
import ctypes as C
import random
import threading

import numpy as np
import pytest

import filter_cases as cases
import randgen
from golden_runner import split_rel
from page_keys import class_positions, page_key

pytestmark = pytest.mark.gpu

EINVAL, EPRECOND, E2BIG = -1, -5, -7
MUST_MATCH, MUST_NOT_MATCH = 1, 2
TOUCH, DELETE = 0, 2
LIMITS = (1, 2, 7, 1000)


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _load(e, rels, expires=None):
    ups = [(TOUCH, r, (expires or {}).get(r, 0)) for r in rels]
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])


def _pair(zg, schema, rels, expires=None, now=0, **kw):
    d, h = zg.Engine(schema, **kw), zg.Engine(schema, host_only=True)
    for e in (d, h):
        if now:
            e.set_clock(now)
        _load(e, rels, expires)
    return d, h


def _pages(e, limit, **f):
    """Every page of the read: [(lines, expires, cursors, next, more)]."""
    out, cursor = [], None
    while True:
        page = e.read_relationships_page(limit, cursor, **f)
        out.append(page)
        cursor = page[3]
        if not page[4]:
            return out


def _outcome(fn):
    try:
        return ("ok", fn())
    except Exception as ex:  # ZgpuError: code and text must agree too
        return ("error", getattr(ex, "code", None), str(ex))


def _same_pages(d, h, schema, filters, limits=LIMITS):
    pos = class_positions(schema)
    before = d.page_counters()
    served = 0
    for i, f in enumerate(filters):
        for limit in (limits if i % 4 == 0 else limits[1::2]):
            got, want = _outcome(lambda: _pages(d, limit, **f)), _outcome(lambda: _pages(h, limit, **f))
            assert got == want, (f, limit)
            if got[0] != "ok":
                continue
            served += len(got[1])
            lines = [l for p in got[1] for l in p[0]]
            assert sorted(lines) == d.read_relationships(**f), (f, limit)
            keys = [page_key(d, pos, l) for l in lines]
            assert keys == sorted(keys) and len(set(keys)) == len(keys), (f, limit)
    after = d.page_counters()
    assert after["host_pages"] == before["host_pages"], "a page on a current snapshot ran on the host"
    assert after["device_pages"] - before["device_pages"] == served
    assert h.page_counters()["device_pages"] == 0


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas(zg, name):
    rng = random.Random(9410)
    schema = randgen.FIXED_SCHEMAS[name]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=6, n_user=6, density=0.4)
    d, h = _pair(zg, schema, rels)
    _same_pages(d, h, schema, cases.filters_for(rels, split_rel, rng, samples=4))
    c = d.filter_counters()
    assert c["host_filters"] == 0 and c["by_resource"] and c["by_subject"] and c["by_scan"]


@pytest.mark.parametrize("seed", range(3))
def test_random_schemas(zg, seed):
    rng = random.Random(9510 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5, density=0.4)
    d, h = _pair(zg, schema, rels)
    _same_pages(d, h, schema, cases.filters_for(rels, split_rel, rng, samples=3))


@pytest.mark.parametrize("now", [100, 200])
def test_expirations(zg, now):
    rng = random.Random(9610)
    rels = randgen.random_relationships(rng, randgen.model_from_schema(cases.EXP_SCHEMA), n_obj=8, n_user=8, density=0.4)
    rels += ["doc:o0#viewer@user:*", "doc:o1#viewer@user:*"]
    expires = {r: rng.choice([50, 150, 250]) for r in rels if rng.random() < 0.5}
    d, h = _pair(zg, cases.EXP_SCHEMA, rels, expires, now=now)
    _same_pages(d, h, cases.EXP_SCHEMA, cases.filters_for(rels, split_rel, rng, samples=4))
    assert any(x for p in _pages(d, 5, res_type="doc") for x in p[1]), "no expiration came back"


@pytest.mark.parametrize("S", [2, 3, 4])
def test_sharded_handle_pages_equal_a_replica(zg, S):
    rng = random.Random(9710 + S)
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=10, n_user=8, density=0.3)
    d, r = zg.Engine(schema, n_shards=S), zg.Engine(schema)
    _load(d, rels)
    _load(r, rels)
    filters = cases.filters_for(rels, split_rel, rng, samples=3)
    for i, f in enumerate(filters):
        for limit in ((1, 7, 1000) if i % 3 == 0 else (2,)):
            assert _outcome(lambda: _pages(d, limit, **f)) == _outcome(lambda: _pages(r, limit, **f)), (f, limit)
    assert d.page_counters()["host_pages"] == 0 and d.page_counters()["device_pages"] > 0
    # a delete with a limit on the handle: the same survivors as on the replica
    f = {"res_type": "document", "rel": "viewer"}
    n = len(r.read_relationships(**f))
    assert n > 3
    for e in (d, r):
        assert e.delete_relationships_limited(f, limit=3, allow_partial=True) == (3, True)
        with pytest.raises(zg.ZgpuError) as ex:
            e.delete_relationships_limited(f, limit=n - 4)
        assert ex.value.code == EPRECOND
    assert d.read_relationships() == r.read_relationships()
    assert d.page_counters()["host_pages"] == 0


def test_paging_across_interleaved_work(zg):
    """5 x 1 000 writes, a collection and a retirement with id reuse between the pages of one read: the relationships
    that exist unchanged throughout appear exactly once, and nothing appears twice."""
    rng = random.Random(9810)
    schema = """
use expiration
definition user {}
definition doc {
  relation viewer: user with expiration
  relation owner: user
}
"""
    d = zg.Engine(schema)
    d.set_clock(800)
    stable = [f"doc:s{i:04d}#viewer@user:u{i % 50}" for i in range(3000)]
    churn = [f"doc:c{i:04d}#owner@user:v{i}" for i in range(3000)]
    _load(d, stable)
    _load(d, churn[:1500])
    # bulk-loaded with names (the watch feed does not keep them): expired at 1000, then collected and retired
    xs = np.zeros(500, dtype=zg.TUPLE_DTYPE)
    xs["res"] = [d.intern("doc", f"x{i}") for i in range(500)]
    xs["subj"] = [d.intern("user", f"gone{i}") for i in range(500)]
    xs["rel"], xs["stype"], xs["srel"] = d.slot_id("doc", "viewer"), d.type_id("user"), zg.SREL_NONE
    d.load_tuples(xs, np.full(500, 900, dtype=np.uint32))
    d.publish()
    d.set_clock(1000)
    seen, cursor, step = [], None, 0
    while True:
        lines, _, _, cursor, more = d.read_relationships_page(400, cursor, res_type="doc")
        seen += lines
        if step < 5:  # 1 000 writes: create 500 new, delete 500 old
            ups = [(TOUCH, r, 0) for r in churn[1500 + step * 300:1500 + step * 300 + 500]]
            ups += [(DELETE, r, 0) for r in churn[step * 300:step * 300 + 500]]
            d.write_relationships(ups[:1000])
        elif step == 5:
            assert d.collect_expired(1000) == 500
        elif step == 6:
            assert d.retire_unused_names() == 1000
            _load(d, [f"doc:new{i}#owner@user:fresh{i}" for i in range(300)])  # takes the freed ids
        step += 1
        if not more:
            break
    assert step > 7
    assert len(seen) == len(set(seen))
    assert sorted(s for s in seen if s.startswith("doc:s")) == sorted(stable)
    assert d.page_counters()["host_pages"] == 0


def test_unpublished_changes_take_the_host_path(zg):
    schema = randgen.FIXED_SCHEMAS["nesting"]
    d = zg.Engine(schema)
    d.write_relationships([(TOUCH, "group:g#member@user:a", 0), (TOUCH, "group:g#member@user:b", 0)])
    assert d.read_relationships_page(1, res_type="group")[0] == ["group:g#member@user:a"]
    assert d.page_counters()["device_pages"] == 1
    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = 0, 0, d.slot_id("group", "member"), d.type_id("group"), d.slot_id("group", "member")
    rev = d.stats()["revision"]
    d.load_tuples(t)
    lines = [l for p in _pages(d, 1, res_type="group") for l in p[0]]
    assert lines == ["group:g#member@user:a", "group:g#member@user:b", "group:g#member@group:g#member"]
    c = d.page_counters()
    assert c["device_pages"] == 1 and c["host_pages"] == 3 and d.stats()["revision"] == rev


def test_e2big_leaves_the_cursor_usable(zg):
    schema = randgen.FIXED_SCHEMAS["nesting"]
    rels = [f"group:g#member@user:u{i:03d}" for i in range(300)]
    d, h = _pair(zg, schema, rels)
    for e in (d, h):
        _, _, _, cursor, more = e.read_relationships_page(100, None, res_type="group")
        assert more
        f = e._filter({"res_type": "group"})
        after = C.create_string_buffer(bytes(cursor), 32)
        nxt = C.create_string_buffer(b"\x55" * 32, 32)
        need, n, m = C.c_size_t(0), C.c_uint64(0), C.c_int32(7)
        buf = C.create_string_buffer(16)
        rc = e._L.zg_read_relationships_page(e._h, C.byref(f), 100, after, buf, 16, C.byref(need), C.byref(n), None, None,
                                             nxt, C.byref(m))
        assert rc == E2BIG and n.value == 100 and need.value == sum(len(r) + 1 for r in sorted(rels)[100:200]) + 1
        assert nxt.raw == b"\x55" * 32 and m.value == 7
        assert e.read_relationships_page(100, cursor, res_type="group")[0] == sorted(rels)[100:200]


def test_delete_with_a_limit_against_the_host(zg):
    rng = random.Random(9910)
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=10, n_user=10, density=0.4)
    d, h = _pair(zg, schema, rels)
    exists = dict(zip(("res_type", "res_id"), split_rel(rels[0])[:2]))
    for f in ({"res_type": "document"}, {"subj_type": "user", "subj_id": "u2"}, {"res_type": "folder", "res_id": "o1"},
              {"res_type": "group", "rel": "member"}):
        n = len(h.read_relationships(**f))
        for limit, partial in ((max(n - 1, 1), False), (max(n // 3, 1), True), (n + 5, False)):
            for pre in ([(MUST_NOT_MATCH, exists)], [(MUST_MATCH, exists)]):
                got = _outcome(lambda: d.delete_relationships_limited(f, pre, limit, partial))
                want = _outcome(lambda: h.delete_relationships_limited(f, pre, limit, partial))
                assert got == want, (f, limit, partial)
                assert d.read_relationships() == h.read_relationships()
    assert d.watch_read(0) == h.watch_read(0)
    assert d.page_counters()["host_pages"] == 0 and d.page_counters()["device_pages"] > 0


def test_pagers_beside_a_writer_and_checkers(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    fixed = [f"org:acme#member@user:u{i:03d}" for i in range(200)]
    d = zg.Engine(schema)
    _load(d, fixed)
    stop, errors = threading.Event(), []

    def pager(k):
        try:
            while not stop.is_set():
                got = [l for p in _pages(d, 1 + k * 7, res_type="org", res_id="acme") for l in p[0]]
                assert [g for g in got if g in set(fixed)] == fixed and len(got) == len(set(got))
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    def checker():
        try:
            while not stop.is_set():
                assert list(d.check_bulk_str([("org", "acme", "member", "user", "u001", "")])) == [2]
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    ths = [threading.Thread(target=pager, args=(k,)) for k in range(16)] + [threading.Thread(target=checker) for _ in range(2)]
    for t in ths:
        t.start()
    for i in range(60):
        d.write_relationships([(TOUCH, f"org:acme#member@user:w{i}", 0)])
    stop.set()
    for t in ths:
        t.join()
    assert not errors, errors[0]
    assert d.page_counters()["host_pages"] == 0


def test_cfg4_against_numpy(zg):
    """cfg4 (2 M relationships): the largest (type, relation) read paged with limits 1 000 and 100 000 against numpy's
    sorted keys over the generated tuples."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.02)
    e = zg.Engine(w.schema)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    pos = class_positions(w.schema)
    sizes = {}
    for g in w.groups:
        sizes[(g.res_type, g.rel)] = sizes.get((g.res_type, g.rel), 0) + g.res.size
    rt, rel = max(sizes, key=sizes.get)
    keys = []
    for g in w.groups:
        if (g.res_type, g.rel) != (rt, rel):
            continue
        p = pos[(rt, rel, g.subj_type, "*" if g.wildcard else (g.srel or ""))]
        subj = np.zeros(g.res.size, dtype=np.uint64) if g.wildcard else g.subj.astype(np.uint64)
        keys.append((g.res.astype(np.uint64) << np.uint64(40)) | (np.uint64(p) << np.uint64(32)) | subj)
    want = np.unique(np.concatenate(keys))
    assert want.size > 100_000
    tid = e.type_id(rt)
    for limit in (1000, 100_000):
        got, cursor, pages = [], None, 0
        while True:
            lines, _, _, cursor, more = e.read_relationships_page(limit, cursor, res_type=rt, rel=rel)
            pages += 1
            for l in lines:
                k = page_key(e, pos, l)
                assert k[0] == tid
                got.append((k[1] << 40) | (k[2] << 32) | k[3])
            if not more:
                break
        assert pages == -(-want.size // limit)
        assert np.array_equal(np.array(got, dtype=np.uint64), want), limit
    assert e.page_counters()["host_pages"] == 0
