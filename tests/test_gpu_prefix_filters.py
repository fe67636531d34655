"""Filters by resource id prefix answered on the GPU (ingress.cuh prefix_match_kernel, then the filter and page kernels
with bitmaps) against a host-only engine holding the same relationships (Store::match, Store::page), byte for byte:
reads, pages, deletes with their watch feed, preconditions, expiry, sharded handles and a standalone shard, churn with
retirement and id reuse, unpublished changes, concurrent readers, and the named workloads."""
import random
import threading

import numpy as np
import pytest

import filter_cases as cases
import randgen
from golden_runner import split_rel

pytestmark = pytest.mark.gpu

EINVAL, EPRECOND = -1, -5
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
    """A device engine and a host-only engine with the same relationships and the same ids. One shard of a sharded
    store (shard_rank / shard_count) keeps the relationships whose resource it owns: the host-only engine is given
    every relationship, so that it interns the same ids, and then loses the others."""
    d, h = zg.Engine(schema, **kw), zg.Engine(schema, host_only=True)
    for e in (d, h):
        if now:
            e.set_clock(now)
    _load(d, rels, expires)
    _load(h, rels, expires)
    if "shard_count" in kw:
        other = [r for r in rels if d.find(*split_rel(r)[:2]) % kw["shard_count"] != kw["shard_rank"]]
        for i in range(0, len(other), 1000):
            h.write_relationships([(DELETE, r, 0) for r in other[i:i + 1000]])
    return d, h


def _outcome(fn):
    try:
        return ("ok", fn())
    except Exception as ex:  # ZgpuError: code and text must agree too
        return ("error", getattr(ex, "code", None), str(ex))


def _pages(e, limit, **f):
    out, cursor = [], None
    while True:
        page = e.read_relationships_page(limit, cursor, **f)
        out.append(page)
        cursor = page[3]
        if not page[4]:
            return out


def _prefix_filters(rels, rng, samples=2):
    """filters_for's filters without a resource id, each with every proper prefix of a sampled resource name, a
    prefix nobody has, and prefixes without a resource type."""
    names = sorted({split_rel(r)[1] for r in rels})
    prefixes = {"zz-nobody-"}
    for name in rng.sample(names, min(2, len(names))):
        prefixes.update(name[:k] for k in range(1, len(name)))
    prefixes = sorted(prefixes)
    out = []
    for f in cases.filters_for(rels, split_rel, rng, samples=samples):
        if f.get("res_id"):
            continue
        for p in rng.sample(prefixes, min(3, len(prefixes))):
            out.append({**f, "res_id_prefix": p})
    out += [{"res_id_prefix": p} for p in prefixes]
    return out


def _same(d, h, filters, limits=LIMITS):
    before = d.prefix_counters()
    for i, f in enumerate(filters):
        got = _outcome(lambda: d.read_relationships(**f))
        assert got == _outcome(lambda: h.read_relationships(**f)), f
        for limit in (limits if i % 5 == 0 else limits[1:2]):
            pd = _outcome(lambda: _pages(d, limit, **f))
            assert pd == _outcome(lambda: _pages(h, limit, **f)), (f, limit)
            if pd[0] == "ok" and got[0] == "ok":
                assert sorted(l for p in pd[1] for l in p[0]) == got[1], (f, limit)
    after = d.prefix_counters()
    assert after["host_filters"] == before["host_filters"], "a prefix filter on a current snapshot ran on the host"
    assert after["device_filters"] > before["device_filters"]


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas(zg, name):
    rng = random.Random(7100)
    schema = randgen.FIXED_SCHEMAS[name]
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=10, n_user=6, density=0.3)
    d, h = _pair(zg, schema, rels)
    _same(d, h, _prefix_filters(rels, rng))
    assert d.filter_counters()["host_filters"] == 0


@pytest.mark.parametrize("seed", range(3))
def test_random_schemas(zg, seed):
    rng = random.Random(7200 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.4)
    d, h = _pair(zg, schema, rels)
    _same(d, h, _prefix_filters(rels, rng))


@pytest.mark.parametrize("now", [100, 200])
def test_expiry(zg, now):
    rng = random.Random(7300)
    rels = randgen.random_relationships(rng, randgen.model_from_schema(cases.EXP_SCHEMA), n_obj=10, n_user=8, density=0.4)
    rels += ["doc:o0#viewer@user:*", "doc:o1#viewer@user:*"]
    expires = {r: rng.choice([50, 150, 250]) for r in rels if rng.random() < 0.5}
    d, h = _pair(zg, cases.EXP_SCHEMA, rels, expires, now=now)
    _same(d, h, _prefix_filters(rels, rng))


def _ns_rels(n_ns=6, n_doc=7, n_user=4):
    return [f"document:ns{i}/d{j}#viewer@user:u{(i + j + k) % n_user}" for i in range(n_ns) for j in range(n_doc)
            for k in range(2)] + [f"org:ns{i}/o#member@user:u{i % n_user}" for i in range(n_ns)]


def test_deletes_preconditions_and_watch(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = _ns_rels()
    d, h = _pair(zg, schema, rels)
    for e in (d, h):  # refused, partial, unlimited, by type and without one
        assert _outcome(lambda: e.delete_relationships_limited({"res_type": "document", "res_id_prefix": "ns0/"},
                                                               limit=5))[1] == EPRECOND
    steps = [lambda e: e.delete_relationships_limited({"res_type": "document", "res_id_prefix": "ns0/"}, limit=5,
                                                      allow_partial=True),
             lambda e: e.delete_relationships({"res_id_prefix": "ns1/"}),
             lambda e: e.delete_relationships({"res_type": "document", "res_id_prefix": "ns2"},
                                              [(MUST_MATCH, {"res_id_prefix": "ns2/"})]),
             lambda e: e.delete_relationships({"res_id_prefix": "ns3/"}, [(MUST_NOT_MATCH, {"res_id_prefix": "ns3/"})]),
             lambda e: e.write_relationships([(TOUCH, "document:ns9/x#viewer@user:u0", 0)],
                                             [(MUST_MATCH, {"res_id_prefix": "ns4/"}),
                                              (MUST_NOT_MATCH, {"res_type": "org", "res_id_prefix": "ns9"})]),
             lambda e: e.write_relationships([(TOUCH, "document:ns9/y#viewer@user:u0", 0)],
                                             [(MUST_MATCH, {"res_id_prefix": "zz"})]),
             lambda e: e.delete_relationships_limited({"res_id_prefix": "ns"}, limit=1000)]
    for step in steps:
        assert _outcome(lambda: step(d)) == _outcome(lambda: step(h))
        assert d.read_relationships() == h.read_relationships()
    assert d.watch_read(0) == h.watch_read(0)
    assert d.read_relationships() == []
    assert d.prefix_counters()["host_filters"] == 0


@pytest.mark.parametrize("kw", [{"n_shards": 2}, {"n_shards": 3}, {"n_shards": 4}, {"shard_rank": 1, "shard_count": 3}],
                         ids=["S2", "S3", "S4", "standalone"])
def test_sharded(zg, kw):
    rng = random.Random(7400 + len(str(kw)))
    schema = randgen.FIXED_SCHEMAS["docs"]
    rels = _ns_rels(n_ns=8)
    rels += randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=10, n_user=6, density=0.3)
    d, h = _pair(zg, schema, rels, **kw)
    if "n_shards" in kw:  # a replica holds the same relationships as the handle
        h = zg.Engine(schema)
        _load(h, rels)
    _same(d, h, _prefix_filters(rels, rng)[::3])
    f = {"res_type": "document", "res_id_prefix": "ns5/"}
    assert _outcome(lambda: d.delete_relationships_limited(f, limit=3, allow_partial=True)) == \
        _outcome(lambda: h.delete_relationships_limited(f, limit=3, allow_partial=True))
    assert d.delete_relationships({"res_id_prefix": "ns6"}) == h.delete_relationships({"res_id_prefix": "ns6"})
    assert d.read_relationships() == h.read_relationships()


def test_churn_collection_and_retirement(zg):
    schema = """
use expiration
definition user {}
definition doc {
  relation viewer: user with expiration
  relation owner: user
}
"""
    d, h = _pair(zg, schema, [f"doc:keep/{i:04d}#owner@user:u{i % 9}" for i in range(500)], now=800)
    rng = random.Random(7500)
    for rnd in range(5):
        ups = [(TOUCH, f"doc:r{rnd}/{i:04d}#viewer@user:u{rng.randrange(50)}", rng.choice([0, 700, 900]))
               for i in range(1000)]
        for e in (d, h):
            e.write_relationships(ups)
        for f in ({"res_id_prefix": f"r{rnd}/"}, {"res_type": "doc", "res_id_prefix": "r"},
                  {"res_id_prefix": "keep/00", "rel": "owner", "res_type": "doc"}):
            assert d.read_relationships(**f) == h.read_relationships(**f), f
            assert _pages(d, 7, **f) == _pages(h, 7, **f), f
    assert d.collect_expired(800) == h.collect_expired(800)
    assert d.read_relationships(res_id_prefix="r") == h.read_relationships(res_id_prefix="r")
    # a retirement, then new names that take the freed ids
    for e in (d, h):
        e.delete_relationships({"res_id_prefix": "r0/"})
        e.intern("doc", "gone/a")
    # the watch feed keeps r0's names; the interned name without a relationship is retired
    assert d.retire_unused_names() == h.retire_unused_names() >= 1
    syncs = d.prefix_counters()["mirror_syncs"]
    for e in (d, h):
        e.write_relationships([(TOUCH, "doc:new/a#owner@user:u1", 0)])
    assert d.find("doc", "new/a") == h.find("doc", "new/a")
    for p in ("new/", "gone", "r1/", "keep/"):
        assert d.read_relationships(res_id_prefix=p) == h.read_relationships(res_id_prefix=p), p
    assert d.prefix_counters()["mirror_syncs"] > syncs, "the mirror was not rebuilt after the retirement"
    assert d.prefix_counters()["host_filters"] == 0


def test_unpublished_changes_use_the_host(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    d = zg.Engine(schema)
    _load(d, _ns_rels())
    before = d.prefix_counters()
    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"] = d.intern("document", "ns0/late"), d.find("user", "u0")
    t["rel"], t["stype"], t["srel"] = d.slot_id("document", "viewer"), d.type_id("user"), zg.SREL_NONE
    d.load_tuples(t)  # loaded, not published
    got = d.read_relationships(res_id_prefix="ns0/")
    assert "document:ns0/late#viewer@user:u0" in got
    c = d.prefix_counters()
    assert c["host_filters"] == before["host_filters"] + 1 and c["device_filters"] == before["device_filters"]
    d.publish()
    assert d.read_relationships(res_id_prefix="ns0/") == got
    assert d.prefix_counters()["device_filters"] == c["device_filters"] + 1


def test_readers_beside_a_writer(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    d = zg.Engine(schema)
    stable = [f"document:s{i % 10}/d{i:05d}#viewer@user:u{i % 7}" for i in range(5000)]
    _load(d, stable)
    want = {p: d.read_relationships(res_id_prefix=p) for p in ("s3/", "s7/d0")}
    errors = []

    def reader(k):
        try:
            for _ in range(20):
                p = "s3/" if k % 2 else "s7/d0"
                got = d.read_relationships(res_id_prefix=p)
                assert got == want[p]
                lines = [l for pg in _pages(d, 97, res_id_prefix=p) for l in pg[0]]
                assert sorted(lines) == want[p]
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    def writer():
        for i in range(20):
            d.write_relationships([(TOUCH, f"document:w/{i}#viewer@user:u0", 0)])
            d.delete_relationships({"res_id_prefix": "w/"})

    threads = [threading.Thread(target=reader, args=(k,)) for k in range(16)] + [threading.Thread(target=writer)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]


def test_named_cfg2_namespace_delete(zg):
    """Full-size named cfg2: deleting `ns00042/` removes exactly its pods' relationships; checks and lookups on the
    rest still equal the oracle's."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg2()
    e = zg.Engine(w.schema, device=0)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    g = w.groups[0]
    assert g.res_type == "pod"
    gone = (g.res >= 42000) & (g.res < 43000)
    n_gone = len({(int(r), int(s)) for r, s in zip(g.res[gone], g.subj[gone])})
    assert len(e.read_relationships(res_type="pod", res_id_prefix="ns00042/")) == n_gone
    assert e.delete_relationships({"res_id_prefix": "ns00042/"}) == n_gone
    assert e.read_relationships(res_id_prefix="ns00042/") == []
    o = Oracle(w.schema)
    o.add_bulk("pod", g.rel, g.subj_type, g.res[~gone], g.subj[~gone])
    items = w.check_items(e, zg.CHECK_DTYPE)
    assert np.array_equal(e.check_bulk(items), o.check_bulk(items))
    for rt, perm, st, u in w.lookups[:4]:
        assert np.array_equal(e.lookup_resources_ids(rt, perm, st, u), o.lookup_resources_ids(rt, perm, st, u))
    c = e.prefix_counters()
    assert c["device_filters"] >= 3 and c["host_filters"] == 0 and c["matched"] >= 3000


def test_named_cfg4_digit_prefixes(zg):
    """Named cfg4 at about 2 M relationships: digit prefixes of each resource type's names against numpy."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.02)
    e = zg.Engine(w.schema, device=0)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    assert w.n_tuples() > 1_500_000
    for rt in sorted({g.res_type for g in w.groups}):
        for digits in ("0000", "00012", "000123"):
            prefix = f"{rt}{digits}"
            lo = int(digits.ljust(7, "0"))
            hi = lo + 10 ** (7 - len(digits))
            keys = set()
            for gi, g in enumerate(w.groups):
                if g.res_type != rt:
                    continue
                m = (g.res >= lo) & (g.res < hi)
                cls = (g.rel, g.subj_type, g.srel, g.wildcard)
                keys.update((cls, int(r), 0 if g.wildcard else int(s)) for r, s in zip(g.res[m], g.subj[m]))
            got = e.read_relationships(res_type=rt, res_id_prefix=prefix)
            assert len(got) == len(keys), (prefix, len(got), len(keys))
            assert all(split_rel(l)[1].startswith(prefix) for l in got)
            page = e.read_relationships_page(100, None, res_id_prefix=prefix)
            assert page[0] == [l for l in _pages(e, 1000, res_id_prefix=prefix)[0][0]][:100]
    assert e.prefix_counters()["host_filters"] == 0
