"""zg_import_relationships on the GPU (csrc/import.cuh): names resolved and deduplicated, keys sorted and duplicates
found on the device. The property: after every import, ids, reads and the watch feed equal a host-only engine's that
ran the same imports (the host path), and checks and LookupResources equal those of an engine that wrote the same
relationships in the same order through zg_write_relationships. Also: failures leave the device mirror, the snapshot
and the revision untouched; duplicates against the resident snapshot (an expired one not yet collected included);
ZGPU_VERIFY_BUILD=1; sharded handles against a replica; a standalone shard; device ingress of the new names;
concurrent checkers."""
import random
import threading

import numpy as np
import pytest

import filter_cases as cases
import randgen as R
import test_import_host as th

pytestmark = pytest.mark.gpu

CREATE = 1
EINVAL, EEXIST = -1, -2
NO_OBJECT = 0xFFFFFFFF


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _dev(zg, schema=cases.EXP_SCHEMA, clock=100, **kw):
    e = zg.Engine(schema, device=0, **kw)
    e.set_clock(clock)
    return e


def _checks(rels):
    """Check texts over the objects the relationships name: every doc against every user and group member."""
    docs = sorted({th._split(r)[1] for r, _ in rels if r.startswith("doc:")})[:25]
    users = sorted({th._split(r)[4] for r, _ in rels if "@user:" in r and not r.endswith("@user:*")})[:20]
    return [("doc", d, p, "user", u, "") for d in docs for u in users + ["nobody"] for p in ("view", "viewer")]


def _lookups(e, rels):
    users = sorted({th._split(r)[4] for r, _ in rels if "@user:" in r and not r.endswith("@user:*")})[:8]
    return [sorted(e.lookup_resources_str("doc", "view", "user", u)) for u in users]


def _compare(zg, dev, host, wr, every, r0):
    assert th._ids(zg, dev, every) == th._ids(zg, host, every) == th._ids(zg, wr, every)
    assert dev.read_relationships() == host.read_relationships() == wr.read_relationships()
    assert th._feed(dev, r0[0]) == th._feed(host, r0[1])
    assert list(dev.iter_relationships(97)) == list(host.iter_relationships(97))
    c = _checks(every)
    assert np.array_equal(dev.check_bulk_str(c), wr.check_bulk_str(c))
    assert _lookups(dev, every) == _lookups(wr, every)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_imports_equal_host_path_and_writes(zg, seed):
    rng = random.Random(seed)
    dev, host, wr = _dev(zg), th._engine(zg), _dev(zg)
    if seed == 3:  # into a populated store
        pre = th._exp_rels(rng, 150, "p")
        for e in (dev, host, wr):
            th._write(zg, e, pre)
    r0 = (dev.stats()["revision"], host.stats()["revision"])
    every = [] if seed != 3 else list(pre)
    for k in range(3):
        rels = [r for r in th._exp_rels(rng, 250, f"c{k % 2}") if r[0] not in dict(every)]
        assert dev.import_relationships(dev.import_groups(rels)) == len(rels)
        host.import_relationships(host.import_groups(rels))
        order = th._call_order(zg, rels)
        th._write(zg, wr, order)
        every += order
        _compare(zg, dev, host, wr, every, r0)
    assert dev.import_counters()["device"] == 3 and dev.import_counters()["host"] == 0


def test_expirations_at_two_clocks(zg):
    rng = random.Random(5)
    rels = th._exp_rels(rng, 300)
    dev, wr = _dev(zg), _dev(zg)
    dev.import_relationships(dev.import_groups(rels))
    th._write(zg, wr, th._call_order(zg, rels))
    for clock in (100, 40):
        dev.set_clock(clock)
        wr.set_clock(clock)
        c = _checks(rels)
        assert np.array_equal(dev.check_bulk_str(c), wr.check_bulk_str(c))


def test_failures_leave_the_device_untouched(zg):
    rng = random.Random(9)
    e = _dev(zg)
    base = th._exp_rels(rng, 200)
    e.import_relationships(e.import_groups(base))
    probe = (["new0", "new39", "bad", "x"], ["nu0", "nu39", "x", "nu3"])
    e.check_bulk_packed_ingress("doc", "viewer", "user", *probe)  # the mirror holds every name of the store
    ing = e.ingress_counters()
    rev, reads = e.stats()["revision"], e.read_relationships()
    row = e.debug_row("doc", "viewer", e.find("doc", "d1"))
    fresh = [(f"doc:new{i}#viewer@user:nu{i}", 0) for i in range(40)]
    cases_ = [(fresh[:20] + [("doc:bad!#viewer@user:x", 0)] + fresh[20:], EINVAL, 20),
              (fresh + [base[5]], EEXIST, 40),  # against the snapshot
              (fresh[:7] + [fresh[3]], EEXIST, 7),  # within the call
              (fresh + [("doc:x#banned@user:*", 0)], EINVAL, None)]
    expired = [(r, x) for r, x in base if x == 50 and r.startswith("doc:") and "#viewer@user:" in r]
    if expired:
        cases_.append((fresh[:3] + [(expired[0][0], 0)], EEXIST, 3))
    for rels, code, at in cases_:
        groups = [(*th._lit(r), [th._split(r)[1]], [th._split(r)[4]], [x] if x else None) for r, x in rels]
        with pytest.raises(zg.ZgpuError) as ex:
            e.import_relationships(groups)
        assert ex.value.code == code
        if at is not None:
            assert f"relationship {at}" in str(ex.value)
        assert e.stats()["revision"] == rev and e.read_relationships() == reads
        assert np.array_equal(e.debug_row("doc", "viewer", e.find("doc", "d1")), row)
        assert e.find("doc", "new0") == NO_OBJECT and e.find("user", "nu0") == NO_OBJECT
    # the failed imports' names reached neither the store nor the device mirror: a sync after them uploads nothing
    assert e.resolve_checks_packed("doc", "viewer", "user", *probe)["res"].tolist() == [NO_OBJECT] * 4
    assert (e.check_bulk_packed_ingress("doc", "viewer", "user", *probe) == 1).all()
    after = e.ingress_counters()
    for k in ("names", "device_bytes", "sync_uploads", "rebuilds"):
        assert after[k] == ing[k], k
    assert e.import_counters()["device"] == 1
    assert e.import_last_times()["total"] > 0  # the successful import's, not clobbered by the failures


def test_verify_build(zg, monkeypatch):
    monkeypatch.setenv("ZGPU_VERIFY_BUILD", "1")
    rng = random.Random(4)
    e = _dev(zg)
    for k in range(2):
        e.import_relationships(e.import_groups(th._exp_rels(rng, 300, f"v{k}")))
    e.write_relationships([(CREATE, "doc:after#viewer@user:v0u1", 0)])


@pytest.mark.parametrize("shards", [2, 3, 4])
def test_sharded_handle_against_a_replica(zg, shards):
    rng = random.Random(shards)
    h, rep = _dev(zg, n_shards=shards), _dev(zg)
    every = []
    for k in range(2):
        rels = [r for r in th._exp_rels(rng, 250, f"s{k}") if r[0] not in dict(every)]
        h.import_relationships(h.import_groups(rels))
        rep.import_relationships(rep.import_groups(rels))
        every += rels
        assert th._ids(zg, h, every) == th._ids(zg, rep, every)
        assert h.read_relationships() == rep.read_relationships()
        c = _checks(every)
        assert np.array_equal(h.check_bulk_str(c), rep.check_bulk_str(c))
    with pytest.raises(zg.ZgpuError) as ex:
        h.import_relationships(h.import_groups([every[-1]]))
    assert ex.value.code == EEXIST


def test_standalone_shard_refuses(zg):
    e = zg.Engine(cases.EXP_SCHEMA, device=0, shard_rank=0, shard_count=2)
    with pytest.raises(zg.ZgpuError) as ex:
        e.import_relationships(e.import_groups([("doc:a#viewer@user:u", 0)]))
    assert ex.value.code == EINVAL
    assert e.find("doc", "a") == NO_OBJECT


def test_device_ingress_resolves_new_names(zg):
    e = _dev(zg)
    e.write_relationships([(CREATE, "doc:seed#viewer@user:seed", 0)])
    e.check_bulk_packed_ingress("doc", "view", "user", ["seed"], "seed")  # builds the mirror
    before = e.ingress_counters()
    rels = [(f"doc:i{i}#viewer@user:iu{i % 17}", 0) for i in range(300)]
    e.import_relationships(e.import_groups(rels))
    res = [f"i{i}" for i in range(300)]
    subj = [f"iu{(i + (i % 3 == 0)) % 17}" for i in range(300)]
    got = e.check_bulk_packed_ingress("doc", "view", "user", res, subj)
    assert np.array_equal(got, e.check_bulk_packed("doc", "view", "user", res, subj))
    assert (got == 2).sum() == sum(1 for i in range(300) if i % 3)  # HAS_PERMISSION where the subject matches
    assert e.ingress_counters()["rebuilds"] == before["rebuilds"]


def test_checkers_see_one_revision_or_the_next(zg):
    e = _dev(zg)
    e.write_relationships([(CREATE, "doc:c#viewer@user:base", 0)])
    rels = [(f"doc:c{i}#viewer@user:cc", 0) for i in range(2000)]
    items = [("doc", f"c{i}", "view", "user", "cc", "") for i in range(0, 2000, 7)]
    seen, errors, stop = set(), [], threading.Event()

    def checker():
        while not stop.is_set():
            try:
                seen.add(tuple(int(x) for x in set(e.check_bulk_str(items).tolist())))
            except Exception as ex:  # noqa: BLE001
                errors.append(ex)
                return

    threads = [threading.Thread(target=checker) for _ in range(16)]
    for t in threads:
        t.start()
    e.import_relationships(e.import_groups(rels))
    stop.set()
    for t in threads:
        t.join()
    assert not errors
    assert seen <= {(1,), (2,)}  # all NO_PERMISSION (before) or all HAS_PERMISSION (after), never a mix
    assert set(e.check_bulk_str(items).tolist()) == {2}


def test_scale_calls_of_many(zg):
    rng = np.random.default_rng(0)
    n_docs, n_users, n = 40_000, 20_000, 300_000
    pairs = np.unique(rng.integers(0, n_docs, n) * n_users + rng.integers(0, n_users, n))
    res, subj = pairs // n_users, pairs % n_users
    order = rng.permutation(pairs.size)
    res, subj = res[order], subj[order]
    e, host = _dev(zg), th._engine(zg)
    for lo in range(0, pairs.size, 100_000):
        g = [("doc", "viewer", "user", "", [f"d{x}" for x in res[lo:lo + 100_000]],
              [f"u{x}" for x in subj[lo:lo + 100_000]], None)]
        e.import_relationships(g)
        host.import_relationships(g)
    assert e.num_tuples() == pairs.size
    rid = np.array([e.find("doc", f"d{x}") for x in range(0, n_docs, 97)])
    assert np.array_equal(rid, [host.find("doc", f"d{x}") for x in range(0, n_docs, 97)])
    # the page order is K: (resource id, subject id) -- numpy's sorted keys over the same ids
    ids_r = np.array([e.find("doc", f"d{x}") for x in range(n_docs)], dtype=np.int64)
    ids_s = np.array([e.find("user", f"u{x}") for x in range(n_users)], dtype=np.int64)
    want = np.sort(ids_r[res] * (1 << 32) + ids_s[subj])
    lines, _, _, _, _ = e.read_relationships_page(5000)
    got = [(e.find("doc", l.split("#")[0][4:]) << 32) + e.find("user", l.split("@user:")[1]) for l in lines]
    assert np.array_equal(np.array(got, dtype=np.int64), want[:5000])
    assert list(e.iter_relationships(50_000)) == list(host.iter_relationships(50_000))


def test_empty_import(zg):
    e = _dev(zg)
    r0 = e.stats()["revision"]
    assert e.import_relationships([("doc", "viewer", "user", "", [], [], None)]) == 0
    assert e.stats()["revision"] == r0 + 1 and e.read_relationships() == []
    assert e.import_relationships(e.import_groups([("doc:a#viewer@user:u", 0)])) == 1
    assert e.read_relationships() == ["doc:a#viewer@user:u"]


def _named(t, i):
    return "%s%d" % (t[:2], i)


@pytest.mark.parametrize("seed", [0, 1, 4])
def test_shaped_schemas_against_the_oracle(zg, seed):
    """randgen's generated schemas (every relation layout and class position of its plans), imported by name in two
    calls (the second into a populated store). Checks equal the oracle's at two clocks; LookupResources and
    LookupSubjects equal those of an engine that loaded the same relationships by id with the same names."""
    from oracle.pyoracle import Oracle

    rng = random.Random(seed)
    text, plan = R.shaped_schema(rng, **({"n_pairs": seed + 1} if seed < 5 else {}))
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan)
    o = Oracle(text)
    R.load_shaped(o, store)
    e = _dev(zg, text, clock=store["now"])
    seen = set()  # a class's relationships appear once however many groups hold them
    for half in (0, 1):
        groups = []
        for rt, rel, st, res, subj, srel, ex in store["groups"]:
            k = res.size // 2
            sl = slice(0, k) if half == 0 else slice(k, res.size)
            keep = [j for j in range(sl.start, sl.stop) if (rt, rel, st, srel, int(res[j]), int(subj[j])) not in seen]
            seen.update((rt, rel, st, srel, int(res[j]), int(subj[j])) for j in keep)
            if not keep:
                continue
            groups.append((rt, rel, st, "" if srel in (None, "*") else srel, [_named(rt, int(res[j])) for j in keep],
                           ["*"] * len(keep) if srel == "*" else [_named(st, int(subj[j])) for j in keep],
                           None if ex is None else ex[keep]))
        e.import_relationships(groups)
    ref = _dev(zg, text, clock=store["now"])  # the same names at the oracle's ids, loaded by id
    top = {}
    for rt, rel, st, res, subj, srel, ex in store["groups"]:
        top[rt] = max(top.get(rt, 0), int(res.max()) + 1)
        if srel != "*":
            top[st] = max(top.get(st, 0), int(subj.max()) + 1)
    for t, n in sorted(top.items()):
        assert ref.intern_packed(t, [_named(t, i) for i in range(n)]).tolist() == list(range(n))
    R.load_shaped(ref, store)
    ref.publish()
    queries, res, subj = R.shaped_checks(rng, store, plan, 4000)
    items = R.shaped_items(o, zg.CHECK_DTYPE, queries, res, subj)
    strs = [(rt, _named(rt, int(r)), perm, st, _named(st, int(u)), sr or "")
            for (rt, perm, st, sr), r, u in zip(queries, res.tolist(), subj.tolist())]
    for now in ((store["now"], store["now"] + 1000) if plan["expiry"] else (store["now"],)):
        e.set_clock(now)
        ref.set_clock(now)
        assert np.array_equal(e.check_bulk_str(strs), o.check_bulk(items, now=now)), (seed, now)
    e.set_clock(store["now"])
    ref.set_clock(store["now"])
    perms = sorted({(rt, perm, st) for rt, perm, st, sr in queries if sr is None})[:4]
    for rt, perm, st in perms:
        for r in range(0, top.get(rt, 1), max(1, top.get(rt, 1) // 6)):
            # answers come in internal-id order, and the two engines' ids differ: compare them as sets
            got, want = (x.lookup_subjects_str(rt, _named(rt, r), perm, st) for x in (e, ref))
            assert (sorted(got[0]), got[1], sorted(got[2])) == (sorted(want[0]), want[1], sorted(want[2]))
        for u in range(0, top.get(st, 1), max(1, top.get(st, 1) // 6)):
            assert sorted(e.lookup_resources_str(rt, perm, st, _named(st, u))) == \
                sorted(ref.lookup_resources_str(rt, perm, st, _named(st, u)))


def test_named_cfg4_in_calls_of_a_million(zg):
    """A named cfg4-shaped store at scale 0.05 (4.8 M relationships) imported in calls of 1 048 576: the page order equals
    numpy's sorted keys over the engine's ids, and checks by name equal those of the same store loaded by id."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.05)
    cls = {}
    for g in w.groups:
        k = (g.res_type, g.rel, g.subj_type, "*" if g.wildcard else (g.srel or ""))
        r, s = cls.get(k, (np.zeros(0, np.int64), np.zeros(0, np.int64)))
        cls[k] = (np.concatenate([r, g.res.astype(np.int64)]), np.concatenate([s, g.subj.astype(np.int64)]))
    for k, (r, s) in cls.items():
        key = np.unique(r * (1 << 32) + s)
        cls[k] = (key >> 32, key & 0xFFFFFFFF)
    flat = [(k, i) for k, (r, _) in cls.items() for i in range(r.size)]
    total = len(flat)
    e = _dev(zg, w.schema)
    call, at = 1 << 20, 0
    keys = list(cls)
    while at < total:
        groups, left, pos = [], call, 0
        for k in keys:
            r, s = cls[k]
            a, b = max(at - pos, 0), min(at - pos + left, r.size)
            if a < b:
                rt, rel, st, sr = k
                groups.append((rt, rel, st, "" if sr == "*" else sr, [workloads.object_name(rt, x) for x in r[a:b].tolist()],
                               ["*"] * (b - a) if sr == "*" else [workloads.object_name(st, x) for x in s[a:b].tolist()], None))
                left -= b - a
            pos += r.size
        assert e.import_relationships(groups) == call - left
        at += call - left
    assert e.num_tuples() == total
    # K order of one relation's pages: (resource id, class position, subject id) over the engine's ids
    rt, rel, st, sr = next(k for k in keys if k[3] == "" and k[0] == "document")
    r, s = cls[(rt, rel, st, sr)]
    rid = e.intern_packed(rt, [workloads.object_name(rt, x) for x in range(int(r.max()) + 1)]).astype(np.int64)
    sid = e.intern_packed(st, [workloads.object_name(st, x) for x in range(int(s.max()) + 1)]).astype(np.int64)
    flt = {"res_type": rt, "rel": rel, "subj_type": st, "subj_rel": "..."}
    lines = list(e.iter_relationships(100_000, **flt))
    got = np.array([(int(rid_of) << 32) | int(sid_of) for rid_of, sid_of in
                    ((e.find(rt, l.split("#")[0].split(":", 1)[1]), e.find(st, l.split("@")[1].split(":", 1)[1])) for l in lines[:20000])])
    want = np.sort(rid[r] * (1 << 32) + sid[s])
    assert len(lines) == r.size and np.array_equal(got, want[:20000])
    ref = zg.Engine(w.schema, device=0)
    workloads.intern_names(w, ref)
    w.load_into(ref)
    ref.publish()
    c = w.checks[0]
    names = [[workloads.object_name(t, int(i)) for i in ids[:20000]] for t, ids in ((c.res_type, c.res), (c.subj_type, c.subj))]
    assert np.array_equal(e.check_bulk_packed(c.res_type, c.perm, c.subj_type, *names),
                          ref.check_bulk_packed(c.res_type, c.perm, c.subj_type, *names))
