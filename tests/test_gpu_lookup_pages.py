"""Pages of LookupResources on the GPU (zg_lookup_resources_page, zg_lookup_resources_page_str; Device::lookup_page):
paged through at several limits, the concatenation equals the unpaged answer and the oracle's; each page holds at most
`limit` ids, `more` is exact, an empty page's next cursor is its `after`, and every per-id cursor resumes after its id.
Also the exhaustive and flat candidate sources, expiry, userset subjects, the depth cap, writes between pages, sharded
handles, concurrency, and the point of the windows: a small page verifies a small share of the candidates."""
import random
import threading

import numpy as np
import pytest

import randgen
import shard_lookup_cases as cases

pytestmark = pytest.mark.gpu

EINVAL, EDEPTH = -1, -9
LIMITS = (1, 2, 7, 100, 1000)
TOUCH, DELETE = 0, 2


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _id_pages(e, q, limit, srel=None, check_cursors=True):
    """Every page of the id form of lookup q = (rt, perm, st, subj) -> the concatenated ids; asserts the page rules."""
    out, cur, first = [], None, True
    while True:
        ids, curs, nxt, more = e.lookup_resources_page(*q, srel=srel, limit=limit, after=cur)
        assert len(ids) <= limit and len(curs) == len(ids)
        if more:
            assert len(ids) == limit, (q, limit)
        if not len(ids):
            assert not more and (first or nxt == cur), (q, limit)
        elif check_cursors:
            assert curs[-1] == nxt
            k = random.Random(len(out)).randrange(len(ids))  # a per-id cursor resumes right after its id
            rest = e.lookup_resources_page(*q, srel=srel, limit=1, after=curs[k])[0]
            if k + 1 < len(ids):
                assert list(rest) == [ids[k + 1]], (q, limit, k)
        out += [int(i) for i in ids]
        cur, first = nxt, False
        if not more:
            return out


def _str_pages(e, q, limit):
    out, cur = [], None
    while True:
        names, curs, nxt, more = e.lookup_resources_page_str(*q, limit=limit, after=cur)
        assert len(names) <= limit and len(curs) == len(names)
        if more:
            assert len(names) == limit
        if not names and cur is not None:
            assert nxt == cur
        out += names
        cur = nxt
        if not more:
            return out


def _agree_ids(e, q, want, limits=LIMITS, srel=None):
    whole = e.lookup_resources_ids(*q, srel=srel) if srel else e.lookup_resources_ids(*q)
    assert np.array_equal(whole, want), q
    for limit in limits:
        got = _id_pages(e, q, limit, srel, check_cursors=limit <= 7)
        assert got == [int(i) for i in want], (q, limit)


@pytest.mark.parametrize("wl,scale", [("cfg2", 0.002), ("cfg3", 0.005), ("cfg4", 0.002)])
def test_workloads_id_and_string_forms(zg, wl, scale):
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    e, o = zg.Engine(w.schema, device=0), Oracle(w.schema)
    workloads.intern_names(w, e)
    w.load_into(e), w.load_into(o)
    e.publish()
    before = e.lookup_page_counters()
    for q in w.lookups:
        want = o.lookup_resources_ids(*q)
        _agree_ids(e, q, want)
        rt, perm, st, u = q
        sq = (rt, perm, st, workloads.object_name(st, u), "")
        names = e.lookup_resources_str(*sq)
        for limit in (1, 7, 1000):
            assert _str_pages(e, sq, limit) == names, (q, limit)
    c = e.lookup_page_counters()
    assert c["windowed_pages"] > before["windowed_pages"] and c["cut_pages"] == 0


def _strings_engine(zg, schema, rels, expires=None, now=0, **kw):
    e = zg.Engine(schema, device=0, **kw)
    if now:
        e.set_clock(now)
    ups = [(TOUCH, r, (expires or {}).get(r, 0)) for r in rels]
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])
    return e


def _agree_strings(zg, schema, rels, lookups, expires=None, now=0, limits=(1, 2, 7, 1000), **kw):
    from oracle.pyoracle import Oracle

    o = Oracle(schema)
    for r in rels:
        o.touch(r, (expires or {}).get(r, 0))
    e = _strings_engine(zg, schema, rels, expires, now, **kw)
    for q in lookups:
        want = cases.oracle_answer(o, q, now)
        try:
            whole = e.lookup_resources_str(*q)
        except zg.ZgpuError as x:
            assert x.code == EDEPTH and want is None, q
            continue
        assert sorted(whole) == want, q
        for limit in limits:
            assert _str_pages(e, q, limit) == whole, (q, limit)
        rt, perm, st, sid, srel = q
        sub = e.find(st, sid)
        if sub != 0xFFFFFFFF:
            ids = e.lookup_resources_ids(rt, perm, st, sub, srel=srel or None)
            for limit in limits:
                assert _id_pages(e, (rt, perm, st, sub), limit, srel or None) == [int(i) for i in ids], (q, limit)
    return e


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas(zg, name):
    schema, rels, lookups = cases.random_case(9800, fixed=name)
    _agree_strings(zg, schema, rels, lookups)


@pytest.mark.parametrize("seed", range(4))
def test_random_schemas(zg, seed):
    schema, rels, lookups = cases.random_case(9810 + seed)
    _agree_strings(zg, schema, rels, lookups)


@pytest.mark.parametrize("seed", range(3))
def test_shaped_schemas(zg, seed):
    from oracle.pyoracle import Oracle

    rng = random.Random(seed)
    text, plan = randgen.shaped_schema(rng, n_pairs=seed + 1)
    store = randgen.shaped_relationships(rng, randgen.model_from_schema(text), plan)
    o = Oracle(text)
    randgen.load_shaped(o, store)
    e = zg.Engine(text, device=0)
    randgen.load_shaped(e, store)
    e.publish()
    e.set_clock(store["now"])
    users = sorted(set(store["split"]))[:6]
    for perm in ("view", "only_l2"):
        for u in users:
            _agree_ids(e, ("doc", perm, "user", u), o.lookup_resources_ids("doc", perm, "user", u, now=store["now"]),
                       limits=(1, 7, 100, 1000))


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_exhaustive_candidates(zg, name, monkeypatch):
    monkeypatch.setenv("ZGPU_NO_RBFS", "1")  # read when the engine is created
    schema, rels, lookups = cases.random_case(9820, fixed=name)
    _agree_strings(zg, schema, rels, lookups)


def test_flat_path_with_repeated_ids(zg):
    """pod#view = viewer + creator is a flat union: the answer is the subject's reverse rows, where a pod that names
    the user as viewer and as creator appears twice. No candidate is verified."""
    from spicedb_kubeapi_proxy_b200 import workloads

    rels = [f"pod:p{i}#viewer@user:a" for i in range(0, 3000, 2)] + [f"pod:p{i}#creator@user:a" for i in range(0, 3000, 3)]
    e = _strings_engine(zg, workloads.CFG2_SCHEMA, rels)
    q = ("pod", "view", "user", e.find("user", "a"))
    want = e.lookup_resources_ids(*q)
    assert len(want) == len({r.split("#")[0] for r in rels})
    _agree_ids(e, q, want)
    c = e.lookup_page_counters()
    assert c["windowed_pages"] > 0 and c["verified"] == 0 and c["windows"] == 0


@pytest.mark.parametrize("now", [100, 200])
def test_expiry(zg, now):
    from test_lookup_subjects import EXP_SCHEMA

    rng = random.Random(9830)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=6, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    _agree_strings(zg, EXP_SCHEMA, rels, cases.random_lookups(rng, model, rels, 10), expires, now)


def test_userset_subjects_written_and_never_written(zg):
    from test_oracle_random import SELF_LOOKUPS, SELF_RELS, SELF_SCHEMA

    lookups = [q for q, _ in SELF_LOOKUPS]
    e = _agree_strings(zg, SELF_SCHEMA, SELF_RELS, lookups)
    # never written doc:9#viewer: no id, its own name after every id, with the cursor past the ids
    q = ("doc", "view", "doc", "9", "viewer")
    assert e.lookup_resources_str(*q) == ["9"]
    names, curs, nxt, more = e.lookup_resources_page_str(*q, limit=1)
    assert names == ["9"] and not more and curs == [nxt]
    assert e.lookup_resources_page_str(*q, limit=1, after=nxt)[:1] == ([],)
    # a written subject with ids and itself: doc:5#viewer -> 3, 5 in id order, 5 by the self candidate
    q = ("doc", "view", "doc", "5", "viewer")
    whole = e.lookup_resources_str(*q)
    assert _str_pages(e, q, 1) == whole and sorted(whole) == ["3", "5"]
    e.write_relationships([(TOUCH, "doc:1#viewer@doc:9#viewer", 0)])  # now doc:9 is written, 1 and 9 answer
    assert _str_pages(e, ("doc", "view", "doc", "9", "viewer"), 1) == e.lookup_resources_str("doc", "view", "doc", "9", "viewer")


def test_depth_cap_fails_only_the_pages_that_reach_it(zg):
    """g0 .. g4 are more than 50 dispatches from user:deep and cannot be decided; they are interned last, so their ids
    follow every decidable group's. The unpaged call fails; pages whose deciding answer comes before them succeed and
    give the oracle's answer in id order; the page that reaches them fails."""
    from oracle.pyoracle import Oracle
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i + 1}#member" for i in range(5, 55)] + ["group:g55#member@user:deep"]
    rels += [f"group:g{i}#member@group:g{i + 1}#member" for i in range(0, 5)]
    e = _strings_engine(zg, CHAIN, rels)
    o = Oracle(CHAIN)
    for r in rels:
        o.touch(r, 0)
    good = sorted(e.find("group", n) for n in o.lookup_resources("group", "member", "user", "deep", ""))
    bad = [e.find("group", f"g{i}") for i in range(5)]
    assert len(good) > 20 and max(good) < min(bad)
    q = ("group", "member", "user", e.find("user", "deep"))
    with pytest.raises(zg.ZgpuError) as x:
        e.lookup_resources_ids(*q)
    assert x.value.code == EDEPTH
    ids, _, nxt, more = e.lookup_resources_page(*q, limit=10)
    assert list(ids) == good[:10] and more
    ids, _, _, more = e.lookup_resources_page(*q, limit=len(good) - 1)
    assert list(ids) == good[:-1] and more
    for limit, after in ((len(good), None), (1000, None), (1000, nxt)):
        with pytest.raises(zg.ZgpuError) as x:
            e.lookup_resources_page(*q, limit=limit, after=after)
        assert x.value.code == EDEPTH, limit
    # paging by one: every page before the undecidable ones succeeds, in order, then the one that reaches them fails
    got, cur = [], None
    with pytest.raises(zg.ZgpuError) as x:
        while True:
            ids, _, cur, more = e.lookup_resources_page(*q, limit=1, after=cur)
            got += [int(i) for i in ids]
            assert more
    assert x.value.code == EDEPTH and got == good[:-1]


def test_paging_across_writes_collections_and_retirements(zg):
    schema = ("use expiration\ndefinition user {}\ndefinition doc {\n  relation viewer: user with expiration\n"
              "  relation editor: user\n  permission view = viewer + editor\n}\n")
    e = zg.Engine(schema, device=0)
    e.set_clock(1000)
    stable = [f"doc:s{i}#editor@user:a" for i in range(3000)]
    for i in range(0, len(stable), 1000):
        e.write_relationships([(TOUCH, r, 0) for r in stable[i:i + 1000]])
    a = e.find("user", "a")
    rng = random.Random(9840)
    seen, cur, rounds = [], None, 0
    churn = []
    while True:
        ids, _, cur, more = e.lookup_resources_page("doc", "view", "user", a, limit=97, after=cur)
        seen += [int(i) for i in ids]
        if rounds < 5:  # 1 000 interleaved writes: new docs, expiring ones, and deletes of the churn
            ups, new = [], []
            for k in range(1000):  # each relationship once per write: deletes only of earlier rounds' docs
                if churn and rng.random() < 0.3:
                    ups.append((DELETE, churn.pop(rng.randrange(len(churn))), 0))
                else:
                    new.append(f"doc:c{rounds}_{k}#viewer@user:a")
                    ups.append((TOUCH, new[-1], rng.choice([0, 1500])))
            churn += new
            e.write_relationships(ups)
        elif rounds == 5:
            e.set_clock(2000)
            e.collect_expired(2000)
            e.retire_unused_names()
        rounds += 1
        if not more:
            break
    assert len(seen) == len(set(seen)) and seen == sorted(seen)
    want = {e.find("doc", f"s{i}") for i in range(3000)}
    assert want <= set(seen)


def test_retirement_between_resolving_and_answering_the_string_form(zg):
    """A retirement forced between resolving and answering the string form: the page runs again and never prints the
    name that took the retired id."""
    from test_gpu_retire import SCHEMA, T, _apply, _hook_once, _retire_and_reuse

    e = zg.Engine(SCHEMA)
    e.set_clock(T)
    _apply(e, ["doc:keep#viewer@user:a", "doc:d1#viewer@user:a"], TOUCH)

    def drop_d1():
        _apply(e, ["doc:d1#viewer@user:a"], DELETE)
        _retire_and_reuse(e, ("doc", "d1"), ("doc", "z"))

    calls = _hook_once(e, drop_d1)
    names, curs, nxt, more = e.lookup_resources_page_str("doc", "view", "user", "a", limit=10)
    e.set_resolve_hook(None)
    assert len(calls) == 2 and names == ["keep"] and not more


@pytest.mark.parametrize("S", [2, 3, 4])
def test_sharded_handles_equal_a_replica(zg, S):
    schema, rels, lookups = cases.random_case(9850 + S, fixed="nesting")
    rep = _strings_engine(zg, schema, rels)
    h = _strings_engine(zg, schema, rels, n_shards=S, handle_lookups=True)
    for q in lookups:
        for limit in (1, 2, 7, 1000):
            cur_r = cur_h = None
            while True:
                try:
                    a = rep.lookup_resources_page_str(*q, limit=limit, after=cur_r)
                except zg.ZgpuError as x:
                    with pytest.raises(zg.ZgpuError):
                        h.lookup_resources_page_str(*q, limit=limit, after=cur_h)
                    break
                b = h.lookup_resources_page_str(*q, limit=limit, after=cur_h)
                assert a == b, (q, limit)
                cur_r, cur_h = a[2], b[2]
                if not a[3]:
                    break
    assert h.lookup_page_counters()["cut_pages"] > 0 and h.lookup_page_counters()["windowed_pages"] == 0


def test_sharded_refusals(zg):
    """A handle without handle_lookups and a standalone shard refuse pages with the unpaged call's code and message."""
    schema, rels, lookups = cases.random_case(9860)
    rt, perm, st = lookups[0][:3]
    for e in (zg.Engine(schema, device=0, n_shards=2), zg.Engine(schema, device=0, shard_rank=0, shard_count=2)):
        out = []
        for fn in (lambda: e.lookup_resources_ids(rt, perm, st, 0), lambda: e.lookup_resources_page(rt, perm, st, 0, limit=3),
                   lambda: e.lookup_resources_str(rt, perm, st, "x"),
                   lambda: e.lookup_resources_page_str(rt, perm, st, "x", limit=3)):
            with pytest.raises(zg.ZgpuError) as x:
                fn()
            out.append((x.value.code, str(x.value)))
        assert out[0] == out[1] and out[2] == out[3] and out[0][0] == EINVAL, out


def test_sixteen_threads_paging_beside_lookups_checks_and_a_writer(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg2", 0.002)
    e = zg.Engine(w.schema, device=0)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    want = {q: [int(i) for i in e.lookup_resources_ids(*q)] for q in w.lookups[:8]}
    items = w.check_items(e, zg.CHECK_DTYPE)[:5000]
    codes = e.check_bulk(items)
    errors, stop = [], threading.Event()

    def pager(k):
        try:
            for i in range(6):
                q = w.lookups[(k + i) % 8]
                assert _id_pages(e, q, (1, 7, 100)[i % 3], check_cursors=False) == want[q]
        except Exception as x:  # noqa: BLE001
            errors.append(repr(x))

    def other():
        try:
            while not stop.is_set():
                assert np.array_equal(e.check_bulk(items), codes)
                q = w.lookups[0]
                assert [int(i) for i in e.lookup_resources_ids(*q)] == want[q]
        except Exception as x:  # noqa: BLE001
            errors.append(repr(x))

    def writer():
        n = 0
        while not stop.is_set():  # a user no lookup asks about: the answers stay as they were
            e.write_relationships([(TOUCH, f"pod:zz{n}#viewer@user:zz", 0)])
            n += 1

    threads = [threading.Thread(target=pager, args=(k,)) for k in range(16)]
    threads += [threading.Thread(target=other), threading.Thread(target=writer)]
    for t in threads:
        t.start()
    for t in threads[:16]:
        t.join()
    stop.set()
    for t in threads[16:]:
        t.join()
    assert not errors, errors[:3]


def test_small_page_verifies_few_candidates_on_cfg4(zg):
    """cfg4 at full size (scale 1, 95 M relationships): the first page of 100 equals the first 100 of the unpaged answer and
    verifies far fewer candidates than follow the cursor; a limit as large as the answer verifies them all."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=1.0)
    e = zg.Engine(w.schema, device=0)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    sizes = [(len(e.lookup_resources_ids(*q)), q) for q in w.lookups]
    n, q = max(sizes)
    assert n > 1000
    whole = e.lookup_resources_ids(*q)
    c0 = e.lookup_page_counters()
    ids, _, _, more = e.lookup_resources_page(*q, limit=100)
    c1 = e.lookup_page_counters()
    assert np.array_equal(ids, whole[:100]) and more
    after, verified = c1["after_cursor"] - c0["after_cursor"], c1["verified"] - c0["verified"]
    assert verified * 10 < after, (verified, after)
    ids, _, _, more = e.lookup_resources_page(*q, limit=n)
    c2 = e.lookup_page_counters()
    assert np.array_equal(ids, whole) and not more
    assert c2["verified"] - c1["verified"] == c2["after_cursor"] - c1["after_cursor"]
