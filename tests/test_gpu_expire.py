"""zg_collect_expired on the GPU: the scan of the resident snapshot (csrc/filter.cuh filter_expired_kernel), the
DELETEs and the merge-publish. The property: at clocks T, T + 1 and T + 10^6 every check, LookupResources,
LookupSubjects and ReadRelationships answer the same before and after collect_expired(T), and as the oracle does. Also
the count against a host-only engine, the device and host paths, sharded handles, a standalone shard, two devices,
the proxy's idempotency keys, incremental writes and concurrent callers."""
import random
import threading

import pytest

import filter_cases as cases
import randgen
from golden_runner import split_rel

pytestmark = pytest.mark.gpu

TOUCH, DELETE = 0, 2
T = 1_000_000
CLOCKS = (T, T + 1, T + 10 ** 6)

# owner may not carry an expiration: its rows are never scanned
SCHEMA = """
use expiration
definition user {}
definition group { relation member: user with expiration | group#member with expiration }
definition doc {
  relation viewer: user with expiration | user:* with expiration | group#member with expiration
  relation owner: user | user:* | group#member
  relation banned: user with expiration
  permission view = viewer + owner - banned
  permission edit = owner & view
}
"""


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _with_expiration(schema, rng):
    """A random schema with `with expiration` on about half of every relation's allowed subject types."""
    out = ["use expiration"]
    for line in schema.splitlines():
        if line.strip().startswith("relation "):
            head, types = line.split(": ", 1)
            line = head + ": " + " | ".join(t + (" with expiration" if rng.random() < 0.6 else "") for t in types.split(" | "))
        out.append(line)
    return "\n".join(out) + "\n"


def _expirations(rng, schema_text, rels):
    """T - 2 .. T + 2 and T + 10^6 (+1) on the relationships whose class allows it, none on the rest."""
    allowed, where = set(), None
    for line in schema_text.splitlines():
        if line.startswith("definition "):
            where = line.split()[1].rstrip("{")
        if "relation " not in line:
            continue
        for part in line.split("relation ")[1:]:  # "definition group { relation member: ... }" on one line too
            rel, types = part.split(":", 1)
            for t in types.split("}")[0].split(" | "):
                if t.strip().endswith(" with expiration"):
                    allowed.add((where, rel.strip(), t.strip()[: -len(" with expiration")].strip()))
    ex = {}
    for r in rels:
        rt, rid, rel, st, sid, srel = split_rel(r)
        kind = st + (":*" if sid == "*" else (f"#{srel}" if srel else ""))
        if (rt, rel, kind) in allowed and rng.random() < 0.75:
            ex[r] = rng.choice([T - 2, T - 1, T, T, T + 1, T + 2, T + 10 ** 6, T + 10 ** 6 + 1])
    return ex


def _write(e, rels, expires):
    ups = [(TOUCH, r, expires.get(r, 0)) for r in rels]
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])


def _queries(model, n_obj, n_user):
    types = model["types"]
    tnames = model.get("tnames", list(types))
    users = [f"u{i}" for i in range(n_user)] + ["nobody"]  # an id no relationship names: only wildcards grant it
    checks, lookups, subjects = [], [], []
    for t in tnames:
        perms = list(types[t]["perms"])
        for o in range(n_obj):
            for p in perms + list(types[t]["rels"]):
                checks += [f"{t}:o{o}#{p}@user:{u}" for u in users]
                for st in tnames:  # userset subjects
                    for sr in list(types[st]["rels"])[:2]:
                        checks.append(f"{t}:o{o}#{p}@{st}:o{(o + 1) % n_obj}#{sr}")
            subjects += [(t, f"o{o}", p, "user", "") for p in perms]
        lookups += [(t, p, "user", u, "") for p in perms for u in users]
    return checks, lookups, subjects


def _answers(e, queries, clock, subjects_too=True):
    checks, lookups, subjects = queries
    e.set_clock(clock)
    got = {"checks": [int(x) for x in e.check_bulk_str([split_rel(c) for c in checks])],
           "lookups": [sorted(e.lookup_resources_str(*q)) for q in lookups],
           "read": e.read_relationships()}
    if subjects_too:
        got["subjects"] = [e.lookup_subjects_str(*q) for q in subjects]
    return got


def _oracle(schema, rels, expires):
    from oracle.pyoracle import Oracle

    o = Oracle(schema)
    for r in rels:
        o.touch(r, expires.get(r, 0))
    return o


def _invariance(zg, schema, model, rels, expires, n_obj, n_user, **kw):
    """Answers at every clock of CLOCKS before and after collect_expired(T) on a device engine (kw) equal, and equal
    the oracle's checks; the count equals a host-only engine's; the tuple count drops by it."""
    d, h = zg.Engine(schema, **kw), zg.Engine(schema, host_only=True)
    for e in (d, h):
        e.set_clock(T - 10)
        _write(e, rels, expires)
    q = _queries(model, n_obj, n_user)
    subjects_too = "n_shards" not in kw or kw.get("handle_subjects", False)
    before = {c: _answers(d, q, c, subjects_too) for c in CLOCKS}
    o = _oracle(schema, rels, expires)
    for c in CLOCKS:
        want = [o.check(*split_rel(x), c) for x in q[0]]
        assert before[c]["checks"] == want, c
        for lk, got in zip(q[1], before[c]["lookups"]):
            assert got == sorted(o.lookup_resources(*lk, c)), (lk, c)
    tuples, fc = d.stats()["tuples"], d.filter_counters()
    d.set_clock(T)
    h.set_clock(T)
    n = d.collect_expired(T)
    assert n == h.collect_expired(T) == sum(1 for r in set(rels) if 0 < expires.get(r, 0) <= T)
    assert d.stats()["tuples"] == tuples - n
    fc2 = d.filter_counters()
    assert fc2["host_filters"] == fc["host_filters"] and fc2["device_filters"] == fc["device_filters"] + 1
    assert fc2["by_scan"] == fc["by_scan"] + 1
    for c in CLOCKS:
        assert _answers(d, q, c, subjects_too) == before[c], c
    d.set_clock(1)
    h.set_clock(1)
    assert d.read_relationships() == h.read_relationships()
    return d, h, n


@pytest.mark.parametrize("seed", range(3))
def test_invariance_fixed_schema(zg, seed):
    rng = random.Random(11000 + seed)
    model = randgen.model_from_schema(SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5, density=0.4)
    rels = list(dict.fromkeys(rels + ["doc:o0#viewer@user:*", "doc:o1#owner@user:*", "doc:o2#viewer@user:*"]))
    ex = _expirations(rng, SCHEMA, rels)
    ex["doc:o0#viewer@user:*"], ex["doc:o2#viewer@user:*"] = T, T + 1
    _, _, n = _invariance(zg, SCHEMA, model, rels, ex, 5, 5)
    assert n > 0


@pytest.mark.parametrize("seed", range(5))
def test_invariance_random_schemas(zg, seed):
    rng = random.Random(11100 + seed)
    schema, model = randgen.random_schema(rng)
    schema = _with_expiration(schema, rng)
    rels = randgen.random_relationships(rng, model, n_obj=4, n_user=4, density=0.4)
    _invariance(zg, schema, model, rels, _expirations(rng, schema, rels), 4, 4)


def test_invariance_exp_schema_and_verified_merge(zg, monkeypatch):
    """Under ZGPU_VERIFY_BUILD=1 every publish, the collection's merge included, is compared array by array with a
    rebuild on the host."""
    monkeypatch.setenv("ZGPU_VERIFY_BUILD", "1")
    rng = random.Random(11200)
    model = randgen.model_from_schema(cases.EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=6, density=0.4) + ["doc:o1#viewer@user:*"]
    d, _, n = _invariance(zg, cases.EXP_SCHEMA, model, rels, _expirations(rng, cases.EXP_SCHEMA, rels), 6, 6)
    assert n > 0 and d.stats()["delta_publishes"] >= 1


def test_device_and_host_paths_remove_the_same(zg):
    rng = random.Random(11300)
    model = randgen.model_from_schema(SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=8, density=0.4)
    ex = _expirations(rng, SCHEMA, rels)
    a, b = zg.Engine(SCHEMA), zg.Engine(SCHEMA)
    for e in (a, b):
        e.set_clock(T - 10)
        _write(e, rels, ex)
        e.set_clock(T)
    # b: a change left unpublished (a relationship without expiration) sends the collection to the host scan
    import numpy as np

    t = np.zeros(1, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = b.intern("doc", "extra"), b.intern("user", "u0"), \
        b.slot_id("doc", "owner"), b.type_id("user"), 0xFFFF
    b.load_tuples(t)
    a.write_relationships([(TOUCH, "doc:extra#owner@user:u0", 0)])
    fa, fb = a.filter_counters(), b.filter_counters()
    na, nb = a.collect_expired(T), b.collect_expired(T)
    assert na == nb > 0
    ga, gb = a.filter_counters(), b.filter_counters()
    assert (ga["device_filters"] - fa["device_filters"], ga["host_filters"] - fa["host_filters"]) == (1, 0)
    assert (gb["device_filters"] - fb["device_filters"], gb["host_filters"] - fb["host_filters"]) == (0, 1)
    for e in (a, b):
        e.set_clock(1)
    assert a.read_relationships() == b.read_relationships()
    # nothing left to collect: one count launch, no publish
    rev = a.stats()["revision"]
    a.set_clock(T)
    assert a.collect_expired(T) == 0 and a.stats()["revision"] == rev


def _shard_rels(rng):
    model = randgen.model_from_schema(SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=6, density=0.4) + ["doc:o3#viewer@user:*"]
    return model, rels, _expirations(rng, SCHEMA, rels)


@pytest.mark.parametrize("S", [2, 3, 4])
def test_sharded_handle_against_a_replica(zg, S):
    rng = random.Random(11400 + S)
    model, rels, ex = _shard_rels(rng)
    d, _, n = _invariance(zg, SCHEMA, model, rels, ex, 8, 6, n_shards=S, handle_lookups=True, handle_subjects=True)
    r, _, m = _invariance(zg, SCHEMA, model, rels, ex, 8, 6)
    assert n == m > 0
    for e in (d, r):
        e.set_clock(T + 5)
    q = _queries(model, 8, 6)
    assert _answers(d, q, T + 5) == _answers(r, q, T + 5)


def test_standalone_shard(zg):
    rng = random.Random(11500)
    _, rels, ex = _shard_rels(rng)
    d = zg.Engine(SCHEMA, shard_rank=1, shard_count=3)
    d.set_clock(T - 10)
    _write(d, rels, ex)
    owned = [r for r in rels if d.find(*split_rel(r)[:2]) % 3 == 1]
    h = zg.Engine(SCHEMA, host_only=True)
    h.set_clock(T - 10)
    _write(h, owned, ex)
    for e in (d, h):
        e.set_clock(T)
    fc = d.filter_counters()
    assert d.collect_expired(T) == h.collect_expired(T) == sum(1 for r in set(owned) if 0 < ex.get(r, 0) <= T) > 0
    assert d.filter_counters()["device_filters"] == fc["device_filters"] + 1
    for e in (d, h):
        e.set_clock(1)
    assert d.read_relationships() == h.read_relationships()


def test_two_devices(zg):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = random.Random(11600)
    model, rels, ex = _shard_rels(rng)
    _invariance(zg, SCHEMA, model, rels, ex, 8, 6, n_devices=2)


def test_proxy_idempotency_keys(zg):
    """The proxy's dual write: every WriteRelationships carries workflow:<id>#idempotency_key@activity:<hash> with a
    24 h expiration. 10 000 writes, the clock advanced 24 h: every key goes, everything else stays and answers as
    before."""
    from spicedb_kubeapi_proxy_b200 import workloads

    schema = workloads.BOOTSTRAP_SCHEMA
    e = zg.Engine(schema)
    t0 = 1_700_000_000
    e.set_clock(t0)
    other = []
    for i in range(10_000):
        ns, pod = f"ns{i % 97}", f"ns{i % 97}/pod{i}"
        rel = f"pod:{pod}#namespace@namespace:{ns}" if i % 2 else f"namespace:{ns}#creator@user:u{i % 31}"
        other.append(rel)
        e.write_relationships([(TOUCH, rel, 0), (TOUCH, f"workflow:w{i}#idempotency_key@activity:h{i}", t0 + i // 100 + 86_400)])
    keep = sorted(set(other))
    checks = [("namespace", f"ns{k}", "view", "user", f"u{k % 31}", "") for k in range(97)]
    checks += [("pod", f"ns{k}/pod{k + 97}", "view", "user", f"u{k % 31}", "") for k in range(97)]
    e.set_clock(t0 + 200_000)
    before_checks = list(e.check_bulk_str(checks))
    before_read = e.read_relationships(res_type="namespace")
    tuples = e.stats()["tuples"]
    assert e.collect_expired(t0 + 86_400 + 100) == 10_000
    assert e.stats()["tuples"] == tuples - 10_000 == len(keep)
    assert list(e.check_bulk_str(checks)) == before_checks
    assert e.read_relationships(res_type="namespace") == before_read
    e.set_clock(1)
    assert e.read_relationships(res_type="workflow") == []
    assert sorted(e.read_relationships()) == keep


def test_interleaved_with_incremental_writes(zg):
    rng = random.Random(11700)
    model = randgen.model_from_schema(SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=80, n_user=80, density=0.2)
    rng.shuffle(rels)
    ex = _expirations(rng, SCHEMA, rels)
    d, h = zg.Engine(SCHEMA), zg.Engine(SCHEMA, host_only=True)
    base = rels[: len(rels) // 2]
    for e in (d, h):
        e.set_clock(T - 10)
        _write(e, base, ex)
    live, rest = list(base), rels[len(rels) // 2:]
    clock = T
    for r in range(5):
        ups = [(TOUCH, x, ex[x] + r if x in ex else 0) for x in rest[r * 500:(r + 1) * 500]]
        ups += [(DELETE, x, 0) for x in live[r * 500:(r + 1) * 500]]
        assert len(ups) == 1000
        for e in (d, h):
            e.set_clock(T - 10)
            e.write_relationships(ups)
            e.set_clock(clock)
        assert d.collect_expired(clock) == h.collect_expired(clock)
        clock += 1
    assert d.stats()["delta_publishes"] >= 5
    for e in (d, h):
        e.set_clock(1)
    assert d.read_relationships() == h.read_relationships()
    assert d.filter_counters()["host_filters"] == 0


def test_checkers_and_a_writer_beside_a_collector(zg):
    """14 checkers and a writer on 16 threads while a collector removes expired grants: the fixed grants (no expiration)
    always answer HAS, the expired ones always NO (clock T + 10), and nothing fails."""
    e = zg.Engine(SCHEMA)
    e.set_clock(T - 100)
    fixed = [f"doc:d{i}#owner@user:u{i}" for i in range(50)]
    _write(e, fixed, {})
    e.set_clock(T + 10)
    stop, errors = threading.Event(), []

    def checker(k):
        try:
            while not stop.is_set():
                got = list(e.check_bulk_str([("doc", f"d{k}", "view", "user", f"u{k}", ""), ("doc", f"d{k}", "viewer", "user", "x", "")]))
                assert got == [2, 1], got
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    def writer():
        try:
            for i in range(200):
                e.write_relationships([(TOUCH, f"doc:d{i % 14}#viewer@user:x", T - 50 + i % 40)])
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    removed = []

    def collector():
        try:
            while not stop.is_set():
                removed.append(e.collect_expired(T))
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    ths = [threading.Thread(target=checker, args=(k,)) for k in range(14)] + [threading.Thread(target=collector)]
    w = threading.Thread(target=writer)
    for t in ths + [w]:
        t.start()
    w.join()
    stop.set()
    for t in ths:
        t.join()
    assert not errors, errors[0]
    removed.append(e.collect_expired(T))
    e.set_clock(1)
    assert e.read_relationships(res_type="doc", rel="viewer") == []
    assert sum(removed) >= 14
