"""LookupSubjects answered by a sharded handle (zg_config.n_shards = S with ZG_FLAG_HANDLE_SUBJECTS): the forward walk
runs on every shard of the one engine, each discovery written into its owner's inbox through peer memory, and both
verifications run on the handle's own check protocol. Every answer is compared with a replica engine fed the same
relationships (the same ids), and with the LookupSubjects oracle where the store is small. With one GPU the shards are
virtual: they share device 0."""
import ctypes
import os
import random
import threading

import numpy as np
import pytest

import randgen
import shard_lookup_cases as slc
import shard_subjects_cases as cases
import zgpu
from lookup_subjects_oracle import EXCLUDE, INCLUDE

pytestmark = pytest.mark.gpu

EINVAL, E2BIG, EDEPTH = -1, -7, -9  # include/zgpu.h


@pytest.fixture(scope="module")
def zg():
    return zgpu


def _pair(zg, schema, S, loader, now=None, **flags):
    """(flagged handle, replica), both loaded by loader(engine) and published."""
    h = zg.Engine(schema, device=0, n_shards=S, handle_subjects=True, **flags)
    rep = zg.Engine(schema, device=0)
    for e in (h, rep):
        loader(e)
        e.publish()
        if now is not None:
            e.set_clock(now)
    return h, rep


def _ans(e, rt, res, perm, st, srel=None, opt=INCLUDE):
    """zg_lookup_subjects -> (ids, wildcard, excluded), or None for ZG_EDEPTH."""
    try:
        return e.lookup_subjects_ids(rt, int(res), perm, st, srel or None, wildcards=opt)
    except zgpu.ZgpuError as ex:
        if ex.code == EDEPTH:
            return None
        raise


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2])


def _names_case(zg, schema, rels, lookups, S, expires=None, now=None, **flags):
    """lookups: ((rt, rid, perm, st, srel), option) by name. Each is asked of a flagged handle and a replica, whose
    answers must be equal; -> (the handle's answers by name, the oracle's, the handle)."""
    names = slc.intern(rels)
    h, rep = _pair(zg, schema, S, lambda e: slc.load(e, rels, names, expires), now, **flags)
    got = []
    for q, opt in lookups:
        rt, rid, perm, st, srel = q
        res = names.get((rt, rid), cases.NEVER_WRITTEN)
        a, b = _ans(h, rt, res, perm, st, srel, opt), _ans(rep, rt, res, perm, st, srel, opt)
        assert _same(a, b), f"S={S} {q} opt={opt}: handle={a} replica={b}"
        got.append(cases.names_of(names, st, a))
    c = cases.oracle(schema, rels, expires)
    return got, [cases.oracle_answer(c, q, opt, now or 0) for q, opt in lookups], h


@pytest.mark.parametrize("S", [2, 3, 4, 8])
def test_hand_table(zg, S):
    from test_lookup_subjects import HAND, HAND_EXPIRES, HAND_RELS, HAND_TABLE

    lookups = cases.with_options([q for q, _, _ in HAND_TABLE])
    got, want, h = _names_case(zg, HAND, HAND_RELS, lookups, S, expires=HAND_EXPIRES, now=100)
    cases.agree(got, want, lookups)
    for q, opt, expect in HAND_TABLE:  # the fenced divergence row d4 included
        assert got[lookups.index((q, opt))] == (None if expect == "EDEPTH" else expect), q
    c = h.handle_subjects_counters()
    assert c["lookups"] == len(lookups)  # the never-written resource and the failed lookups included
    assert c["levels"] > 0 and c["candidates"] > 0 and c["inbox_entries"] > 0 and c["nowild_items"] > 0


@pytest.mark.parametrize("S", [2, 3, 4])
def test_no_wildcards_holds_in_the_sub_queries_raised_to_other_shards(zg, S):
    """doc:d#view reaches a `user:*` only through folder:f, owned by another shard: the no-wildcards verification
    must hold in the pass that evaluates the sub-query raised there, or bob (editor, not member2) is listed."""
    names = slc.intern(cases.REMOTE_WILD_RELS)
    assert names[("doc", "d")] % S != names[("folder", "f")] % S
    lookups = cases.with_options(cases.REMOTE_WILD_QUERIES)
    got, want, h = _names_case(zg, cases.REMOTE_WILD, cases.REMOTE_WILD_RELS, lookups, S)
    cases.agree(got, want, lookups)
    assert got[:2] == [([], True, []), ([], False, [])]
    assert h.handle_subjects_counters()["nowild_items"] > 0


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("S", [2, 3])
def test_random_and_fixed_schemas(zg, seed, S):
    """Plain and userset (#member-like) subject types, never-written resources included."""
    fixed = sorted(randgen.FIXED_SCHEMAS)[seed % len(randgen.FIXED_SCHEMAS)] if seed % 2 else None
    schema, rels, queries = cases.random_case(9700 + seed, fixed=fixed)
    assert any(q[4] for q in queries), "userset subject types"
    lookups = cases.with_options(queries)
    got, want, _ = _names_case(zg, schema, rels, lookups, S)
    cases.agree(got, want, lookups)


@pytest.mark.parametrize("S", [2, 4])
def test_userset_subjects(zg, S):
    rels = ["group:g1#member@group:g2#member", "group:g2#member@user:frank", "doc:d#viewer@group:g1#member",
            "doc:d#viewer@group:g3#member", "group:g3#member@user:ann", "doc:e#viewer@user:ann"]
    schema = """
definition user {}
definition group { relation member: user | group#member }
definition doc {
  relation viewer: user | group#member
  permission view = viewer
}
"""
    lookups = cases.with_options([("doc", "d", "view", "group", "member"), ("doc", "d", "view", "user", ""),
                                  ("group", "g1", "member", "group", "member"), ("doc", "e", "view", "group", "member")])
    got, want, _ = _names_case(zg, schema, rels, lookups, S)
    cases.agree(got, want, lookups)
    assert got[0] == (["g1", "g2", "g3"], False, [])


@pytest.mark.parametrize("S", [2, 4])
def test_expiry_at_two_clocks(zg, S):
    from lookup_subjects_oracle import subject_queries
    from test_lookup_subjects import EXP_SCHEMA

    rng = random.Random(9800)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    lookups = cases.with_options(subject_queries(model, rng, 6, per_type=3))
    answers = []
    for now in (100, 200):
        got, want, _ = _names_case(zg, EXP_SCHEMA, rels, lookups, S, expires=expires, now=now)
        cases.agree(got, want, lookups)
        answers.append(got)
    assert answers[0] != answers[1]


@pytest.mark.parametrize("S", [2, 3])
def test_depth_cap_fails_that_call_and_the_next_is_answered(zg, S):
    from test_lookup_subjects import HAND, HAND_RELS

    names = slc.intern(HAND_RELS)
    h, rep = _pair(zg, HAND, S, lambda e: slc.load(e, HAND_RELS, names))
    with pytest.raises(zg.ZgpuError, match="could not be decided") as ex:
        h.lookup_subjects_ids("group", names[("group", "c0")], "member", "user")
    assert ex.value.code == EDEPTH
    for q in (("doc", "d1", "view"), ("group", "g1", "member")):
        a = _ans(h, q[0], names[q[:2]], q[2], "user")
        assert a is not None and _same(a, _ans(rep, q[0], names[q[:2]], q[2], "user")), q


BIG_SCHEMA = """
definition user {}
definition group { relation member: user | group#member }
definition doc {
  relation viewer: user | user:* | group#member
  relation banned: user
  permission view = viewer - banned
}
"""


def _big_rels():
    rels = [f"doc:big#viewer@user:u{i}" for i in range(5000)] + ["doc:big#banned@user:u7", "doc:w#viewer@user:*"]
    rels += [f"doc:w#banned@user:u{i}" for i in range(0, 3000, 3)] + [f"group:g#member@user:u{i}" for i in range(2000)]
    rels += ["doc:gd#viewer@group:g#member", "doc:small#viewer@user:u1"]
    return rels


def test_forced_fallback_verifies_every_subject(zg, monkeypatch):
    """ZGPU_LOOKUP_BATCH_CAP=1 (raised to its floor, 1 024): a walk whose outbox passes it verifies every object of
    the subject type the shard owns. Answers unchanged."""
    rels = _big_rels()
    names = slc.intern(rels)
    rep = zg.Engine(BIG_SCHEMA, device=0)
    slc.load(rep, rels, names)
    rep.publish()
    monkeypatch.setenv("ZGPU_LOOKUP_BATCH_CAP", "1")
    h = zg.Engine(BIG_SCHEMA, device=0, n_shards=3, handle_subjects=True)
    slc.load(h, rels, names)
    h.publish()
    for rid in ("big", "w", "gd", "small"):
        for opt in (INCLUDE, EXCLUDE):
            a = _ans(h, "doc", names[("doc", rid)], "view", "user", opt=opt)
            assert _same(a, _ans(rep, "doc", names[("doc", rid)], "view", "user", opt=opt)), (rid, opt)
    assert _ans(h, "doc", names[("doc", "big")], "view", "user")[0].size == 4999
    c = h.handle_subjects_counters()
    assert c["fallbacks"] > 0 and c["fallbacks"] < c["lookups"], c


def test_no_rbfs_verifies_every_subject(zg, monkeypatch):
    schema, rels, queries = cases.random_case(9900, fixed="nesting")
    monkeypatch.setenv("ZGPU_NO_RBFS", "1")
    lookups = cases.with_options(queries)
    got, want, h = _names_case(zg, schema, rels, lookups, 3)
    cases.agree(got, want, lookups)
    c = h.handle_subjects_counters()
    assert c["levels"] == 0 and c["fallbacks"] == c["lookups"] > 0


def test_string_form_and_a_never_written_resource(zg):
    from test_lookup_subjects import HAND, HAND_RELS

    h, rep = _pair(zg, HAND, 3, lambda e: e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in HAND_RELS]))
    for rid, perm in (("d1", "view"), ("d2", "view2"), ("d4", "diverge"), ("nope", "view"), ("never", "view2")):
        for opt in (INCLUDE, EXCLUDE):
            assert h.lookup_subjects_str("doc", rid, perm, "user", wildcards=opt) == \
                rep.lookup_subjects_str("doc", rid, perm, "user", wildcards=opt), (rid, opt)
    assert h.lookup_subjects_str("doc", "d1", "view", "user") == (["alice"], True, ["bob"])
    assert h.lookup_subjects_str("doc", "never", "view", "user") == ([], False, [])
    assert h.lookup_subjects_str("group", "g1", "member", "group", "member") == \
        rep.lookup_subjects_str("group", "g1", "member", "group", "member")


def test_e2big_for_ids_and_for_exclusions(zg):
    rels = [f"doc:d#viewer@user:u{i}" for i in range(40)] + ["doc:d#viewer@user:*"]
    rels += [f"doc:d#banned@user:b{i}" for i in range(30)]
    h, rep = _pair(zg, BIG_SCHEMA, 4, lambda e: e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels]))
    L = h._L
    args = (h.slot_id("doc", "view"), h.find("doc", "d"), h.type_id("user"), zg._lib.SREL_NONE, INCLUDE)
    n, nx, wild = ctypes.c_uint64(0), ctypes.c_uint64(0), ctypes.c_int32(0)
    ids, ex = np.zeros(64, dtype=np.uint32), np.zeros(64, dtype=np.uint32)
    # ids too small, exclusions large enough; then the other way round: both sizes are reported each time
    for cap, ex_cap in ((1, 64), (64, 1)):
        rc = L.zg_lookup_subjects(h._h, *args, ids.ctypes.data, cap, ctypes.byref(n), ex.ctypes.data, ex_cap,
                                  ctypes.byref(nx), ctypes.byref(wild))
        assert rc == E2BIG and n.value == 40 and nx.value == 30 and wild.value == 1, (cap, ex_cap)
    rc = L.zg_lookup_subjects(h._h, *args, ids.ctypes.data, 64, ctypes.byref(n), ex.ctypes.data, 64, ctypes.byref(nx),
                              ctypes.byref(wild))
    assert rc == 0
    want = rep.lookup_subjects_ids("doc", h.find("doc", "d"), "view", "user")
    assert np.array_equal(ids[:n.value], want[0]) and np.array_equal(ex[:nx.value], want[2]) and want[1]
    buf, need, cnt = ctypes.create_string_buffer(8), ctypes.c_size_t(0), ctypes.c_uint64(0)
    rc = L.zg_lookup_subjects_str(h._h, b"doc", b"d", b"view", b"user", b"", INCLUDE, buf, 8, ctypes.byref(need),
                                  ctypes.byref(cnt))
    assert rc == E2BIG and cnt.value == 40 + 1 + 30
    assert h.lookup_subjects_str("doc", "d", "view", "user") == rep.lookup_subjects_str("doc", "d", "view", "user")


def test_client_lookup_subjects_equals_a_replica_client(zg):
    from test_lookup_subjects import HAND, HAND_EXPIRES, HAND_RELS, HAND_TABLE

    C = zg.client
    cl = C.PermissionsClient(HAND, engine=zg.Engine(HAND, n_shards=3, handle_subjects=True))
    rep = C.PermissionsClient(HAND)
    ups = [C.RelationshipUpdate(C.OPERATION_TOUCH, C.Relationship.parse(r)) for r in HAND_RELS if r not in HAND_EXPIRES]
    for c in (cl, rep):
        c.WriteRelationships(C.WriteRelationshipsRequest(ups))
    for (rt, rid, perm, st, srel), _, _ in HAND_TABLE:
        for opt in (C.WILDCARD_OPTION_INCLUDE_WILDCARDS, C.WILDCARD_OPTION_EXCLUDE_WILDCARDS):
            req = C.LookupSubjectsRequest(C.ObjectReference(rt, rid), perm, st, srel, opt)

            def run(client):
                try:
                    return [(r.subject.subject_object_id, [x.subject_object_id for x in r.excluded_subjects])
                            for r in client.LookupSubjects(req)]
                except C.RpcError as ex:
                    return ("error", ex.code)

            assert run(cl) == run(rep), (rid, perm, opt)
    got = [r.subject.subject_object_id for r in cl.LookupSubjects(C.LookupSubjectsRequest(C.ObjectReference("doc", "d1"), "view", "user"))]
    assert got == ["alice", "*"]


def _workload_lookups(w, n, seed, usersets=False):
    rng = np.random.default_rng(seed)
    out = []
    for c in w.checks[:2]:
        for r in rng.choice(np.unique(c.res), size=min(n, np.unique(c.res).size), replace=False):
            out += [(c.res_type, int(r), c.perm, c.subj_type, None, opt) for opt in (INCLUDE, EXCLUDE)]
            if usersets:
                out.append((c.res_type, int(r), c.perm, "group", "member", INCLUDE))
    return out


def _agree_with_replica(h, rep, lookups):
    for rt, r, p, st, srel, opt in lookups:
        a = _ans(h, rt, r, p, st, srel, opt)
        assert a is not None and _same(a, _ans(rep, rt, r, p, st, srel, opt)), (rt, r, p, st, srel, opt)


@pytest.mark.parametrize("wl,scale", [("cfg2", 0.002), ("cfg3", 0.002), ("cfg4", 0.001)])
@pytest.mark.parametrize("S", [2, 4])
def test_workloads_agree_with_a_replica(zg, wl, scale, S):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    h, rep = _pair(zg, w.schema, S, w.load_into)
    _agree_with_replica(h, rep, _workload_lookups(w, 8, 5, usersets=wl == "cfg4"))
    c = h.handle_subjects_counters()
    assert c["levels"] > 0 and c["inbox_entries"] > 0


def test_cfg4_full_size_scale_agrees_with_a_replica(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=float(os.environ.get("ZGPU_FULLSIZE_SCALE", "0.25")))
    h, rep = _pair(zg, w.schema, 4, w.load_into)
    rng = np.random.default_rng(11)
    docs = np.unique(np.concatenate([c.res for c in w.checks if c.res_type == "document"]))
    lookups = [("document", int(r), p, "user", None, opt) for p in ("view", "restricted_view")
               for r in rng.choice(docs, size=8, replace=False) for opt in (INCLUDE, EXCLUDE)]
    _agree_with_replica(h, rep, lookups)


def test_handle_equals_the_multi_engine_driver_and_a_replica(zg):
    from spicedb_kubeapi_proxy_b200 import dist as zdist
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.002)
    S = 4
    h, rep = _pair(zg, w.schema, S, w.load_into)
    ts = zdist.LocalDeviceTransport.cluster(S)
    engines = [zg.Engine(w.schema, device=0, shard_rank=r, shard_count=S) for r in range(S)]
    for e in engines:
        w.load_into(e)
        e.publish()
    lookups = _workload_lookups(w, 6, 13)
    e0 = engines[0]
    reqs = [(e0.type_id(rt), r, e0.slot_id(rt, p), e0.type_id(st), slc.SREL_NONE, opt) for rt, r, p, st, _, opt in lookups]
    out, _ = cases.run_sharded(engines, ts, [reqs] + [[] for _ in range(S - 1)], walk_cap=1 << 22)
    for (rt, r, p, st, srel, opt), d in zip(lookups, out[0]):
        a = _ans(h, rt, r, p, st, srel, opt)
        assert a is not None and _same(a, d) and _same(a, _ans(rep, rt, r, p, st, srel, opt)), (rt, r, p, opt)


def test_answers_follow_5x1000_updates_merged_into_every_shard(zg):
    from lookup_subjects_oracle import subject_queries

    schema = randgen.FIXED_SCHEMAS["nesting"]
    rng = random.Random(9920)
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=40, n_user=25, density=0.12)
    pool = randgen.random_relationships(rng, model, n_obj=80, n_user=50, density=0.3)
    assert len(pool) >= 1000
    queries = subject_queries(model, rng, 40, per_type=4)
    h = zg.Engine(schema, device=0, n_shards=3, handle_subjects=True)
    rep = zg.Engine(schema, device=0)
    for e in (h, rep):
        e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels])
    for _ in range(5):
        ups = [((zg._lib.OP_DELETE if rng.random() < 0.3 else zg._lib.OP_TOUCH), r, 0) for r in rng.sample(pool, 1000)]
        for e in (h, rep):
            e.write_relationships(ups)
        for rt, rid, perm, st, srel in queries:
            for opt in (INCLUDE, EXCLUDE):
                assert h.lookup_subjects_str(rt, rid, perm, st, srel, opt) == rep.lookup_subjects_str(rt, rid, perm, st, srel, opt)
    assert h.stats()["delta_publishes"] > 0 or h.stats()["full_publishes"] > 0


def test_threads_look_up_subjects_while_others_check_look_up_resources_and_write(zg):
    schema = randgen.FIXED_SCHEMAS["nesting"]
    rng = random.Random(9910)
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.15)
    churn = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.05)
    from lookup_subjects_oracle import subject_queries

    subj_q = subject_queries(model, rng, 30, per_type=4)
    res_q = slc.random_lookups(rng, model, rels, 20)
    checks = [r for r in rels if "#" not in r.split("@")[1]][:64]
    h, rep = _pair(zg, schema, 4, lambda e: e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels]),
                   handle_lookups=True)
    for e in (h, rep):  # intern the churn's names in the same order on both engines
        e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in churn])
        e.write_relationships([(zg._lib.OP_DELETE, r, 0) for r in churn if r not in rels])
    moving = [r for r in churn if r not in rels]
    assert moving
    stop, errs, last = threading.Event(), [], {}

    def writer():
        i = 0
        while not stop.is_set():
            r = moving[i % len(moving)]
            op = zg._lib.OP_TOUCH if (i // len(moving)) % 2 == 0 else zg._lib.OP_DELETE
            h.write_relationships([(op, r, 0)])
            last[r] = op
            i += 1

    def guard(fn):
        def run(t):
            try:
                fn(t)
            except Exception as ex:  # noqa: BLE001
                if getattr(ex, "code", 0) != EDEPTH:
                    errs.append(repr(ex))
        return run

    @guard
    def subjects(t):
        for j in range(4):
            rt, rid, perm, st, srel = subj_q[(t + j * 7) % len(subj_q)]
            h.lookup_subjects_str(rt, rid, perm, st, srel, INCLUDE if j % 2 else EXCLUDE)

    @guard
    def resources(t):
        for j in range(3):
            rt, perm, st, sid, srel = res_q[(t + j * 5) % len(res_q)]
            h.lookup_resources_str(rt, perm, st, sid, srel)

    @guard
    def check(t):
        h.check_bulk_str(checks)

    wt = threading.Thread(target=writer)
    wt.start()
    ths = [threading.Thread(target=f, args=(t,)) for t in range(24) for f in (subjects, resources, check)]
    [x.start() for x in ths]
    [x.join() for x in ths]
    stop.set()
    wt.join()
    assert not errs, errs[:5]
    for r, op in last.items():  # the writer's last state, replayed on the replica
        rep.write_relationships([(op, r, 0)])
    assert sorted(rep.read_relationships()) == sorted(h.read_relationships())
    for rt, rid, perm, st, srel in subj_q:
        for opt in (INCLUDE, EXCLUDE):
            assert h.lookup_subjects_str(rt, rid, perm, st, srel, opt) == rep.lookup_subjects_str(rt, rid, perm, st, srel, opt)
    for rt, perm, st, sid, srel in res_q:
        assert h.lookup_resources_str(rt, perm, st, sid, srel) == rep.lookup_resources_str(rt, perm, st, sid, srel)


def test_flag_combinations(zg):
    import torch

    from spicedb_kubeapi_proxy_b200 import workloads

    rel = "pod:ns/p1#viewer@user:a"
    only = zg.Engine(workloads.BOOTSTRAP_SCHEMA, n_shards=2, handle_subjects=True)
    both = zg.Engine(workloads.BOOTSTRAP_SCHEMA, n_shards=2, handle_subjects=True, handle_lookups=True)
    rep = zg.Engine(workloads.BOOTSTRAP_SCHEMA)
    for e in (only, both, rep):
        e.write_relationships([(zg._lib.OP_TOUCH, rel, 0)])
    # handle_subjects alone: LookupSubjects answered, LookupResources and the pre-filter refused as without the flag
    assert only.lookup_subjects_str("pod", "ns/p1", "view", "user") == (["a"], False, [])
    for call in (lambda: only.lookup_resources_ids("pod", "view", "user", only.find("user", "a")),
                 lambda: only.lookup_resources_str("pod", "view", "user", "a"),
                 lambda: only.list_prefilter(b'{"items": [{"metadata": {"name": "p1", "namespace": "ns"}}]}',
                                             only.list_template("pod", "view", "user", "a"))):
        with pytest.raises(zg.ZgpuError, match="LookupResources, LookupSubjects and the list pre-filter are not served") as ex:
            call()
        assert ex.value.code == EINVAL
    # both flags: both calls served
    assert both.lookup_subjects_str("pod", "ns/p1", "view", "user") == rep.lookup_subjects_str("pod", "ns/p1", "view", "user")
    assert both.lookup_resources_str("pod", "view", "user", "a") == ["ns/p1"]
    assert both.handle_subjects_counters()["lookups"] == 1 and both.handle_lookup_counters()["rounds"] == 1
    # the device-buffer, ingress and zg_shard_*_dev calls stay refused under either flag
    d_items = torch.zeros(16 * 4, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(4, dtype=torch.uint8, device="cuda")
    for h in (only, both):
        calls = {
            "device": (lambda: h.check_bulk_device(d_items.data_ptr(), 4, d_out.data_ptr()), "device buffers"),
            "ingress": (lambda: h.check_bulk_packed_ingress("pod", "view", "user", ["ns/p1"], ["a"]), "device-ingress"),
            "shard pass": (lambda: h.shard_pass_dev(d_items.data_ptr(), 4, 0), "zg_shard_"),
            "shard nowild": (lambda: h.shard_pass_nowild_dev(d_items.data_ptr(), 4, 0), "zg_shard_"),
            "shard subjects": (lambda: h.shard_subjects_candidates_dev(False, 0, 0), "zg_shard_"),
        }
        for what, (call, msg) in calls.items():
            with pytest.raises(zg.ZgpuError, match=msg) as ex:
                call()
            assert ex.value.code == EINVAL, what
            assert "sharded handle" in str(ex.value), what
    assert list(only.check_bulk_str(["pod:ns/p1#view@user:a", "pod:ns/p1#view@user:b"])) == [2, 1]


def test_shards_on_several_devices(zg):
    import torch

    from spicedb_kubeapi_proxy_b200 import workloads

    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs >= 2 GPUs")
    w = workloads.cfg4(scale=0.005)
    h = zg.Engine(w.schema, device=0, n_devices=n_dev, n_shards=2 * n_dev, handle_subjects=True)
    rep = zg.Engine(w.schema, device=0)
    for e in (h, rep):
        w.load_into(e)
        e.publish()
    _agree_with_replica(h, rep, _workload_lookups(w, 4, 17))
