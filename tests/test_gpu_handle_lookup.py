"""LookupResources and the list pre-filter answered by a sharded handle (zg_config.n_shards = S with
ZG_FLAG_HANDLE_LOOKUPS): the reverse walk runs on every shard of the one engine, its frontier and answer keys cross the
shards through peer memory, and the candidates are verified by the handle's own check protocol. Every answer is
compared with a replica engine fed the same relationships (the same ids), and with the oracle where the store is
small. With one GPU the shards are virtual: they share device 0."""
import ctypes
import json
import os
import random
import threading

import numpy as np
import pytest

import randgen
import shard_lookup_cases as cases
import zgpu
from golden_runner import run_case, split_rel

pytestmark = pytest.mark.gpu

EINVAL, E2BIG, EDEPTH = -1, -7, -9  # include/zgpu.h


@pytest.fixture(scope="module")
def zg():
    return zgpu


def _pair(zg, schema, S, loader, now=None):
    """(flagged handle, replica), both loaded by loader(engine) and published."""
    h = zg.Engine(schema, device=0, n_shards=S, handle_lookups=True)
    rep = zg.Engine(schema, device=0)
    for e in (h, rep):
        loader(e)
        e.publish()
        if now is not None:
            e.set_clock(now)
    return h, rep


def _ids(e, rt, perm, st, subj, srel=None):
    """zg_lookup_resources -> ascending ids, or None for ZG_EDEPTH."""
    try:
        return e.lookup_resources_ids(rt, perm, st, subj, srel)
    except zgpu.ZgpuError as ex:
        if ex.code == EDEPTH:
            return None
        raise


def _same(a, b):
    return (a is None and b is None) or (a is not None and b is not None and np.array_equal(a, b))


def _string_case(zg, schema, rels, lookups, S, expires=None, now=None):
    """The lookups (names) on a flagged handle and a replica: -> (handle's names, replica's names, oracle's names)."""
    from oracle.pyoracle import Oracle

    names = cases.intern(rels)
    h, rep = _pair(zg, schema, S, lambda e: cases.load(e, rels, names, expires), now)
    o = Oracle(schema)
    for r in rels:
        o.touch(r, (expires or {}).get(r, 0))
    got, rgot = [], []
    for rt, perm, st, sid, srel in lookups:
        subj = names[(st, sid)]
        a, b = _ids(h, rt, perm, st, subj, srel or None), _ids(rep, rt, perm, st, subj, srel or None)
        assert _same(a, b), f"{(rt, perm, st, sid, srel)}: handle={a} replica={b}"
        got.append(cases.names_of(names, rt, a))
        rgot.append(cases.names_of(names, rt, b))
    return got, rgot, [cases.oracle_answer(o, q, now or 0) for q in lookups], h


@pytest.mark.parametrize("wl,scale", [("cfg2", 0.002), ("cfg3", 0.002), ("cfg4", 0.001)])
@pytest.mark.parametrize("S", [2, 3, 4, 8])
def test_workloads_equal_a_replica_and_the_oracle(zg, wl, scale, S):
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    h, rep = _pair(zg, w.schema, S, w.load_into)
    o = Oracle(w.schema)
    w.load_into(o)
    rng = np.random.default_rng(7)
    n_users = max(int(g.subj.max()) + 1 for g in w.groups if g.subj_type == "user" and not g.wildcard and g.subj.size)
    rt, perm = w.lookups[0][:2]
    lookups = [q + (None,) for q in w.lookups] + [(rt, perm, "user", int(u), None) for u in rng.integers(0, n_users, 8)]
    if wl == "cfg4":  # userset subjects
        lookups += [("document", "view", "group", g, "member") for g in (0, 1, 5)]
    before = h.handle_lookup_counters()
    for q in lookups:  # a repeated lookup is answered from the lookup cache
        a = _ids(h, *q)
        assert a is not None and np.array_equal(a, _ids(rep, *q)), f"{wl} S={S} {q}"
        if q[4] is None:
            assert np.array_equal(a, o.lookup_resources_ids(*q[:4])), f"{wl} S={S} {q}"
    c = h.handle_lookup_counters()
    assert c["rounds"] - before["rounds"] >= len(set(lookups)) and c["levels"] > before["levels"] and c["candidates"] > 0


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("S", [2, 3, 4])
def test_random_and_fixed_schemas(zg, seed, S):
    fixed = sorted(randgen.FIXED_SCHEMAS)[seed % len(randgen.FIXED_SCHEMAS)] if seed % 2 else None
    schema, rels, lookups = cases.random_case(9700 + seed, fixed=fixed, n_lookups=16)
    got, _, want, _ = _string_case(zg, schema, rels, lookups, S)
    assert got == want, schema


@pytest.mark.parametrize("S", [2, 3, 4])
def test_userset_subject_itself_written_and_never_written(zg, S):
    from test_oracle_random import SELF_LOOKUPS, SELF_RELS, SELF_SCHEMA

    lookups = [q for q, _ in SELF_LOOKUPS if q[3] != "9"]
    got, _, want, h = _string_case(zg, SELF_SCHEMA, SELF_RELS, lookups, S)
    assert got == want
    assert got[0] == ["3", "5"] and got[2] == ["5"] and got[4] == []
    # by name, the never-written subject naming itself included: engines loaded by name
    h, rep = _pair(zg, SELF_SCHEMA, S, lambda e: e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in SELF_RELS]))
    for q, _ in SELF_LOOKUPS:
        assert h.lookup_resources_str(*q) == rep.lookup_resources_str(*q), q
    assert h.lookup_resources_str("doc", "view", "doc", "9", "viewer") == ["9"]


@pytest.mark.parametrize("S", [2, 4])
def test_expiry_at_two_clocks(zg, S):
    from test_lookup_subjects import EXP_SCHEMA

    rng = random.Random(9800)
    model = randgen.model_from_schema(EXP_SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.4)
    expires = {r: rng.choice([50, 150]) for r in rels if rng.random() < 0.5}
    lookups = cases.random_lookups(rng, model, rels, 12)
    answers = []
    for now in (100, 200):
        got, _, want, _ = _string_case(zg, EXP_SCHEMA, rels, lookups, S, expires=expires, now=now)
        assert got == want
        answers.append(got)
    assert answers[0] != answers[1]


@pytest.mark.parametrize("S", [2, 3])
def test_depth_cap_fails_only_that_lookup_of_a_group(zg, S):
    """Concurrent callers share one round: exactly the lookup with the undecidable candidate gets ZG_EDEPTH."""
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i+1}#member" for i in range(55)] + ["group:g55#member@user:deep"]
    rels += ["group:x#member@user:v", "folder:f0#viewer@user:v", "folder:f1#parent@folder:f0"]
    lookups = [("group", "member", "user", "deep", ""), ("group", "member", "user", "v", ""),
               ("folder", "view", "user", "v", "")] * 4
    names = cases.intern(rels)
    h, rep = _pair(zg, CHAIN, S, lambda e: cases.load(e, rels, names))
    out, errs = [None] * len(lookups), []
    gate = threading.Barrier(len(lookups))

    def call(i):
        try:
            rt, perm, st, sid, _ = lookups[i]
            gate.wait()
            out[i] = _ids(h, rt, perm, st, names[(st, sid)])
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))

    th = [threading.Thread(target=call, args=(i,)) for i in range(len(lookups))]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs
    for i, (rt, perm, st, sid, _) in enumerate(lookups):
        want = _ids(rep, rt, perm, st, names[(st, sid)])
        assert _same(out[i], want), lookups[i]
        assert (out[i] is None) == (sid == "deep")


OVF_SCHEMA = """
definition user {}
definition group { relation member: user | group#member }
definition doc {
  relation viewer: user | group#member
  permission view = viewer
}
"""


def _overflow_rels():
    rels = [f"doc:a{i}#viewer@user:big" for i in range(5000)]
    rels += [f"doc:s{j}_{i}#viewer@user:s{j}" for j in range(16) for i in range(700)]
    rels += [f"group:g{j}#member@user:s{j}" for j in range(4)] + [f"doc:gd{i}#viewer@group:g{i % 4}#member" for i in range(40)]
    return rels


def test_forced_overflow_halves_a_group_and_falls_back_for_one_lookup(zg, monkeypatch):
    """ZGPU_LOOKUP_BATCH_CAP=1024 (its floor): a group of lookups whose candidates pass it on a shard is redone in
    halves; the one lookup whose own candidates pass it verifies every resource of the type. Answers unchanged."""
    rels = _overflow_rels()
    names = cases.intern(rels)
    rep = zg.Engine(OVF_SCHEMA, device=0)
    cases.load(rep, rels, names)
    rep.publish()
    monkeypatch.setenv("ZGPU_LOOKUP_BATCH_CAP", "1024")
    h = zg.Engine(OVF_SCHEMA, device=0, n_shards=2, handle_lookups=True)
    cases.load(h, rels, names)
    h.publish()
    uid = lambda u: names[("user", u)]  # noqa: E731
    c0 = h.handle_lookup_counters()
    big = _ids(h, "doc", "view", "user", uid("big"))
    assert np.array_equal(big, _ids(rep, "doc", "view", "user", uid("big"))) and big.size == 5000
    c1 = h.handle_lookup_counters()
    assert c1["fallbacks"] > c0["fallbacks"] and c1["halvings"] == c0["halvings"]
    users = [f"s{j}" for j in range(16)] * 3
    out, errs = [None] * len(users), []
    gate = threading.Barrier(len(users))

    def call(i):
        try:
            gate.wait()
            out[i] = _ids(h, "doc", "view", "user", uid(users[i]))
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))

    th = [threading.Thread(target=call, args=(i,)) for i in range(len(users))]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs
    for u, a in zip(users, out):
        want = _ids(rep, "doc", "view", "user", uid(u))
        assert np.array_equal(a, want) and a.size >= 700, u
    c2 = h.handle_lookup_counters()
    assert c2["halvings"] > c1["halvings"], c2
    assert h.stats()["lookup_batches"] > 0


def test_no_rbfs_verifies_every_resource(zg, monkeypatch):
    schema, rels, lookups = cases.random_case(9900, fixed="nesting", n_lookups=12)
    monkeypatch.setenv("ZGPU_NO_RBFS", "1")
    got, _, want, h = _string_case(zg, schema, rels, lookups, 3)
    assert got == want
    c = h.handle_lookup_counters()
    assert c["levels"] == 0 and c["fallbacks"] == c["rounds"] > 0


def test_concurrent_callers_form_groups_while_a_thread_writes(zg):
    schema = randgen.FIXED_SCHEMAS["nesting"]
    rng = random.Random(9910)
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.15)
    churn = randgen.random_relationships(rng, model, n_obj=30, n_user=20, density=0.05)
    lookups = cases.random_lookups(rng, model, rels, 40)
    h, rep = _pair(zg, schema, 4, lambda e: e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels]))
    for e in (h, rep):  # intern the churn's names in the same order on both engines
        e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in churn])
        e.write_relationships([(zg._lib.OP_DELETE, r, 0) for r in churn if r not in rels])
    names = {(st, sid): rep.find(st, sid) for _, _, st, sid, _ in lookups}
    stop, errs, last = threading.Event(), [], {}
    b0 = h.stats()["lookup_batches"]
    moving = [r for r in churn if r not in rels]
    assert moving

    def writer():
        i = 0
        while not stop.is_set():
            r = moving[i % len(moving)]
            op = zg._lib.OP_TOUCH if (i // len(moving)) % 2 == 0 else zg._lib.OP_DELETE
            h.write_relationships([(op, r, 0)])
            last[r] = op
            i += 1

    def caller(t):
        try:
            for j in range(4):
                rt, perm, st, sid, srel = lookups[(t + j * 7) % len(lookups)]
                h.lookup_resources_ids(rt, perm, st, names[(st, sid)], srel or None)
        except Exception as ex:  # noqa: BLE001
            if getattr(ex, "code", 0) != EDEPTH:
                errs.append(repr(ex))

    wt = threading.Thread(target=writer)
    wt.start()
    ths = [threading.Thread(target=caller, args=(t,)) for t in range(96)]
    [x.start() for x in ths]
    [x.join() for x in ths]
    stop.set()
    wt.join()
    assert not errs, errs[:5]
    assert h.stats()["lookup_batches"] > b0, "concurrent callers must have shared rounds"
    # the writer's last state, replayed on the replica
    for r, op in last.items():
        rep.write_relationships([(op, r, 0)])
    assert sorted(rep.read_relationships()) == sorted(h.read_relationships())
    for rt, perm, st, sid, srel in lookups:
        q = (rt, perm, st, names[(st, sid)], srel or None)
        assert _same(_ids(h, *q), _ids(rep, *q)), q


def test_answers_follow_5x1000_updates_merged_into_every_shard(zg):
    schema = randgen.FIXED_SCHEMAS["nesting"]
    rng = random.Random(9920)
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=40, n_user=25, density=0.12)
    pool = randgen.random_relationships(rng, model, n_obj=80, n_user=50, density=0.3)
    assert len(pool) >= 1000
    lookups = cases.random_lookups(rng, model, rels, 30)
    h = zg.Engine(schema, device=0, n_shards=3, handle_lookups=True)
    rep = zg.Engine(schema, device=0)
    for e in (h, rep):
        e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels])
    for w in range(5):
        ups = [((zg._lib.OP_DELETE if rng.random() < 0.3 else zg._lib.OP_TOUCH), r, 0) for r in rng.sample(pool, 1000)]
        first = rels[w].split("#")[0].split(":")
        pre = [(zg._lib.PRECOND_MUST_MATCH, {"res_type": rels[0].split(":")[0]})]
        for e in (h, rep):
            e.write_relationships(ups, pre)
            e.delete_relationships({"res_type": first[0], "res_id": first[1]})
    assert h.stats()["delta_publishes"] > 0 or h.stats()["full_publishes"] > 0
    for rt, perm, st, sid, srel in lookups:
        subj = rep.find(st, sid)
        if subj == zg._lib.NO_OBJECT:
            continue
        q = (rt, perm, st, subj, srel or None)
        assert _same(_ids(h, *q), _ids(rep, *q)), q


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
    lookups = [q + (None,) for q in w.lookups] + [("document", "view", "group", g, "member") for g in (0, 2)]
    e0 = engines[0]
    reqs = [(e0.type_id(a), e0.slot_id(a, p), e0.type_id(s), u, cases.SREL_NONE if sr is None else e0.slot_id(s, sr))
            for a, p, s, u, sr in lookups]
    out, _ = cases.run_sharded(engines, ts, [reqs] + [[] for _ in range(S - 1)])
    for q, d in zip(lookups, out[0]):
        a, b = _ids(h, *q), _ids(rep, *q)
        assert a is not None and np.array_equal(a, b) and np.array_equal(a, d), q


def test_e2big_retry_is_served_from_the_cache(zg):
    rels = [f"doc:d{i}#viewer@user:u{i % 3}" for i in range(300)]
    h, rep = _pair(zg, OVF_SCHEMA, 2, lambda e: e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels]))
    names = {("user", "u1"): rep.find("user", "u1")}
    L = h._L
    args = (h.type_id("doc"), h.slot_id("doc", "view"), h.type_id("user"), names[("user", "u1")], zg._lib.SREL_NONE)
    n = ctypes.c_uint64(0)
    one = np.zeros(1, dtype=np.uint32)
    assert L.zg_lookup_resources(h._h, *args, one.ctypes.data, 1, ctypes.byref(n)) == E2BIG and n.value == 100
    rounds = h.handle_lookup_counters()["rounds"]
    out = np.zeros(n.value, dtype=np.uint32)
    assert L.zg_lookup_resources(h._h, *args, out.ctypes.data, n.value, ctypes.byref(n)) == 0
    assert np.array_equal(out, rep.lookup_resources_ids("doc", "view", "user", names[("user", "u1")]))
    buf, need, cnt = ctypes.create_string_buffer(8), ctypes.c_size_t(0), ctypes.c_uint64(0)
    rc = L.zg_lookup_resources_str(h._h, b"doc", b"view", b"user", b"u1", b"", buf, 8, ctypes.byref(need), ctypes.byref(cnt))
    assert rc == E2BIG and cnt.value == 100
    assert h.lookup_resources_str("doc", "view", "user", "u1") == rep.lookup_resources_str("doc", "view", "user", "u1")
    assert h.handle_lookup_counters()["rounds"] == rounds, "the retries are answered from the cache"


class _FlaggedBackend:
    """The golden cases through client.PermissionsClient over a flagged handle: LookupResources answered by the handle
    itself, and compared with a replica fed the same writes."""

    def __init__(self, zg, schema):
        self.C = zg.client
        self.cl = self.C.PermissionsClient(schema, engine=zg.Engine(schema, n_shards=3, handle_lookups=True))
        self.rep = self.C.PermissionsClient(schema)

    def write(self, rel):
        C = self.C
        req = C.WriteRelationshipsRequest([C.RelationshipUpdate(C.OPERATION_TOUCH, C.Relationship.parse(rel))])
        self.cl.WriteRelationships(req)
        self.rep.WriteRelationships(req)

    def check(self, rt, rid, perm, st, sid, srel=""):
        C = self.C
        try:
            r = self.cl.CheckPermission(C.CheckPermissionRequest(
                C.ObjectReference(rt, rid), perm, C.SubjectReference(C.ObjectReference(st, sid), srel)))
        except C.RpcError:
            return 255
        return r.permissionship

    def bulk(self, rels):
        C = self.C
        items = [C.CheckBulkPermissionsRequestItem(C.ObjectReference(rt, rid), perm, C.SubjectReference(C.ObjectReference(st, sid), srel))
                 for rt, rid, perm, st, sid, srel in (split_rel(r) for r in rels)]
        resp = self.cl.CheckBulkPermissions(C.CheckBulkPermissionsRequest(items))
        return [255 if p.GetError() else p.GetItem().permissionship for p in resp.pairs]

    def lookup(self, rt, perm, st, sid, srel):
        C = self.C
        req = C.LookupResourcesRequest(rt, perm, C.SubjectReference(C.ObjectReference(st, sid), srel))
        got = [r.resource_object_id for r in self.cl.LookupResources(req)]
        assert got == [r.resource_object_id for r in self.rep.LookupResources(req)]
        return got

    def read(self, res_type="", res_id="", rel="", **_):
        C = self.C
        return [r.relationship.text() for r in self.cl.ReadRelationships(
            C.ReadRelationshipsRequest(C.RelationshipFilter(res_type, res_id, rel)))]


def test_golden_cases_through_the_client(zg, golden):
    for case in golden["cases"]:
        run_case(_FlaggedBackend(zg, golden["schemas"][case["schema"]]), case)


def test_list_prefilter_equals_a_replica_byte_for_byte(zg):
    from spicedb_kubeapi_proxy_b200 import _lib, workloads
    from test_listfilter_protobuf import pod, pod_list

    schema = workloads.BOOTSTRAP_SCHEMA + """
definition team {
  relation member: user | team#member
  permission view = member
}
"""
    rels = [f"pod:ns{i % 3}/p{i}#viewer@user:u{i % 7}" for i in range(300)] + \
           [f"pod:ns{i % 3}/p{i}#creator@user:u{i % 5}" for i in range(0, 300, 4)] + ["namespace:ns1#creator@user:u1"]
    rels += ["team:a#member@user:u1", "team:b#member@team:a#member"]
    h, rep = zg.Engine(schema, n_shards=3, handle_lookups=True), zg.Engine(schema)
    for e in (h, rep):
        e.write_relationships([(_lib.OP_TOUCH, r, 0) for r in rels])
    pods = [(f"p{i}", f"ns{i % 3}") for i in range(0, 320, 2)]
    body = json.dumps({"kind": "PodList", "items": [{"metadata": {"name": n, "namespace": s}} for n, s in pods]}).encode()
    table = json.dumps({"kind": "Table", "rows": [{"cells": [n], "object": {"metadata": {"name": n, "namespace": s}}}
                                                  for n, s in pods]}).encode()
    proto = pod_list([pod(n, s) for n, s in pods])
    teams = json.dumps({"kind": "List", "items": [{"metadata": {"name": t}} for t in ("a", "b", "c", "zz")]}).encode()
    for u in ("u1", "u4", "nobody"):
        for b, mode in ((body, _lib.LIST_ITEMS), (table, _lib.LIST_TABLE_ROWS), (proto, _lib.LIST_PROTOBUF)):
            got = h.list_prefilter(b, h.list_template("pod", "view", "user", u), mode)
            assert got == rep.list_prefilter(b, rep.list_template("pod", "view", "user", u), mode), (u, mode)
    # userset subjects, the never-written one ("zz") naming itself
    for t in ("a", "b", "zz"):
        tpl = dict(res_type="team", permission="view", subj_type="team", subj_id=t, subj_rel="member")
        got = h.list_prefilter(teams, h.list_template(**tpl))
        assert got == rep.list_prefilter(teams, rep.list_template(**tpl)), t
    assert [i["metadata"]["name"] for i in json.loads(h.list_prefilter(teams, h.list_template(
        res_type="team", permission="view", subj_type="team", subj_id="zz", subj_rel="member")))["items"]] == ["zz"]


def test_flagged_handle_still_refuses_the_rest(zg):
    import torch

    from spicedb_kubeapi_proxy_b200 import workloads

    h = zg.Engine(workloads.BOOTSTRAP_SCHEMA, n_shards=2, handle_lookups=True)
    h.write_relationships([(zg._lib.OP_TOUCH, "pod:ns/p1#viewer@user:a", 0)])
    d_items = torch.zeros(16 * 4, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(4, dtype=torch.uint8, device="cuda")
    calls = {
        "lookup subjects": (lambda: h.lookup_subjects_ids("pod", h.find("pod", "ns/p1"), "view", "user"), "LookupSubjects"),
        "lookup subjects str": (lambda: h.lookup_subjects_str("pod", "ns/p1", "view", "user"), "LookupSubjects"),
        "device": (lambda: h.check_bulk_device(d_items.data_ptr(), 4, d_out.data_ptr()), "device buffers"),
        "ingress": (lambda: h.check_bulk_packed_ingress("pod", "view", "user", ["ns/p1"], ["a"]), "device-ingress"),
        "shard pass": (lambda: h.shard_pass_dev(d_items.data_ptr(), 4, 0), "zg_shard_"),
        "shard lookup": (lambda: h.shard_lookup_candidates_dev(False, 0, 0), "zg_shard_"),
    }
    for what, (call, msg) in calls.items():
        with pytest.raises(zg.ZgpuError, match=msg) as ex:
            call()
        assert ex.value.code == EINVAL, what
        assert "sharded handle" in str(ex.value), what
    assert h.lookup_resources_str("pod", "view", "user", "a") == ["ns/p1"]
    assert list(h.check_bulk_str(["pod:ns/p1#view@user:a", "pod:ns/p1#view@user:b"])) == [2, 1]


def test_cfg4_full_size_scale_agrees_with_a_replica(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=float(os.environ.get("ZGPU_FULLSIZE_SCALE", "0.25")))
    h, rep = _pair(zg, w.schema, 4, w.load_into)
    users = [u for _, _, _, u in w.lookups]
    lookups = [("document", p, "user", u, None) for p in ("view", "restricted_view") for u in users]
    lookups += [("document", "view", "group", g, "member") for g in (0, 1, 7)]
    for q in lookups:
        a = _ids(h, *q)
        assert a is not None and np.array_equal(a, _ids(rep, *q)), q


def test_shards_on_several_devices(zg):
    import torch

    from spicedb_kubeapi_proxy_b200 import workloads

    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs >= 2 GPUs")
    w = workloads.cfg4(scale=0.005)
    h = zg.Engine(w.schema, device=0, n_devices=n_dev, n_shards=2 * n_dev, handle_lookups=True)
    rep = zg.Engine(w.schema, device=0)
    for e in (h, rep):
        w.load_into(e)
        e.publish()
    for q in w.lookups:
        a = _ids(h, *q)
        assert a is not None and np.array_equal(a, _ids(rep, *q)), q
