"""GPU tests of the host-side paths added after the last GPU session of round 1 (DESIGN.md section 9): the string
path through the batcher, the fused list post-filter, the watch feed against a live snapshot. Kept in the file
that sorts last so that a surprise here cannot hide the kernel parity results under `pytest -x`."""
import json

import numpy as np
import pytest

import zgpu  # noqa: F401
from spicedb_kubeapi_proxy_b200 import client as cl, postfilter as pf

pytestmark = pytest.mark.gpu

REQ = pf.RequestInfo(verb="list")


def pod(name, ns="default", **extra):
    return {"metadata": {"name": name, "namespace": ns}, **extra}


@pytest.fixture(scope="module")
def zg():
    return zgpu


def test_gpu_filter_through_engine():
    """The whole post-filter through the real engine: cfg1-like schema, one bulk call, one launch."""
    schema = """
    definition user {}
    definition namespace { relation viewer: user  permission view = viewer }
    definition pod { relation namespace: namespace  relation viewer: user | user:*
                     permission view = viewer + namespace->view }
    """
    c = cl.PermissionsClient(schema, ["namespace:team-a#viewer@user:alice", "pod:team-a/p1#namespace@namespace:team-a",
                                      "pod:team-b/p2#namespace@namespace:team-b", "pod:team-b/p3#viewer@user:alice",
                                      "pod:team-b/p4#viewer@user:*"])
    body = json.dumps({"kind": "PodList", "items": [pod("p1", "team-a"), pod("p2", "team-b"), pod("p3", "team-b"),
                                                    pod("p4", "team-b"), pod("p5", "team-b")]}).encode()
    tpl = "pod:{{namespacedName}}#view@user:{{user.name}}"
    before = c.engine.stats()["launches"]
    out = json.loads(pf.filter_list_response(body, [tpl], REQ, pf.UserInfo(name="alice"), c))
    assert [i["metadata"]["name"] for i in out["items"]] == ["p1", "p3", "p4"]
    assert c.engine.stats()["launches"] > before
    out = json.loads(pf.filter_list_response(body, [tpl], REQ, pf.UserInfo(name="bob"), c))
    assert [i["metadata"]["name"] for i in out["items"]] == ["p4"]
    # the fused C entry point gives the same bytes as the mirror, with one call and one launch
    for who in ("alice", "bob"):
        fused = c.engine.list_postfilter(body, [c.engine.list_template("pod", "view", "user", who)])
        assert fused == pf.filter_list_response(body, [tpl], REQ, pf.UserInfo(name=who), c)
    both = [c.engine.list_template("pod", "view", "user", "alice"), c.engine.list_template("pod", "viewer", "user", "alice")]
    assert [i["metadata"]["name"] for i in json.loads(c.engine.list_postfilter(body, both))["items"]] == ["p3", "p4"]
    # the pre-filter path over the same store: LookupResources -> allowed set -> list
    res = pf.run_lookup_resources(c, ("pod", "$", "view", "user", "alice", ""), REQ)
    assert res.allowed_results == {("team-a", "p1"), ("team-b", "p3"), ("team-b", "p4")}
    assert [i["metadata"]["name"] for i in json.loads(pf.filter_list(body, res))["items"]] == ["p1", "p3", "p4"]
    # ... and the same in one C call (LookupResources on the GPU + scan + keep + splice), list and table
    for who in ("alice", "bob", "nobody"):
        r = pf.run_lookup_resources(c, ("pod", "$", "view", "user", who, ""), REQ)
        t = c.engine.list_template("pod", "view", "user", who)
        assert c.engine.list_prefilter(body, t) == pf.filter_list(body, r)
        table = json.dumps({"kind": "Table", "rows": [{"cells": [i["metadata"]["name"]], "object": i}
                                                       for i in json.loads(body)["items"]]}).encode()
        assert c.engine.list_prefilter(table, t, zgpu._lib.LIST_TABLE_ROWS) == pf.filter_table(table, r)
    # the watch path: a write shows up on the feed and is re-checked against the new snapshot
    stream = c.Watch(cl.WatchRequest(["pod"]))
    c.WriteRelationships(cl.WriteRelationshipsRequest([
        cl.RelationshipUpdate(cl.OPERATION_TOUCH, cl.Relationship.parse("pod:team-b/p2#viewer@user:alice")),
        cl.RelationshipUpdate(cl.OPERATION_DELETE, cl.Relationship.parse("pod:team-b/p3#viewer@user:alice"))]))
    assert pf.run_watch(stream, c, ("pod", "$", "view", "user", "alice", "")) == [
        pf.ResultChange(True, ("team-b", "p2")), pf.ResultChange(False, ("team-b", "p3"))]


def test_concurrent_string_callers_share_launches_and_see_writes(zg):
    """zg_check_bulk_str resolves under the engine lock and then takes the batcher like zg_check_bulk: concurrent
    string callers (what the Go shim issues) get exactly their own answers while a writer keeps publishing."""
    import threading

    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    schema = workloads.BOOTSTRAP_SCHEMA
    OP_TOUCH, OP_DELETE = zg._lib.OP_TOUCH, zg._lib.OP_DELETE
    e, o = zg.Engine(schema), Oracle(schema)
    rels = [f"pod:ns{i % 7}/p{i}#viewer@user:u{i % 13}" for i in range(400)] + \
           [f"namespace:ns{i}#creator@user:u{i}" for i in range(7)]
    for k in range(0, len(rels), 500):
        e.write_relationships([(OP_TOUCH, r, 0) for r in rels[k:k + 500]])
    for r in rels:
        o.touch(r)
    queries = [("pod", f"ns{i % 7}/p{i % 450}", "view", "user", f"u{(i * 5) % 15}", "") for i in range(3000)]
    want = np.array([o.check(*q[:5]) for q in queries], dtype=np.uint8)
    assert 0 < (want == 2).sum() < want.size
    errors, stop = [], threading.Event()

    def reader(tid):
        rng = np.random.default_rng(tid)
        try:
            for _ in range(30):
                lo = int(rng.integers(0, len(queries) - 1))
                n = int(rng.integers(1, min(400, len(queries) - lo)))
                got = e.check_bulk_str(queries[lo:lo + n])
                if not np.array_equal(got, want[lo:lo + n]):
                    errors.append((tid, lo, n))
        except Exception as ex:  # noqa: BLE001
            errors.append((tid, repr(ex)))

    def writer():
        i = 0
        try:
            while not stop.is_set():  # relationships no query looks at: answers must not move
                e.write_relationships([(OP_TOUCH if i % 2 == 0 else OP_DELETE, f"workflow:w{i // 2 % 50}#idempotency_key@activity:a",
                                        4_000_000_000 if i % 2 == 0 else 0)])
                i += 1
        except Exception as ex:  # noqa: BLE001
            errors.append(("writer", repr(ex)))

    before = e.stats()
    wt = threading.Thread(target=writer)
    wt.start()
    threads = [threading.Thread(target=reader, args=(t,)) for t in range(16)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    stop.set()
    wt.join()
    assert not errors, errors[:3]
    st = e.stats()
    assert st["checks"] > before["checks"] and st["revision"] > before["revision"]
    # a write is visible to the very next string check (FullyConsistent)
    assert e.check_bulk_str([("pod", "ns0/new", "view", "user", "late", "")])[0] == 1
    e.write_relationships([(OP_TOUCH, "pod:ns0/new#viewer@user:late", 0)])
    assert e.check_bulk_str([("pod", "ns0/new", "view", "user", "late", "")])[0] == 2
    print("coalesced", st["coalesced_requests"], "string calls into", st["coalesced_launches"], "launches")


@pytest.mark.gpu
def test_lookup_resources_agrees_with_check_for_userset_subjects():
    """LookupResources(T, P, T:x#r) contains x whenever Check(T:x#P @ T:x#r) is HAS -- for every relation r inlined
    into P's union, not only r == P, written or never written (round-1 advisor finding): same table as the oracle
    test (tests/test_oracle_random.py), through the client mirror."""
    import zgpu
    from test_oracle_random import SELF_LOOKUPS, SELF_RELS, SELF_SCHEMA

    C = zgpu.client
    cl = C.PermissionsClient(SELF_SCHEMA)
    cl.WriteRelationships(C.WriteRelationshipsRequest(
        [C.RelationshipUpdate(C.OPERATION_TOUCH, C.Relationship.parse(r)) for r in SELF_RELS]))
    for (rt, perm, st, sid, srel), want in SELF_LOOKUPS:
        if srel == "editor":
            want = ["5"]
        got = sorted(r.resource_object_id for r in cl.LookupResources(C.LookupResourcesRequest(
            rt, perm, C.SubjectReference(C.ObjectReference(st, sid), srel))))
        assert got == want, f"{rt}#{perm}@{st}:{sid}#{srel}: {got} != {want}"


def test_two_level_meet_over_every_range_size_and_membership_count():
    """Same sweep as the emulator test of the same name (tests/test_kernel_emulation.py), on the real kernel: ranges of
    1 .. 70 children against subjects with 1 .. 17 memberships, answers against the oracle."""
    import zgpu
    from oracle.pyoracle import Oracle

    schema = """definition user {}
definition group { relation member: user }
definition team { relation member: group#member }
definition namespace { relation viewer: team#member  permission view = viewer }"""
    rng = np.random.default_rng(11)
    rels, checks = [], []
    n_teams = 400
    for g in range(300):
        for t in rng.choice(n_teams, 1 + g % 12, replace=False):
            rels.append(f"team:t{t}#member@group:g{g}#member")
    sizes = [1, 2, 3, 15, 16, 17, 31, 32, 33, 63, 64, 65, 70]
    for i, nf in enumerate(sizes):
        for t in rng.choice(n_teams, nf, replace=False):
            rels.append(f"namespace:n{i}#viewer@team:t{t}#member")
    for u in range(1, 18):
        for g in rng.choice(300, u, replace=False):
            rels.append(f"group:g{g}#member@user:u{u}")
    for i in range(len(sizes)):
        for u in range(1, 18):
            checks.append(f"namespace:n{i}#view@user:u{u}")
    C = zgpu.client
    c = C.PermissionsClient(schema)
    for i in range(0, len(rels), 1000):  # a write carries at most 1 000 updates (pkg/spicedb/spicedb.go:34)
        c.WriteRelationships(C.WriteRelationshipsRequest(
            [C.RelationshipUpdate(C.OPERATION_TOUCH, C.Relationship.parse(r)) for r in rels[i:i + 1000]]))
    o = Oracle(schema)
    for r in rels:
        o.touch(r)
    got = c.engine.check_bulk_str(checks)
    want = np.array([o.check_rel(q) for q in checks], dtype=np.uint8)
    assert np.array_equal(got, want), [checks[i] for i in np.flatnonzero(got != want)[:5]]
    assert 0.1 < (got == 2).mean() < 0.9


def test_prefilter_of_a_protobuf_encoded_list():
    """zg_list_prefilter with ZG_LIST_PROTOBUF: LookupResources on the GPU, then the items of a protobuf-encoded PodList
    (what kube clients receive for built-in types) whose namespace/name it returned are kept, byte for byte
    (pkg/authz/responsefilterer.go:241-313,:376-400). Encoder / decoder: tests/test_listfilter_protobuf.py."""
    import test_listfilter_protobuf as P
    import zgpu
    from spicedb_kubeapi_proxy_b200 import _lib

    schema = """definition user {}
definition namespace { relation viewer: user  permission view = viewer }
definition pod { relation namespace: namespace  relation viewer: user  permission view = viewer + namespace->view }"""
    c = zgpu.client.PermissionsClient(schema, ["namespace:n1#viewer@user:alice", "pod:n1/a#namespace@namespace:n1",
                                               "pod:n1/b#namespace@namespace:n1", "pod:n2/c#namespace@namespace:n2",
                                               "pod:n2/d#viewer@user:alice", "pod:n2/e#viewer@user:bob"])
    pods = [P.pod("a", "n1"), P.pod("b", "n1"), P.pod("c", "n2"), P.pod("d", "n2"), P.pod("e", "n2"), P.pod("ghost", "n1")]
    body = P.pod_list(pods)
    tpl = c.engine.list_template("pod", "view", "user", "alice")
    out = c.engine.list_prefilter(body, tpl, _lib.LIST_PROTOBUF)
    assert P.decode_items(out) == [("n1", "a"), ("n1", "b"), ("n2", "d")]
    assert out == P.pod_list([pods[0], pods[1], pods[3]])
    nobody = c.engine.list_template("pod", "view", "user", "nobody")
    assert P.decode_items(c.engine.list_prefilter(body, nobody, _lib.LIST_PROTOBUF)) == []
