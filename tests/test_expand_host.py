"""ExpandPermissionTree on the CPU: the Python restatement (expand_oracle.py) against Check, by the defining property,
over both oracles on random schemas at two clocks and on hand-written shapes; the C ABI's argument errors and the
host-only refusal; the client mirror over a stub engine."""
import random
import re

import numpy as np
import pytest

import randgen
import zgpu
from expand_oracle import DepthError, contains, expand_tree, lines
from oracle.mini_oracle import MiniOracle
from oracle.pyoracle import Oracle
from spicedb_kubeapi_proxy_b200 import client

HAS = 2
T0, T1 = 1_000, 2_000  # the two clocks: every expiration sits between them or past both


def expiring(schema: str) -> str:
    """The schema with every allowed subject `with expiration`."""
    return "use expiration\n" + re.sub(
        r"(relation \w+: )([^\n}]*)",
        lambda m: m.group(1) + " | ".join(p.strip() + " with expiration" for p in m.group(2).split("|")) + " ", schema)


def _stores(schema, rels, expires):
    o, m = Oracle(schema), MiniOracle(schema)
    for r in rels:
        o.touch(r, expires.get(r, 0))
        m.write(r, expires.get(r, 0))
    return o, m


def _violations(schema, o, m, rt, rid, perm, subjects, now):
    """Subjects on which the restated tree and Check (C oracle and MiniOracle) disagree."""
    tree = expand_tree(m, rt, rid, perm, now)
    bad = []
    for st, sid in subjects:
        got = contains(tree, st, sid, lambda t, i, r: o.check(t, i, r, st, sid, "", now) == HAS)
        got_m = contains(tree, st, sid, lambda t, i, r: m.check(t, i, r, st, sid, "", now) == HAS)
        want = o.check(rt, rid, perm, st, sid, "", now) == HAS
        if got != want or got_m != (m.check(rt, rid, perm, st, sid, "", now) == HAS):
            bad.append((rt, rid, perm, st, sid, now, got, want))
    return bad


@pytest.mark.parametrize("seed", range(24))
def test_restatement_has_the_defining_property_on_random_schemas(seed):
    rng = random.Random(seed)
    schema, model = randgen.random_schema(rng)
    schema = expiring(schema)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5)
    expires = {r: rng.choice((T0 + 500, T1 + 500)) for r in rels if rng.random() < 0.3}
    o, m = _stores(schema, rels, expires)
    subjects = [("user", f"u{i}") for i in range(6)] + [("user", "!probe")]
    subjects += [(t, f"o{i}") for t in model["tnames"] for i in range(3)]
    bad = []
    for t in model["tnames"]:
        d = model["types"][t]
        for name in list(d["rels"]) + list(d["perms"]):
            for rid in ("o0", "o3", "o4", "o9"):  # o9: never written
                for now in (T0, T1):
                    bad += _violations(schema, o, m, t, rid, name, subjects, now)
    assert not bad, bad[:5]


DOCS = randgen.FIXED_SCHEMAS["docs"]


def _docs():
    rels = ["document:d#viewer@user:a", "document:d#viewer@group:g#member", "document:d#owner@user:*",
            "document:d#banned@user:b", "document:d#parent@folder:f", "document:d#org@org:o", "folder:f#viewer@user:c",
            "folder:f#parent@folder:root", "folder:root#owner@user:e", "group:g#member@user:g1", "org:o#member@user:a"]
    m = MiniOracle(DOCS)
    for r in rels:
        m.write(r)
    return m


def test_restatement_shapes_on_cfg4():
    got = lines(expand_tree(_docs(), "document", "d", "view"))
    assert got == [
        "0 X document:d#view",
        "1 U document:d#view",
        "2 L document:d#viewer user:a group:g#member",
        "2 U document:d#edit",
        "3 L document:d#owner user:*",
        "3 L document:d#editor",
        "2 U document:d#view",
        "3 U folder:f#view",
        "4 L folder:f#viewer user:c",
        "4 L folder:f#owner",
        "4 U folder:f#view",
        "5 U folder:root#view",
        "6 L folder:root#viewer",
        "6 L folder:root#owner user:e",
        "6 U folder:root#view",
        "1 L document:d#banned user:b",
    ]
    assert lines(expand_tree(_docs(), "document", "d", "restricted_view"))[:2] == [
        "0 I document:d#restricted_view", "1 X document:d#view"]
    assert lines(expand_tree(_docs(), "document", "d", "edit")) == [
        "0 U document:d#edit", "1 L document:d#owner user:*", "1 L document:d#editor"]
    # never written: empty leaves and childless arrow unions
    assert lines(expand_tree(_docs(), "document", "nope", "view"))[-2:] == ["2 U document:nope#view",
                                                                           "1 L document:nope#banned"]


def test_restatement_nesting_rules():
    schema = """definition user {}
definition other { relation x: user }
definition doc {
  relation a: user
  relation b: user
  relation c: user
  relation d: user
  relation t: other | user | user:*
  permission chain = a + (b + c) + d
  permission inter = a & b & (c & d)
  permission excl = a - b - c
  permission nested = (a + b) & (c - d)
  permission bare = a
  permission none = nil
  permission arrow = t->x + t->missing
}
"""
    m = MiniOracle(schema)
    for r in ("doc:r#t@other:o", "doc:r#t@user:u", "doc:r#t@user:*", "other:o#x@user:v"):
        m.write(r)
    ex = lambda p: lines(expand_tree(m, "doc", "r", p))
    assert ex("chain") == ["0 U doc:r#chain"] + [f"1 L doc:r#{x}" for x in "abcd"]
    assert ex("inter") == ["0 I doc:r#inter"] + [f"1 L doc:r#{x}" for x in "abcd"]
    assert ex("excl") == ["0 X doc:r#excl", "1 X doc:r#excl", "2 L doc:r#a", "2 L doc:r#b", "1 L doc:r#c"]
    assert ex("nested") == ["0 I doc:r#nested", "1 U doc:r#nested", "2 L doc:r#a", "2 L doc:r#b", "1 X doc:r#nested",
                            "2 L doc:r#c", "2 L doc:r#d"]
    assert ex("bare") == ["0 U doc:r#bare", "1 L doc:r#a"]
    assert ex("none") == ["0 U doc:r#none", "1 L doc:r#none"]
    # arrow: one child per non-wildcard tupleset relationship; a subject type without the permission: empty leaf
    assert ex("arrow") == ["0 U doc:r#arrow", "1 U doc:r#arrow", "2 L other:o#x user:v", "2 L doc:r#arrow",
                           "1 U doc:r#arrow", "2 L doc:r#arrow", "2 L doc:r#arrow"]


def test_restatement_depth_cap():
    schema = "definition user {}\ndefinition folder {\n  relation parent: folder\n  relation viewer: user\n" \
             "  permission view = viewer + parent->view\n}\n"
    for hops, ok in ((50, True), (51, False)):
        m = MiniOracle(schema)
        for i in range(hops):
            m.write(f"folder:f{i}#parent@folder:f{i + 1}")
        m.write(f"folder:f{hops}#viewer@user:u")
        if ok:
            t = expand_tree(m, "folder", "f0", "view")
            assert contains(t, "user", "u", lambda *a: False)
        else:
            with pytest.raises(DepthError):
                expand_tree(m, "folder", "f0", "view")
    m = MiniOracle(schema)
    m.write("folder:a#parent@folder:b")
    m.write("folder:b#parent@folder:a")
    with pytest.raises(DepthError):
        expand_tree(m, "folder", "a", "view")


def test_host_only_engine_refuses():
    e = zgpu.Engine(DOCS, host_only=True)
    e.write_relationships([(zgpu._lib.OP_TOUCH, "document:d#viewer@user:a", 0)])
    with pytest.raises(zgpu.ZgpuError) as x:
        e.expand_permission_tree_str("document", "d", "view")
    assert x.value.code == -4 and "host-only" in str(x.value)
    with pytest.raises(zgpu.ZgpuError) as x:
        e.expand_permission_trees([("document", e.find("document", "d"), "view")])
    assert x.value.code == -4


def test_argument_errors():
    e = zgpu.Engine(DOCS, host_only=True)
    e.write_relationships([(zgpu._lib.OP_TOUCH, "document:d#viewer@user:a", 0)])
    e.publish()
    for args, msg in ((("nope", "d", "view"), "object definition `nope` not found"),
                      (("document", "d", "nope"), "relation/permission `nope` not found under definition `document`")):
        with pytest.raises(zgpu.ZgpuError) as x:
            e.expand_permission_tree_str(*args)
        assert x.value.code == -1 and msg in str(x.value)
    L, h = e._L, e._h
    cap = int(L.zg_object_capacity(h, e.type_id("document")))
    for perm, res, msg in ((e.slot_id("document", "view"), cap + 5, "past the capacity of document"),
                           (L.zg_num_slots(h), 0, "unknown relation or permission")):
        req = np.zeros(1, dtype=zgpu._lib.EXPAND_REQUEST_DTYPE)
        req[0] = (perm, 0, res)
        st, nn, ns = np.zeros(1, dtype=np.int32), zgpu._lib.C.c_uint64(0), zgpu._lib.C.c_uint64(0)
        rc = L.zg_expand_permission_trees(h, req.ctypes.data, 1, st.ctypes.data, None, 0, zgpu._lib.C.byref(nn), None, 0,
                                          zgpu._lib.C.byref(ns))
        assert rc == -1 and msg in L.zg_last_error().decode()


class _StubEngine:
    def __init__(self, out):
        self.out, self.calls = out, []

    def expand_permission_tree_str(self, rt, rid, perm):
        self.calls.append((rt, rid, perm))
        if isinstance(self.out, Exception):
            raise self.out
        return self.out


def test_client_mirror():
    tree = expand_tree(_docs(), "document", "d", "view")
    stub = _StubEngine(lines(tree))
    c = client.PermissionsClient(DOCS, engine=stub)
    r = c.ExpandPermissionTree(client.ExpandPermissionTreeRequest(client.ObjectReference("document", "d"), "view"))
    assert stub.calls == [("document", "d", "view")]
    root = r.tree_root
    assert root.expanded_object == client.ObjectReference("document", "d") and root.expanded_relation == "view"
    assert root.leaf is None and root.intermediate.operation == client.OPERATION_EXCLUSION
    union, banned = root.intermediate.children
    assert banned.leaf.subjects == [client.SubjectReference(client.ObjectReference("user", "b"))]
    viewer = union.intermediate.children[0]
    assert viewer.expanded_relation == "viewer" and viewer.leaf.subjects == [
        client.SubjectReference(client.ObjectReference("user", "a")),
        client.SubjectReference(client.ObjectReference("group", "g"), "member")]
    owner = union.intermediate.children[1].intermediate.children[0]
    assert owner.leaf.subjects == [client.SubjectReference(client.ObjectReference("user", "*"))]
    arrow = union.intermediate.children[2]
    assert arrow.intermediate.operation == client.OPERATION_UNION
    assert arrow.intermediate.children[0].expanded_object == client.ObjectReference("folder", "f")
    # ZG_EDEPTH is the error LookupSubjects raises for an undecidable answer
    stub.out = zgpu.ZgpuError(-9, "passes the maximum depth")
    with pytest.raises(client.RpcError) as x:
        c.ExpandPermissionTree(client.ExpandPermissionTreeRequest(client.ObjectReference("folder", "a"), "view"))
    assert x.value.code == client._rpc(zgpu.ZgpuError(-9, "")).code
    assert zgpu._lib.parse_expand_lines(lines(tree)) == tree
