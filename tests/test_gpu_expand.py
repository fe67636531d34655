"""ExpandPermissionTree on the GPU, through the C ABI: the trees equal the restatement (expand_oracle.py) line for line,
in the engine's leaf order, and satisfy the defining property against the oracle's checks, on fixed and random schemas,
at two clocks and after incremental writes, collection and id reuse; the id and string forms agree; the leaf order is
the resident rows'; the depth cap, arrow cycles and a mixed batch; the ZG_E2BIG retry and the node cap; the client
mirror; the refusals; concurrent callers; cfg4 at the full-size tests' scale."""
import ctypes as C
import os
import random
import threading

import numpy as np
import pytest

import randgen
from expand_oracle import DepthError, GroupRows, canonical, contains, expand_tree, group_order, id_tree_lines, lines
from oracle.mini_oracle import MiniOracle
from oracle.pyoracle import Oracle
from test_expand_host import DOCS, expiring

pytestmark = pytest.mark.gpu
HAS = 2


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _load(zg, schema, rels, now=0, expires=None):
    e, m, o = zg.Engine(schema, device=0), MiniOracle(schema), Oracle(schema)
    if now:
        e.set_clock(now)
    ups = []
    for r in rels:
        ex = (expires or {}).get(r, 0)
        m.write(r, ex)
        o.touch(r, ex)
        ups.append((zg._lib.OP_TOUCH, r, ex))
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])
    e.publish()
    return e, m, o


def _want(e, m, rt, rid, perm, now):
    try:
        return lines(expand_tree(m, rt, rid, perm, now, order=lambda t, i: e.find(t, i)))
    except DepthError:
        return "EDEPTH"


def _got(zg, e, rt, rid, perm):
    try:
        return e.expand_permission_tree_str(rt, rid, perm)
    except zg.ZgpuError as x:
        assert x.code == -9, x
        return "EDEPTH"


def _compare(zg, e, m, o, queries, now=0, subjects=()):
    for rt, rid, perm in queries:
        want, got = _want(e, m, rt, rid, perm, now), _got(zg, e, rt, rid, perm)
        assert got == want, f"{rt}:{rid}#{perm} now={now}\ngpu={got}\nwant={want}"
        if got == "EDEPTH":
            continue
        tree = zg._lib.parse_expand_lines(got)
        assert canonical(tree) == canonical(expand_tree(m, rt, rid, perm, now))
        for st, sid in subjects:
            has = contains(tree, st, sid, lambda t, i, r: o.check(t, i, r, st, sid, "", now) == HAS)
            assert has == (o.check(rt, rid, perm, st, sid, "", now) == HAS), (rt, rid, perm, st, sid, now)


def _queries(model, ids=("o0", "o2", "o4", "o9")):
    return [(t, rid, name) for t in model["tnames"] for name in list(model["types"][t]["rels"]) +
            list(model["types"][t]["perms"]) for rid in ids]


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas(zg, name):
    schema = randgen.FIXED_SCHEMAS[name]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(random.Random(7), model, n_obj=6, n_user=6)
    e, m, o = _load(zg, schema, rels)
    _compare(zg, e, m, o, _queries(model), subjects=[("user", f"u{i}") for i in range(7)])


@pytest.mark.parametrize("seed", range(12))
def test_random_schemas_at_two_clocks(zg, seed):
    rng = random.Random(100 + seed)
    schema, model = randgen.random_schema(rng)
    schema = expiring(schema)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5)
    expires = {r: rng.choice((1_500, 2_500)) for r in rels if rng.random() < 0.3}
    e, m, o = _load(zg, schema, rels, now=1_000, expires=expires)
    subjects = [("user", f"u{i}") for i in range(6)] + [(t, "o1") for t in model["tnames"]]
    for now in (1_000, 2_000):
        e.set_clock(now)
        _compare(zg, e, m, o, _queries(model), now=now, subjects=subjects)


def test_id_and_string_forms_agree_and_leaves_follow_the_rows(zg):
    schema = randgen.FIXED_SCHEMAS["docs"]
    rng = random.Random(3)
    rels = randgen.random_relationships(rng, randgen.model_from_schema(schema), n_obj=8, n_user=40, density=0.5)
    e, m, _ = _load(zg, schema, rels)
    reqs = [("document", e.find("document", f"o{i}"), p) for i in range(8) for p in ("view", "restricted_view", "owner")]
    trees = e.expand_permission_trees(reqs)
    for (rt, res, perm), tree in zip(reqs, trees):
        by_str = zg._lib.parse_expand_lines(e.expand_permission_tree_str(rt, e.object_name(rt, res), perm))
        stack = [(tree, by_str)]
        while stack:
            a, b = stack.pop()
            assert a["op"] == b["op"]
            assert f"{a['type']}:{e.object_name(a['type'], a['object'])}" == b["object"] and a["relation"] == b["relation"]
            subs = [f"{t}:" + ("*" if r == "*" else e.object_name(t, i)) + (f"#{r}" if r and r != "*" else "")
                    for t, i, r in a["subjects"]]
            assert subs == b["subjects"]
            if a["op"] == "L" and a["relation"] in ("owner", "viewer", "editor", "banned"):
                # class order, then ascending id: the resident row of each class in turn
                rel = e.slot_id(a["type"], a["relation"])
                row = []
                for k in range(8):
                    out, n = np.zeros(4096, dtype=np.uint32), C.c_uint64(0)
                    if e._L.zg_debug_row(e._h, rel, a["object"], k, out.ctypes.data, out.size, C.byref(n)) != 0:
                        break
                    row += [int(x) for x in out[: n.value]]
                assert [i for _, i, _ in a["subjects"]] == row
            assert len(a["children"]) == len(b["children"])
            stack += list(zip(a["children"], b["children"]))


CHAIN = "definition user {}\ndefinition folder {\n  relation parent: folder\n  relation viewer: user\n" \
        "  permission view = viewer + parent->view\n}\n"


def test_depth_cap_cycles_and_a_mixed_batch(zg):
    rels = [f"folder:a{i}#parent@folder:a{i + 1}" for i in range(50)] + ["folder:a50#viewer@user:u"]
    rels += [f"folder:b{i}#parent@folder:b{i + 1}" for i in range(51)] + ["folder:b51#viewer@user:u"]
    rels += ["folder:c0#parent@folder:c1", "folder:c1#parent@folder:c0", "folder:c1#viewer@user:v"]
    e, m, o = _load(zg, CHAIN, rels)
    _compare(zg, e, m, o, [("folder", x, "view") for x in ("a0", "a1", "b0", "b1", "c0", "c1")],
             subjects=[("user", "u"), ("user", "v")])
    reqs = [("folder", e.find("folder", x), "view") for x in ("a0", "b0", "c1", "a1", "b0")]
    got = e.expand_permission_trees(reqs)
    assert [isinstance(t, zg.ZgpuError) for t in got] == [False, True, True, False, True]
    assert all(t.code == -9 for t in got if isinstance(t, zg.ZgpuError))
    alone = e.expand_permission_trees([reqs[0], reqs[3]])
    assert got[0] == alone[0] and got[3] == alone[1]


def test_e2big_retry_and_the_node_cap(zg, monkeypatch):
    model = randgen.model_from_schema(DOCS)
    rels = randgen.random_relationships(random.Random(5), model, n_obj=8, n_user=30, density=0.6)
    e, m, o = _load(zg, DOCS, rels)
    reqs = [("document", e.find("document", f"o{i}"), "view") for i in range(8)]
    big = e.expand_permission_trees(reqs)
    assert e.expand_permission_trees(reqs, node_cap=1, subj_cap=1) == big  # ZG_E2BIG, then the retry
    n_nodes = e.expand_counters()["nodes"]
    monkeypatch.setenv("ZGPU_EXPAND_CAP", "10")
    with pytest.raises(zg.ZgpuError) as x:
        e.expand_permission_trees(reqs)
    assert x.value.code == -8 and "ZGPU_EXPAND_CAP" in str(x.value)
    monkeypatch.delenv("ZGPU_EXPAND_CAP")
    assert e.expand_permission_trees(reqs) == big
    c = e.expand_counters()
    assert c["trees"] >= 24 and c["nodes"] > n_nodes and c["levels"] > 0
    assert e.expand_last_times().shape[1] == 3


def test_incremental_writes_collection_and_id_reuse(zg):
    rng = random.Random(11)
    model = randgen.model_from_schema(expiring(DOCS))
    schema = expiring(DOCS)
    e, m, o = _load(zg, schema, [], now=1_000)
    live = {}
    for round_ in range(5):
        ups, in_call = [], set()
        while len(ups) < 1000:
            t = rng.choice(["document", "folder", "group"])
            rel = rng.choice(list(model["types"][t]["rels"]))
            st, sr = rng.choice(model["types"][t]["rels"][rel])
            res = rng.randrange(1, 30)
            # a folder's parent is the folder below it: a chain, not a cycle or a DAG whose trees grow exponentially
            sid = "*" if sr == "*" else f"u{rng.randrange(60)}" if st == "user" else f"o{res - 1 if st == t else rng.randrange(30)}"
            r = f"{t}:o{res}#{rel}@{st}:{sid}" + (f"#{sr}" if sr and sr != "*" else "")
            if r in in_call:  # one update per relationship in a call
                continue
            in_call.add(r)
            if r in live and rng.random() < 0.3:
                ups.append((zg._lib.OP_DELETE, r, 0))
                live.pop(r)
                m.write(r, delete=True)
                o.delete(r)
                continue
            ex = rng.choice((0, 0, 1_500))
            ups.append((zg._lib.OP_TOUCH, r, ex))
            live[r] = ex
            m.write(r, ex)
            o.touch(r, ex)
        e.write_relationships(ups)
        _compare(zg, e, m, o, [("document", f"o{i}", "view") for i in range(0, 30, 7)] +
                 [("folder", f"o{i}", "view") for i in range(0, 30, 9)], now=1_000)
    e.set_clock(2_000)
    n = C.c_uint64(0)
    assert e._L.zg_collect_expired(e._h, 1_999, C.byref(n)) == 0 and n.value > 0
    for r, ex in list(live.items()):
        if ex:
            live.pop(r)
            m.write(r, delete=True)
            o.delete(r)
    _compare(zg, e, m, o, [("document", f"o{i}", "view") for i in range(0, 30, 5)], now=2_000)
    # retire the names nobody mentions any more, then hand their ids to new names
    assert e._L.zg_retire_unused_names(e._h, C.byref(n)) == 0
    new = [f"document:fresh{i}#viewer@user:new{i}" for i in range(20)]
    e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in new])
    for r in new:
        m.write(r)
        o.touch(r)
    _compare(zg, e, m, o, [("document", f"fresh{i}", "view") for i in range(0, 20, 4)] +
             [("document", f"o{i}", "view") for i in range(0, 30, 6)], now=2_000)


def test_client(zg):
    from spicedb_kubeapi_proxy_b200 import client

    c = client.PermissionsClient(DOCS, relationships=["document:d#viewer@user:a", "document:d#parent@folder:f",
                                                      "folder:f#owner@group:g#member"], device=0)
    r = c.ExpandPermissionTree(client.ExpandPermissionTreeRequest(client.ObjectReference("document", "d"), "view"))
    root = r.tree_root
    assert root.intermediate.operation == client.OPERATION_EXCLUSION
    union = root.intermediate.children[0]
    assert union.intermediate.children[0].leaf.subjects == [client.SubjectReference(client.ObjectReference("user", "a"))]
    folder = union.intermediate.children[2].intermediate.children[0]
    assert folder.expanded_object == client.ObjectReference("folder", "f")
    assert folder.intermediate.children[1].leaf.subjects == [
        client.SubjectReference(client.ObjectReference("group", "g"), "member")]


def test_refusals(zg):
    rels = [(zg._lib.OP_TOUCH, "document:d#viewer@user:a", 0)]
    e = zg.Engine(DOCS, device=0, shard_rank=0, shard_count=2)
    e.write_relationships(rels)
    with pytest.raises(zg.ZgpuError) as x:
        e.expand_permission_tree_str("document", "d", "view")
    assert x.value.code == -1
    try:
        h = zg.Engine(DOCS, device=0, n_shards=2)
    except zg.ZgpuError as err:
        pytest.skip(f"no sharded handle here: {err}")
    h.write_relationships(rels)
    with pytest.raises(zg.ZgpuError) as x:
        h.expand_permission_tree_str("document", "d", "view")
    assert x.value.code == -1 and "ExpandPermissionTree" in str(x.value)


def test_two_devices_answer_on_the_first(zg):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one device")
    e = zg.Engine(DOCS, device=0, n_devices=2)
    e.write_relationships([(zg._lib.OP_TOUCH, "document:d#viewer@user:a", 0)])
    assert e.expand_permission_tree_str("document", "d", "viewer") == ["0 L document:d#viewer user:a"]


def test_concurrent_callers(zg):
    model = randgen.model_from_schema(DOCS)
    rels = randgen.random_relationships(random.Random(9), model, n_obj=10, n_user=20)
    e, m, o = _load(zg, DOCS, rels)
    want = {f"o{i}": _want(e, m, "document", f"o{i}", "view", 0) for i in range(10)}
    errors, stop = [], threading.Event()

    def expander(k):
        try:
            for j in range(30):
                rid = f"o{(k + j) % 10}"
                got = e.expand_permission_tree_str("document", rid, "view")
                if got != want[rid]:
                    errors.append((rid, got))
        except Exception as x:  # noqa: BLE001
            errors.append(x)

    def writer():
        i = 0
        while not stop.is_set():  # relationships on objects the expanders never read
            e.write_relationships([(zg._lib.OP_TOUCH, f"document:w{i}#viewer@user:x{i}", 0)])
            i += 1

    def checker():
        while not stop.is_set():
            e.check_bulk_str([("document", "o1", "view", "user", "u1", "")])

    side = [threading.Thread(target=writer), threading.Thread(target=checker)]
    ts = [threading.Thread(target=expander, args=(k,)) for k in range(16)]
    for t in side + ts:
        t.start()
    for t in ts:
        t.join()
    stop.set()
    for t in side:
        t.join()
    assert not errors, errors[:3]


def _contains_ids(tree, stype, sid, has):
    if tree["op"] == "L":
        return any((t == stype and r is None and i == sid) or (t == stype and r == "*") or
                   (r not in (None, "*") and has[(t, i, r)]) for t, i, r in tree["subjects"])
    kids = [_contains_ids(c, stype, sid, has) for c in tree["children"]]
    return any(kids) if tree["op"] == "U" else all(kids) if tree["op"] == "I" else kids[0] and not any(kids[1:])


def _usersets(tree, out):
    out.update((t, i, r) for t, i, r in tree["subjects"] if r not in (None, "*"))
    for c in tree["children"]:
        _usersets(c, out)
    return out


def _property_on_sample(zg, e, o, res_type, perm, trees, res_ids, stype, users, now=0):
    """contains(tree, user) == Check(res#perm @ user) for every sampled tree and user, userset leaves decided by the
    oracle's checks."""
    for tree, res in zip(trees, res_ids):
        assert not isinstance(tree, zg.ZgpuError), tree
        us = sorted(_usersets(tree, set()))
        q = np.zeros(len(us) * len(users) + len(users), dtype=zg.CHECK_DTYPE)
        for k, u in enumerate(users):
            for j, (t, i, r) in enumerate(us):
                q[k * len(us) + j] = (i, u, o.slot_id(t, r), o.type_id(stype), zg.SREL_NONE, 0)
            q[len(us) * len(users) + k] = (res, u, o.slot_id(res_type, perm), o.type_id(stype), zg.SREL_NONE, 0)
        codes = o.check_bulk(q, now=now)
        for k, u in enumerate(users):
            has = {x: codes[k * len(us) + j] == HAS for j, x in enumerate(us)}
            assert _contains_ids(tree, stype, u, has) == (codes[len(us) * len(users) + k] == HAS), (res, perm, u)


@pytest.mark.parametrize("name,scale", [("cfg2", 0.002), ("cfg3", 0.002), ("cfg4", 0.001)])
def test_workloads_at_small_scale(zg, name, scale):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(name, scale=scale)
    e, o = zg.Engine(w.schema, device=0), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    c = w.checks[0]
    res = np.unique(c.res)[:24]
    trees = e.expand_permission_trees([(c.res_type, int(r), c.perm) for r in res])
    users = sorted({int(x) for x in c.subj[:40]} | {0})
    _property_on_sample(zg, e, o, c.res_type, c.perm, trees, res, c.subj_type, users)
    rows = GroupRows(w.schema, w.groups)  # the restatement, line for line and canonically
    for r, tree in zip(res, trees):
        want = expand_tree(rows, c.res_type, str(int(r)), c.perm, order=group_order)
        assert id_tree_lines(tree) == lines(want)
        assert canonical(zg._lib.parse_expand_lines(id_tree_lines(tree))) == canonical(want)


@pytest.mark.parametrize("seed,wide", [(0, False), (1, False), (2, True), (3, True)])
def test_shaped_stores(zg, seed, wide):
    """randgen.shaped_schema stores, 16-bit (wide False) and 32-bit closure-index seeds: trees line for line and
    canonically against the restatement at two clocks, and the property on a sample."""
    rng = random.Random(500 + seed)
    text, plan = randgen.shaped_schema(rng)
    store = randgen.shaped_relationships(rng, randgen.model_from_schema(text), plan, wide=wide)
    e, o = zg.Engine(text, device=0), Oracle(text)
    randgen.load_shaped(e, store)
    randgen.load_shaped(o, store)
    e.publish()
    rows = GroupRows(text, store["groups"])
    ex = [int(x) for g in store["groups"] if g[6] is not None for x in g[6][:1000]]
    model = randgen.model_from_schema(text)
    for now in (1, int(np.median(ex)) if ex else 2):
        e.set_clock(now)
        for t in model["tnames"]:
            for perm in list(model["types"][t]["perms"]):
                reqs = [(t, i, perm) for i in (0, 1, 7)]
                for (_, i, _), tree in zip(reqs, e.expand_permission_trees(reqs)):
                    want = expand_tree(rows, t, str(i), perm, now, order=group_order)
                    assert id_tree_lines(tree) == lines(want), (t, i, perm, now)
                    assert canonical(zg._lib.parse_expand_lines(id_tree_lines(tree))) == canonical(want)
        if now == 1:
            continue
        queries, res, subj = randgen.shaped_checks(random.Random(seed), store, plan, n=400)
        rt, perm, st, _ = next(q for q in queries if q[3] is None)
        pick = [i for i, q in enumerate(queries) if q == (rt, perm, st, None)][:8]
        res_ids = sorted({int(res[i]) for i in pick})
        trees = e.expand_permission_trees([(rt, r, perm) for r in res_ids])
        _property_on_sample(zg, e, o, rt, perm, trees, res_ids, st, sorted({int(subj[i]) for i in pick}), now=now)


def test_cfg4_full_size_batched(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    scale = float(os.environ.get("ZGPU_FULLSIZE_SCALE", "0.25"))
    w = workloads.cfg4(scale=scale)
    e = zg.Engine(w.schema, device=0)
    w.load_into(e)
    e.publish()
    c = w.checks[0]
    docs = np.unique(c.res)[:4096]
    assert c.res_type == "document" and docs.size == 4096
    trees = e.expand_permission_trees([("document", int(d), "view") for d in docs])
    assert sum(isinstance(t, zg.ZgpuError) for t in trees) == 0
    o = Oracle(w.schema)
    w.load_into(o)
    pick = np.random.default_rng(0).choice(4096, 16, replace=False)
    users = [int(u) for u in np.random.default_rng(1).choice(int(c.subj.max()) + 1, 24, replace=False)]
    _property_on_sample(zg, e, o, "document", "view", [trees[i] for i in pick], docs[pick], c.subj_type, users)
