"""The sharded handle (zg_config.n_shards): ONE engine holding every shard of an object-hash sharded store, checks
crossing the shards in-process. Every answer is compared bit for bit with the oracle, a replica engine and the
multi-engine protocol (dist.DeviceShardedChecker). With one GPU the shards are virtual: they share device 0."""
import os
import random
import threading

import numpy as np
import pytest

import randgen
from golden_runner import run_case, split_rel

pytestmark = pytest.mark.gpu

EINVAL, EPRECOND = -1, -5  # include/zgpu.h
FULL_SCALE = float(os.environ.get("ZGPU_FULLSIZE_SCALE", "0.25"))  # as tests/test_gpu_fullsize.py: 0.25 = 24 M


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _load_strings(e, rels, expires=None):
    ups = [(0, r, (expires or {}).get(r, 0)) for r in rels]
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])
    if not ups:
        e.publish()


def _items(e, checks):
    """Interned items for 'type:id#perm@stype:sid[#srel]' strings (names the engine never saw read as unknown ids)."""
    from spicedb_kubeapi_proxy_b200 import _lib

    items = np.zeros(len(checks), dtype=_lib.CHECK_DTYPE)
    for i, q in enumerate(checks):
        rt, rid, perm, st, sid, srel = split_rel(q)
        items["perm"][i] = e.slot_id(rt, perm)
        items["stype"][i] = e.type_id(st)
        items["srel"][i] = e.slot_id(st, srel) if srel else _lib.SREL_NONE
        r, u = e.find(rt, rid), e.find(st, sid)
        items["res"][i] = r
        items["subj"][i] = u if u != _lib.NO_OBJECT else (_lib.NO_OBJECT if (r == _lib.NO_OBJECT and rt == st and rid == sid)
                                                          else _lib.NO_OBJECT - 1)
    return items


@pytest.mark.parametrize("S,name,scale", [(2, "cfg2", 0.01), (3, "cfg3", 0.005), (4, "cfg4", 0.001), (8, "cfg4", 0.002),
                                          (8, "cfg3", 0.003), (2, "cfg4", 0.001)])
def test_handle_equals_oracle_and_replica_on_workloads(zg, S, name, scale):
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = getattr(workloads, name)(scale=scale)
    h, rep, o = zg.Engine(w.schema, n_shards=S), zg.Engine(w.schema), Oracle(w.schema)
    for t in (h, rep, o):
        w.load_into(t)
    h.publish(), rep.publish()
    items = w.check_items(h, zg.CHECK_DTYPE)
    got = h.check_bulk(items)
    assert np.array_equal(got, o.check_bulk(items))
    assert np.array_equal(got, rep.check_bulk(items))
    st = h.stats()
    assert st["shards"] == S and st["devices"] == 1 and st["last_levels"] >= 1 and st["last_round_trips"] >= 3
    assert st["tuples"] == rep.stats()["tuples"], "the shards hold the store's relationships between them"


@pytest.mark.parametrize("S", [2, 3, 4, 8])
@pytest.mark.parametrize("seed", range(4))
def test_handle_equals_oracle_and_replica_on_random_graphs(zg, S, seed):
    from oracle.pyoracle import Oracle

    rng = random.Random(9000 + 10 * S + seed)
    if seed % 2:
        schema, model = randgen.random_schema(rng)
    else:
        schema = randgen.FIXED_SCHEMAS[sorted(randgen.FIXED_SCHEMAS)[(seed // 2 + S) % len(randgen.FIXED_SCHEMAS)]]
        model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=9, n_user=6, density=0.35)
    checks = randgen.random_checks(rng, model, 800, n_obj=9, n_user=6)
    h, rep, o = zg.Engine(schema, n_shards=S), zg.Engine(schema), Oracle(schema)
    _load_strings(h, rels), _load_strings(rep, rels)
    for r in rels:
        o.touch(r)
    got = h.check_bulk_str(checks)
    assert list(got) == [o.check(*split_rel(q)) for q in checks], schema
    assert np.array_equal(got, rep.check_bulk_str(checks))


def test_depth_cap_and_cycles_across_shards(zg):
    from oracle.pyoracle import Oracle
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i+1}#member" for i in range(51)] + ["group:g51#member@user:deep"]
    rels += ["group:a#member@group:b#member", "group:b#member@group:a#member", "group:b#member@user:x"]
    rels += [f"folder:f{i}#parent@folder:f{i+1}" for i in range(51)] + ["folder:f0#viewer@user:v"]
    checks = ["group:g0#member@user:deep", "group:g1#member@user:deep", "group:g2#member@user:nobody",
              "group:a#member@user:x", "group:a#member@user:y", "folder:f0#view@user:v", "folder:f0#view@user:w",
              "folder:f0#not_view@user:v", "folder:f0#not_view@user:w", "folder:f40#view@user:v"]
    o = Oracle(CHAIN)
    for r in rels:
        o.touch(r)
    h = zg.Engine(CHAIN, n_shards=3)
    _load_strings(h, rels)
    got = h.check_bulk_str(checks)
    assert list(got) == [o.check(*split_rel(q)) for q in checks]
    assert list(got[:5]) == [255, 2, 1, 2, 255]
    assert h.stats()["last_levels"] > 20, "the 51-hop chain must cross shards level by level"


def test_expiry_at_two_clocks(zg):
    from oracle.pyoracle import Oracle

    schema = """
use expiration
definition user {}
definition group { relation member: user | group#member }
definition doc {
  relation viewer: user | user:* | group#member
  relation temp: user with expiration
  relation wtemp: user:* with expiration
  permission view = viewer + temp + wtemp
  permission strict = view - temp
}
"""
    rels = ["doc:d1#temp@user:t", "doc:d2#viewer@user:*", "doc:d3#viewer@group:eng#member", "group:eng#member@user:e1",
            "doc:d4#wtemp@user:*", "group:eng#member@group:sub#member", "group:sub#member@user:s1", "doc:d5#temp@user:t"]
    expires = {"doc:d1#temp@user:t": 1000, "doc:d4#wtemp@user:*": 2000, "doc:d5#temp@user:t": 3000}
    checks = ["doc:d1#view@user:t", "doc:d1#strict@user:t", "doc:d2#view@user:anyone", "doc:d3#view@user:e1",
              "doc:d3#view@user:s1", "doc:d4#view@user:who", "doc:d5#view@user:t", "doc:d5#strict@user:t",
              "doc:d3#view@group:sub#member", "doc:never#view@user:never"]
    o = Oracle(schema)
    for r in rels:
        o.touch(r, expires.get(r, 0))
    h = zg.Engine(schema, n_shards=4)
    _load_strings(h, rels, expires)
    for now in (999, 2001):
        h.set_clock(now)
        assert list(h.check_bulk_str(checks)) == [o.check(*split_rel(q), now) for q in checks], now


def _dist_run(zg, schema, load, items, world):
    """dist.DeviceShardedChecker over LocalDeviceTransport on `world` one-shard engines of this GPU: the answers, rank 0's
    levels and the sub-queries every rank sent."""
    import torch

    from spicedb_kubeapi_proxy_b200 import dist as zdist

    ts = zdist.LocalDeviceTransport.cluster(world)
    engines = [zg.Engine(schema, shard_rank=r, shard_count=world) for r in range(world)]
    for e in engines:
        load(e)
        e.publish()
    bounds = [zdist.shard_bounds(items.size, r, world) for r in range(world)]
    out, errs, stats = [None] * world, [], [None] * world

    def run(r):
        try:
            lo, hi = bounds[r]
            d = torch.from_numpy(np.ascontiguousarray(items[lo:hi]).view(np.uint8).copy()).cuda()
            ck = zdist.DeviceShardedChecker(engines[r], ts[r])
            out[r] = ck.check_bulk(d, hi - lo).cpu().numpy()
            stats[r] = ck.stats
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))
            ts[r]._s["bar"].abort()

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errs, errs
    return np.concatenate(out), stats[0]["levels"], sum(s["subqueries_sent"] for s in stats)


@pytest.mark.parametrize("S,name,scale", [(3, "cfg4", 0.001), (4, "cfg3", 0.003), (8, "deep_nonpure", 0)])
def test_handle_equals_the_multi_engine_protocol(zg, S, name, scale):
    """Same answers and levels as dist.DeviceShardedChecker on S one-shard engines, and the same sub-queries sent up to the
    check kernel's order dependence: which checks share a warp decides short circuits and the lossy path memo, and both
    drivers place routed queries with atomics, so either's count moves by a fraction of a percent between runs."""
    from spicedb_kubeapi_proxy_b200 import workloads

    if name in randgen.FIXED_SCHEMAS:
        schema = randgen.FIXED_SCHEMAS[name]
        rng = random.Random(31)
        model = randgen.model_from_schema(schema)
        rels = randgen.random_relationships(rng, model, n_obj=9, n_user=6, density=0.35)
        checks = randgen.random_checks(rng, model, 3000, n_obj=9, n_user=6)

        def load(e):
            _load_strings(e, rels)

        h = zg.Engine(schema, n_shards=S)
        load(h)
        items = _items(h, checks)
    else:
        w = getattr(workloads, name)(scale=scale)
        schema = w.schema

        def load(e):
            w.load_into(e)

        h = zg.Engine(schema, n_shards=S)
        load(h)
        h.publish()
        items = w.check_items(h, zg.CHECK_DTYPE)
    got = h.check_bulk(items)
    st = h.stats()
    want, levels, sent = _dist_run(zg, schema, load, items, S)
    assert np.array_equal(got, want)
    assert st["last_levels"] == levels
    assert abs(st["last_subqueries"] - sent) <= max(2, sent // 100), (st["last_subqueries"], sent)
    assert st["last_round_trips"] == levels + 2, "one host round trip per level, plus routing in and answers out"


def test_full_size_cfg4_against_a_replica(zg):
    """cfg4 at the suite's full-size scale (0.25: 24 M relationships), 1 M checks, 4 virtual shards."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=FULL_SCALE)
    h, rep = zg.Engine(w.schema, n_shards=4), zg.Engine(w.schema)
    for e in (h, rep):
        w.load_into(e)
        e.publish()
    items = w.check_items(h, zg.CHECK_DTYPE)[: 1 << 20]
    assert items.size == 1 << 20
    got = h.check_bulk(items)
    assert np.array_equal(got, rep.check_bulk(items))
    assert (got == zg.HAS_PERMISSION).any() and (got == zg.NO_PERMISSION).any()


def test_subquery_overflow_splits_and_stays_exact(zg):
    from oracle.pyoracle import Oracle

    rng = random.Random(77)
    schema = randgen.FIXED_SCHEMAS["deep_nonpure"]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=6, density=0.35)
    checks = randgen.random_checks(rng, model, 1500, n_obj=8, n_user=6)
    o = Oracle(schema)
    for r in rels:
        o.touch(r)
    small, big = zg.Engine(schema, n_shards=3, subquery_capacity=48), zg.Engine(schema, n_shards=3)
    _load_strings(small, rels), _load_strings(big, rels)
    want = [o.check(*split_rel(q)) for q in checks]
    assert list(big.check_bulk_str(checks)) == want
    assert list(small.check_bulk_str(checks)) == want
    assert small.stats()["split_batches"] > 0 and big.stats()["split_batches"] == 0


def test_writes_merge_on_every_shard(zg, monkeypatch):
    """5 x 1 000 updates (TOUCH, DELETE, preconditions, delete-by-filter) with checks after every write: equal to a replica,
    every shard merges (no rebuild), and under ZGPU_VERIFY_BUILD=1 every shard's arrays equal its host rebuild."""
    from spicedb_kubeapi_proxy_b200 import _lib

    monkeypatch.setenv("ZGPU_VERIFY_BUILD", "1")
    rng = random.Random(5)
    schema = randgen.FIXED_SCHEMAS["docs"]
    model = randgen.model_from_schema(schema)
    pool = randgen.random_relationships(rng, model, n_obj=120, n_user=80, density=0.25)
    checks = randgen.random_checks(rng, model, 4000, n_obj=120, n_user=80)
    S = 4
    h, rep = zg.Engine(schema, n_shards=S), zg.Engine(schema)
    first = pool[: len(pool) // 2]
    _load_strings(h, first), _load_strings(rep, first)
    before = h.stats()
    assert before["full_publishes"] == S
    live = set(first)
    for step in range(5):
        ups = []
        for r in rng.sample(pool, 1000):
            op = _lib.OP_DELETE if (r in live and rng.random() < 0.5) else _lib.OP_TOUCH
            ups.append((op, r, 0))
            (live.discard if op == _lib.OP_DELETE else live.add)(r)
        anchor = rng.choice(sorted(live))
        pre = [(_lib.PRECOND_MUST_MATCH, {"res_type": anchor.split(":")[0], "res_id": anchor.split(":")[1].split("#")[0]})]
        for e in (h, rep):
            e.write_relationships(ups, pre)
        assert np.array_equal(h.check_bulk_str(checks), rep.check_bulk_str(checks)), step
        # a failing precondition writes nothing on either
        for e in (h, rep):
            with pytest.raises(zg.ZgpuError) as ex:
                e.write_relationships([(_lib.OP_TOUCH, pool[0], 0)],
                                      [(_lib.PRECOND_MUST_NOT_MATCH, {"res_type": anchor.split(":")[0],
                                                                       "res_id": anchor.split(":")[1].split("#")[0]})])
            assert ex.value.code == EPRECOND
        victim = rng.choice(sorted(live))
        flt = {"res_type": victim.split(":")[0], "res_id": victim.split(":")[1].split("#")[0]}
        assert h.delete_relationships(flt) == rep.delete_relationships(flt)
        live = {r for r in live if not r.startswith(f"{flt['res_type']}:{flt['res_id']}#")}
        assert np.array_equal(h.check_bulk_str(checks), rep.check_bulk_str(checks)), step
        assert sorted(h.read_relationships()) == sorted(rep.read_relationships())
    st = h.stats()
    assert st["full_publishes"] == before["full_publishes"], "writes merge into every shard, no rebuild"
    assert st["delta_publishes"] >= S * 10
    assert h.watch_read(0) == rep.watch_read(0)


def test_shard_arrays_equal_one_shard_engines(zg):
    """For every shard k: the handle's rows equal those of an engine built as shard_rank = k, shard_count = S."""
    rng = random.Random(12)
    schema = randgen.FIXED_SCHEMAS["docs"]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=10, n_user=7, density=0.5)
    S = 3
    h = zg.Engine(schema, n_shards=S)
    one = [zg.Engine(schema, shard_rank=k, shard_count=S) for k in range(S)]
    for e in [h] + one:
        _load_strings(e, rels)
    for k in range(S):
        for t, d in model["types"].items():
            for r, allowed in d["rels"].items():
                for c in range(len(allowed)):
                    for i in range(12):
                        for rev in (False, True):
                            assert np.array_equal(h.debug_row(t, r, i, c, reverse=rev, shard=k),
                                                  one[k].debug_row(t, r, i, c, reverse=rev)), (k, t, r, c, i, rev)


def test_concurrent_callers_while_a_writer_publishes(zg):
    """32 threads call zg_check_bulk while a writer publishes relationships none of their checks can see: every answer
    is exact and the callers share groups."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import _lib, workloads

    w = workloads.cfg4(scale=0.002)
    h, o = zg.Engine(w.schema, n_shards=4), Oracle(w.schema)
    w.load_into(h), w.load_into(o)
    h.publish()
    items = w.check_items(h, zg.CHECK_DTYPE)
    want = o.check_bulk(items)
    checked = set(int(x) for x in items["res"])
    free = [d for d in range(1, 200000) if d not in checked][:400]
    stop, errs = threading.Event(), []

    def writer():
        up = np.zeros(1, dtype=_lib.UPDATE_DTYPE)
        up["rel"], up["stype"], up["srel"] = h.slot_id("document", "banned"), h.type_id("user"), _lib.SREL_NONE
        i = 0
        while not stop.is_set():
            up["res"], up["subj"], up["op"] = free[i % len(free)], i % 97, _lib.OP_TOUCH if (i // len(free)) % 2 == 0 else _lib.OP_DELETE
            h.apply_updates(up)
            h.publish()
            i += 1

    def caller(t):
        try:
            for j in range(6):
                lo = ((t * 6 + j) * 1000) % (items.size - 2000)
                n = 500 + (t * 37 + j * 11) % 1500
                got = h.check_bulk(items[lo:lo + n])
                if not np.array_equal(got, want[lo:lo + n]):
                    errs.append((t, j))
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))

    c0 = h.stats()["coalesced_launches"]
    wt = threading.Thread(target=writer)
    wt.start()
    ths = [threading.Thread(target=caller, args=(t,)) for t in range(32)]
    [x.start() for x in ths]
    [x.join() for x in ths]
    stop.set()
    wt.join()
    assert not errs, errs[:5]
    assert h.stats()["coalesced_launches"] > c0


class _HandleBackend:
    """The golden cases through client.PermissionsClient over a sharded handle. LookupResources is refused by the handle
    (the deployment delegates it), so lookups are answered by a replica fed the same writes."""

    def __init__(self, zg, schema):
        self.C = zg.client
        self.cl = self.C.PermissionsClient(schema, engine=zg.Engine(schema, n_shards=3))
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
        with pytest.raises(C.RpcError, match="sharded handle"):
            list(self.cl.LookupResources(req))
        return [r.resource_object_id for r in self.rep.LookupResources(req)]

    def read(self, res_type="", res_id="", rel="", **_):
        C = self.C
        return [r.relationship.text() for r in self.cl.ReadRelationships(
            C.ReadRelationshipsRequest(C.RelationshipFilter(res_type, res_id, rel)))]


def test_golden_cases_through_the_client(zg, golden):
    for case in golden["cases"]:
        run_case(_HandleBackend(zg, golden["schemas"][case["schema"]]), case)


def test_string_packed_and_postfilter_calls_equal_a_replica(zg):
    import json

    from spicedb_kubeapi_proxy_b200 import _lib, workloads

    schema = workloads.BOOTSTRAP_SCHEMA
    rels = [f"pod:ns{i % 3}/p{i}#viewer@user:u{i % 7}" for i in range(300)] + \
           [f"pod:ns{i % 3}/p{i}#creator@user:u{i % 5}" for i in range(0, 300, 4)] + ["namespace:ns1#creator@user:u1"]
    h, rep = zg.Engine(schema, n_shards=3), zg.Engine(schema)
    _load_strings(h, rels), _load_strings(rep, rels)
    checks = [f"pod:ns{i % 3}/p{i}#view@user:u{i % 9}" for i in range(0, 400, 3)] + ["pod:nope#view@user:u1", "nope:x#view@user:u1"]
    assert np.array_equal(h.check_bulk_str(checks), rep.check_bulk_str(checks))
    res_ids = [f"ns{i % 3}/p{i}" for i in range(350)]
    subjects = [f"u{i % 8}" for i in range(350)]
    assert np.array_equal(h.check_bulk_packed("pod", "view", "user", res_ids, subjects),
                          rep.check_bulk_packed("pod", "view", "user", res_ids, subjects))
    body = json.dumps({"kind": "PodList", "items": [{"metadata": {"name": f"p{i}", "namespace": f"ns{i % 3}"}}
                                                    for i in range(0, 320, 2)]}).encode()
    for u in ("u1", "u4", "nobody"):
        tpl = [h.list_template("pod", "view", "user", u)]
        assert h.list_postfilter(body, tpl) == rep.list_postfilter(body, [rep.list_template("pod", "view", "user", u)])


def test_refused_entry_points_say_so(zg):
    import torch

    from spicedb_kubeapi_proxy_b200 import _lib, workloads

    schema = workloads.BOOTSTRAP_SCHEMA
    h = zg.Engine(schema, n_shards=2)
    _load_strings(h, ["pod:ns/p1#viewer@user:a"])
    d_items = torch.zeros(16 * 4, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(4, dtype=torch.uint8, device="cuda")
    calls = {
        "lookup resources": (lambda: h.lookup_resources_ids("pod", "view", "user", h.find("user", "a")), "LookupResources"),
        "lookup subjects": (lambda: h.lookup_subjects_ids("pod", h.find("pod", "ns/p1"), "view", "user"), "LookupResources"),
        "pre-filter": (lambda: h.list_prefilter(b'{"items": []}', h.list_template("pod", "view", "user", "a")), "pre-filter"),
        "device": (lambda: h.check_bulk_device(d_items.data_ptr(), 4, d_out.data_ptr()), "device buffers"),
        "ingress": (lambda: h.check_bulk_packed_ingress("pod", "view", "user", ["ns/p1"], ["a"]), "device-ingress"),
        "shard pass": (lambda: h.shard_pass_dev(d_items.data_ptr(), 4, 0), "zg_shard_"),
        "shard route": (lambda: h.shard_route_dev(d_items.data_ptr(), 4, 0, 2, d_items.data_ptr(), d_out.data_ptr()), "zg_shard_"),
        "shard lookup": (lambda: h.shard_lookup_candidates_dev(False, 0, 0), "zg_shard_"),
    }
    for what, (call, msg) in calls.items():
        with pytest.raises(zg.ZgpuError, match=msg) as ex:
            call()
        assert ex.value.code == EINVAL, what
        assert "sharded handle" in str(ex.value), what
    # the handle still answers checks afterwards
    assert list(h.check_bulk_str(["pod:ns/p1#view@user:a", "pod:ns/p1#view@user:b"])) == [2, 1]


def test_shards_on_several_devices(zg):
    import torch

    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs >= 2 GPUs")
    w = workloads.cfg4(scale=0.005)
    S = 2 * n_dev
    h, o = zg.Engine(w.schema, device=0, n_devices=n_dev, n_shards=S), Oracle(w.schema)
    w.load_into(h), w.load_into(o)
    h.publish()
    st = h.stats()
    assert st["devices"] == n_dev and st["shards"] == S
    items = w.check_items(h, zg.CHECK_DTYPE)
    assert np.array_equal(h.check_bulk(items), o.check_bulk(items))
