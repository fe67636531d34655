"""Parity tests proper: the CUDA path, called through the C ABI (libzgpu.so), against
the CPU oracle on the same inputs -- bit-exact (integer/boolean work).

  * golden cases G1..G14 restated from the reference's own tests (tests/golden/)
  * random schemas/graphs covering the operators the reference never pins
    (& - -> usersets wildcards expiration depth cap): "parity unpinned" vs SpiceDB,
    exact vs the oracle
  * the BASELINE.json configurations at oracle-sized scale, bit-exact
  * the full-size configurations through size-independent properties
"""
import random

import numpy as np
import pytest

import randgen
from golden_runner import run_case, split_rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


class EngineBackend:
    """Drives the golden cases through the v1.PermissionsServiceClient mirror."""

    def __init__(self, zg, schema):
        self.C = zg.client
        self.cl = self.C.PermissionsClient(schema)

    def write(self, rel):
        C = self.C
        self.cl.WriteRelationships(C.WriteRelationshipsRequest(
            [C.RelationshipUpdate(C.OPERATION_TOUCH, C.Relationship.parse(rel))]))

    def _item(self, rt, rid, perm, st, sid, srel):
        C = self.C
        return C.CheckBulkPermissionsRequestItem(C.ObjectReference(rt, rid), perm,
                                                 C.SubjectReference(C.ObjectReference(st, sid), srel))

    def check(self, rt, rid, perm, st, sid, srel=""):
        C = self.C
        try:
            r = self.cl.CheckPermission(C.CheckPermissionRequest(
                C.ObjectReference(rt, rid), perm, C.SubjectReference(C.ObjectReference(st, sid), srel)))
        except C.RpcError:
            return 255
        return r.permissionship

    def bulk(self, rels):
        resp = self.cl.CheckBulkPermissions(self.C.CheckBulkPermissionsRequest([self._item(*split_rel(r)) for r in rels]))
        assert len(resp.pairs) == len(rels)  # pkg/authz/check.go:54-57 relies on this
        return [255 if p.GetError() else p.GetItem().permissionship for p in resp.pairs]

    def lookup(self, rt, perm, st, sid, srel):
        C = self.C
        return [r.resource_object_id for r in self.cl.LookupResources(C.LookupResourcesRequest(
            rt, perm, C.SubjectReference(C.ObjectReference(st, sid), srel)))]

    def read(self, res_type="", res_id="", rel="", **_):
        C = self.C
        return [r.relationship.text() for r in self.cl.ReadRelationships(
            C.ReadRelationshipsRequest(C.RelationshipFilter(res_type, res_id, rel)))]


def test_golden_cases_through_the_client(zg, golden):
    for case in golden["cases"]:
        run_case(EngineBackend(zg, golden["schemas"][case["schema"]]), case)


def _compare_strings(zg, schema, rels, checks, lookups=(), now=0, expires=None):
    from oracle.pyoracle import Oracle

    o = Oracle(schema)
    e = zg.Engine(schema)
    if now:
        e.set_clock(now)
    ups = []
    for r in rels:
        ex = (expires or {}).get(r, 0)
        o.touch(r, ex)
        ups.append((zg._lib.OP_TOUCH, r, ex))
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])
    if not ups:
        e.publish()
    got = e.check_bulk_str(checks)
    want = [o.check(*split_rel(q), now) for q in checks]
    bad = [(q, int(g), w) for q, g, w in zip(checks, got, want) if g != w]
    assert not bad, f"{len(bad)} mismatches, first: {bad[:5]}\n{schema}\n" + "\n".join(rels)
    for (rt, perm, st, sid, srel) in lookups:
        a = sorted(e.lookup_resources_str(rt, perm, st, sid, srel))
        b = sorted(o.lookup_resources(rt, perm, st, sid, srel, now))
        assert a == b, f"lookup {rt}#{perm}@{st}:{sid}#{srel}: gpu={a} oracle={b}"
    return e, o


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
@pytest.mark.parametrize("seed", range(3))
def test_fixed_schemas_random_graphs(zg, name, seed):
    rng = random.Random(500 + seed)
    schema = randgen.FIXED_SCHEMAS[name]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=7, n_user=6, density=0.3)
    checks = randgen.random_checks(rng, model, 600, n_obj=7, n_user=6)
    lookups = [(t, p, "user", f"u{rng.randint(0, 6)}", "") for t, d in model["types"].items() for p in list(d["perms"])[:3]]
    _compare_strings(zg, schema, rels, checks, lookups)


@pytest.mark.parametrize("seed", range(30))
def test_random_schemas_random_graphs(zg, seed):
    rng = random.Random(seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.35)
    checks = randgen.random_checks(rng, model, 400, n_obj=6, n_user=5)
    lookups = [(t, p, "user", f"u{rng.randint(0, 5)}", "") for t in model["tnames"]
               for p in list(model["types"][t]["perms"])[:2]]
    _compare_strings(zg, schema, rels, checks, lookups)


def test_depth_cap_cycles_and_error_propagation(zg):
    """pkg/spicedb/spicedb.go:33: the 51st dispatch is an error; Kleene propagation."""
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i+1}#member" for i in range(51)] + ["group:g51#member@user:deep"]
    rels += ["group:a#member@group:b#member", "group:b#member@group:a#member", "group:b#member@user:x"]
    rels += [f"folder:f{i}#parent@folder:f{i+1}" for i in range(51)] + ["folder:f0#viewer@user:v"]
    checks = ["group:g0#member@user:deep", "group:g1#member@user:deep", "group:g2#member@user:nobody",
              "group:a#member@user:x", "group:a#member@user:y", "folder:f0#view@user:v", "folder:f0#view@user:w",
              "folder:f0#not_view@user:v", "folder:f0#not_view@user:w", "folder:f1#view@user:v", "folder:f40#view@user:v"]
    e, o = _compare_strings(zg, CHAIN, rels, checks)
    assert list(e.check_bulk_str(checks[:5])) == [255, 2, 1, 2, 255]


def test_expiration_wildcards_userset_subjects_unknown_names(zg):
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
            "doc:d4#wtemp@user:*", "group:eng#member@group:sub#member", "group:sub#member@user:s1"]
    expires = {"doc:d1#temp@user:t": 1000, "doc:d4#wtemp@user:*": 2000}
    checks = ["doc:d1#view@user:t", "doc:d1#strict@user:t", "doc:d2#view@user:anyone-at-all", "doc:d2#view@group:g#member",
              "doc:d3#view@user:e1", "doc:d3#view@group:eng#member", "doc:d3#viewer@group:eng#member",
              "doc:d3#view@group:ops#member", "group:eng#member@group:eng#member", "group:zzz#member@group:zzz#member",
              "doc:never#view@user:never", "doc:d4#view@user:who", "doc:d3#view@user:s1", "doc:d3#view@group:sub#member",
              "doc:d3#nope@user:e1", "nope:d3#view@user:e1", "doc:d3#view@user:e1#member", "doc:d3#view@nope:x"]
    lookups = [("doc", "view", "user", "t", ""), ("doc", "view", "user", "e1", ""), ("doc", "strict", "user", "zz", ""),
               ("doc", "view", "group", "eng", "member"), ("group", "member", "group", "sub", "member"),
               ("group", "member", "group", "nowhere", "member")]
    for now in (999, 1000, 1999, 2001):
        _compare_strings(zg, schema, rels, checks, lookups, now=now, expires=expires)


def test_bulk_contract_and_edge_cases(zg):
    """empty batch, one item, ragged sizes around the 32-check batch, out-of-range ids."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg2(scale=0.002)
    e, o = zg.Engine(w.schema), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(e, zg.CHECK_DTYPE)
    assert np.array_equal(items, w.check_items(o, zg.CHECK_DTYPE))
    assert e.check_bulk(items[:0]).size == 0
    for n in (1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, items.size):
        assert np.array_equal(e.check_bulk(items[:n]), o.check_bulk(items[:n])), n
    # ids beyond every row table, invalid slots/types -> NO / ERROR exactly like the oracle
    bad = items[:8].copy()
    bad["res"][0] = 0xFFFFFFFF
    bad["subj"][1] = 0xFFFFFFFE
    bad["res"][2] = 10**9
    bad["perm"][3] = 999
    bad["stype"][4] = 77
    bad["srel"][5] = 999
    bad["flags"][6] = 0xFFFF  # flags are ignored on caller items
    assert np.array_equal(e.check_bulk(bad), o.check_bulk(bad))
    # pinned caller buffers take the no-staging path
    pin_in = zg._lib.PinnedArray(items.size, zg.CHECK_DTYPE)
    pin_out = zg._lib.PinnedArray(items.size, np.uint8)
    pin_in.array[:] = items
    e.check_bulk_ptr(pin_in.ptr, items.size, pin_out.ptr)
    assert np.array_equal(pin_out.array, o.check_bulk(items))
    # results are answered per item, in order: a permutation permutes the answers
    perm = np.random.default_rng(0).permutation(items.size)
    assert np.array_equal(e.check_bulk(items[perm]), e.check_bulk(items)[perm])


@pytest.mark.parametrize("forward_only", [False, True])
@pytest.mark.parametrize("name,scale", [("cfg1", 1.0), ("cfg2", 0.01), ("cfg2-zipf", 0.01), ("cfg3", 0.002), ("cfg3", 0.01),
                                        ("cfg4", 0.0005), ("cfg4", 0.002)])
def test_baseline_configs_scaled_bit_exact(zg, name, scale, forward_only):
    """Both probe strategies (direction-optimised from the subject's reverse rows, and
    forward-only binary search) must agree with the oracle bit for bit."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(name, scale)
    e, o = zg.Engine(w.schema, forward_only=forward_only), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(e, zg.CHECK_DTYPE)
    got, want = e.check_bulk(items), o.check_bulk(items)
    assert np.array_equal(got, want), f"{name}: {(got != want).sum()} of {items.size} differ"
    assert 0.05 < (want == 2).mean() < 0.95, "workload should mix HAS and NO"
    for (rt, perm, st, subj) in w.lookups[:4]:
        a = e.lookup_resources_ids(rt, perm, st, subj)
        b = o.lookup_resources_ids(rt, perm, st, subj)
        assert np.array_equal(a, b), f"{name} lookup {rt}#{perm}@{st}:{subj}: {a.size} vs {b.size}"
    # the instrumented variant answers identically and reports a plausible byte count
    nbytes = e.count_alg_bytes(items)
    assert nbytes >= 17 * items.size
    assert e.num_tuples() == o_num_unique(w)


def o_num_unique(w):
    tot = 0
    for g in w.groups:
        key = g.res.astype(np.uint64) << np.uint64(32) | (0 if g.wildcard else g.subj.astype(np.uint64))
        tot += np.unique(key).size
    # groups sharing (relation, subject kind) could overlap; generators never do that
    return tot


def test_device_pointer_entry_matches_host_entry(zg):
    import torch
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3(scale=0.002)
    e = zg.Engine(w.schema)
    w.load_into(e)
    e.publish()
    items = w.check_items(e, zg.CHECK_DTYPE)
    d_items = torch.from_numpy(items.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(items.size, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    e.check_bulk_device(d_items.data_ptr(), items.size, d_out.data_ptr(), s.cuda_stream)
    s.synchronize()
    assert np.array_equal(d_out.cpu().numpy(), e.check_bulk(items))


def test_full_size_cfg2_properties(zg):
    """BASELINE config 2 at full size: every stored relationship checks HAS (direct
    and through the union), LookupResources equals the stored set, answers are
    invariant under permutation and identical between host and device entry points."""
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg2()
    e = zg.Engine(w.schema)
    w.load_into(e)
    e.publish()
    g = w.groups[0]
    idx = np.random.default_rng(5).integers(0, g.res.size, 200_000)
    items = np.zeros(idx.size, dtype=zg.CHECK_DTYPE)
    items["res"], items["subj"] = g.res[idx], g.subj[idx]
    items["stype"], items["srel"] = e.type_id("user"), 0xFFFF
    for perm in ("viewer", "view"):
        items["perm"] = e.slot_id("pod", perm)
        assert (e.check_bulk(items) == 2).all()
    items["perm"] = e.slot_id("pod", "creator")
    assert (e.check_bulk(items) == 1).all()
    for (rt, perm, st, u) in w.lookups[:6]:
        want = np.unique(g.res[g.subj == u])
        assert np.array_equal(e.lookup_resources_ids(rt, perm, st, u), want)
    base = w.check_items(e, zg.CHECK_DTYPE)
    r1 = e.check_bulk(base)
    pm = np.random.default_rng(6).permutation(base.size)
    assert np.array_equal(e.check_bulk(base[pm]), r1[pm])


def test_full_size_cfg3_properties(zg):
    """BASELINE config 3 at full size (10M tuples, 1M checks): the half of the batch
    built by walking stored edges must be HAS; a sample agrees with the oracle."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3()
    e = zg.Engine(w.schema)
    w.load_into(e)
    e.publish()
    items = w.check_items(e, zg.CHECK_DTYPE)
    got = e.check_bulk(items)
    assert 0.45 < (got == 2).mean() < 0.75 and not (got == 255).any()
    o = Oracle(w.schema)
    w.load_into(o)
    sample = np.random.default_rng(7).choice(items.size, 20_000, replace=False)
    assert np.array_equal(got[sample], o.check_bulk(items[sample]))
    st = e.stats()
    assert st["tuples"] == e.num_tuples() and st["launches"] >= 1


def test_concurrent_callers_are_coalesced_and_exact(zg):
    """The proxy calls the boundary from many goroutines at once (pkg/authz/check.go:77-93,
    pkg/authz/postfilter.go:127-134). Concurrent zg_check_bulk calls must each get exactly
    their own answers, in order, while the batcher folds them into shared launches."""
    import threading

    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.001)
    e, o = zg.Engine(w.schema), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(e, zg.CHECK_DTYPE)
    want = o.check_bulk(items)
    errors = []

    def client(tid):
        rng = np.random.default_rng(tid)
        try:
            for _ in range(40):
                lo = int(rng.integers(0, items.size - 1))
                n = int(rng.integers(1, min(3000, items.size - lo)))  # 1-item and list-sized calls
                got = e.check_bulk(items[lo:lo + n])
                if not np.array_equal(got, want[lo:lo + n]):
                    errors.append((tid, lo, n))
        except Exception as ex:  # noqa: BLE001
            errors.append((tid, repr(ex)))

    before = e.stats()
    threads = [threading.Thread(target=client, args=(t,)) for t in range(24)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors[:3]
    st = e.stats()
    assert st["checks"] > before["checks"]
    # informational: how many calls shared a launch
    print("coalesced", st["coalesced_requests"], "calls into", st["coalesced_launches"], "launches")


@pytest.mark.parametrize("name,scale", [("cfg2", 0.02), ("cfg3", 0.01), ("cfg4", 0.002)])
def test_lookup_resources_reverse_bfs_equals_exhaustive_and_oracle(zg, name, scale, monkeypatch):
    """LookupResources = reverse-BFS candidates (a superset) verified by the check kernel.
    It must equal both the exhaustive scan of every resource of the type and the oracle's
    definition (pkg/authz/lookups.go:49-88 consumes it as a set)."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(name, scale)
    e = zg.Engine(w.schema)
    monkeypatch.setenv("ZGPU_NO_RBFS", "1")
    e_ex = zg.Engine(w.schema)
    monkeypatch.delenv("ZGPU_NO_RBFS")
    o = Oracle(w.schema)
    for t in (e, e_ex, o):
        w.load_into(t)
    e.publish(), e_ex.publish()
    rng = np.random.default_rng(11)
    rt, perm, st, _ = w.lookups[0]
    perms = [perm] + (["restricted_view", "edit"] if name == "cfg4" else [])
    n_users = max(g.subj.max() for g in w.groups if g.subj_type == st and not g.wildcard) + 1
    nonempty = 0
    for p in perms:
        for u in list(rng.integers(0, n_users, 12)) + [n_users + 5]:  # incl. a never-written subject
            a = e.lookup_resources_ids(rt, p, st, int(u))
            b = e_ex.lookup_resources_ids(rt, p, st, int(u))
            c = o.lookup_resources_ids(rt, p, st, int(u))
            assert np.array_equal(a, b) and np.array_equal(a, c), (name, p, u, a.size, b.size, c.size)
            nonempty += a.size > 0
    assert nonempty > 0
    if name == "cfg4":  # userset subject: group:g#member
        for g in rng.integers(0, 50, 4):
            a = e.lookup_resources_ids("document", "view", "group", int(g), srel="member")
            c = o.lookup_resources_ids("document", "view", "group", int(g), srel="member")
            assert np.array_equal(a, c)


def _layered_dag(layers, width, fan, seed):
    """group layers: every group of layer l includes `fan` random groups of layer l+1 (as
    group#member usersets); users sit in the last layer. Path multiplicity ~ fan**layers."""
    rng = np.random.default_rng(seed)
    par, chi = [], []
    for l in range(layers - 1):
        for g in range(width):
            for c in rng.choice(width, size=fan, replace=False):
                par.append(l * width + g)
                chi.append((l + 1) * width + int(c))
    last = (layers - 1) * width
    gm_g = np.repeat(np.arange(last, last + width), 2)
    gm_u = rng.integers(0, 64, gm_g.size)
    return np.array(par, np.uint32), np.array(chi, np.uint32), gm_g.astype(np.uint32), gm_u.astype(np.uint32)


NEST = "definition user {}\ndefinition group { relation member: user | group#member }\n"


def test_path_memo_keeps_dag_blowup_exact(zg, monkeypatch):
    """Cache-off forward evaluation multiplies work by the number of PATHS. With the memo
    switched on early the GPU must still equal the oracle bit for bit (moderate DAG the
    oracle can finish), i.e. skipping repeated (job, slot, object, depth) visits is exact."""
    from oracle.pyoracle import Oracle

    par, chi, gm_g, gm_u = _layered_dag(layers=7, width=8, fan=3, seed=1)  # ~3^6 = 729 paths / check
    monkeypatch.setenv("ZGPU_MEMO_AFTER", "4")
    e = zg.Engine(NEST)
    monkeypatch.delenv("ZGPU_MEMO_AFTER")
    e_plain, o = zg.Engine(NEST), Oracle(NEST)
    for t in (e, e_plain, o):
        t.add_bulk("group", "member", "group", par, chi, srel="member")
        t.add_bulk("group", "member", "user", gm_g, gm_u)
    e.publish(), e_plain.publish()
    items = np.zeros(8 * 80, dtype=zg.CHECK_DTYPE)
    items["res"] = np.repeat(np.arange(8), 80)  # top-layer groups
    items["subj"] = np.tile(np.arange(80), 8)   # users 64..79 are members of nothing
    items["perm"], items["stype"], items["srel"] = e.slot_id("group", "member"), e.type_id("user"), 0xFFFF
    want = o.check_bulk(items)
    assert np.array_equal(e.check_bulk(items), want)
    assert np.array_equal(e_plain.check_bulk(items), want)
    assert 0.05 < (want == 2).mean() < 0.999


def test_path_memo_bounds_work_on_deep_dags(zg):
    """3^14 = 4.8 M paths per check: far beyond what path enumeration finishes inside the work
    budget, but only 15 x 8 distinct (object, depth) nodes. Ground truth is plain
    reachability (numpy); the engine must answer every check, without budget errors."""
    L, Wd = 15, 8
    par, chi, gm_g, gm_u = _layered_dag(layers=L, width=Wd, fan=3, seed=2)
    e = zg.Engine(NEST)
    e.add_bulk("group", "member", "group", par, chi, srel="member")
    e.add_bulk("group", "member", "user", gm_g, gm_u)
    e.publish()
    n = L * Wd
    reach = np.zeros((n, 80), dtype=bool)
    reach[gm_g, gm_u] = True
    for l in range(L - 2, -1, -1):  # propagate memberships up the layers
        for p_, c_ in zip(par, chi):
            if p_ // Wd == l:
                reach[p_] |= reach[c_]
    items = np.zeros(Wd * 80, dtype=zg.CHECK_DTYPE)
    items["res"] = np.repeat(np.arange(Wd), 80)
    items["subj"] = np.tile(np.arange(80), Wd)
    items["perm"], items["stype"], items["srel"] = e.slot_id("group", "member"), e.type_id("user"), 0xFFFF
    got = e.check_bulk(items)
    want = np.where(reach[items["res"], items["subj"]], 2, 1)
    assert not (got == 255).any(), "work budget hit: the path memo did not bound the expansion"
    assert np.array_equal(got, want)


def test_subquery_buffer_overflow_splits_the_batch(zg):
    """Edges into non-pure permissions raise sub-queries; when a pass raises more than the
    buffer holds the batch is answered in halves (checks are independent) - same answers."""
    from oracle.pyoracle import Oracle

    rng = random.Random(77)
    schema = randgen.FIXED_SCHEMAS["deep_nonpure"]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=6, density=0.35)
    checks = randgen.random_checks(rng, model, 1500, n_obj=8, n_user=6)
    o = Oracle(schema)
    small, big = zg.Engine(schema, subquery_capacity=48), zg.Engine(schema)
    for r in rels:
        o.touch(r)
    for e in (small, big):
        ups = [(zg._lib.OP_TOUCH, r, 0) for r in rels]
        for i in range(0, len(ups), 1000):
            e.write_relationships(ups[i:i + 1000])
    want = np.array([o.check(*split_rel(q)) for q in checks], dtype=np.uint8)
    assert np.array_equal(big.check_bulk_str(checks), want)
    assert np.array_equal(small.check_bulk_str(checks), want)
    assert big.stats()["passes"] > 0, "this schema must exercise sub-query passes"


def test_many_direct_classes_and_flat_lookup(zg):
    """A subject type with more invertible classes than the per-check set tracks (12 > 11)
    falls back to forward probes; flat unions of direct relations answer LookupResources
    straight from the reverse rows. Both must equal the oracle."""
    from oracle.pyoracle import Oracle

    rels = [f"r{i}" for i in range(13)]
    schema = "definition user {}\ndefinition group { relation member: user | group#member }\ndefinition doc {\n" + \
        "".join(f"  relation {r}: user | user:*\n" for r in rels) + \
        "  relation g: group#member\n" + \
        "  permission any = " + " + ".join(rels) + "\n  permission deep = any + g\n}\n"
    rng = np.random.default_rng(3)
    e, o = zg.Engine(schema), Oracle(schema)
    for t in (e, o):
        for r in rels:
            n = 300
            t.add_bulk("doc", r, "user", rng.integers(0, 200, n), rng.integers(0, 50, n))
        t.add_bulk("doc", "r3", "user", [7, 9], [0, 0], wildcard=True)
        t.add_bulk("doc", "g", "group", rng.integers(0, 200, 100), rng.integers(0, 10, 100), srel="member")
        t.add_bulk("group", "member", "user", rng.integers(0, 10, 60), rng.integers(0, 50, 60))
        rng = np.random.default_rng(3)  # same data for the second target
    e.publish()
    items = np.zeros(4000, dtype=zg.CHECK_DTYPE)
    r2 = np.random.default_rng(4)
    items["res"], items["subj"] = r2.integers(0, 205, 4000), r2.integers(0, 55, 4000)
    items["stype"], items["srel"] = e.type_id("user"), 0xFFFF
    for perm in ("any", "deep", "r3"):
        items["perm"] = e.slot_id("doc", perm)
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items)), perm
        for u in (0, 1, 17, 49, 54, 10**6):
            assert np.array_equal(e.lookup_resources_ids("doc", perm, "user", u),
                                  o.lookup_resources_ids("doc", perm, "user", u)), (perm, u)


def test_gpu_snapshot_build_equals_host_build(zg, monkeypatch):
    """The CSR is built on the GPU (cub radix sorts + scans, csrc/build.cu). With
    ZGPU_VERIFY_BUILD=1 every publish also runs the host builder and compares row_ptr, col,
    exp, the reverse CSR, the per-type resource lists and the class-emptiness flags."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    monkeypatch.setenv("ZGPU_VERIFY_BUILD", "1")
    for w in (workloads.cfg2(scale=0.01, zipf=True), workloads.cfg3(scale=0.01), workloads.cfg4(scale=0.002)):
        e = zg.Engine(w.schema)
        w.load_into(e)
        g = w.groups[0]  # duplicates inside a bulk load must fold (TOUCH)
        e.add_bulk(g.res_type, g.rel, g.subj_type, g.res[:500], g.subj[:500], srel=g.srel, wildcard=g.wildcard)
        e.publish()  # raises if the GPU-built arrays differ from the host-built ones
        o = Oracle(w.schema)
        w.load_into(o)
        items = w.check_items(e, zg.CHECK_DTYPE)[:20000]
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items))
    # tombstones, expirations and empty stores through the write API
    C = zg.client
    cl = C.PermissionsClient(workloads.BOOTSTRAP_SCHEMA)
    up = lambda op, rel, exp=0: C.RelationshipUpdate(op, C.Relationship.parse(rel, exp))
    cl.engine.publish()  # empty store
    for i in range(30):
        cl.WriteRelationships(C.WriteRelationshipsRequest([
            up(C.OPERATION_TOUCH, f"namespace:n{i % 7}#viewer@user:u{i % 5}"),
            up(C.OPERATION_TOUCH, f"workflow:w{i % 3}#idempotency_key@activity:a{i % 4}", 4_000_000_000 + i)]))
        if i % 4 == 3:
            cl.WriteRelationships(C.WriteRelationshipsRequest([up(C.OPERATION_DELETE, f"namespace:n{i % 7}#viewer@user:u{i % 5}")]))
    assert len(list(cl.ReadRelationships(C.ReadRelationshipsRequest(C.RelationshipFilter("namespace"))))) > 0


def _items_from_strings(e, zg, checks):
    """Interned zg_check items for 'type:id#perm@stype:sid[#srel]' strings (no interning of new names)."""
    items = np.zeros(len(checks), dtype=zg.CHECK_DTYPE)
    for i, q in enumerate(checks):
        rt, rid, perm, st, sid, srel = split_rel(q)
        items["perm"][i] = e.slot_id(rt, perm)
        items["stype"][i] = e.type_id(st)
        items["srel"][i] = e.slot_id(st, srel) if srel else 0xFFFF
        r, u = e.find(rt, rid), e.find(st, sid)
        items["res"][i] = r
        items["subj"][i] = u if u != 0xFFFFFFFF else (0xFFFFFFFF if (r == 0xFFFFFFFF and rt == st and rid == sid) else 0xFFFFFFFE)
    return items


def test_interleaved_writes_and_checks_stay_consistent(zg):
    """FullyConsistent (every call site in the reference sets it: pkg/authz/check.go:42-44):
    after each WriteRelationships / DeleteRelationships returns, checks and lookups observe it.
    Random TOUCH / DELETE / delete-by-filter sequence on the engine and on the oracle in lockstep."""
    from oracle.pyoracle import Oracle

    schema = randgen.FIXED_SCHEMAS["docs"]
    model = randgen.model_from_schema(schema)
    rng = random.Random(4242)
    pool = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.6)
    checks = randgen.random_checks(rng, model, 120, n_obj=6, n_user=5)
    e, o = zg.Engine(schema), Oracle(schema)
    e.publish()
    live = set()
    for step in range(60):
        op = rng.random()
        if op < 0.6 or not live:
            batch = rng.sample(pool, rng.randint(1, 6))
            e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in batch])
            for r in batch:
                o.touch(r)
            live.update(batch)
        elif op < 0.9:
            batch = rng.sample(sorted(live), min(len(live), rng.randint(1, 4)))
            e.write_relationships([(zg._lib.OP_DELETE, r, 0) for r in batch])
            for r in batch:
                o.delete(r)
            live.difference_update(batch)
        else:  # delete by filter: every relationship of one resource
            rt, rid = split_rel(rng.choice(sorted(live)))[:2]
            n = e.delete_relationships({"res_type": rt, "res_id": rid})
            gone = {r for r in live if split_rel(r)[:2] == (rt, rid)}
            assert n == len(gone)
            for r in gone:
                o.delete(r)
            live -= gone
        assert sorted(e.read_relationships()) == sorted(live) == sorted(o.read())
        got = e.check_bulk_str(checks)
        want = [o.check(*split_rel(q)) for q in checks]
        assert list(got) == want, f"step {step}"
        u = f"u{rng.randint(0, 4)}"
        assert sorted(e.lookup_resources_str("document", "view", "user", u)) == sorted(o.lookup_resources("document", "view", "user", u))


def test_known_divergence_same_object_permission_hops_vs_the_depth_cap(zg):
    """FENCE for the one documented semantic divergence (DESIGN.md 2): a permission that refers to another
    permission of the SAME object is inlined here and costs no dispatch, while SpiceDB dispatches it. In
        reach = member + next->via ;  via = reach
    every link of a chain costs 1 hop here and 2 dispatches there. With the 50-dispatch cap
    (pkg/spicedb/spicedb.go:33):
        chain of <= 25 links : HAS here, HAS in SpiceDB                       (agree)
        26 .. 50 links       : HAS here, SpiceDB would report max depth       (MAY DIFFER: the fenced band)
        >= 51 links          : ERROR here, error in SpiceDB                   (agree)
    Outside that band -- and for every schema without same-object permission references, which includes all
    BASELINE configurations -- hop counting is identical. The oracle counts like the engine (it is the checker of
    the engine, not of this divergence)."""
    from oracle.pyoracle import Oracle

    schema = ("definition user {}\ndefinition node {\n  relation next: node\n  relation member: user\n"
              "  permission reach = member + next->via\n  permission via = reach\n}\n")
    e, o = zg.Engine(schema), Oracle(schema)
    n = 60
    for t in (e, o):
        t.add_bulk("node", "next", "node", np.arange(n - 1, dtype=np.uint32), np.arange(1, n, dtype=np.uint32))
        t.add_bulk("node", "member", "user", np.array([n - 1], np.uint32), np.array([7], np.uint32))
    e.publish()
    items = np.zeros(n, dtype=zg.CHECK_DTYPE)
    items["res"] = np.arange(n)
    items["subj"] = 7
    items["perm"], items["stype"], items["srel"] = e.slot_id("node", "reach"), e.type_id("user"), 0xFFFF
    got = e.check_bulk(items)
    links = (n - 1) - np.arange(n)  # arrows between the checked node and the member's node
    assert np.array_equal(got, o.check_bulk(items))
    assert (got[links <= 50] == 2).all() and (got[links >= 51] == 255).all()
    band = (links >= 26) & (links <= 50)
    assert band.sum() == 25 and (got[band] == 2).all()  # the answers SpiceDB may replace by a depth error


def _random_updates(zg, e, w, rng, n, new_objects=True):
    """n interned updates against workload w: deletes and touches of loaded relationships, inserts between
    existing objects, and (new_objects) inserts on objects the store has never seen."""
    ups = np.zeros(n, dtype=zg.UPDATE_DTYPE)
    for i in range(n):
        g = w.groups[rng.integers(0, len(w.groups))]
        k = rng.integers(0, g.res.size)
        kind = rng.random()
        ups["rel"][i] = e.slot_id(g.res_type, g.rel)
        ups["stype"][i] = e.type_id(g.subj_type)
        ups["srel"][i] = 0xFFFE if g.wildcard else (0xFFFF if g.srel is None else e.slot_id(g.subj_type, g.srel))
        ups["res"][i], ups["subj"][i] = g.res[k], 0 if g.wildcard else g.subj[k]
        if kind < 0.35:
            ups["op"][i] = 2  # DELETE (maybe already deleted by an earlier batch: a no-op then)
        elif kind < 0.45:
            ups["op"][i] = 0  # TOUCH of an existing relationship
        else:
            ups["op"][i] = 0  # TOUCH of a new pairing
            ups["res"][i] = g.res[rng.integers(0, g.res.size)]
            if new_objects and kind > 0.85:
                ups["res"][i] = int(g.res.max()) + 1 + rng.integers(0, 50)
            if not g.wildcard:
                ups["subj"][i] = g.subj[rng.integers(0, g.subj.size)]
    # one update per relationship in a batch (as WriteRelationships requires)
    key = np.stack([ups["rel"], ups["res"], ups["stype"], ups["srel"], ups["subj"]], axis=1)
    _, first = np.unique(key, axis=0, return_index=True)
    return ups[np.sort(first)]


def test_incremental_publish_equals_rebuild_and_oracle(zg, monkeypatch):
    """A write does not rebuild the snapshot: its updates are merged into the resident CSR on the device
    (csrc/build.cu gpu_apply_delta). With ZGPU_VERIFY_BUILD=1 every array after every merge is compared with the host
    builder's; answers are compared with the oracle, which applies the same updates."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    monkeypatch.setenv("ZGPU_VERIFY_BUILD", "1")
    rng = np.random.default_rng(7)
    for w in (workloads.cfg4(scale=0.002), workloads.cfg3(scale=0.01)):
        e, o = zg.Engine(w.schema), Oracle(w.schema)
        w.load_into(e), w.load_into(o)
        e.publish()
        items = w.check_items(e, zg.CHECK_DTYPE)[:8000]
        for step in range(6):
            ups = _random_updates(zg, e, w, rng, [3, 40, 400, 1000, 1, 1000][step])
            e.apply_updates(ups)
            e.publish()  # raises if a merged array differs from the rebuilt one
            o.apply_updates(ups)
            # checks on touched objects and on the standing batch
            probe = items.copy()
            probe["res"][: ups.size] = ups["res"][: probe.size][: ups.size] if w.name == "cfg3" else probe["res"][: ups.size]
            assert np.array_equal(e.check_bulk(probe), o.check_bulk(probe)), f"{w.name} step {step}"
        st = e.stats()
        assert st["delta_publishes"] >= 5, st  # a batch that outgrows an object capacity may rebuild
        e.close()


@pytest.mark.parametrize("cap", [0, 4096])
def test_concurrent_lookups_share_launches_and_equal_the_oracle(zg, monkeypatch, cap):
    """One LookupResources per list request, concurrently (pkg/authz/responsefilterer.go:165): queued lookups are
    answered K at a time by one multi-source reverse walk + one verification launch. Every answer equals the
    oracle's; with a tiny batch buffer (cap=4096) the batch overflows and is answered in halves, same answers."""
    import threading

    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    if cap:
        monkeypatch.setenv("ZGPU_LOOKUP_BATCH_CAP", str(cap))
    w = workloads.cfg4(scale=0.003)
    e, o = zg.Engine(w.schema), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    rng = np.random.default_rng(5)
    n_users = int(max(g.subj.max() for g in w.groups if g.subj_type == "user" and not g.wildcard)) + 1
    users = rng.integers(0, n_users, 96)
    perms = ["view" if i % 3 else "restricted_view" for i in range(users.size)]
    want = [o.lookup_resources_ids("document", p, "user", int(u)) for u, p in zip(users, perms)]
    got = [None] * users.size
    errs = []

    def run(lo, hi):
        try:
            for i in range(lo, hi):
                got[i] = e.lookup_resources_ids("document", perms[i], "user", int(users[i]))
        except Exception as ex:  # noqa: BLE001
            errs.append(ex)

    ths = [threading.Thread(target=run, args=(i, i + 3)) for i in range(0, users.size, 3)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    assert not errs, errs
    for i in range(users.size):
        assert np.array_equal(got[i], want[i]), f"lookup {i}: {got[i].size} ids vs {want[i].size}"
    st = e.stats()
    assert st["lookups_batched"] > 0 and st["lookup_batches"] < st["lookups_batched"], st
    assert sum(x.size for x in want) > 1000
    e.close()


def test_one_engine_owning_several_gpus_equals_a_single_gpu_engine(zg):
    """zg_config.n_devices: ONE handle, every device holds a replica and answers its slice of each bulk call
    (the proxy keeps a single client: pkg/proxy/options.go:81-82). Needs >= 2 GPUs."""
    import threading

    import torch

    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    n_dev = torch.cuda.device_count()
    if n_dev < 2:
        pytest.skip("needs >= 2 GPUs")
    w = workloads.cfg4(scale=0.005)
    multi, o = zg.Engine(w.schema, device=0, n_devices=n_dev), Oracle(w.schema)
    w.load_into(multi), w.load_into(o)
    multi.publish()
    assert multi.stats()["devices"] == n_dev
    items = w.check_items(multi, zg.CHECK_DTYPE)
    want = o.check_bulk(items)
    assert np.array_equal(multi.check_bulk(items), want)
    # a write reaches every replica before it returns
    doc, user = int(items["res"][0]), 123
    rel = zg.UPDATE_DTYPE
    up = np.zeros(1, dtype=rel)
    up["res"], up["subj"], up["rel"], up["stype"], up["srel"], up["op"] = doc, user, multi.slot_id("document", "banned"), \
        multi.type_id("user"), 0xFFFF, 0
    multi.apply_updates(up), multi.publish()
    o.write_ids(0, up["rel"][0], doc, up["stype"][0], user)
    probe = np.repeat(items[:1], 20000)
    probe["subj"] = user
    assert np.array_equal(multi.check_bulk(probe), o.check_bulk(probe))
    # concurrent small callers and concurrent lookups are spread over the devices
    got = [None] * 16
    def run(i):
        got[i] = multi.check_bulk(items[i * 5000:(i + 1) * 5000])
    ths = [threading.Thread(target=run, args=(i,)) for i in range(16)]
    [t.start() for t in ths], [t.join() for t in ths]
    for i in range(16):
        assert np.array_equal(got[i], o.check_bulk(items[i * 5000:(i + 1) * 5000]))
    rt, perm, st, u = w.lookups[0]
    lk = [None] * 8
    def look(i):
        lk[i] = multi.lookup_resources_ids(rt, perm, st, int(u) + i)
    ths = [threading.Thread(target=look, args=(i,)) for i in range(8)]
    [t.start() for t in ths], [t.join() for t in ths]
    for i in range(8):
        assert np.array_equal(lk[i], o.lookup_resources_ids(rt, perm, st, int(u) + i))
    multi.close()


def _run_sharded_device(zg, schema, load, items, world=3):
    """The device-resident protocol (dist.DeviceShardedChecker) on `world` virtual shards of this one GPU: every
    rank brings a slice of the batch as a CUDA tensor and gets that slice's answers back. Returns the answers, the
    relationships held over all shards and rank 0's checker stats."""
    import threading

    import torch

    from spicedb_kubeapi_proxy_b200 import dist as zdist

    ts = zdist.LocalDeviceTransport.cluster(world)
    engines = [zg.Engine(schema, shard_rank=r, shard_count=world) for r in range(world)]
    for e in engines:
        load(e)
        e.publish()
    bounds = [zdist.shard_bounds(items.size, r, world) for r in range(world)]
    out, errs, checkers = [None] * world, [], [None] * world

    def run(r):
        try:
            lo, hi = bounds[r]
            mine = np.ascontiguousarray(items[lo:hi])
            d = torch.from_numpy(mine.view(np.uint8).copy()).cuda()
            ck = zdist.DeviceShardedChecker(engines[r], ts[r])
            checkers[r] = ck
            out[r] = ck.check_bulk(d, hi - lo).cpu().numpy()
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))
            ts[r]._s["bar"].abort()

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errs, errs
    return np.concatenate(out), sum(e.num_tuples() for e in engines), checkers[0].stats


@pytest.mark.parametrize("name,scale", [("cfg3", 0.005), ("cfg4", 0.001)])
def test_device_resident_sharded_store_equals_oracle_on_workloads(zg, name, scale):
    """Object-hash sharded store (north-star's multi-GPU mode): relationships are split by
    resource id % 3 over three engines, sub-queries cross shards between passes, and the answers
    equal the oracle's on the whole store."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(name, scale)
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(o, zg.CHECK_DTYPE)[:6000]
    got, total, stats = _run_sharded_device(zg, w.schema, w.load_into, items)
    assert np.array_equal(got, o.check_bulk(items))
    assert total == o_num_unique(w), "every relationship lives on exactly one shard"
    assert stats["subqueries_sent"] > 0 and stats["levels"] >= 2


@pytest.mark.parametrize("seed", range(6))
def test_device_resident_sharded_store_random_schemas(zg, seed):
    """& / - / arrows / usersets / wildcards across shards, incl. the depth cap and cycles."""
    from oracle.pyoracle import Oracle

    rng = random.Random(900 + seed)
    if seed < 3:
        schema = randgen.FIXED_SCHEMAS[sorted(randgen.FIXED_SCHEMAS)[seed]]
        model = randgen.model_from_schema(schema)
    else:
        schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=7, n_user=6, density=0.3)
    checks = randgen.random_checks(rng, model, 500, n_obj=7, n_user=6)
    o = Oracle(schema)
    for r in rels:
        o.touch(r)

    def load(e):
        ups = [(zg._lib.OP_TOUCH, r, 0) for r in rels]
        for i in range(0, len(ups), 1000):
            e.write_relationships(ups[i:i + 1000])

    probe = zg.Engine(schema, host_only=True)
    load(probe)
    items = _items_from_strings(probe, zg, checks)
    got, _, _ = _run_sharded_device(zg, schema, load, items)
    want = np.array([o.check(*split_rel(q)) for q in checks], dtype=np.uint8)
    bad = [(q, int(g), int(x)) for q, g, x in zip(checks, got, want) if g != x]
    assert not bad, bad[:5]


def test_device_resident_sharded_store_depth_cap_across_shards(zg):
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

    def load(e):
        e.write_relationships([(zg._lib.OP_TOUCH, r, 0) for r in rels])

    probe = zg.Engine(CHAIN, host_only=True)
    load(probe)
    items = _items_from_strings(probe, zg, checks)
    got, _, stats = _run_sharded_device(zg, CHAIN, load, items)
    assert list(got) == [o.check(*split_rel(q)) for q in checks]
    assert list(got[:5]) == [255, 2, 1, 2, 255]
    assert stats["levels"] > 20, "the 51-hop chain must cross shards level by level"
