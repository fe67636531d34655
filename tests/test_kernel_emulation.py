"""The product's CUDA kernel source (spicedb-kubeapi-proxy_b200/csrc/kernels.cuh) executed on the CPU by a SIMT emulator
(tests/emu/: every CUDA thread an OS thread, every warp collective a rendezvous) and compared with the oracle.

What this is: a CPU-side check of the kernel's LOGIC -- admission, leaf loop with Kleene short circuit, meet in the
middle (one and two levels), spills, path memo, sub-query passes and folds, batched LookupResources -- available without
a GPU, so a kernel change is exercised before it runs on a GPU. What it is not: a product path (the emulator lives under
tests/, libzgpu.so has no CPU evaluation), a performance statement, or a substitute for the -m gpu parity tests, which
run the same source on the GPU through the C ABI."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import randgen  # noqa: E402
from golden_runner import split_rel  # noqa: E402


@pytest.fixture(scope="module")
def emu():
    import emu as E

    E.lib()
    return E


def _compare_strings(emu, schema, rels, checks, opts=None, now=0, expires=None):
    from oracle.pyoracle import Oracle

    e, o = emu.EmuEngine(schema), Oracle(schema)
    exp = expires or {}
    for r in rels:
        o.touch(r, exp.get(r, 0))
    e.write_rels(rels, split_rel)
    if exp:  # second load with the expirations (TOUCH: last wins)
        t = [r for r in rels if r in exp]
        items = e.items_from_strings([x.replace("#", "#", 1) for x in t], split_rel)  # only to intern nothing new
        del items
        tt = np.zeros(len(t), dtype=emu.TUPLE_DTYPE)
        ex = np.zeros(len(t), dtype=np.uint32)
        for i, r in enumerate(t):
            rt, rid, rel, st, sid, srel = split_rel(r)
            tt["rel"][i], tt["stype"][i] = e.slot_id(rt, rel), e.type_id(st)
            tt["res"][i] = e._id(rt, rid, True)
            tt["srel"][i] = 0xFFFE if sid == "*" else (e.slot_id(st, srel) if srel else 0xFFFF)
            tt["subj"][i] = 0 if sid == "*" else e._id(st, sid, True)
            ex[i] = exp[r]
        e.load_tuples(tt, ex)
    e.publish()
    ok_checks = [q for q in checks if e.type_id(split_rel(q)[0]) >= 0 and e.type_id(split_rel(q)[3]) >= 0]
    items = e.items_from_strings(ok_checks, split_rel)
    o_ = opts or emu.default_opts()
    o_.now = now
    got = e.check_bulk(items, o_)
    want = np.array([o.check(*split_rel(q), now) for q in ok_checks], dtype=np.uint8)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{[ok_checks[i] for i in bad[:5]]}: emu={got[bad[:5]]} oracle={want[bad[:5]]}\n{schema}"
    return e, o


@pytest.mark.parametrize("name", sorted(randgen.FIXED_SCHEMAS))
def test_fixed_schemas_random_graphs_under_the_emulator(emu, name):
    rng = random.Random(500)
    schema = randgen.FIXED_SCHEMAS[name]
    model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=7, n_user=6, density=0.3)
    checks = randgen.random_checks(rng, model, 400, n_obj=7, n_user=6)
    _compare_strings(emu, schema, rels, checks)


@pytest.mark.parametrize("seed", range(12))
def test_random_schemas_under_the_emulator(emu, seed):
    rng = random.Random(seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=6, n_user=5, density=0.35)
    checks = randgen.random_checks(rng, model, 300, n_obj=6, n_user=5)
    # alternate the variants: forward only, tiny sub-query buffer (split), memo from the first round, streamed admission
    opts = [emu.default_opts(), emu.default_opts(invert=0), emu.default_opts(subq_cap=24), emu.default_opts(memo_after=0),
            emu.default_opts(streamed=1), emu.default_opts(grid=1, spill_cap=64)][seed % 6]
    _compare_strings(emu, schema, rels, checks, opts)


def test_depth_cap_cycles_and_error_propagation_under_the_emulator(emu):
    from test_oracle_random import CHAIN

    rels = [f"group:g{i}#member@group:g{i+1}#member" for i in range(51)] + ["group:g51#member@user:deep"]
    rels += ["group:a#member@group:b#member", "group:b#member@group:a#member", "group:b#member@user:x"]
    rels += [f"folder:f{i}#parent@folder:f{i+1}" for i in range(51)] + ["folder:f0#viewer@user:v"]
    checks = ["group:g0#member@user:deep", "group:g1#member@user:deep", "group:g2#member@user:nobody",
              "group:a#member@user:x", "group:a#member@user:y", "folder:f0#view@user:v", "folder:f0#view@user:w",
              "folder:f0#not_view@user:v", "folder:f0#not_view@user:w", "folder:f1#view@user:v", "folder:f40#view@user:v"]
    for o in (emu.default_opts(), emu.default_opts(invert=0)):
        e, _ = _compare_strings(emu, CHAIN, rels, checks, o)
        assert list(e.check_bulk(e.items_from_strings(checks[:5], split_rel), o)) == [255, 2, 1, 2, 255]


def test_expiration_wildcards_userset_subjects_under_the_emulator(emu):
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
              "doc:d3#nope@user:e1", "doc:d3#view@user:e1#member"]
    for now in (999, 1000, 1999, 2001):
        _compare_strings(emu, schema, rels, checks, now=now, expires=expires)


def test_two_level_meet_over_every_range_size_and_membership_count_under_the_emulator(emu):
    """The two-level meet (batch_l2) answers ranges of <= 64 children against a 128-bit filter of each: ranges of
    1 .. 70 children (beyond 64: the walk takes over), subjects with 1 .. 17 memberships (beyond 16: the per-check set
    overflows and the meet reads them from the subject's reverse row), hits on the first / last child, near misses
    (filter false positives must die in the search)."""
    schema = """definition user {}
definition group { relation member: user }
definition team { relation member: group#member }
definition namespace { relation viewer: team#member  permission view = viewer }"""
    rng = np.random.default_rng(11)
    rels, checks = [], []
    n_teams = 400
    for g in range(300):  # every group sits in 1 .. 12 teams
        for t in rng.choice(n_teams, 1 + g % 12, replace=False):
            rels.append(f"team:t{t}#member@group:g{g}#member")
    sizes = [1, 2, 3, 15, 16, 17, 31, 32, 33, 63, 64, 65, 70]
    for i, nf in enumerate(sizes):
        for t in rng.choice(n_teams, nf, replace=False):
            rels.append(f"namespace:n{i}#viewer@team:t{t}#member")
    for u in range(1, 18):  # user u<k> is a member of k groups
        for g in rng.choice(300, u, replace=False):
            rels.append(f"group:g{g}#member@user:u{u}")
    for i in range(len(sizes)):
        for u in range(1, 18):
            checks.append(f"namespace:n{i}#view@user:u{u}")
    e, o = _compare_strings(emu, schema, rels, checks)
    got = e.check_bulk(e.items_from_strings(checks, split_rel))
    assert 0.1 < (got == 2).mean() < 0.9  # both answers occur


@pytest.mark.parametrize("wl,scale,n", [("cfg2", 0.01, 2000), ("cfg3", 0.003, 3000), ("cfg4", 0.001, 3000)])
def test_baseline_workloads_scaled_under_the_emulator(emu, wl, scale, n):
    """The BASELINE shapes (scaled): cfg3 resolves every namespace -> team -> group range by the two-level meet in the
    middle (far fewer bytes than forward probing, same answers), cfg4 runs its 2-3 leaves per check in one pass with
    the boolean short circuit."""
    import zgpu  # noqa: F401  (registers the package: the workload generators live in it; libzgpu.so is not used)
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    e, o = emu.EmuEngine(w.schema), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(o, emu.CHECK_DTYPE)[:n]
    want = o.check_bulk(items)
    assert np.array_equal(e.check_bulk(items), want)
    assert np.array_equal(e.check_bulk(items, emu.default_opts(invert=0)), want)
    assert np.array_equal(e.check_bulk(items, emu.default_opts(memo_after=0, grid=1)), want)
    assert np.array_equal(e.check_bulk(items, emu.default_opts(streamed=1)), want)
    e2 = emu.EmuEngine(w.schema)
    w.load_into(e2), e2.publish()
    e2.check_bulk(items, count=True)
    inv_bytes = e2.stat("alg_bytes")
    e3 = emu.EmuEngine(w.schema)
    w.load_into(e3), e3.publish()
    e3.check_bulk(items, emu.default_opts(invert=0), count=True)
    fwd_bytes = e3.stat("alg_bytes")
    if wl == "cfg3":
        assert inv_bytes * 2 < fwd_bytes, (inv_bytes, fwd_bytes)  # the meet in the middle is doing the work (fan-outs shrink with scale)
    assert 0.05 < (want == 2).mean() < 0.95


def test_subquery_passes_split_and_fold_under_the_emulator(emu):
    """cfg4 with a non-pure folder#view: sub-queries level after level up the folder chain; a pass buffer smaller than
    one batch's sub-queries forces the batch to be answered in halves."""
    import zgpu  # noqa: F401
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.001, nonpure_folders=True)
    e, o = emu.EmuEngine(w.schema), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(o, emu.CHECK_DTYPE)[:2500]
    want = o.check_bulk(items)
    assert np.array_equal(e.check_bulk(items), want)
    assert e.stat("passes") >= 2
    assert np.array_equal(e.check_bulk(items, emu.default_opts(subq_cap=300)), want)
    assert e.stat("splits") > 0


def test_batched_lookup_resources_under_the_emulator(emu):
    """K lookups in one multi-source reverse walk + one verification pass + one sort == the oracle's LookupResources."""
    import zgpu  # noqa: F401
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    for w in (workloads.cfg4(scale=0.001), workloads.cfg3(scale=0.003)):
        e, o = emu.EmuEngine(w.schema), Oracle(w.schema)
        w.load_into(e), w.load_into(o)
        e.publish()
        rt, perm, st, _ = w.lookups[0]
        rng = np.random.default_rng(3)
        n_users = int(max(g.subj.max() for g in w.groups if g.subj_type == st and not g.wildcard)) + 1
        users = [int(u) for u in rng.integers(0, n_users, 24)]
        perms = [perm] * 24
        if w.name == "cfg4":
            perms = [perm if i % 2 else "restricted_view" for i in range(24)]
        reqs = [(e.type_id(rt), e.slot_id(rt, p), e.type_id(st), u, 0xFFFF) for u, p in zip(users, perms)]
        got = e.lookup_batch(reqs)
        total = 0
        for u, p, g in zip(users, perms, got):
            want = o.lookup_resources_ids(rt, p, st, u)
            assert g is not None and np.array_equal(g, want), f"{w.name} {p} user {u}: {g.size if g is not None else None} vs {want.size}"
            total += want.size
        assert total > 50


def test_warp_stack_spills_to_its_overflow_area_under_the_emulator(emu):
    """More than 64 pending edge ranges per warp: 32 checks x 6 userset relations x nested groups. The stack spills
    halves to the per-warp overflow area and refills; answers unchanged; a too small overflow area reports the
    overflow flag (the host call fails with ZG_ENOMEM) instead of corrupting anything."""
    from oracle.pyoracle import Oracle

    rels_decl = "".join(f"  relation r{i}: group#member\n" for i in range(6))
    schema = ("definition user {}\ndefinition group { relation member: user | group#member }\ndefinition doc {\n" + rels_decl +
              "  permission view = " + " + ".join(f"r{i}" for i in range(6)) + "\n}\n")
    rng = np.random.default_rng(9)
    e, o = emu.EmuEngine(schema), Oracle(schema)
    n_doc, n_grp, n_user = 64, 200, 300
    for t in (e, o):
        r = np.random.default_rng(9)
        for i in range(6):
            t.add_bulk("doc", f"r{i}", "group", r.integers(0, n_doc, 400), r.integers(100, n_grp, 400), srel="member")
        # groups 100.. nest groups 0..99 (acyclic), which hold the users
        t.add_bulk("group", "member", "group", r.integers(100, n_grp, 600), r.integers(0, 100, 600), srel="member")
        t.add_bulk("group", "member", "user", r.integers(0, 100, 500), r.integers(0, n_user, 500))
    e.publish()
    items = np.zeros(2000, dtype=emu.CHECK_DTYPE)
    items["res"] = rng.integers(0, n_doc, 2000)
    items["subj"] = rng.integers(0, n_user, 2000)
    items["perm"], items["stype"], items["srel"] = e.slot_id("doc", "view"), e.type_id("user"), 0xFFFF
    want = o.check_bulk(items)
    for opts in (emu.default_opts(invert=0), emu.default_opts()):
        assert np.array_equal(e.check_bulk(items, opts), want)
    assert e.stat("spills") > 0
    e.check_bulk(items, emu.default_opts(invert=0, spill_cap=32))
    assert e.stat("flags") & 1  # overflow of the overflow area is reported, not ignored
    assert 0.05 < (want == 2).mean() < 0.95


def _random_updates(E, e, w, rng, n, new_objects=True):
    """n interned updates against workload w: deletes and touches of loaded relationships, inserts between existing
    objects, and (new_objects) inserts on objects the store has never seen. One update per relationship."""
    ups = np.zeros(n, dtype=E.UPDATE_DTYPE)
    for i in range(n):
        g = w.groups[rng.integers(0, len(w.groups))]
        k = rng.integers(0, g.res.size)
        kind = rng.random()
        ups["rel"][i] = e.slot_id(g.res_type, g.rel)
        ups["stype"][i] = e.type_id(g.subj_type)
        ups["srel"][i] = 0xFFFE if g.wildcard else (0xFFFF if g.srel is None else e.slot_id(g.subj_type, g.srel))
        ups["res"][i], ups["subj"][i] = g.res[k], 0 if g.wildcard else g.subj[k]
        if kind < 0.35:
            ups["op"][i] = 2
        elif kind >= 0.45:
            ups["res"][i] = g.res[rng.integers(0, g.res.size)]
            if new_objects and kind > 0.85:
                ups["res"][i] = int(g.res.max()) + 1 + rng.integers(0, 50)
            if not g.wildcard:
                ups["subj"][i] = g.subj[rng.integers(0, g.subj.size)]
    key = np.stack([ups["rel"], ups["res"], ups["stype"], ups["srel"], ups["subj"]], axis=1)
    _, first = np.unique(key, axis=0, return_index=True)
    return ups[np.sort(first)]


@pytest.mark.parametrize("wl,scale", [("cfg4", 0.001), ("cfg3", 0.004)])
def test_incremental_publish_kernels_equal_a_rebuild_under_the_emulator(emu, wl, scale):
    """csrc/delta.cuh: locate the delta in the old arrays, re-emit the edge arrays in one pass (constant-shift tiles),
    add the running insert/delete counts to the row tables in place -- forward and reverse. After every merge every
    array equals a fresh host build of the store, and the checks equal the oracle's (which applies the same updates)."""
    import zgpu  # noqa: F401
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    e, o = emu.EmuEngine(w.schema), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    rng = np.random.default_rng(21)
    items = w.check_items(o, emu.CHECK_DTYPE)[:1500]
    merged = 0
    for step, n in enumerate([1, 3, 40, 400, 1000, 7]):
        ups = _random_updates(emu, e, w, rng, n, new_objects=step % 2 == 1)
        e.apply_updates(ups)
        merged += e.merge_and_verify() == 0
        o.apply_updates(ups)
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items)), f"{wl} step {step}"
    assert merged >= 4


def test_incremental_publish_with_expirations_and_empty_classes_under_the_emulator(emu):
    """TOUCH of an existing relationship only changes its expiration (patched in place); a class that receives its
    first relationship, or loses its last one, changes the program's steps."""
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    schema = workloads.BOOTSTRAP_SCHEMA
    e, o = emu.EmuEngine(schema), Oracle(schema)
    e.publish()  # empty store
    U = emu.UPDATE_DTYPE

    def up(op, rt, rel, res, st, subj, exp=0):
        u = np.zeros(1, dtype=U)
        u["op"], u["rel"], u["res"], u["stype"], u["subj"], u["srel"], u["expires_at"] = op, e.slot_id(rt, rel), res, e.type_id(st), subj, 0xFFFF, exp
        return u

    script = [up(0, "namespace", "viewer", 3, "user", 1), up(0, "workflow", "idempotency_key", 2, "activity", 5, 1000),
              up(0, "workflow", "idempotency_key", 2, "activity", 5, 2000),  # expiration only
              up(0, "namespace", "creator", 3, "user", 2), up(2, "namespace", "viewer", 3, "user", 1),
              up(2, "namespace", "creator", 3, "user", 2), up(0, "namespace", "viewer", 4000, "user", 7)]
    items = np.zeros(4, dtype=emu.CHECK_DTYPE)
    items["res"], items["subj"] = [3, 3, 4000, 3], [1, 2, 7, 9]
    items["perm"], items["stype"], items["srel"] = e.slot_id("namespace", "view"), e.type_id("user"), 0xFFFF
    for i, u in enumerate(script):
        e.apply_updates(u)
        e.merge_and_verify()
        o.write_ids(int(u["op"][0]), int(u["rel"][0]), int(u["res"][0]), int(u["stype"][0]), int(u["subj"][0]), 0xFFFF, int(u["expires_at"][0]))
        for now in (500, 1500):
            opts = emu.default_opts(now=now)
            assert np.array_equal(e.check_bulk(items, opts), o.check_bulk(items, now=now)), f"step {i} now {now}"


def _run_sharded_emulated(emu, schema, load, items, world=3):
    """dist.DeviceShardedChecker -- the product's own protocol driver -- over `world` emulated shards: CPU tensors
    change hands by reference, the kernels (raise of remote edges, routing, fold in routed order) run emulated."""
    import threading

    import torch

    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200 import dist as zdist

    cpu = torch.device("cpu")
    ts = zdist.LocalDeviceTransport.cluster(world, device=cpu)
    engines = [emu.EmuEngine(schema, shard_rank=r, shard_count=world) for r in range(world)]
    for e in engines:
        load(e)
        e.publish()
    bounds = [zdist.shard_bounds(items.size, r, world) for r in range(world)]
    out, errs, cks = [None] * world, [], [None] * world

    def run(r):
        try:
            lo, hi = bounds[r]
            d = torch.from_numpy(np.ascontiguousarray(items[lo:hi]).view(np.uint8).copy())
            cks[r] = zdist.DeviceShardedChecker(engines[r], ts[r])
            out[r] = cks[r].check_bulk(d, hi - lo).numpy().copy()
        except Exception as ex:  # noqa: BLE001
            import traceback

            errs.append(traceback.format_exc())
            ts[r]._s["bar"].abort()

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert not errs, errs[0]
    return np.concatenate(out), cks[0].stats


@pytest.mark.parametrize("wl,scale,n", [("cfg4", 0.001, 1500), ("cfg3", 0.002, 600)])
def test_device_resident_sharded_protocol_under_the_emulator(emu, wl, scale, n):
    import zgpu  # noqa: F401
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(wl, scale)
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(o, emu.CHECK_DTYPE)[:n]
    got, stats = _run_sharded_emulated(emu, w.schema, w.load_into, items)
    assert np.array_equal(got, o.check_bulk(items))
    assert stats["subqueries_sent"] > 0 and stats["levels"] >= 2


def test_sharded_protocol_with_boolean_operators_and_depth_cap_under_the_emulator(emu):
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
    probe = emu.EmuEngine(CHAIN)
    probe.write_rels(rels, split_rel)
    names = dict(probe._names)

    def load(e):
        e._names = dict(names)  # the same interning on every shard
        e.write_rels(rels, split_rel)

    items = probe.items_from_strings(checks, split_rel)
    got, stats = _run_sharded_emulated(emu, CHAIN, load, items)
    assert list(got) == [o.check(*split_rel(q)) for q in checks]
    assert list(got[:5]) == [255, 2, 1, 2, 255]
    assert stats["levels"] > 20
