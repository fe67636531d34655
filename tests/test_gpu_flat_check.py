"""The lean flat-check kernel (csrc/kernels.cuh flat_check_kernel) on the GPU: a permission whose checks are direct
probes and two-level meets over set-tabled closure indexes (SF_FLAT) is answered one check per thread, and every other
item by check_kernel through the residual list. Answers against the oracle and against engines with the lean kernel off
(ZGPU_FLAT_CHECK=0), on cfg3, generated schemas, a multi-pass program, and after writes; and the configurations that
must leave no slot flat."""
import random

import numpy as np
import pytest

import randgen as R

pytestmark = pytest.mark.gpu


def _engine(schema, load, monkeypatch, **env):
    import zgpu

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    e = zgpu.Engine(schema, device=0)
    load(e), e.publish()
    for k in env:
        monkeypatch.delenv(k, raising=False)
    return e


def _device(e, items):
    import torch

    import zgpu

    d_items = torch.from_numpy(np.ascontiguousarray(items, dtype=zgpu.CHECK_DTYPE).view(np.uint8).copy()).cuda()
    d_out = torch.zeros(items.size, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    e.check_bulk_device(d_items.data_ptr(), items.size, d_out.data_ptr(), s.cuda_stream)
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


@pytest.mark.parametrize("scale", [0.1, 1.0])
def test_cfg3_against_the_oracle_and_the_generic_kernel(scale, monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3(scale=scale)
    e = _engine(w.schema, w.load_into, monkeypatch)
    st = e.stats()
    assert st["flat_slots"] >= 1, st
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    r0 = e.stats()["flat_residual"]
    got = e.check_bulk(items)
    assert e.stats()["flat_residual"] == r0  # every cfg3 check is answered by the lean kernel
    assert np.array_equal(got, _device(e, items))
    alg = e.count_alg_bytes(items)
    del e
    f = _engine(w.schema, w.load_into, monkeypatch, ZGPU_FLAT_CHECK="0")
    assert f.stats()["flat_slots"] == 0
    assert np.array_equal(got, f.check_bulk(items))
    assert alg == f.count_alg_bytes(items)  # the byte model of the generic kernel
    del f
    o = Oracle(w.schema)
    w.load_into(o)
    assert np.array_equal(got, o.check_bulk(items))


@pytest.mark.parametrize("env", [{"ZGPU_CLOSURE_CAP": "0"}, {"ZGPU_CLOSURE_TABLE": "0"}, {"ZGPU_NO_INVERT": "1"},
                                 {"ZGPU_FLAT_CHECK": "0"}])
def test_configurations_without_flat_slots(env, monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3(scale=0.02)
    e = _engine(w.schema, w.load_into, monkeypatch, **env)
    assert e.stats()["flat_slots"] == 0, env
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    o = Oracle(w.schema)
    w.load_into(o)
    assert np.array_equal(e.check_bulk(items), o.check_bulk(items))


@pytest.mark.parametrize("seed,wide", [(0, False), (1, False), (2, False), (3, True), (4, False), (9, True)])
def test_shaped_schemas(seed, wide, monkeypatch):
    """Generated schemas with probes (expiring direct subjects, wildcards) next to the meets: answers at two clocks equal
    the oracle's and the generic kernel's, from the host and the device entry points; 32-bit pairs have no set table and
    leave no slot flat."""
    import zgpu
    from oracle.pyoracle import Oracle

    rng = random.Random(seed)
    text, plan = R.shaped_schema(rng, **({"n_pairs": seed + 1} if seed < 5 else {}))
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan, wide=wide)
    o = Oracle(text)
    R.load_shaped(o, store)
    lean = _engine(text, lambda e: R.load_shaped(e, store), monkeypatch)
    generic = _engine(text, lambda e: R.load_shaped(e, store), monkeypatch, ZGPU_FLAT_CHECK="0")
    assert (lean.stats()["flat_slots"] == 0) if wide else (lean.stats()["flat_slots"] >= 1)
    queries, res, subj = R.shaped_checks(rng, store, plan, 20000)
    items = R.shaped_items(o, zgpu.CHECK_DTYPE, queries, res, subj)
    for now in ((store["now"], store["now"] + 1000) if plan["expiry"] else (store["now"],)):
        want = o.check_bulk(items, now=now)
        for e in (lean, generic):
            e.set_clock(now)
            assert np.array_equal(e.check_bulk(items), want), (seed, now)
        assert np.array_equal(_device(lean, items), want)
    print(f"seed {seed}: flat slots {lean.stats()['flat_slots']}, residual {lean.stats()['flat_residual']}")


NONPURE = """definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member
  relation banned: user
  relation parent: namespace
  permission view = viewer
  permission allowed = viewer - banned
  permission inherited = parent->allowed + viewer
}
"""


def test_multi_pass_program_with_a_residual(monkeypatch):
    """A program with non-pure permissions runs in passes: level 0 takes the lean kernel for `view` and check_kernel
    for the rest through the residual list, whose items raise sub-queries (`inherited` into `allowed`) that are folded
    back into their own (query, leaf): the list's indices reach val and subq_parent."""
    import zgpu
    from oracle.pyoracle import Oracle

    rng = np.random.default_rng(21)
    nu, ng, nt, nn = 400, 80, 30, 120
    gm = np.unique(np.stack([rng.integers(0, ng, 2500), rng.integers(0, nu, 2500)], 1), axis=0)
    tm = np.unique(np.stack([rng.integers(0, nt, 200), rng.integers(0, ng, 200)], 1), axis=0)
    nv = np.unique(np.stack([rng.integers(0, nn, 300), rng.integers(0, nt, 300)], 1), axis=0)
    nb = np.unique(np.stack([rng.integers(0, nn, 200), rng.integers(0, nu, 200)], 1), axis=0)
    npar = np.stack([np.arange(1, nn), [rng.integers(0, i) for i in range(1, nn)]], 1)  # acyclic
    rels = [("group", "member", "user", gm, None), ("team", "member", "group", tm, "member"),
            ("namespace", "viewer", "team", nv, "member"), ("namespace", "banned", "user", nb, None),
            ("namespace", "parent", "namespace", npar, None)]

    def load(x):
        for rt, rel, st, a, srel in rels:
            x.add_bulk(rt, rel, st, a[:, 0].astype(np.uint32), a[:, 1].astype(np.uint32), srel=srel)

    o = Oracle(NONPURE)
    load(o)
    e = _engine(NONPURE, load, monkeypatch)
    assert e.stats()["flat_slots"] >= 1
    n = 5003
    items = np.zeros(n, dtype=zgpu.CHECK_DTYPE)
    items["res"] = rng.integers(0, nn, n)
    items["subj"] = rng.integers(0, nu, n)
    perms = [o.slot_id("namespace", p) for p in ("view", "allowed", "inherited")]
    items["perm"] = np.array(perms, dtype=np.uint16)[rng.integers(0, 3, n)]
    items["stype"], items["srel"] = o.type_id("user"), zgpu.SREL_NONE
    want = o.check_bulk(items)
    r0 = e.stats()["flat_residual"]
    got = e.check_bulk(items)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    assert e.stats()["flat_residual"] - r0 == int((items["perm"] != perms[0]).sum())
    assert e.stats()["passes"] > 0
    assert np.array_equal(_device(e, items), want)


def test_writes_recompute_the_flags(monkeypatch):
    """5 x 1000 writes to group#member and team#member: every publish recomputes SF_FLAT, and the answers of the lean
    kernel equal the oracle's after each."""
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.02)
    e, o = zgpu.Engine(w.schema, device=0), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    rng = np.random.default_rng(17)
    for step in range(5):
        ups = np.zeros(1000, dtype=zgpu.UPDATE_DTYPE)
        for i in range(ups.size):
            g = w.groups[int(rng.integers(0, 2))]
            ups["rel"][i], ups["stype"][i] = e.slot_id(g.res_type, g.rel), e.type_id(g.subj_type)
            ups["srel"][i] = zgpu.SREL_NONE if g.srel is None else e.slot_id(g.subj_type, g.srel)
            k = int(rng.integers(0, g.res.size))
            if rng.random() < 0.5:
                ups["res"][i], ups["subj"][i], ups["op"][i] = g.res[k], g.subj[k], 2
            else:
                ups["res"][i] = g.res[int(rng.integers(0, g.res.size))]
                ups["subj"][i], ups["op"][i] = g.subj[k], 0
        key = np.stack([ups["rel"], ups["res"], ups["stype"], ups["srel"], ups["subj"]], axis=1)
        ups = ups[np.sort(np.unique(key, axis=0, return_index=True)[1])]
        e.apply_updates(ups), o.apply_updates(ups)
        e.publish()
        assert e.stats()["flat_slots"] >= 1
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items)), f"step {step}"


PROBES = """use expiration
definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member | user with expiration | user:*
  relation reader: team#member | user:* with expiration
  permission view = viewer
  permission read = reader
}
"""


def test_flat_slots_with_probes(monkeypatch):
    """Flat slots whose meets follow expiring direct subjects and wildcards (with and without expiry): checks at two
    clocks from the host and device entry points equal the oracle's and the generic kernel's, and LookupSubjects (whose
    verification hides the wildcards) equals the oracle's checks on every user."""
    import zgpu
    from oracle.pyoracle import Oracle

    rng = np.random.default_rng(41)
    nu, ng, nt, nn, t0 = 3000, 300, 60, 400, 1_000_000
    rows = []  # (res_type, rel, subj_type, srel, res, subj, expires_at)
    for g, u in {(int(a), int(b)) for a, b in zip(rng.integers(0, ng, 20000), rng.integers(0, nu, 20000))}:
        rows.append(("group", "member", "user", None, g, u, 0))
    for t, g in {(int(a), int(b)) for a, b in zip(rng.integers(0, nt, 900), rng.integers(0, ng, 900))}:
        rows.append(("team", "member", "group", "member", t, g, 0))
    for rel in ("viewer", "reader"):
        for n_, t in {(int(a), int(b)) for a, b in zip(rng.integers(0, nn, 800), rng.integers(0, nt, 800))}:
            rows.append(("namespace", rel, "team", "member", n_, t, 0))
    exps = [0, t0 - 10, t0 + 500, t0 + 5000]
    for n_, u in {(int(a), int(b)) for a, b in zip(rng.integers(0, nn, 3000), rng.integers(0, nu, 3000))}:
        rows.append(("namespace", "viewer", "user", None, n_, u, exps[int(rng.integers(0, 4))]))
    for n_ in (3, 7, 50):
        rows.append(("namespace", "viewer", "user", "*", n_, 0, 0))
    for n_, x in ((2, 0), (5, t0 + 500), (11, t0 - 10)):
        rows.append(("namespace", "reader", "user", "*", n_, 0, x))

    o = Oracle(PROBES)

    def updates(x):
        u = np.zeros(len(rows), dtype=zgpu.UPDATE_DTYPE)
        for i, (rt, rel, st, srel, r, sj, ex) in enumerate(rows):
            u["rel"][i], u["stype"][i], u["res"][i], u["subj"][i], u["expires_at"][i] = \
                x.slot_id(rt, rel), x.type_id(st), r, sj, ex
            u["srel"][i] = zgpu.SREL_WILDCARD if srel == "*" else (zgpu.SREL_NONE if srel is None else x.slot_id(st, srel))
        return u

    o.apply_updates(updates(o))
    lean = _engine(PROBES, lambda e: e.apply_updates(updates(e)), monkeypatch)
    generic = _engine(PROBES, lambda e: e.apply_updates(updates(e)), monkeypatch, ZGPU_FLAT_CHECK="0")
    assert lean.stats()["flat_slots"] >= 2
    n = 30000
    items = np.zeros(n, dtype=zgpu.CHECK_DTYPE)
    items["res"], items["subj"] = rng.integers(0, nn, n), rng.integers(0, nu, n)
    dv = [(r, sj) for rt, rel, st, srel, r, sj, ex in rows if rel == "viewer" and st == "user" and srel is None]
    own = np.flatnonzero(rng.random(n) < 0.3)
    pick = rng.integers(0, len(dv), own.size)
    items["res"][own] = [dv[k][0] for k in pick]
    items["subj"][own] = [dv[k][1] for k in pick]
    items["perm"] = np.array([o.slot_id("namespace", "view"), o.slot_id("namespace", "read")],
                             dtype=np.uint16)[rng.integers(0, 2, n)]
    items["stype"], items["srel"] = o.type_id("user"), zgpu.SREL_NONE
    for now in (t0, t0 + 1000):
        want = o.check_bulk(items, now=now)
        r0 = lean.stats()["flat_residual"]
        for e in (lean, generic):
            e.set_clock(now)
            assert np.array_equal(e.check_bulk(items), want), now
        assert lean.stats()["flat_residual"] - r0 < n // 10  # the lean kernel answered (nearly) all of them
        assert np.array_equal(_device(lean, items), want)
    lean.set_clock(t0)
    q = np.zeros(nu, dtype=zgpu.CHECK_DTYPE)
    q["subj"], q["stype"], q["srel"] = np.arange(nu), o.type_id("user"), zgpu.SREL_NONE
    for res in (3, 5, 11, 50, 100):
        for perm in ("view", "read"):
            ids, wild, ex = lean.lookup_subjects_ids("namespace", res, perm, "user")
            w = np.full(nu, 2 if wild else 1, dtype=np.uint8)
            w[ids], w[ex] = 2, 1
            q["res"], q["perm"] = res, o.slot_id("namespace", perm)
            assert np.array_equal(o.check_bulk(q, now=t0), w), (res, perm)
