"""The check kernel's specialised paths (csrc/kernels.cuh) on generated schemas whose stores reach them, on the GPU,
against the oracle: tests/randgen.py shaped_schema composes a schema from units that compile into each step kind
(leaf meets, two-level meets over a closure index or batch_l2, SF_NO_RSET slots, a fifth two-level pair past
kMaxClosure, expiring classes, wildcards, sub-query passes, a leaf meet two subject types reach), and
shaped_relationships fills it with rows at the kernel's thresholds. Every case is answered by four engines -- the
default, forward_only, ZGPU_CLOSURE_CAP=0 (no index: no SF_NO_RSET, every two-level step through batch_l2) and
ZGPU_MEMO_AFTER=0 -- and each targeted path is shown reached by a counter or by buckets computed from the data.
Emulator twin: tests/test_step_shapes_emulation.py."""
import random

import numpy as np
import pytest

import randgen as R
from lookup_subjects_oracle import property_violations
from test_step_shapes_emulation import (CHAIN, _fail, assert_buckets, assert_hub_buckets, chain_items, chain_store,
                                        hub_schema, hub_store)

pytestmark = pytest.mark.gpu

HAS, ERR = 2, 255
N_CHECKS = 20000
# seeds 0 .. 4 take 1 .. 5 two-level pairs, the rest draw; "wide" puts the pair types' ids past 65 536
CASES = [(s, {"n_pairs": s + 1} if s < 5 else {}, s in (3, 9)) for s in range(12)]


def _engines(text, load, monkeypatch):
    """default, forward_only, no closure index, path memo from the first round (the environment is read when the
    engine is created and when it publishes)."""
    import zgpu

    out = {}
    for label, env, kw in (("default", {}, {}), ("forward", {}, {"forward_only": True}),
                           ("no_index", {"ZGPU_CLOSURE_CAP": "0"}, {}), ("memo", {"ZGPU_MEMO_AFTER": "0"}, {})):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e = zgpu.Engine(text, device=0, **kw)
        load(e)
        e.publish()
        for k in env:
            monkeypatch.delenv(k)
        out[label] = e
    return out


@pytest.mark.parametrize("seed,plan_kw,wide", CASES, ids=[f"seed{s}{'-wide' if w else ''}" for s, _, w in CASES])
def test_shaped_schemas_against_the_oracle(seed, plan_kw, wide, monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle

    rng = random.Random(seed)
    text, plan = R.shaped_schema(rng, **plan_kw)
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan, wide=wide)
    assert_buckets(store)
    o = Oracle(text)
    R.load_shaped(o, store)
    eng = _engines(text, lambda e: R.load_shaped(e, store), monkeypatch)
    # the index: the first kMaxClosure pairs, 32-bit entries when a pair type's ids pass 65 536
    n_idx = min(len(plan["pairs"]), R.MAX_CLOSURE)
    c = eng["default"].closure_index_counters()
    assert c["indexed"] == n_idx and c["over_budget"] == 0, (seed, c)
    for k in range(n_idx):
        assert eng["default"].closure_index_info(k)["width"] == (4 if wide else 2), (seed, k)
    # the device's index of the first pair has the rows computed from the data (every size at every offset mod 16)
    # (the device's rows run to the user type's capacity: the users past the data have empty rows)
    crow = R.closure_rows(store, plan["pairs"][0])[0]
    dev = [eng["default"].closure_index(k)[0] for k in range(n_idx)]
    assert any(r.size >= crow.size and np.array_equal(r[:crow.size], crow) and (r[crow.size:] == crow[-1]).all()
               for r in dev), (seed, crow.size, [(r.size, r[:4], r[-4:]) for r in dev], crow[-4:])
    assert eng["no_index"].closure_index_counters()["indexed"] == 0
    assert eng["forward"].closure_index_counters()["indexed"] == 0
    queries, res, subj = R.shaped_checks(rng, store, plan, N_CHECKS)
    items = R.shaped_items(o, zgpu.CHECK_DTYPE, queries, res, subj)
    assert np.array_equal(items, R.shaped_items(eng["default"], zgpu.CHECK_DTYPE, queries, res, subj))
    clocks = (store["now"], store["now"] + 1000) if plan["expiry"] else (store["now"],)
    answers, passes = [], 0
    for now in clocks:
        want = o.check_bulk(items, now=now)
        answers.append(want)
        assert 0.05 < (want == HAS).mean() < 0.95
        for label, e in eng.items():
            e.set_clock(now)
            got = e.check_bulk(items)
            assert np.array_equal(got, want), _fail(seed, text, got, want, queries, res, subj, f"{label} now={now}")
            passes += e.stats()["passes"]
    if plan["expiry"]:  # the second clock expires relationships the first one held
        assert not np.array_equal(answers[0], answers[1])
    assert passes > 0  # doc#nonpure_target reaches folder#strict: sub-query passes
    # the event counters describe the last launch: one launch of the pure permissions' checks per engine
    pure = np.array([q[0] == "folder" and q[1] == "view" or q[1] in plan["pure"] for q in queries])
    st = {}
    for label, e in eng.items():
        assert np.array_equal(e.check_bulk(items[pure]), answers[-1][pure]), label
        st[label] = e.stats()
    assert st["memo"]["memo_batches"] > 0, st["memo"]
    assert sum(x["stack_spills"] for x in st.values()) > 0, {k: x["stack_spills"] for k, x in st.items()}
    # LookupResources for users of every membership bucket, LookupSubjects for docs of every range size
    e = eng["default"]
    e.set_clock(clocks[0])
    by_split = {}
    for u, s in store["split"].items():
        by_split.setdefault(s, u)
    users = sorted(by_split.values())[:10] + sorted(store["closure"])[:4]
    for perm in ("view", "only_l2"):
        for u in users:
            got = e.lookup_resources_ids("doc", perm, "user", u)
            want = o.lookup_resources_ids("doc", perm, "user", u, now=clocks[0])
            assert np.array_equal(got, want), (seed, perm, u, got[:10], want[:10])
    for d in range(0, len(R.RANGE_SIZES) * 2, 3):
        for perm in ("view", "reader"):
            ids, wild, ex = e.lookup_subjects_ids("doc", d, perm, "user")
            bad = property_violations(lambda it: o.check_bulk(it, now=clocks[0]), zgpu.CHECK_DTYPE, d,
                                      e.slot_id("doc", perm), e.type_id("user"), zgpu.SREL_NONE, store["n"]["user"],
                                      ids, wild, ex)
            assert not bad, (seed, d, perm, bad[:5])


def test_rsetless_slots_equal_the_run_without_index(monkeypatch):
    """SF_NO_RSET: doc#only_l2 and doc#minus_rsetless were built to qualify (every root push an indexed two-level
    step, no invertible probe); with 5 pairs, doc#with5 reaches the fifth, unindexed pair and must keep the set. Their
    answers equal the ZGPU_CLOSURE_CAP=0 run's (no index, no flag) and the oracle's."""
    import zgpu
    from oracle.pyoracle import Oracle

    rng = random.Random(100)
    text, plan = R.shaped_schema(rng, n_pairs=5)
    assert set(plan["rsetless"]) <= set(plan["perms"]) and "with5" in plan["perms"]
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan)
    o = Oracle(text)
    R.load_shaped(o, store)
    eng = _engines(text, lambda e: R.load_shaped(e, store), monkeypatch)
    assert eng["default"].closure_index_counters()["indexed"] == R.MAX_CLOSURE
    n_user = store["n"]["user"]
    users = np.concatenate([np.array(sorted(store["closure"])), np.arange(0, n_user, 7), [n_user, n_user + 1]])
    for perm in plan["rsetless"] + ["with5", "l2"]:
        items = np.zeros(users.size * store["n"]["doc"], dtype=zgpu.CHECK_DTYPE)
        items["res"] = np.repeat(np.arange(store["n"]["doc"]), users.size)
        items["subj"] = np.tile(users, store["n"]["doc"])
        items["perm"], items["stype"], items["srel"] = o.slot_id("doc", perm), o.type_id("user"), zgpu.SREL_NONE
        want = o.check_bulk(items, now=store["now"])
        assert (want == HAS).any() and (want != HAS).any(), perm
        for label in ("default", "no_index"):
            eng[label].set_clock(store["now"])
            assert np.array_equal(eng[label].check_bulk(items), want), (perm, label)


def test_depth_cap_through_each_meet(monkeypatch):
    """A folder#parent chain: leaf meets at depth 49 and 50, two-level meets at 48 and 49, indexed and through
    batch_l2: HAS where the path fits ZG_MAX_DEPTH, the oracle's answer (ERROR) one hop further."""
    import zgpu
    from oracle.pyoracle import Oracle

    groups = chain_store()

    def load(t):
        for rt, rel, st, res, subj, srel in groups:
            t.add_bulk(rt, rel, st, np.asarray(res), np.asarray(subj), srel=srel)

    o = Oracle(CHAIN)
    load(o)
    items = chain_items(o, zgpu.CHECK_DTYPE)
    want = o.check_bulk(items)
    for k in (0, 1):
        assert (want[k::3] == HAS).any() and (want[k::3] == ERR).any(), want[k::3]
    eng = _engines(CHAIN, load, monkeypatch)
    assert eng["default"].closure_index_counters()["indexed"] == 1
    for label, e in eng.items():
        assert np.array_equal(e.check_bulk(items), want), (label, e.check_bulk(items), want)


@pytest.mark.parametrize("k", [2, 3, R.MAX_INV_CLASSES, R.MAX_INV_CLASSES + 1])
def test_admission_at_the_set_cap_split_over_classes(k, monkeypatch):
    """Memberships 0 .. 24 spread over k invertible classes, 16 and 17 with the cap inside a later class; k = 12 is one
    class past kMaxInvClasses."""
    import zgpu
    from oracle.pyoracle import Oracle

    text = hub_schema(k)
    groups, n_user, n_doc = hub_store(k, seed=k)
    assert_hub_buckets(groups, k, n_user)

    def load(t):
        for rt, rel, st, res, subj, srel in groups:
            t.add_bulk(rt, rel, st, np.asarray(res), np.asarray(subj), srel=srel)

    o = Oracle(text)
    load(o)
    eng = _engines(text, load, monkeypatch)
    items = np.zeros(n_doc * n_user, dtype=zgpu.CHECK_DTYPE)
    items["res"], items["subj"] = np.repeat(np.arange(n_doc), n_user), np.tile(np.arange(n_user), n_doc)
    items["perm"], items["stype"], items["srel"] = o.slot_id("doc", "view"), o.type_id("user"), zgpu.SREL_NONE
    want = o.check_bulk(items)
    assert 0.05 < (want == HAS).mean() < 0.95
    for label, e in eng.items():
        got = e.check_bulk(items)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"k={k} {label}: first (doc, user) {[(int(items['res'][i]), int(items['subj'][i])) for i in bad[:6]]}"
