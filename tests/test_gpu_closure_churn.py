"""Closure indexes, signatures and set tables through every kind of publish, against tests/closure_restate.py's
restatement from the relationships (csrc/device.cu publish_delta / build_closures / finish_publish).

After every publish of a churned store: each pair's index, signatures and table equal the restatement; on a delta
publish the pairs the round did not touch are byte-identical to before and only the touched ones were rebuilt; the
answers and a few lookups equal the oracle's; and fresh engines loaded from the same relationships (with and without
the lean flat kernel) hold the same structures and answer the same. Every engine verifies its CSR
(ZGPU_VERIFY_BUILD=1)."""
import random

import numpy as np
import pytest

import closure_restate as CR
import randgen as R

pytestmark = pytest.mark.gpu

GM = ("group", "member", "user", None)
SMALL = """definition user {}
definition group { relation member: user }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member | user
  permission view = viewer
}
"""
SMALL_STEPS = [(("namespace", "viewer", "team", "member"), GM, ("team", "member", "group", "member"))]


def shaped_steps(plan):
    """The two-level steps of randgen.shaped_schema in step order: team's through folder#viewer, doc#tm and doc#l2,
    then the other pair types' through doc#l2, the fifth's through doc#l2x."""
    out = []
    for i, p in enumerate(plan["pairs"]):
        tgc = (p, "member", "group", "member")
        vias = [("doc", "l2x" if i >= R.MAX_CLOSURE else "l2", p, "member")]
        if p == "team":
            vias = [("folder", "viewer", "team", "member"), ("doc", "tm", "team", None)] + vias
        out += [(v, GM, tgc) for v in vias]
    return out


def _structures(e):
    """Every pair of the published snapshot: (info, signature info, table info, index, signatures, table)."""
    c = e.closure_index_counters()
    out = []
    for k in range(c["indexed"] + c["over_budget"]):
        info, si, ti = e.closure_index_info(k), e.closure_signature_info(k), e.closure_table_info(k)
        idx = e.closure_index(k) if info["built"] else None
        sig = e.closure_signature(k) if si["built"] else None
        tab = e.closure_table(k) if ti["built"] else None
        out.append((info, si, ti, idx, sig, tab))
    return out


def _same(a, b):
    """Two pairs' structures byte-identical (build times and allocation sizes aside: a rebuilt index reuses the
    buffers of the one it replaces, which may be larger)."""
    key = lambda s: (s[0]["built"], s[0]["width"], s[0]["entries"], s[1]["words"], s[2]["buckets"])  # noqa: E731
    if key(a) != key(b):
        return False
    for x, y in zip(a[3:], b[3:]):
        if (x is None) != (y is None):
            return False
        if x is not None:
            xs, ys = (x, y) if isinstance(x, tuple) else ((x,), (y,))
            if not all(np.array_equal(u, v) for u, v in zip(xs, ys)):
                return False
    return True


def _match(e, restated):
    """Engine pair k -> restated pair, matched by the index's content (over-budget pairs by elimination), after
    asserting each equals its restatement. Returns the engine's pairs' tgc classes in order and its structures."""
    st = _structures(e)
    assert e.closure_index_counters() | CR.counters(restated) == e.closure_index_counters()
    assert len(st) == len(restated)
    free = list(range(len(restated)))
    tgcs = [None] * len(st)
    for k, (info, si, ti, idx, sig, tab) in enumerate(st):
        if not info["built"]:
            continue
        hits = [j for j in free if restated[j]["built"] and np.array_equal(idx[0], restated[j]["row_ptr"])
                and np.array_equal(idx[1], restated[j]["col"])]
        assert hits, f"pair {k}: index equals no restated pair"
        p = restated[hits[0]]
        free.remove(hits[0])
        tgcs[k] = p["tgc"]
        assert info["width"] == p["width"] and info["entries"] == p["col"].size, (k, info)
        assert si["built"] and si["words"] == p["words"] and np.array_equal(sig, p["sig"]), (k, si)
        assert (p["table"] is None) == (not ti["built"]), (k, ti, p["tgc"])
        if p["table"] is not None:
            assert np.array_equal(tab[0], p["table"][0]) and np.array_equal(tab[1], p["table"][1]), k
    rest = [restated[j]["tgc"] for j in free]
    assert all(not restated[j]["built"] for j in free)
    for k in range(len(st)):
        if tgcs[k] is None:
            tgcs[k] = rest.pop(0)
    return tgcs, st


class Churn:
    """An engine, the model of its relationships, and the checks run after each of its publishes."""

    def __init__(self, text, steps, model, monkeypatch, checks, lookups, cap=None, now=1000, expiry=False):
        import zgpu

        self.zgpu, self.text, self.steps, self.model, self.mp = zgpu, text, steps, model, monkeypatch
        self.cap, self.now, self.expiry = cap, now, expiry
        # checks [(res_type, perm, subj_type, res ids, subj ids)], lookups [(res_type, perm, subj_type, users)]
        self.checks, self.lookups = checks, lookups
        monkeypatch.setenv("ZGPU_VERIFY_BUILD", "1")
        if cap is not None:
            monkeypatch.setenv("ZGPU_CLOSURE_CAP", str(cap))
        self.e = self.fresh()
        self.pairs, self.st, self.stats = None, None, None
        self.touched = set()
        self.log = []
        self.verify("load")

    def fresh(self, flat=True):
        if not flat:
            self.mp.setenv("ZGPU_FLAT_CHECK", "0")
        e = self.zgpu.Engine(self.text, device=0)
        self.mp.delenv("ZGPU_FLAT_CHECK", raising=False)
        e.set_clock(self.now)
        R.load_shaped(e, {"groups": self.model.groups()})
        e.publish()
        return e

    def write(self, ops):
        """[(op, class, res, subj, expires)]: applied to the engine and the model; the classes count as touched."""
        zg = self.zgpu
        ups = np.zeros(len(ops), dtype=zg.UPDATE_DTYPE)
        for i, (op, (rt, rel, st, srel), res, subj, ex) in enumerate(ops):
            ups[i]["rel"], ups[i]["stype"] = self.e.slot_id(rt, rel), self.e.type_id(st)
            ups[i]["srel"] = zg.SREL_NONE if srel is None else self.e.slot_id(st, srel)
            ups[i]["res"], ups[i]["subj"], ups[i]["op"], ups[i]["expires_at"] = res, subj, op, ex
            self.model.write(op, (rt, rel, st, srel), res, subj, ex)
            self.touched.add((rt, rel, st, srel))
        self.e.apply_updates(ups)

    def oracle(self):
        from oracle.pyoracle import Oracle

        o = Oracle(self.text)
        R.load_shaped(o, {"groups": self.model.groups()})
        return o

    def items(self, o):
        out = []
        for rt, perm, st, res, subj in self.checks:
            it = np.zeros(res.size, dtype=self.zgpu.CHECK_DTYPE)
            it["perm"], it["stype"], it["srel"] = o.slot_id(rt, perm), o.type_id(st), 0xFFFF
            it["res"], it["subj"] = res, subj
            out.append(it)
        return np.concatenate(out)

    def answers(self, e, items):
        got = []
        for now in ((self.now, self.now + 1000) if self.expiry else (self.now,)):
            e.set_clock(now)
            got.append(e.check_bulk(items))
        e.set_clock(self.now)
        return got

    def verify(self, kind):
        """Everything a publish must hold; returns what it saw (delta / full, builds, the pairs' tgc classes)."""
        e, m = self.e, self.model
        m.publish()
        pairs = CR.pairs(m, self.steps)
        restated = CR.restate(m, pairs, self.cap)
        stats, builds = e.stats(), e.closure_index_counters()["builds"]
        tgcs, st = _match(e, restated)
        assert {t: e.object_capacity(t) for t in m.cap} == m.cap, kind
        assert tgcs == [t for _, t in pairs], (kind, tgcs, pairs)
        saw = {"kind": kind, "tgcs": tgcs, "indexed": sum(p["built"] for p in restated)}
        if self.stats is not None:
            full = stats["full_publishes"] > self.stats["full_publishes"]
            delta = stats["delta_publishes"] > self.stats["delta_publishes"]
            old = {t: (inner, s) for (inner, t), s in zip(self.pairs, self.st)}
            if full:
                want = len(pairs)
            else:
                assert delta, kind
                hit = {t for t, (inner, _) in old.items() if inner in self.touched or t in self.touched}
                want = len(hit) + sum(t not in old for _, t in pairs)
                for k, (inner, t) in enumerate(pairs):
                    if t in old and t not in hit:  # kept as it was
                        assert _same(st[k], old[t][1]), (kind, t)
            assert builds - self.builds == want, (kind, builds - self.builds, want, full)
            saw.update(full=full, delta=delta and not full, builds=builds - self.builds)
        self.pairs, self.st, self.stats, self.builds = pairs, st, stats, builds
        self.touched = set()
        # answers: the oracle's, and a fresh engine's with and without the flat kernel
        o = self.oracle()
        items = self.items(o)
        got = self.answers(e, items)
        for g, now in zip(got, (self.now, self.now + 1000)):
            assert np.array_equal(g, o.check_bulk(items, now=now)), (kind, now, np.flatnonzero(g != o.check_bulk(items, now=now))[:8])
        f = self.fresh()
        fm = CR.Model()
        fm.load(m.groups())
        fm.publish()
        ftgcs, fst = _match(f, CR.restate(fm, CR.pairs(fm, self.steps), self.cap))
        assert ftgcs == tgcs
        if all(fm.cap[t] == m.cap[t] for t in fm.cap):  # same capacities: the same bytes
            assert all(_same(a, b) for a, b in zip(st, fst)), kind
        for g, h in zip(got, self.answers(f, items)):
            assert np.array_equal(g, h), kind
        del f
        f = self.fresh(flat=False)
        for g, h in zip(got, self.answers(f, items)):
            assert np.array_equal(g, h), kind
        del f
        for rt, perm, st_, users in self.lookups:
            for u in users:
                assert np.array_equal(e.lookup_resources_ids(rt, perm, st_, int(u)),
                                      o.lookup_resources_ids(rt, perm, st_, int(u), now=self.now)), (kind, perm, u)
        self.log.append(saw)
        return saw


def _shaped(seed, n_pairs, expiry, monkeypatch, cap=None):
    rng = random.Random(seed)
    text, plan = R.shaped_schema(rng, n_pairs=n_pairs, expiry=expiry)
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan, n_user=1000, n_bot=100, n_group=300,
                                   n_crew=50, n_pair=120, n_folder=40, n_doc=200)
    m = CR.Model()
    m.load(store["groups"])
    q, res, subj = R.shaped_checks(rng, store, plan, 4000)
    checks = [(rt, perm, st, res[i:i + 1], subj[i:i + 1]) for i, (rt, perm, st, sr) in enumerate(q) if sr is None]
    by = {}
    for rt, perm, st, r, s in checks:  # one group per query kind
        by.setdefault((rt, perm, st), ([], []))
        by[(rt, perm, st)][0].append(r[0]), by[(rt, perm, st)][1].append(s[0])
    checks = [(rt, perm, st, np.array(a, np.uint32), np.array(b, np.uint32)) for (rt, perm, st), (a, b) in by.items()]
    users = sorted(store["closure"])[:: 37][:3]
    lookups = [("doc", "only_l2", "user", users), ("doc", "view", "user", users[:1])]
    c = Churn(text, shaped_steps(plan), m, monkeypatch, checks, lookups, cap=cap, now=store["now"], expiry=expiry)
    return c, plan, store, rng


def _subjects(c, res, perm="only_l2"):
    """lookup_subjects_ids of a doc against the oracle's checks over every user."""
    o = c.oracle()
    n = c.model.cap["user"]
    ids, wild, ex = c.e.lookup_subjects_ids("doc", int(res), perm, "user")
    q = np.zeros(n, dtype=c.zgpu.CHECK_DTYPE)
    q["res"], q["subj"] = int(res), np.arange(n)
    q["perm"], q["stype"], q["srel"] = o.slot_id("doc", perm), o.type_id("user"), 0xFFFF
    assert np.array_equal(ids, np.flatnonzero(o.check_bulk(q, now=c.now) == 2)) and ex.size == 0


def _tgc_writes(c, rng, p, n=20):
    """Deletes and inserts in pair type p's class, within _shaped's 120 objects per pair type and 300 groups."""
    cls = (p, "member", "group", "member")
    have = sorted(c.model.rels.get(cls, {}))
    ops = [(2, cls, t, g, 0) for t, g in rng.sample(have, min(n // 2, len(have)))]
    ops += [(0, cls, rng.randrange(120), rng.randrange(300), 0) for _ in range(n - len(ops))]
    return ops


@pytest.mark.parametrize("n_pairs", [2, 3, 4, 5])
@pytest.mark.parametrize("expiry", [False, True])
def test_multi_pair_churn(n_pairs, expiry, monkeypatch):
    seed = 700 + 10 * n_pairs + expiry
    c, plan, store, rng = _shaped(seed, n_pairs, expiry, monkeypatch)
    idx = plan["pairs"][:R.MAX_CLOSURE]
    kinds = ["tgc", "inner", "none", "empty", "refill", "import", "retire", "relayout"] + (["collect"] if expiry else [])
    rng.shuffle(kinds)
    for a, b in (("empty", "refill"), ("import", "retire")):
        if kinds.index(a) > kinds.index(b):
            i, j = kinds.index(a), kinds.index(b)
            kinds[i], kinds[j] = kinds[j], kinds[i]
    emptied = None

    def live():
        return [p for p in idx if c.model.live((p, "member", "group", "member"))]
    for r, kind in enumerate(kinds):
        if kind == "tgc":
            c.write(_tgc_writes(c, rng, rng.choice(live())))
            c.e.publish()
            saw = c.verify(kind)
            assert saw["delta"] and saw["builds"] == 1, saw
        elif kind == "inner":
            have = sorted(c.model.rels[GM])
            ops = [(2, GM, g, u, 0) for g, u in rng.sample(have, 10)]
            ops += [(0, GM, rng.randrange(300), rng.randrange(1000), 0) for _ in range(10)]
            c.write(ops)
            c.e.publish()
            saw = c.verify(kind)
            assert saw["delta"] and saw["builds"] == len(c.pairs) >= 1, saw
        elif kind == "none":
            c.write([(0, ("doc", "owner", "user", None), rng.randrange(200), rng.randrange(1000), 0) for _ in range(20)])
            c.e.publish()
            saw = c.verify(kind)
            assert saw["delta"] and saw["builds"] == 0, saw
        elif kind == "empty":
            p = rng.choice(live())
            cls = (p, "member", "group", "member")
            emptied = (cls, sorted(c.model.rels[cls]))
            c.write([(2, cls, t, g, 0) for t, g in emptied[1]])
            c.e.publish()
            saw = c.verify(kind)
            assert saw["delta"] and cls not in saw["tgcs"] and len(saw["tgcs"]) == min(n_pairs - 1, R.MAX_CLOSURE), saw
        elif kind == "refill":
            cls, rows = emptied
            c.write([(0, cls, t, g, 0) for t, g in rows])
            c.e.publish()
            saw = c.verify(kind)
            assert saw["delta"] and cls in saw["tgcs"] and len(saw["tgcs"]) == min(n_pairs, R.MAX_CLOSURE), saw
        elif kind == "import":
            before = c.e.import_counters()["relationships"]
            names = [(f"ig{seed}_{i}", f"iu{seed}_{i}") for i in range(12)]
            c.e.import_relationships([("group", "member", "user", None, [g for g, _ in names], [u for _, u in names], None)])
            assert c.e.import_counters()["relationships"] == before + 12
            for g, u in names:
                gi, ui = c.e.find("group", g), c.e.find("user", u)
                c.model.named("group", gi), c.model.named("user", ui)
                c.model.write(0, GM, gi, ui)
            c.touched.add(GM)
            c.e.publish()
            c.verify(kind)
        elif kind == "retire":
            # names no watch change mentions (interned, written and deleted by raw updates) are retired
            olds = [(c.e.intern("group", f"og{seed}_{i}"), c.e.intern("user", f"ou{seed}_{i}")) for i in range(8)]
            for g, u in olds:
                c.model.named("group", g), c.model.named("user", u)
            c.write([(0, GM, g, u, 0) for g, u in olds])
            c.e.publish()
            c.verify(kind)
            c.write([(2, GM, g, u, 0) for g, u in olds])
            c.e.publish()
            c.verify(kind)
            freed = {("group", g) for g, _ in olds} | {("user", u) for _, u in olds}
            assert c.e.retire_unused_names() == len(freed)
            news = [(f"rg{seed}_{i}", f"ru{seed}_{i}") for i in range(5)]
            for g, u in news:  # names interned anew take the freed ids, lowest first
                gi, ui = c.e.intern("group", g), c.e.intern("user", u)
                assert ("group", gi) in freed and ("user", ui) in freed
                c.model.named("group", gi), c.model.named("user", ui)
            c.write([(0, GM, c.e.find("group", g), c.e.find("user", u), 0) for g, u in news])
            c.e.publish()
            saw = c.verify(kind)
            assert saw["delta"], saw
        elif kind == "relayout":
            p = rng.choice(live())
            cls = (p, "member", "group", "member")
            t = c.model.cap[p] + 3
            c.write([(0, cls, t, rng.randrange(300), 0)])
            c.e.publish()
            saw = c.verify(kind)
            assert saw["full"] and c.model.cap[p] > t, saw
        elif kind == "collect":
            c.now += 600
            c.e.set_clock(c.now)
            n = c.model.collect(c.now)
            assert n > 0 and c.e.collect_expired(c.now) == n
            c.e.publish()
            saw = c.verify(kind)
            assert saw["builds"] == 0, saw
        if r % 3 == 0:
            docs = sorted({d for d, _ in c.model.rels.get(("doc", "l2", idx[0], "member"), {})})
            _subjects(c, docs[r % len(docs)])
    assert {s["kind"] for s in c.log} == {"load"} | set(kinds)
    print(f"churn n_pairs={n_pairs} expiry={expiry}: " + ", ".join(
        f"{s['kind']}:{'full' if s.get('full') else 'delta' if s.get('delta') else 'load'}/{s.get('builds', '-')}"
        for s in c.log))


def test_budget_crossing(monkeypatch):
    """ZGPU_CLOSURE_CAP lets every index fit; inserts push team's over it (no index, the stale flags of the last full
    publish stay live) and deletes bring it back."""
    rng = random.Random(800)
    text, plan = R.shaped_schema(rng, n_pairs=2, expiry=False)
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan, n_user=1000, n_bot=100, n_group=300,
                                   n_crew=50, n_pair=120, n_folder=40, n_doc=200)
    m = CR.Model()
    m.load(store["groups"])
    m.publish()
    steps = shaped_steps(plan)
    pre = [p["pre"] for p in CR.restate(m, CR.pairs(m, steps))]
    cap = max(pre) + 5
    q, res, subj = R.shaped_checks(rng, store, plan, 3000)
    checks = [("doc", perm, "user", res[i:i + 1], subj[i:i + 1]) for i, (rt, perm, st, sr) in enumerate(q)
              if rt == "doc" and st == "user"]
    checks = [(rt, p, st, np.concatenate([x[3] for x in checks if x[1] == p]), np.concatenate([x[4] for x in checks if x[1] == p]))
              for p in sorted({x[1] for x in checks}) for rt, st in [("doc", "user")]]
    users = sorted(store["closure"])[:2]
    c = Churn(text, steps, m, monkeypatch, checks, [("doc", "only_l2", "user", users)], cap=cap)
    assert c.log[-1]["indexed"] == 2
    j = int(np.argmax(pre))  # the pair closest to the cap goes over it
    tm = c.pairs[j][1]
    members = {}
    for g, u in c.model.rels[GM]:
        members[g] = members.get(g, 0) + 1
    g = max(members, key=members.get)
    add = [t for t in range(120) if (t, g) not in c.model.rels[tm]]
    k = (cap - pre[j]) // members[g] + 1
    assert k <= len(add)
    c.write([(0, tm, t, g, 0) for t in add[:k]])
    c.e.publish()
    saw = c.verify("over")
    assert saw["delta"] and saw["indexed"] == 1 and c.e.closure_index_counters()["over_budget"] == 1, saw
    assert not c.e.closure_index_info(j)["built"]
    assert c.e.stats()["flat_slots"] > 0  # the marks of the last full publish are still live
    _subjects(c, 0)
    c.write([(2, tm, t, g, 0) for t in add[:k]])
    c.e.publish()
    saw = c.verify("under")
    assert saw["delta"] and saw["indexed"] == 2 and c.e.closure_index_counters()["over_budget"] == 0, saw


def _small(monkeypatch, max_team, group0_teams, n_users=50, seed=0):
    """SMALL: user 0 in group 0, whose teams are `group0_teams`; users 1.. in groups 1..20, each in a few teams;
    team `max_team` exists (it sets the capacity); namespaces view teams."""
    rng = np.random.default_rng(seed)
    gu = [(0, 0)] + [(int(g), int(u)) for u in range(1, n_users) for g in rng.choice(np.arange(1, 21), 2, replace=False)]
    tg = [(int(t), 0) for t in group0_teams] + [(int(t), int(g)) for g in range(1, 21)
                                                for t in rng.choice(max_team, 30, replace=False)] + [(max_team, 1)]
    nv = [(n, int(t)) for n in range(30) for t in rng.choice(max_team + 1, 40, replace=False)]
    nv += [(30, int(t)) for t in list(group0_teams)[:: max(1, len(group0_teams) // 50)]] + [(31, max_team)]
    m = CR.Model()
    m.load([("group", "member", "user", np.array([g for g, _ in gu]), np.array([u for _, u in gu]), None, None),
            ("team", "member", "group", np.array([t for t, _ in tg]), np.array([g for _, g in tg]), "member", None),
            ("namespace", "viewer", "team", np.array([n for n, _ in nv]), np.array([t for _, t in nv]), "member", None)])
    res = np.repeat(np.arange(33, dtype=np.uint32), n_users + 2)
    subj = np.tile(np.arange(n_users + 2, dtype=np.uint32), 33)
    c = Churn(SMALL, SMALL_STEPS, m, monkeypatch, [("namespace", "view", "user", res, subj)],
              [("namespace", "view", "user", [0, 1])])
    return c


def test_set_table_lost_and_regained_through_a_delta(monkeypatch):
    """Group 0's teams (user 0's closure row) grow across the table's bucket limit and back, one delta each."""
    from test_closure_set_emulation import np_choose

    order = np.random.default_rng(3).permutation(20000)
    row = lambda L: np.sort(order[:L]).astype(np.int64)  # noqa: E731
    first = next(L for L in range(3000, 16400, 100) if np_choose(row(L)) is None)
    first = next(L for L in range(first - 100, first + 1) if np_choose(row(L)) is None)
    c = _small(monkeypatch, 19999, order[:100])
    tm = ("team", "member", "group", "member")
    assert c.e.closure_table_info(0)["built"] == 1
    have = 100
    seen = []
    for L in (first - 1, first, 16383, 16384, 16385, 100):
        if L > have:
            c.write([(0, tm, int(t), 0, 0) for t in order[have:L]])
        else:
            c.write([(2, tm, int(t), 0, 0) for t in order[L:have]])
        have = L
        c.e.publish()
        saw = c.verify(f"row {L}")
        built = c.e.closure_table_info(0)["built"]
        assert saw["delta"] and not saw["full"] and c.e.closure_signature_info(0)["built"] == 1, saw
        assert built == (np_choose(row(L)) is not None), (L, built)
        seen.append((L, built))
    assert [b for _, b in seen] == [1, 0, 0, 0, 0, 1], seen
    print(f"set table through deltas (row length, built): {seen}, first unplaceable length {first}")


@pytest.mark.parametrize("cap", [65535, 65536, 65537])
def test_sixteen_bit_boundary(cap, monkeypatch):
    """Target capacities 65 535 (16-bit, table), 65 536 (16-bit, no table) and 65 537 (32-bit); the first store then
    grows across the boundary."""
    need = next(n for n in range(50000, 60000) if CR.next_capacity(0, n) == cap)
    c = _small(monkeypatch, need - 1, np.arange(0, need, 997))
    info, ti = c.e.closure_index_info(0), c.e.closure_table_info(0)
    assert c.e.object_capacity("team") == cap == c.model.cap["team"]
    assert (info["width"], ti["built"]) == {65535: (2, 1), 65536: (2, 0), 65537: (4, 0)}[cap], (info, ti)
    if cap == 65535:
        c.write([(0, ("team", "member", "group", "member"), 65535, 0, 0), (0, ("namespace", "viewer", "team", "member"), 31, 65535, 0)])
        c.e.publish()
        saw = c.verify("across")
        assert saw["full"] and c.e.closure_index_info(0)["width"] == 4 and c.e.closure_table_info(0)["built"] == 0


def test_fifth_pair_takes_an_emptied_slot(monkeypatch):
    """n_pairs = 5: team's class emptied (org, club, guild, band indexed), refilled (team back, band out)."""
    c, plan, store, rng = _shaped(900, 5, False, monkeypatch)
    tgc = {p: (p, "member", "group", "member") for p in plan["pairs"]}
    assert c.log[-1]["tgcs"] == [tgc[p] for p in plan["pairs"][:4]]
    rows = sorted(c.model.rels[tgc["team"]])
    c.write([(2, tgc["team"], t, g, 0) for t, g in rows])
    c.e.publish()
    saw = c.verify("team emptied")
    assert saw["tgcs"] == [tgc[p] for p in plan["pairs"][1:]] and saw["builds"] == 2, saw
    _subjects(c, 1, "with5")
    c.write([(0, tgc["team"], t, g, 0) for t, g in rows])
    c.e.publish()
    saw = c.verify("team refilled")
    assert saw["tgcs"] == [tgc[p] for p in plan["pairs"][:4]] and saw["builds"] == 1, saw
