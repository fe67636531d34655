"""Range records of the lean check kernel (csrc/build.cu gpu_build_flat_records, csrc/device.cu build_flat_records /
publish_delta / finish_publish) through every kind of publish, against a restatement from the relationships
(tests/closure_restate.py's Model).

After each publish of a churned store, the records of namespace#viewer (the push step class of the flat slot
namespace#view) equal the restatement: per namespace, its row's length and teams in row order, 0xFFFF after them, or
0xFFFF alone for a row longer than a record holds. Rows cross the 31 children a record holds in both directions. The
answers equal the oracle's and those of an engine built without records (ZGPU_FLAT_RECORDS=0)."""
import numpy as np
import pytest

import closure_restate as CR
import randgen as R

pytestmark = pytest.mark.gpu

TEXT = """definition user {}
definition group { relation member: user }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member
  permission view = viewer
}
definition doc { relation owner: user }
"""
VR = ("namespace", "viewer", "team", "member")
GM = ("group", "member", "user", None)
TM = ("team", "member", "group", "member")
DO = ("doc", "owner", "user", None)
SLOTS = 32            # closure_sig.cuh kRecSlots
LONG = 0xFFFF         # closure_sig.cuh kRecLong
N_USER, N_GROUP, N_TEAM, N_NS = 400, 80, 120, 200
LENGTHS = [0, 1, 8, 9, 16, 17, 30, 31, 32, 33, 100]


def restate(m):
    """The records of namespace#viewer at the model's namespace capacity."""
    n = m.cap["namespace"]
    out = np.full((n, SLOTS), LONG, dtype=np.uint16)
    rows = {}
    for ns, t in m.rels.get(VR, {}):
        rows.setdefault(ns, []).append(t)
    out[:, 0] = 0
    for ns, ts in rows.items():
        ts = sorted(ts)
        if len(ts) < SLOTS:
            out[ns, 0] = len(ts)
            out[ns, 1:1 + len(ts)] = ts
        else:
            out[ns, 0] = LONG
    return out


def records(e):
    """Every range record array of the published snapshot: [(info, records)]."""
    import zgpu

    out = []
    for k in range(8):
        try:
            info = e.flat_record_info(k)
        except zgpu.ZgpuError:
            break
        out.append((info, e.flat_records(k) if info["built"] else None))
    return out


class Store:
    def __init__(self, monkeypatch, rng):
        import zgpu

        self.zgpu, self.mp, self.rng = zgpu, monkeypatch, rng
        monkeypatch.setenv("ZGPU_VERIFY_BUILD", "1")
        m = CR.Model()
        gm = [(g, u) for u in range(N_USER) for g in rng.choice(N_GROUP, 3, replace=False)]
        tm = [(t, g) for t in range(N_TEAM) for g in rng.choice(N_GROUP, 4, replace=False)]
        vr = []
        for ns in range(N_NS):
            n = LENGTHS[ns % len(LENGTHS)] if ns < 3 * len(LENGTHS) else int(rng.integers(0, 28))
            vr += [(ns, t) for t in rng.choice(N_TEAM, min(n, N_TEAM), replace=False)]
        do = [(d, int(rng.integers(0, N_USER))) for d in range(50)]
        for cls, pairs in ((GM, gm), (TM, tm), (VR, vr), (DO, do)):
            a = np.array(pairs, dtype=np.uint32)
            m.load([(cls[0], cls[1], cls[2], a[:, 0], a[:, 1], cls[3], None)])
        self.m = m
        self.e = self.fresh()
        self.last = None

    def fresh(self, records=True):
        if not records:
            self.mp.setenv("ZGPU_FLAT_RECORDS", "0")
        e = self.zgpu.Engine(TEXT, device=0)
        self.mp.delenv("ZGPU_FLAT_RECORDS", raising=False)
        R.load_shaped(e, {"groups": self.m.groups()})
        e.publish()
        return e

    def write(self, ops):
        zg = self.zgpu
        ups = np.zeros(len(ops), dtype=zg.UPDATE_DTYPE)
        for i, (op, (rt, rel, st, srel), res, subj) in enumerate(ops):
            ups[i]["rel"], ups[i]["stype"] = self.e.slot_id(rt, rel), self.e.type_id(st)
            ups[i]["srel"] = zg.SREL_NONE if srel is None else self.e.slot_id(st, srel)
            ups[i]["res"], ups[i]["subj"], ups[i]["op"] = res, subj, op
            self.m.write(op, (rt, rel, st, srel), res, subj)
        self.e.apply_updates(ups)

    def verify(self, kind, range_touched):
        from oracle.pyoracle import Oracle

        e, m = self.e, self.m
        m.publish()
        recs = records(e)
        if m.live(VR):
            assert len(recs) == 1, (kind, recs)
            info, got = recs[0]
            want = restate(m)
            assert info["built"] == 1 and info["objects"] == want.shape[0], (kind, info)
            assert info["long_rows"] == int((want[:, 0] == LONG).sum()), (kind, info)
            bad = np.flatnonzero((got != want).any(axis=1))
            assert bad.size == 0, (kind, bad[:8], got[bad[:2]], want[bad[:2]])
            if self.last is not None and not range_touched and self.last.shape == got.shape:
                assert np.array_equal(self.last, got), kind
            self.last = got
        else:
            assert recs == [], (kind, recs)  # no push step over an empty class: no flat slot records
            self.last = None
        o = Oracle(TEXT)
        R.load_shaped(o, {"groups": m.groups()})
        it = np.zeros(6000, dtype=self.zgpu.CHECK_DTYPE)
        it["perm"], it["stype"], it["srel"] = o.slot_id("namespace", "view"), o.type_id("user"), 0xFFFF
        it["res"] = self.rng.integers(0, m.cap["namespace"], it.size)
        it["subj"] = self.rng.integers(0, N_USER, it.size)
        got = e.check_bulk(it)
        want = o.check_bulk(it)
        assert np.array_equal(got, want), (kind, np.flatnonzero(got != want)[:8])
        f = self.fresh(records=False)
        assert records(f) == [] or all(not i["built"] for i, _ in records(f))
        assert np.array_equal(f.check_bulk(it), got), kind
        del f


def _cross(s, up):
    """Inserts (up) or deletes that move rows across the 31 children a record holds."""
    rows = {}
    for ns, t in s.m.rels.get(VR, {}):
        rows.setdefault(ns, set()).add(t)
    ops = []
    for ns, ts in sorted(rows.items()):
        if up and len(ts) in (30, 31):
            free = [t for t in range(N_TEAM) if t not in ts][: 32 - len(ts)]
            ops += [(0, VR, ns, t) for t in free]
        elif not up and len(ts) in (32, 33):
            ops += [(2, VR, ns, t) for t in sorted(ts)[: len(ts) - 31]]
    return ops


def test_flat_records_through_publishes(monkeypatch):
    rng = np.random.default_rng(11)
    s = Store(monkeypatch, rng)
    s.verify("load", True)
    stats = s.e.stats()
    rounds = [
        ("cross up", lambda: _cross(s, True), True),
        ("cross down", lambda: _cross(s, False), True),
        ("range", lambda: [(0, VR, int(rng.integers(0, N_NS)), int(rng.integers(0, N_TEAM))) for _ in range(40)]
         + [(2, VR, ns, t) for ns, t in sorted(s.m.rels[VR])[::50]], True),
        ("group#member", lambda: [(0, GM, int(rng.integers(0, N_GROUP)), int(rng.integers(0, N_USER))) for _ in range(30)],
         False),
        ("team#member", lambda: [(0, TM, int(rng.integers(0, N_TEAM)), int(rng.integers(0, N_GROUP))) for _ in range(30)],
         False),
        ("unrelated", lambda: [(0, DO, int(rng.integers(0, 50)), int(rng.integers(0, N_USER))) for _ in range(30)], False),
    ]
    for kind, ops, touched in rounds:
        s.write(ops())
        s.e.publish()
        st = s.e.stats()
        assert st["delta_publishes"] > stats["delta_publishes"], kind
        stats = st
        s.verify(kind, touched)
    # a class emptied and refilled: the flat slot and its records go and come back
    rows = sorted(s.m.rels[VR])
    s.write([(2, VR, ns, t) for ns, t in rows])
    s.e.publish()
    s.verify("empty", True)
    s.write([(0, VR, ns, t) for ns, t in rows])
    s.e.publish()
    s.verify("refill", True)
    # an import of named namespaces and teams
    names = [(f"ns_{i}", f"tm_{i % 7}") for i in range(40)]
    s.e.import_relationships([("namespace", "viewer", "team", "member", [a for a, _ in names], [b for _, b in names],
                               None)])
    for a, b in names:
        ni, ti = s.e.find("namespace", a), s.e.find("team", b)
        s.m.named("namespace", ni), s.m.named("team", ti)
        s.m.write(0, VR, ni, ti)
    s.e.publish()
    s.verify("import", True)
    # a namespace past the capacity: the snapshot is laid out again
    cap = s.e.object_capacity("namespace")
    s.write([(0, VR, cap + 5, t) for t in range(3)])
    s.e.publish()
    assert s.e.object_capacity("namespace") > cap
    s.verify("growth", True)
    s.write([(0, VR, 3, 0), (0, GM, 1, 2)])
    s.e.publish()
    s.verify("after growth", True)
