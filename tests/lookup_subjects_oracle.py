"""LookupSubjects defined by Check, twice: once over the C oracle (oracle/pyoracle.py) and once, written
separately, over the pure-Python oracle (oracle/mini_oracle.py). TEST INFRASTRUCTURE.

Semantics (DESIGN.md §2, "LookupSubjects"), for resource T:r, permission P, subject type ST, optional subject
relation SR and a wildcard option:

  * candidates C: every object id of ST named by a stored relationship (resource or subject side), plus r
    itself when ST == T (userset self-membership, as LookupResources);
  * the probe: Check(T:r#P @ ST:<a never-written id>[#SR]). It stands for every subject outside C. ERROR fails
    the call (ZG_EDEPTH); HAS with SR unset means the wildcard is granted;
  * any candidate whose Check is ERROR fails the call;
  * concrete answer: candidates with Check = HAS; when the wildcard is granted, only those that also check HAS
    with every wildcard relationship invisible (Check_nowild; its ERROR only means "not listed");
  * wildcard entry: present iff granted and the option is INCLUDE; its exclusions are the candidates with
    Check = NO;
  * a resource id that no relationship ever named gives an empty answer.
"""
from __future__ import annotations

from golden_runner import split_rel
from oracle.mini_oracle import MiniOracle
from oracle.pyoracle import Oracle

HAS, NO, ERR = 2, 1, 255
INCLUDE, EXCLUDE = 0, 1
PROBE_ID = "!probe"  # '!' is outside SpiceDB's object-id charset: never written


class DepthError(Exception):
    """The answer cannot be decided (ZG_EDEPTH)."""


class COracleSubjects:
    """Over the C oracle: a second oracle instance holds every relationship except the wildcard ones."""

    def __init__(self, schema: str):
        self.schema = schema
        self.o = Oracle(schema)
        self.rels = {}      # relationship text -> expires_at
        self.seen = set()   # (type, id) ever written
        self._nw = None

    def touch(self, rel: str, expires_at: int = 0):
        self.o.touch(rel, expires_at)
        self.rels[rel] = expires_at
        rt, rid, _, st, sid, _ = split_rel(rel)
        self.seen.add((rt, rid))
        if sid != "*":
            self.seen.add((st, sid))
        self._nw = None

    def delete(self, rel: str):
        self.o.delete(rel)
        self.rels.pop(rel, None)
        self._nw = None

    def _nowild(self) -> Oracle:
        if self._nw is None:
            self._nw = Oracle(self.schema)
            for r, ex in self.rels.items():
                if split_rel(r)[4] != "*":
                    self._nw.touch(r, ex)
        return self._nw

    def lookup_subjects(self, rt, rid, perm, st, srel="", wildcards=INCLUDE, now=0):
        """-> (sorted concrete ids, wildcard entry present, sorted excluded ids); raises DepthError."""
        if (rt, rid) not in self.seen:
            return [], False, []
        cands = set()
        for r in self.rels:
            a, aid, _, b, bid, _ = split_rel(r)
            if a == st:
                cands.add(aid)
            if b == st and bid != "*":
                cands.add(bid)
        if st == rt:
            cands.add(rid)
        cands = sorted(cands)
        probe = self.o.check(rt, rid, perm, st, PROBE_ID, srel, now)
        codes = [self.o.check(rt, rid, perm, st, s, srel, now) for s in cands]
        if probe == ERR or ERR in codes:
            raise DepthError(f"{rt}:{rid}#{perm}@{st}#{srel}")
        has = [s for s, c in zip(cands, codes) if c == HAS]
        if srel or probe != HAS:
            return has, False, []
        nw = self._nowild()
        concrete = [s for s in has if nw.check(rt, rid, perm, st, s, srel, now) == HAS]
        if wildcards != INCLUDE:
            return concrete, False, []
        return concrete, True, [s for s, c in zip(cands, codes) if c == NO]


def mini_lookup_subjects(m: MiniOracle, seen, rt, rid, perm, st, srel="", wildcards=INCLUDE, now=0):
    """The same definition over the pure-Python oracle's rows; `seen` = {(type, id)} ever written."""
    if (rt, rid) not in seen:
        return [], False, []
    objs = {rid} if st == rt else set()
    for (t, i, _rel), row in m.rows.items():
        if row and t == st:
            objs.add(i)
        objs.update(sid for (s, sid, _sr) in row if s == st and sid != "*")
    probe = m.check(rt, rid, perm, st, PROBE_ID, srel, now)
    if probe == ERR:
        raise DepthError("probe")
    verdict = {}
    for s in sorted(objs):
        verdict[s] = m.check(rt, rid, perm, st, s, srel, now)
        if verdict[s] == ERR:
            raise DepthError(s)
    granted = probe == HAS and srel in ("", None)
    listed = sorted(s for s, v in verdict.items() if v == HAS)
    if not granted:
        return listed, False, []
    bare = MiniOracle.__new__(MiniOracle)
    bare.defs = m.defs
    bare.rows = {k: {sk: ex for sk, ex in row.items() if sk[1] != "*"} for k, row in m.rows.items()}
    listed = [s for s in listed if bare.check(rt, rid, perm, st, s, srel, now) == HAS]
    if wildcards != INCLUDE:
        return listed, False, []
    return listed, True, sorted(s for s, v in verdict.items() if v == NO)


def subject_queries(model, rng, n_obj, per_type=2):
    """(rt, rid, perm, st, srel) queries over a randgen model: user subjects and userset subjects."""
    out = []
    tn = [t for t in model["tnames"] if model["types"][t]["rels"] or model["types"][t]["perms"]]
    for t in tn:
        d = model["types"][t]
        names = list(d["perms"]) + list(d["rels"])
        for _ in range(per_type):
            name = rng.choice(names)
            rid = f"o{rng.randint(0, n_obj)}"  # o{n_obj}: never written
            out.append((t, rid, name, "user", ""))
            st = rng.choice(tn)
            sd = model["types"][st]
            out.append((t, rid, name, st, rng.choice(list(sd["rels"]) + list(sd["perms"]))))
            out.append((t, rid, name, st, ""))
    return out


def property_violations(check_fn, dtype, res, perm, stype, srel, n_subjects, ids, wildcard, excluded, limit=None):
    """The answer's defining property, by one bulk Check over every subject id of the type and the probe:
    every listed subject checks HAS, every excluded one NO, every other one HAS exactly when the wildcard entry
    is present (INCLUDE). check_fn(items) -> codes. Returns the violations [(subject, code, expected)]."""
    import numpy as np

    subj = np.arange(n_subjects if limit is None else min(n_subjects, limit), dtype=np.uint32)
    subj = np.concatenate([subj, np.array([0xFFFFFFFE], dtype=np.uint32)])
    items = np.zeros(subj.size, dtype=dtype)
    items["res"], items["subj"], items["perm"], items["stype"], items["srel"] = res, subj, perm, stype, srel
    codes = np.asarray(check_fn(items))
    want = np.full(subj.size, HAS if wildcard else NO, dtype=np.uint8)
    listed = np.isin(subj, np.asarray(ids, dtype=np.uint32))
    want[listed] = HAS
    want[np.isin(subj, np.asarray(excluded, dtype=np.uint32))] = NO
    bad = np.nonzero(codes != want)[0]
    return [(int(subj[i]), int(codes[i]), int(want[i])) for i in bad[:20]]
