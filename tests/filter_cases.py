"""Relationship-filter cases shared by the emulator suite (test_filter_emulation.py) and the GPU suite
(test_gpu_filters.py): filters as dicts of the six v1.RelationshipFilter fields ("" = unset), derived from a list of
relationship strings so that every combination of set and unset fields is exercised on data that matches and on data
that does not."""
from __future__ import annotations

import random

FIELDS = ("res_type", "res_id", "rel", "subj_type", "subj_id", "subj_rel")

EXP_SCHEMA = """
use expiration
definition user {}
definition group { relation member: user with expiration | group#member with expiration }
definition doc {
  relation viewer: user with expiration | user:* with expiration | group#member with expiration
  relation banned: user with expiration
  permission view = viewer - banned
}
"""


def _sides():
    """The valid set/unset combinations of one side (type, id, relation): an id or a relation needs the type."""
    return [(0, 0, 0), (1, 0, 0), (1, 1, 0), (1, 0, 1), (1, 1, 1)]


def field_matrix(rel_parts):
    """Every valid combination of set and unset fields taken from one relationship (25 filters). A subject without a
    relation filters on "..." when the subject relation is set."""
    rt, rid, rel, st, sid, srel = rel_parts
    out = []
    for a in _sides():
        for b in _sides():
            out.append({"res_type": rt if a[0] else "", "res_id": rid if a[1] else "", "rel": rel if a[2] else "",
                        "subj_type": st if b[0] else "", "subj_id": sid if b[1] else "",
                        "subj_rel": (srel or "...") if b[2] else ""})
    return out


def filters_for(rels, split_rel, rng: random.Random, samples=8):
    """Filters over `rels`: the field matrix of sampled relationships (every wildcard relationship and one of every
    relation included), the same with an id nobody wrote, wildcard and concrete subject ids swapped, and the
    filters that name nothing or a type only."""
    parts = [split_rel(r) for r in rels]
    picked, seen = [], set()
    for p in parts:  # one relationship of every (relation, subject kind), wildcards included
        key = (p[0], p[2], p[3], p[5], p[4] == "*")
        if key not in seen:
            seen.add(key)
            picked.append(p)
    rng.shuffle(picked)
    picked = [p for p in picked if p[4] == "*"] + [p for p in picked if p[4] != "*"][:samples]
    out = [{}]
    for p in picked:
        out += field_matrix(p)
        rt, rid, rel, st, sid, srel = p
        out.append({"res_type": rt, "res_id": "never-written"})
        out.append({"res_type": rt, "res_id": "never-written", "rel": rel, "subj_type": st})
        out.append({"subj_type": st, "subj_id": "never-written"})
        out.append({"res_type": rt, "res_id": rid, "subj_type": st, "subj_id": "never-written"})
        out.append({"res_type": rt, "rel": rel, "subj_type": st, "subj_id": "*"})
        out.append({"subj_type": st, "subj_id": "*"})
        out.append({"res_type": rt, "res_id": rid, "subj_type": st, "subj_id": "*"})
        if sid == "*":  # a concrete id never matches a wildcard relationship
            other = next((q[4] for q in parts if q[3] == st and q[4] != "*"), "u0")
            out.append({"res_type": rt, "res_id": rid, "rel": rel, "subj_type": st, "subj_id": other})
            out.append({"rel": rel, "res_type": rt, "subj_type": st, "subj_id": other})
        out.append({"subj_type": st, "subj_rel": "..."})
        out.append({"res_type": rt, "res_id": rid, "subj_type": st, "subj_rel": "..."})
    uniq, keys = [], set()
    for f in out:
        k = tuple(f.get(x, "") for x in FIELDS)
        if k not in keys:
            keys.add(k)
            uniq.append({x: v for x, v in zip(FIELDS, k)})
    return uniq


def matches(f, rel_parts):
    """Python statement of Store::match for one relationship (expiry aside)."""
    rt, rid, rel, st, sid, srel = rel_parts
    if f.get("res_type") and f["res_type"] != rt:
        return False
    if f.get("res_id") and f["res_id"] != rid:
        return False
    if f.get("rel") and f["rel"] != rel:
        return False
    if f.get("subj_type") and f["subj_type"] != st:
        return False
    if f.get("subj_id") and f["subj_id"] != sid:
        return False
    if f.get("subj_rel"):
        want = "" if f["subj_rel"] == "..." else f["subj_rel"]
        if sid == "*" or (srel or "") != want:
            return False
    return True
