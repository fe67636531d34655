"""ExpandPermissionTree restated in Python over MiniOracle.rows, and the tree evaluated for a subject. TEST
INFRASTRUCTURE (DESIGN.md §2, "ExpandPermissionTree").

A tree node is what _lib.parse_expand_lines builds from the engine's string form: {"op": U|I|X|L, "object": "type:id",
"relation": str, "subjects": ["type:id" | "type:id#rel" | "type:*"], "children": [...]}.

  * a relation: one leaf listing its live relationships, classes in schema order, then ids in `order` within a class
    (the engine's interned ids; by default the id strings);
  * a permission: the node of its expression at (T:r, P). A chain of + or & is one n-ary node, - stays binary, a bare
    operand is a one-child union. `ref n` is Expand(T:r, n); `nil` an empty leaf at (T:r, P); an arrow a union at
    (T:r, P) with one child per live non-wildcard relationship of the tupleset: Expand(S:s, p) when S defines p, else
    an empty leaf at (T:r, P);
  * a subtree reached through more than MAX_DEPTH arrows raises DepthError.
"""
from __future__ import annotations

MAX_DEPTH = 50


class DepthError(Exception):
    """The tree would hold a subtree deeper than MAX_DEPTH arrow hops (ZG_EDEPTH)."""


def _node(op, rt, rid, rel, subjects=(), children=()):
    return {"op": op, "object": f"{rt}:{rid}", "relation": rel, "subjects": list(subjects), "children": list(children)}


def _flatten(e, op, out):
    if e[0] == op:
        _flatten(e[1], op, out)
        _flatten(e[2], op, out)
    else:
        out.append(e)
    return out


class Expander:
    def __init__(self, mo, now=0, order=None):
        self.mo, self.defs, self.now = mo, mo.defs, now
        self.order = order or (lambda t, i: i)

    def rows(self, rt, rid, rel):
        """Live (stype, sid, srel) of rt:rid#rel in the engine's leaf order."""
        cls = {}
        for i, (st, sr, _ex) in enumerate(self.defs[rt]["relations"][rel]):
            cls.setdefault((st, sr), i)
        live = self.mo._live(rt, rid, rel, self.now)
        return sorted(live, key=lambda k: (cls[(k[0], "*" if k[1] == "*" else k[2])], self.order(k[0], k[1])))

    def expand(self, rt, rid, name, depth=0):
        d = self.defs[rt]
        if name in d["relations"]:
            subs = [f"{st}:{sid}" + (f"#{sr}" if sr else "") for st, sid, sr in self.rows(rt, rid, name)]
            return _node("L", rt, rid, name, subs)
        return self._expr(d["permissions"][name], rt, rid, name, depth)

    def _expr(self, e, rt, rid, at, depth):
        if e[0] in ("+", "&"):
            kids = [self._operand(o, rt, rid, at, depth) for o in _flatten(e, e[0], [])]
            return _node("U" if e[0] == "+" else "I", rt, rid, at, children=kids)
        if e[0] == "-":
            return _node("X", rt, rid, at, children=[self._operand(e[1], rt, rid, at, depth),
                                                     self._operand(e[2], rt, rid, at, depth)])
        return _node("U", rt, rid, at, children=[self._operand(e, rt, rid, at, depth)])

    def _operand(self, e, rt, rid, at, depth):
        k = e[0]
        if k in ("+", "&", "-"):
            return self._expr(e, rt, rid, at, depth)
        if k == "ref":
            return self.expand(rt, rid, e[1], depth)
        if k == "nil":
            return _node("L", rt, rid, at)
        kids = []
        for st, sid, _sr in self.rows(rt, rid, e[1]):
            if sid == "*":
                continue
            sd = self.defs[st]
            if e[2] in sd["relations"] or e[2] in sd["permissions"]:
                if depth + 1 > MAX_DEPTH:
                    raise DepthError(f"{rt}:{rid}#{at}")
                kids.append(self.expand(st, sid, e[2], depth + 1))
            else:
                kids.append(_node("L", rt, rid, at))
        return _node("U", rt, rid, at, children=kids)


def expand_tree(mo, rt, rid, name, now=0, order=None):
    """Expand(rt:rid, name) over MiniOracle `mo` at clock `now`; raises DepthError."""
    return Expander(mo, now, order).expand(rt, rid, name)


def contains(tree, st, sid, check):
    """Whether the tree grants the plain subject st:sid. check(ut, uid, urel) -> Check(ut:uid#urel @ st:sid) == HAS."""
    op = tree["op"]
    if op == "L":
        for x in tree["subjects"]:
            t, rest = x.split(":", 1)
            i, _, rel = rest.partition("#")
            if t == st and (i == sid or i == "*") and not rel:
                return True
            if rel and check(t, i, rel):
                return True
        return False
    kids = [contains(c, st, sid, check) for c in tree["children"]]
    if op == "U":
        return any(kids)
    if op == "I":
        return all(kids)
    return kids[0] and not any(kids[1:])


def lines(tree, depth=0):
    """The string form's lines of a tree (pre-order, children in order)."""
    out = [" ".join([str(depth), tree["op"], f"{tree['object']}#{tree['relation']}"] + tree["subjects"])]
    for c in tree["children"]:
        out += lines(c, depth + 1)
    return out


def canonical(tree):
    """The tree with every leaf's subjects and every union's children sorted by their text: independent of id order."""
    kids = [canonical(c) for c in tree["children"]]
    if tree["op"] == "U":
        kids.sort(key=lambda c: "\n".join(lines(c)))
    return {**tree, "subjects": sorted(tree["subjects"]), "children": kids}


class GroupRows:
    """The rows of relationship groups of dense ids in the shape Expander reads from MiniOracle, found by binary search:
    a sample of trees of a full-size store without a copy of it in Python objects. groups: workloads.RelGroup, or the
    (res_type, rel, subj_type, res, subj, srel or "*", expirations or None) tuples of randgen.shaped_relationships.
    Object ids are the decimal strings of the dense ids; use order=group_order."""

    def __init__(self, schema, groups):
        import numpy as np

        from oracle.mini_oracle import parse_schema

        self.defs = parse_schema(schema)
        self.index = {}
        for g in groups:
            if isinstance(g, tuple):
                rt, rel, st, res, subj, srel, ex = g
            else:
                rt, rel, st, res, subj, srel, ex = g.res_type, g.rel, g.subj_type, g.res, g.subj, g.srel, None
                srel = "*" if g.wildcard else srel
            o = np.argsort(res, kind="stable")
            ex = np.zeros(res.size, np.uint32) if ex is None else np.asarray(ex, np.uint32)
            self.index.setdefault((rt, rel), []).append((res[o], subj[o], ex[o], st, srel or None))

    def _live(self, rt, rid, rl, now):
        import numpy as np

        out = set()
        for res, subj, ex, st, srel in self.index.get((rt, rl), []):
            if not rid.isdigit():
                continue
            lo, hi = np.searchsorted(res, int(rid), "left"), np.searchsorted(res, int(rid), "right")
            for s, x in zip(subj[lo:hi], ex[lo:hi]):
                if x == 0 or now == 0 or x > now:
                    out.add((st, "*", None) if srel == "*" else (st, str(int(s)), srel))
        return list(out)


def group_order(t, i):
    return -1 if i == "*" else int(i)


def id_tree_lines(tree, depth=0):
    """Engine.expand_permission_trees' tree (dense ids) -> the string form's lines, objects named by their ids."""
    subs = [f"{t}:" + ("*" if r == "*" else f"{i}" + (f"#{r}" if r else "")) for t, i, r in tree["subjects"]]
    out = [" ".join([str(depth), tree["op"], f"{tree['type']}:{tree['object']}#{tree['relation']}"] + subs)]
    for c in tree["children"]:
        out += id_tree_lines(c, depth + 1)
    return out
