"""What a published snapshot's closure indexes, signatures and set tables should hold, restated from the store's live
relationships alone (csrc/build.cu gpu_build_closure / _sig / _table, csrc/device.cu build_closures / finish_publish,
csrc/store.cc Store::layout).

A `Model` mirrors the relationships an engine holds and the object capacities its layouts handed out; `pairs` restates
the two-level pairs a program indexes, and `restate` each pair's index, budget decision, signatures and set table. The
signature and table restatements are the ones the emulator tests pin (np_signature, np_choose, np_table)."""
from __future__ import annotations

import numpy as np

from test_closure_set_emulation import np_choose, np_table
from test_closure_sig_emulation import np_signature

MAX_CLOSURE = 4       # kernels.cuh kMaxClosure
CLOSURE_RATIO = 16    # device.h kClosureRatio: entries before deduplication per relationship of the pair's classes
SIG_MAX_WORDS = 32    # build.cu gpu_build_closure_sig
NARROW = 65536        # ids of a target type whose capacity is at most this fit 16-bit entries


def next_capacity(cap, need):
    """Store::layout: a type's capacity grows only when it no longer holds `need` ids, and then with room to spare."""
    return min(need + need // 8 + 4096, 0xFFFFFFF0) if need > cap else cap


class Model:
    """Live relationships by class (res_type, rel, subj_type, subj_rel) -> {(res, subj): expires}, and per type the
    numeric id extent (max id + 1 ever inserted), the named id extent and the capacity of the last layout."""

    def __init__(self):
        self.rels = {}
        self.n_numeric, self.n_ids, self.cap = {}, {}, {}

    def _saw(self, t, i):
        self.n_numeric[t] = max(self.n_numeric.get(t, 0), int(i) + 1)

    def load(self, groups):
        """Bulk load of shaped groups (randgen.shaped_relationships): later duplicates win, every id counts."""
        for rt, rel, st, res, subj, srel, ex in groups:
            d = self.rels.setdefault((rt, rel, st, srel), {})
            exs = np.zeros(len(res), np.int64) if ex is None else ex
            for r, s, x in zip(np.asarray(res).tolist(), np.asarray(subj).tolist(), np.asarray(exs).tolist()):
                d[(r, 0 if srel == "*" else s)] = int(x)
                self._saw(rt, r)
                if srel != "*":
                    self._saw(st, s)

    def write(self, op, cls, res, subj, expires=0):
        """One TOUCH (op 0) or DELETE (op 2), as Store::apply: only an insert widens the numeric extents."""
        d = self.rels.setdefault(cls, {})
        k = (int(res), int(subj))
        if op == 2:
            d.pop(k, None)
            return
        if k not in d:
            self._saw(cls[0], res)
            self._saw(cls[2], subj)
        d[k] = int(expires)

    def named(self, t, i):
        """A name interned to id i of type t."""
        self.n_ids[t] = max(self.n_ids.get(t, 0), int(i) + 1)

    def collect(self, before):
        """collect_expired: every relationship whose expiration is set and <= before goes; returns how many."""
        n = 0
        for d in self.rels.values():
            gone = [k for k, x in d.items() if 0 < x <= before]
            for k in gone:
                del d[k]
            n += len(gone)
        return n

    def publish(self):
        """The capacities a publish's layout hands out; they never shrink."""
        for t in set(self.n_numeric) | set(self.n_ids):
            need = max(self.n_numeric.get(t, 0), self.n_ids.get(t, 0))
            self.cap[t] = next_capacity(self.cap.get(t, 0), need)

    def live(self, cls):
        return bool(self.rels.get(cls))

    def groups(self):
        """The live relationships as shaped groups (randgen.load_shaped loads them)."""
        out = []
        for (rt, rel, st, srel), d in sorted(self.rels.items(), key=lambda kv: tuple(str(x) for x in kv[0])):
            if not d:
                continue
            keys = sorted(d)
            res = np.array([k[0] for k in keys], np.uint32)
            subj = np.array([k[1] for k in keys], np.uint32)
            ex = np.array([d[k] for k in keys], np.uint32)
            out.append((rt, rel, st, res, subj, srel, ex if ex.any() else None))
        return out

    def expires_somewhere(self):
        return any(x for d in self.rels.values() for x in d.values())


def pairs(model, steps):
    """The indexed pairs of a publish: `steps` lists the program's two-level steps in step order as (via, inner, tgc)
    classes; a step exists while all three classes hold a relationship (an empty class vanishes from the program,
    csrc/schema.cc Schema::blob); pairs are deduplicated by tgc and capped at MAX_CLOSURE (finish_publish)."""
    out = []
    for via, inner, tgc in steps:
        if not (model.live(via) and model.live(inner) and model.live(tgc)):
            continue
        if any(t == tgc for _, t in out) or len(out) == MAX_CLOSURE:
            continue
        out.append((inner, tgc))
    return out


def closure_rows(model, inner, tgc):
    """Row u (u below the capacity of the inner class's subject type) = the union of rrow(g, tgc) over the groups g
    of rrow(u, inner), ascending and distinct; and the entries before deduplication."""
    n = model.cap[inner[2]]
    by_g = {}
    for t, g in model.rels.get(tgc, {}):
        by_g.setdefault(g, []).append(t)
    rows = [set() for _ in range(n)]
    pre = 0
    for g, u in model.rels.get(inner, {}):
        ts = by_g.get(g, ())
        pre += len(ts)
        rows[u].update(ts)
    return [np.array(sorted(r), dtype=np.uint32) for r in rows], pre


def sig_words(nsubj, entries):
    """gpu_build_closure_sig's default: the fewest words (a power of two, at most 32) with 64 x words x rows >= 12 x
    entries."""
    w = 1
    while w < SIG_MAX_WORDS and 64 * w * nsubj < 12 * entries:
        w <<= 1
    return w


_TABLES = {}


def _row_table(r):
    """np_table of one row, without its offset (cached by content: most rows outlive a write)."""
    key = r.tobytes()
    if key not in _TABLES:
        _TABLES[key] = None if np_choose(r.astype(np.int64)) is None else np_table([r.astype(np.int64)])
    return _TABLES[key]


def table(rows):
    """np_table over the rows, or None when some row cannot be placed within the bucket limit."""
    hdr, tabs, off = [], [], 0
    for r in rows:
        t = _row_table(r)
        if t is None:
            return None
        hdr.append(int(t[0][0]) + off)
        tabs.append(t[1])
        off += t[1].shape[0]
    return np.array(hdr, dtype=np.uint64), (np.concatenate(tabs) if tabs else np.zeros((0, 4), np.uint16))


def restate(model, pair_list, cap=None, tables=True):
    """Per pair of `pair_list` (model.publish() done): a dict with inner, tgc, built (False: over the budget), pre
    (entries before deduplication), budget, width, row_ptr, col, words, sig, table (None: no table)."""
    width = 4 if any(model.cap[tgc[0]] > NARROW for _, tgc in pair_list) else 2
    out = []
    for inner, tgc in pair_list:
        rows, pre = closure_rows(model, inner, tgc)
        rels = len(model.rels.get(inner, {})) + len(model.rels.get(tgc, {}))
        budget = CLOSURE_RATIO * rels if cap is None else cap
        p = {"inner": inner, "tgc": tgc, "pre": pre, "budget": budget, "built": pre <= budget, "width": width}
        if p["built"]:
            lens = np.array([r.size for r in rows], dtype=np.int64)
            p["row_ptr"] = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
            p["col"] = np.concatenate(rows).astype(np.uint32) if rows else np.zeros(0, np.uint32)
            p["words"] = sig_words(len(rows), int(lens.sum()))
            p["sig"] = np_signature(rows, p["words"])
            narrow = tables and width == 2 and model.cap[tgc[0]] < NARROW
            p["table"] = table(rows) if narrow else None
        out.append(p)
    return out


def counters(restated):
    """closure_index_counters' indexed / over_budget / entries of a restated publish."""
    built = [p for p in restated if p["built"]]
    return {"indexed": len(built), "over_budget": len(restated) - len(built),
            "entries": sum(int(p["col"].size) for p in built)}
