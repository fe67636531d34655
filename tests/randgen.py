"""Random Zanzibar schemas + relationship graphs for cross-checking implementations.

Used by: test_oracle_random.py (C oracle vs pure-Python oracle) and the GPU parity
tests (CUDA engine vs C oracle). Everything is seeded and deterministic.

Data is generated so that recursive usersets / arrows are ACYCLIC (edges go from a
higher object index to a lower one): forward evaluation with the reference's
cache-off configuration (pkg/spicedb/spicedb.go:44-46) is exponential on cyclic
data up to the depth cap. Cycles and the depth cap get their own small tests.
"""
from __future__ import annotations

import random

FIXED_SCHEMAS = {
    # SURVEY.md 8(d) cfg3
    "nesting": """
definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member | user }
definition namespace {
  relation viewer: team#member | user
  permission view = viewer
}
""",
    # SURVEY.md 8(d) cfg4
    "docs": """
definition user {}
definition group { relation member: user | group#member }
definition org { relation member: user | group#member }
definition folder {
  relation parent: folder
  relation owner: user | group#member
  relation viewer: user | group#member
  permission view = viewer + owner + parent->view
}
definition document {
  relation parent: folder
  relation org: org
  relation owner: user | group#member | user:*
  relation editor: user | group#member | user:*
  relation viewer: user | group#member | user:*
  relation banned: user
  permission edit = owner + editor
  permission view = (viewer + edit + parent->view) - banned
  permission restricted_view = view & org->member
}
""",
    # non-pure permissions reached THROUGH arrows and usersets (sub-query passes)
    "deep_nonpure": """
definition user {}
definition group {
  relation member: user | group#member | group#active
  relation suspended: user
  permission active = member - suspended
}
definition folder {
  relation parent: folder
  relation viewer: user | group#active | group#member
  relation banned: user | group#member
  relation auditor: user
  permission view = (viewer + parent->view) - banned
  permission audit = auditor & view
  permission any = view + audit + parent->audit
}
definition document {
  relation folder: folder
  relation reader: user | folder#view | group#active
  permission read = reader + folder->view
  permission strict = folder->audit & reader
  permission nobody = nil
  permission weird = (read - folder->audit) + strict
}
""",
}


def random_schema(rng: random.Random):
    """-> (schema_text, model) where model describes types for data generation."""
    n_types = rng.randint(2, 4)
    tnames = [f"t{i}" for i in range(n_types)]
    perm_pool = ["p0", "p1", "p2"]
    types = {}
    for ti, t in enumerate(tnames):
        rels = {}
        for ri in range(rng.randint(1, 3)):
            allowed = []
            if rng.random() < 0.8:
                allowed.append(("user", None))
            if rng.random() < 0.25:
                allowed.append(("user", "*"))
            for _ in range(rng.randint(0, 2)):
                ot = rng.choice(tnames)
                allowed.append((ot, "?"))  # subject relation resolved below
            if not allowed:
                allowed.append(("user", None))
            rels[f"r{ri}"] = allowed
        # tupleset relations (object subjects of another type, no relation)
        for ai in range(rng.randint(0, 2)):
            rels[f"a{ai}"] = [(rng.choice(tnames), None)]
        types[t] = {"rels": rels, "perms": {}}
    # permissions: expressions over relations, earlier permissions, arrows
    for t in tnames:
        d = types[t]
        names_so_far = list(d["rels"].keys())
        arrows = [r for r in d["rels"] if r.startswith("a")]
        for p in perm_pool[: rng.randint(1, 3)]:
            def leaf():
                x = rng.random()
                if arrows and x < 0.3:
                    return f"{rng.choice(arrows)}->{rng.choice(perm_pool + ['r0'])}"
                if x < 0.35:
                    return "nil"
                return rng.choice(names_so_far)

            def expr(depth):
                if depth == 0 or rng.random() < 0.35:
                    return leaf()
                op = rng.choice(["+", "+", "&", "-"])
                return f"({expr(depth - 1)} {op} {expr(depth - 1)})"

            d["perms"][p] = expr(rng.randint(1, 3))
            names_so_far.append(p)
    # resolve userset subject relations: any relation/permission of the subject type
    for t in tnames:
        for r, allowed in types[t]["rels"].items():
            out = []
            for (ot, sr) in allowed:
                if sr == "?":
                    cands = list(types[ot]["rels"].keys()) + list(types[ot]["perms"].keys())
                    sr = rng.choice(cands)
                if (ot, sr) not in out:
                    out.append((ot, sr))
            types[t]["rels"][r] = out
    lines = ["definition user {}"]
    for t in tnames:
        lines.append(f"definition {t} {{")
        for r, allowed in types[t]["rels"].items():
            parts = [ot + (":*" if sr == "*" else (f"#{sr}" if sr else "")) for ot, sr in allowed]
            lines.append(f"  relation {r}: {' | '.join(parts)}")
        for p, e in types[t]["perms"].items():
            lines.append(f"  permission {p} = {e}")
        lines.append("}")
    return "\n".join(lines) + "\n", {"types": types, "tnames": tnames}


def model_from_schema(schema_text):
    """Derive the data-generation model from schema text (uses the mini parser)."""
    from oracle.mini_oracle import parse_schema

    defs = parse_schema(schema_text)
    types = {}
    for t, d in defs.items():
        rels = {r: [(st, sr) for (st, sr, _ex) in allowed] for r, allowed in d["relations"].items()}
        types[t] = {"rels": rels, "perms": {p: None for p in d["permissions"]}}
    return {"types": types, "tnames": [t for t in types]}


def random_relationships(rng: random.Random, model, n_obj=6, n_user=6, density=0.35, acyclic=True):
    """-> sorted list of relationship strings. Object ids are o0..o{n-1}, users u0.."""
    rels = set()
    for t, d in model["types"].items():
        for r, allowed in d["rels"].items():
            for (st, sr) in allowed:
                for oi in range(n_obj):
                    if sr == "*":
                        if rng.random() < density * 0.3:
                            rels.add(f"{t}:o{oi}#{r}@{st}:*")
                        continue
                    n_subj = n_user if st == "user" else n_obj
                    for si in range(n_subj):
                        if rng.random() >= density / (1 if st == "user" else 1.5):
                            continue
                        if st != "user" and acyclic and si >= oi:
                            continue  # edges only point to strictly lower indices
                        sname = f"u{si}" if st == "user" else f"o{si}"
                        rels.add(f"{t}:o{oi}#{r}@{st}:{sname}" + (f"#{sr}" if sr else ""))
    return sorted(rels)


def random_checks(rng: random.Random, model, n, n_obj=6, n_user=6):
    """-> list of 'type:id#perm@stype:sid[#srel]' (some with userset subjects,
    some naming unknown objects)."""
    out = []
    tn = [t for t in model["tnames"] if model["types"][t]["rels"] or model["types"][t]["perms"]]
    for _ in range(n):
        t = rng.choice(tn)
        d = model["types"][t]
        name = rng.choice(list(d["rels"].keys()) + list(d["perms"].keys()))
        oid = f"o{rng.randint(0, n_obj)}"  # o{n_obj} never written: unknown object
        if rng.random() < 0.85 or not tn:
            subj = f"user:u{rng.randint(0, n_user)}"
        else:
            st = rng.choice(tn)
            sd = model["types"][st]
            sr = rng.choice(list(sd["rels"].keys()) + list(sd["perms"].keys()))
            subj = f"{st}:o{rng.randint(0, n_obj - 1)}#{sr}"
        out.append(f"{t}:{oid}#{name}@{subj}")
    return out


# ---- shaped schemas: step kinds built on purpose, stores with counts at the check kernel's thresholds ----------------
#
# random_schema draws operators blindly, and random_relationships fills 4-9 objects per type: no row reaches the sizes at
# which the check kernel (csrc/kernels.cuh) changes path. shaped_schema composes a schema from named units, each built
# to compile into one step kind (csrc/schema.cc Schema::blob), and shaped_relationships fills it with rows whose sizes sit
# on either side of the kernel's limits. Ids are numeric (the add_bulk surface of the engine, the emulator and the
# oracle); userset and arrow edges are layered, so the oracle's cost per check is bounded by the product of fan-outs.

RSET_CAP = 16       # kernels.cuh kRsetCap: memberships the per-check set holds
FCAP = 64           # kernels.cuh kFCap: the largest range batch_l2 meets without an index
MAX_CLOSURE = 4     # kernels.cuh kMaxClosure: closure indexes per snapshot
MAX_INV_CLASSES = 11  # kernels.cuh kMaxInvClasses
PAIR_TYPES = ("team", "org", "club", "guild", "band")
RANGE_SIZES = (1, 4, 5, 15, 16, 17, 31, 32, 33, 63, 64, 65, 200)
CLOSURE_SIZES = (1, 15, 16, 17, 31, 32, 33)
# memberships of a user over its invertible classes (group#member, role#member, folder#viewer), in that order
MEMBERSHIP_SPLITS = ((0,), (1,), (4,), (15,), (16,), (17,), (8, 8), (8, 9), (10, 7), (6, 5, 5), (6, 6, 5), (5, 10, 2), (30,))
WIDE_OFFSET = 70000  # pair-type ids past 65 536: the closure index takes 32-bit entries


def shaped_schema(rng: random.Random, n_pairs=None, expiry=None, wildcard=None):
    """-> (schema_text, plan). plan["kinds"] lists the step kinds the schema was built to contain; plan["pairs"] the
    types of its two-level pairs (PAIR_TYPES[:n]), of which the first MAX_CLOSURE in step order can be indexed."""
    n_pairs = rng.randint(1, 5) if n_pairs is None else n_pairs
    expiry = rng.random() < 0.6 if expiry is None else expiry
    wildcard = rng.random() < 0.5 if wildcard is None else wildcard
    pairs = list(PAIR_TYPES[:n_pairs])
    kinds = ["direct_invertible_leaf", "noninvertible_probe", "leaf_push", "l2_push", "leaf_via_arrow", "l2_via_arrow",
             "union", "intersection", "exclusion", "rsetless_slot", "rsetless_exclusion", "nonpure_target",
             "two_subject_types", "folder_chain"]
    lines = ["use expiration" if expiry else "", "definition user {}", "definition bot {}",
             "definition group { relation member: user }", "definition role { relation member: user }",
             "definition crew { relation member: bot }"]
    lines += [f"definition {p} {{ relation member: group#member }}" for p in pairs]
    lines += ["definition folder {", "  relation parent: folder", "  relation viewer: user | group#member | team#member",
              "  relation banned: user"]
    if expiry:
        lines.append("  relation gx: group#member with expiration")
    lines += [f"  permission view = viewer + parent->view{' + gx' if expiry else ''}",
              "  permission strict = view - banned", "}"]
    idx = pairs[:MAX_CLOSURE]
    lines += ["definition doc {", "  relation folder: folder", "  relation grp: group", "  relation tm: team",
              "  relation owner: user | bot",
              f"  relation reader: group#member | role#member | crew#member{' | user:*' if wildcard else ''}",
              f"  relation l2: {' | '.join(p + '#member' for p in idx)}", "  relation banned: group#member",
              "  relation sub: folder#strict"]
    perms = ["arrow_leaf = grp->member", "arrow_l2 = tm->member", "only_l2 = l2",
             "view = owner + reader + l2 + arrow_leaf + arrow_l2 + folder->view", "both = reader & l2",
             "minus = l2 - banned", "minus_rsetless = l2 - arrow_l2", "nonpure_target = sub + reader"]
    if n_pairs > MAX_CLOSURE:
        lines.append(f"  relation l2x: {pairs[MAX_CLOSURE]}#member")
        perms.append("with5 = l2 + l2x")
        kinds.append("unindexed_fifth_pair")
    if expiry:
        lines.append("  relation exp: group#member with expiration | user with expiration")
        perms.append("timed = exp + reader")
        kinds.append("expiring_push")
    if wildcard:
        kinds.append("wildcard")
    lines += [f"  permission {p}" for p in perms] + ["}"]
    text = "\n".join(l for l in lines if l) + "\n"
    perm_names = [p.split(" = ")[0] for p in perms]
    # pure permissions only (one launch of the kernel answers them); doc.nonpure_target reaches folder#strict
    pure = [p for p in perm_names if p not in ("both", "minus", "minus_rsetless", "nonpure_target")]
    rsetless = ["only_l2", "minus_rsetless"]
    return text, {"kinds": kinds, "pairs": pairs, "expiry": expiry, "wildcard": wildcard, "perms": perm_names,
                  "pure": pure, "rsetless": rsetless}


def _distinct(rng, n, k):
    return sorted(rng.sample(range(n), min(n, k)))


def shaped_relationships(rng: random.Random, model, plan, n_user=3000, n_bot=300, n_group=600, n_crew=200, n_pair=150,
                         n_folder=60, n_doc=400, wide=False, now=1000):
    """-> store dict: "groups" [(res_type, rel, subj_type, res, subj, srel, expires)] (numpy arrays; expires None or
    per-tuple deadlines, 0 = never), the counts per type, and the buckets the checks draw from:
      * "split": user -> its memberships per invertible class (MEMBERSHIP_SPLITS, cycled over the users);
      * "closure": user -> its closure row's length for every pair type (CLOSURE_SIZES: one private group each, in
        that many objects of every pair type, and no other group);
      * "range": doc -> its row sizes of reader and l2 (RANGE_SIZES);
      * doc 0's owner row lists two thirds of the users (2 000 at the default size: the probe's binary search).
    Userset and arrow edges are layered: folder i's parent is a folder > i; docs, pair types and groups form layers."""
    assert set(plan["pairs"]) <= set(model["types"])
    groups = []

    def add(rt, rel, st, res, subj, srel=None, expires=None):
        import numpy as np

        res, subj = np.asarray(res, dtype=np.uint32), np.asarray(subj, dtype=np.uint32)
        if res.size:
            groups.append((rt, rel, st, res, subj, srel, None if expires is None else np.asarray(expires, np.uint32)))

    off = WIDE_OFFSET if wide else 0
    # closure users: one private group each and no shared group, so that the group's pair-type objects are exactly
    # the user's closure row (CLOSURE_SIZES[k] entries for every pair type). They are the last users, in 16 rounds of
    # CLOSURE_SIZES: a round's rows hold 145 = 1 (mod 16) entries, so each size's row starts at every offset mod 16.
    n_private = len(CLOSURE_SIZES) * 16
    n_shared = n_group - n_private
    closure = {n_user - n_private + i: CLOSURE_SIZES[i % len(CLOSURE_SIZES)] for i in range(n_private)}
    # group#member@user and role#member@user by the membership buckets; folder#viewer@user is the third class
    gm, rm, fv = [], [], []
    split = {}
    for u in range(n_user):
        s = MEMBERSHIP_SPLITS[u % len(MEMBERSHIP_SPLITS)] if u % 3 else (rng.choice((0, 1, 2, 3)),)
        s = tuple(s) + (0,) * (3 - len(s))
        if u in closure:
            s = (0,) + s[1:]
        split[u] = s
        gm += [(g, u) for g in _distinct(rng, n_shared, s[0])]
        rm += [(r, u) for r in _distinct(rng, n_group // 4, s[1])]
        fv += [(f, u) for f in _distinct(rng, n_folder, s[2])]
    pm = []
    for i, u in enumerate(sorted(closure)):
        g = n_shared + i
        gm.append((g, u))
        split[u] = (1,) + split[u][1:]
        for p in plan["pairs"]:
            pm += [(p, t, g) for t in _distinct(rng, n_pair, closure[u])]
    gm.sort()
    add("group", "member", "user", [g for g, _ in gm], [u for _, u in gm])
    add("role", "member", "user", [r for r, _ in rm], [u for _, u in rm])
    add("crew", "member", "bot", [rng.randrange(n_crew) for _ in range(4 * n_bot)], [rng.randrange(n_bot) for _ in range(4 * n_bot)])
    for p in plan["pairs"]:
        rows = [(t, g) for t in range(n_pair) for g in _distinct(rng, n_shared, rng.choice((1, 2, 3, 5, 8, 17)))]
        rows += [(t, g) for (q, t, g) in pm if q == p]
        add(p, "member", "group", [t + off for t, _ in rows], [g for _, g in rows], "member")
    # folders: a parent chain (layered), viewers of each class
    par = [(f, f + rng.choice((1, 2, 3))) for f in range(n_folder) if rng.random() < 0.8]
    par = [(a, b) for a, b in par if b < n_folder]
    add("folder", "parent", "folder", [a for a, _ in par], [b for _, b in par])
    fv.sort()
    add("folder", "viewer", "user", [f for f, _ in fv], [u for _, u in fv])
    fg = [(f, g) for f in range(n_folder) for g in _distinct(rng, n_group, rng.choice(RANGE_SIZES[:6]))]
    add("folder", "viewer", "group", [f for f, _ in fg], [g for _, g in fg], "member")
    ft = [(f, t) for f in range(n_folder) for t in _distinct(rng, n_pair, rng.choice(RANGE_SIZES[:9]))]
    add("folder", "viewer", "team", [f for f, _ in ft], [t + off for _, t in ft], "member")
    add("folder", "banned", "user", [rng.randrange(n_folder) for _ in range(200)], [rng.randrange(n_user) for _ in range(200)])
    # docs: ranges of every size in RANGE_SIZES, over groups / roles / crews (reader) and pair types (l2)
    # every class of a step has its own range: reader's groups and the first pair's objects take the sizes in turn
    rng_rows = {}
    rd = {"group": [], "role": [], "crew": []}
    l2 = {p: [] for p in plan["pairs"]}
    n_of = {"group": n_group, "role": n_group // 4, "crew": n_crew}
    for d in range(n_doc):
        a, b = RANGE_SIZES[d % len(RANGE_SIZES)], RANGE_SIZES[(d * 7 + 3) % len(RANGE_SIZES)]
        rng_rows[d] = (a, b)
        for st, k in (("group", a), ("role", rng.choice(RANGE_SIZES[:4])), ("crew", rng.choice(RANGE_SIZES[:7]))):
            rd[st] += [(d, x) for x in _distinct(rng, n_of[st], k if st == "group" or rng.random() < 0.5 else 0)]
        for i, p in enumerate(plan["pairs"]):
            k = b if i == 0 else rng.choice(RANGE_SIZES)
            l2[p] += [(d, t) for t in _distinct(rng, n_pair, k if i == 0 or rng.random() < 0.4 else 0)]
    for st, rows in rd.items():
        add("doc", "reader", st, [d for d, _ in rows], [x for _, x in rows], "member")
    for i, p in enumerate(plan["pairs"]):
        rows = l2[p]
        add("doc", "l2x" if i >= MAX_CLOSURE else "l2", p, [d for d, _ in rows], [t + off for _, t in rows], "member")
    if plan["wildcard"]:
        w = _distinct(rng, n_doc, n_doc // 20)
        add("doc", "reader", "user", w, [0] * len(w), "*")  # srel "*": the wildcard user:*
    add("doc", "folder", "folder", list(range(n_doc)), [rng.randrange(n_folder) for _ in range(n_doc)])
    add("doc", "grp", "group", [rng.randrange(n_doc) for _ in range(n_doc)], [rng.randrange(n_group) for _ in range(n_doc)])
    add("doc", "tm", "team", [rng.randrange(n_doc) for _ in range(n_doc)], [rng.randrange(n_pair) + off for _ in range(n_doc)])
    add("doc", "banned", "group", [rng.randrange(n_doc) for _ in range(n_doc)], [rng.randrange(n_group) for _ in range(n_doc)],
        "member")
    big = _distinct(rng, n_user, max(n_user * 2 // 3, 1))
    ow = [(0, u) for u in big] + [(rng.randrange(1, n_doc), rng.randrange(n_user)) for _ in range(n_doc)]
    ow = sorted(set(ow))
    add("doc", "owner", "user", [d for d, _ in ow], [u for _, u in ow])
    add("doc", "owner", "bot", [rng.randrange(n_doc) for _ in range(50)], [rng.randrange(n_bot) for _ in range(50)])
    add("doc", "sub", "folder", [rng.randrange(n_doc) for _ in range(n_doc)], [rng.randrange(n_folder) for _ in range(n_doc)],
        "strict")
    if plan["expiry"]:
        n = 4 * n_doc
        ex = [rng.choice((0, now - 500, now + 500)) for _ in range(n)]
        add("doc", "exp", "group", [rng.randrange(n_doc) for _ in range(n)], [rng.randrange(n_group) for _ in range(n)],
            "member", ex)
        add("doc", "exp", "user", [rng.randrange(n_doc) for _ in range(n)], [rng.randrange(n_user) for _ in range(n)], None, ex)
        add("folder", "gx", "group", [rng.randrange(n_folder) for _ in range(n_folder)],
            [rng.randrange(n_group) for _ in range(n_folder)], "member", [rng.choice((0, now + 500)) for _ in range(n_folder)])
    return {"groups": _dedup(groups), "n": {"user": n_user, "bot": n_bot, "group": n_group, "role": n_group // 4,
                                            "crew": n_crew, "folder": n_folder, "doc": n_doc,
                                            **{p: n_pair + off for p in plan["pairs"]}},
            "split": split, "closure": closure, "range": rng_rows, "now": now, "off": off, "pairs": list(plan["pairs"])}


def _dedup(groups):
    """One tuple per (res, subj) in a group: duplicates would load as one relationship with either deadline."""
    import numpy as np

    out = []
    for rt, rel, st, res, subj, srel, ex in groups:
        _, keep = np.unique(np.stack([res, subj], axis=1), axis=0, return_index=True)
        keep.sort()
        out.append((rt, rel, st, res[keep], subj[keep], srel, None if ex is None else ex[keep]))
    return out


def load_shaped(t, store):
    """Loads a shaped store into an engine, the emulator (add_bulk / load_tuples) or the oracle (add_bulk / write_ids)."""
    import numpy as np

    for rt, rel, st, res, subj, srel, ex in store["groups"]:
        if ex is None:
            t.add_bulk(rt, rel, st, res, subj, srel=None if srel == "*" else srel, wildcard=srel == "*")
        elif hasattr(t, "load_tuples"):
            tup = np.zeros(res.size, dtype=[("res", "<u4"), ("subj", "<u4"), ("rel", "<u2"), ("stype", "<u2"),
                                             ("srel", "<u2"), ("flags", "<u2")])
            tup["res"], tup["subj"], tup["rel"], tup["stype"] = res, subj, t.slot_id(rt, rel), t.type_id(st)
            tup["srel"] = 0xFFFF if srel is None else t.slot_id(st, srel)
            t.load_tuples(tup, ex)
        else:
            sr = 0xFFFF if srel is None else t.slot_id(st, srel)
            for a, b, x in zip(res.tolist(), subj.tolist(), ex.tolist()):
                t.write_ids(1, t.slot_id(rt, rel), a, t.type_id(st), b, sr, x)


def shaped_checks(rng, store, plan, n=20000):
    """-> (queries, res, subj): queries[i] = (res_type, perm, subj_type, srel or None) and numpy res / subj ids. Mixes
    users of every membership and closure bucket, never-written ids, bots, and userset subjects; shuffled, so that one
    warp's lanes take different meet kinds."""
    import numpy as np

    N = store["n"]
    by_split = {}
    for u, s in store["split"].items():
        by_split.setdefault(s, []).append(u)
    closure_users = sorted(store["closure"])
    doc_perms = plan["perms"] + ["reader", "l2", "owner"]
    q, res, subj = [], [], []
    for i in range(n):
        x = rng.random()
        if x < 0.78:
            if x < 0.3:
                u = rng.choice(by_split[rng.choice(sorted(by_split))])
            elif x < 0.45:
                u = rng.choice(closure_users)
            elif x < 0.5:
                u = N["user"] + rng.randrange(4)  # never written
            else:
                u = rng.randrange(N["user"])
            if rng.random() < 0.85:
                q.append(("doc", rng.choice(doc_perms), "user", None))
                res.append(rng.randrange(N["doc"] + 2))
            else:
                q.append(("folder", rng.choice(("view", "strict")), "user", None))
                res.append(rng.randrange(N["folder"]))
            subj.append(u)
        elif x < 0.88:
            q.append(("doc", rng.choice(doc_perms), "bot", None))
            res.append(rng.randrange(N["doc"]))
            subj.append(rng.randrange(N["bot"] + 2))
        elif x < 0.95:
            q.append(("doc", rng.choice(doc_perms), "group", "member"))
            res.append(rng.randrange(N["doc"]))
            subj.append(rng.randrange(N["group"]))
        else:
            p = rng.choice(plan["pairs"])
            q.append(("doc", rng.choice(doc_perms), p, "member"))
            res.append(rng.randrange(N["doc"]))
            subj.append(store["off"] + rng.randrange(N[p] - store["off"]))
    return q, np.asarray(res, dtype=np.uint32), np.asarray(subj, dtype=np.uint32)


def shaped_items(t, dtype, queries, res, subj):
    """CHECK_DTYPE items of shaped_checks' queries, with t's slot and type ids."""
    import numpy as np

    table = {}
    items = np.zeros(len(queries), dtype=dtype)
    for i, k in enumerate(queries):
        if k not in table:
            rt, perm, st, sr = k
            table[k] = (t.slot_id(rt, perm), t.type_id(st), 0xFFFF if sr is None else t.slot_id(st, sr))
        items["perm"][i], items["stype"][i], items["srel"][i] = table[k]
    items["res"], items["subj"] = res, subj
    return items


def closure_rows(store, pair):
    """From the generated data: the closure index of `pair` (row u = the objects of `pair` that user u's groups are
    members of, ascending) as (crow, list of rows), and the doc#l2 ranges of `pair` as (col, ptr)."""
    import numpy as np

    g = {(rt, rel, st): (res, subj) for rt, rel, st, res, subj, srel, ex in store["groups"]}
    gm_g, gm_u = g[("group", "member", "user")]
    pt, pg = g[(pair, "member", "group")]
    g2t = {}
    for t, x in zip(pt.tolist(), pg.tolist()):
        g2t.setdefault(x, set()).add(t)
    rows = [set() for _ in range(store["n"]["user"])]
    for x, u in zip(gm_g.tolist(), gm_u.tolist()):
        rows[u].update(g2t.get(x, ()))
    rows = [np.array(sorted(r), dtype=np.uint32) for r in rows]
    crow = np.zeros(len(rows) + 1, dtype=np.int64)
    crow[1:] = np.cumsum([r.size for r in rows])
    rel = "l2" if pair in PAIR_TYPES[:MAX_CLOSURE] else "l2x"
    lr, lt = g[("doc", rel, pair)]
    order = np.lexsort((lt, lr))
    lr, lt = lr[order], lt[order]
    ptr = np.searchsorted(lr, np.arange(store["n"]["doc"] + 1))
    return crow, rows, lt.astype(np.uint32), ptr
