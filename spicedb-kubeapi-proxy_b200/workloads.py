"""Synthetic Zanzibar-shaped workloads: SURVEY.md section 8(d) / BASELINE.md section 4.

Deterministic (numpy PCG64 seeded per config). Every generator returns a Workload:
schema text, relationship groups as dense u32 id arrays (loadable into the engine
AND the oracle with no string rendering), and a batch of checks. `scale` shrinks
every population proportionally so the parity tests run the same shapes at sizes the
CPU oracle finishes in seconds.

cfg1  bootstrap `namespace` schema (pkg/spicedb/bootstrap.yaml:6-15), 1 000 flat tuples
cfg2  pod#view = viewer + creator, 1M pod#viewer tuples, 100k pods x 10k users, batch 64k
cfg3  user -> group -> team -> namespace nesting, 10M tuples, batch 1M (3 hops)
cfg4  Zanzibar doc schema with + & - -> and user:*, 100M tuples
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

SREL_NONE = 0xFFFF


@dataclass
class RelGroup:
    res_type: str
    rel: str
    subj_type: str
    res: np.ndarray
    subj: np.ndarray
    srel: Optional[str] = None
    wildcard: bool = False


@dataclass
class CheckBatch:
    res_type: str
    perm: str
    subj_type: str
    res: np.ndarray
    subj: np.ndarray


@dataclass
class Workload:
    name: str
    schema: str
    groups: List[RelGroup]
    checks: List[CheckBatch]
    lookups: list = field(default_factory=list)  # [(res_type, perm, subj_type, subj_id)]
    note: str = ""

    def n_tuples(self):
        return int(sum(g.res.size for g in self.groups))

    def n_checks(self):
        return int(sum(c.res.size for c in self.checks))

    def load_into(self, target):
        """target: zgpu.Engine or oracle.pyoracle.Oracle (both expose add_bulk)."""
        for g in self.groups:
            target.add_bulk(g.res_type, g.rel, g.subj_type, g.res, g.subj, srel=g.srel, wildcard=g.wildcard)

    def check_items(self, target, dtype):
        """One interleaved item array (deterministic shuffle) using target's slot ids."""
        parts = []
        for c in self.checks:
            a = np.zeros(c.res.size, dtype=dtype)
            a["res"] = c.res
            a["subj"] = c.subj
            a["perm"] = target.slot_id(c.res_type, c.perm)
            a["stype"] = target.type_id(c.subj_type)
            a["srel"] = SREL_NONE
            parts.append(a)
        items = np.concatenate(parts) if len(parts) > 1 else parts[0]
        if len(parts) > 1:
            items = items[np.random.Generator(np.random.PCG64(99)).permutation(items.size)]
        return items


BOOTSTRAP_SCHEMA = """use expiration

definition cluster {}
definition user {}
definition namespace {
  relation cluster: cluster
  relation creator: user
  relation viewer: user

  permission admin = creator
  permission edit = creator
  permission view = viewer + creator
  permission no_one_at_all = nil
}
definition pod {
  relation namespace: namespace
  relation creator: user
  relation viewer: user
  permission edit = creator
  permission view = viewer + creator
}
definition testresource {
  relation namespace: namespace
  relation creator: user
  relation viewer: user
  permission edit = creator
  permission view = viewer + creator
}
definition lock {
  relation workflow: workflow
}

definition workflow {
  relation idempotency_key: activity with expiration
}

definition activity{}
"""

CFG2_SCHEMA = """definition user {}
definition pod {
  relation viewer: user
  relation creator: user
  permission view = viewer + creator
}
"""

CFG3_SCHEMA = """definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member | user }
definition namespace {
  relation viewer: team#member | user
  permission view = viewer
}
"""

CFG4_SCHEMA = """definition user {}
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
"""


def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed))


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def cfg1(seed=1) -> Workload:
    """1 000 flat namespace#viewer tuples; single checks, 50 % present."""
    r = _rng(seed)
    pairs = r.permutation(100 * 10)[:1000]
    ns, us = _u32(pairs // 10), _u32(pairs % 10)
    # 100 x 10 = 1000 distinct pairs = every pair; keep half so 50 % of checks are present
    keep = r.random(1000) < 0.5
    g = RelGroup("namespace", "viewer", "user", ns[keep], us[keep])
    q = r.permutation(1000)
    c = CheckBatch("namespace", "view", "user", _u32(q // 10), _u32(q % 10))
    return Workload("cfg1", BOOTSTRAP_SCHEMA, [g], [c], note="bootstrap schema, 1k flat tuples (CPU-runnable case)")


def cfg2(seed=2, scale=1.0, zipf=False, batch=65536) -> Workload:
    r = _rng(seed)
    n_pods, n_users, n_t = max(int(100_000 * scale), 16), max(int(10_000 * scale), 8), max(int(1_000_000 * scale), 64)
    pods = r.integers(0, n_pods, n_t, dtype=np.uint32)
    if zipf:
        z = r.zipf(1.1, n_t)
        users = _u32((z - 1) % n_users)
    else:
        users = r.integers(0, n_users, n_t, dtype=np.uint32)
    g = RelGroup("pod", "viewer", "user", pods, users)
    nb = max(int(batch * min(scale * 4, 1.0)), 64) if scale < 1 else batch
    half = nb // 2
    pick = r.integers(0, n_t, half)
    res = np.concatenate([pods[pick], r.integers(0, n_pods, nb - half, dtype=np.uint32)])
    sub = np.concatenate([users[pick], r.integers(0, n_users, nb - half, dtype=np.uint32)])
    perm = r.permutation(nb)
    c = CheckBatch("pod", "view", "user", _u32(res[perm]), _u32(sub[perm]))
    lookups = [("pod", "view", "user", int(u)) for u in r.integers(0, n_users, 16)]
    return Workload("cfg2" + ("-zipf" if zipf else ""), CFG2_SCHEMA, [g], [c], lookups,
                    note=f"1-hop pod#view, {n_t} tuples, {n_pods} pods x {n_users} users, batch {nb}")


def _sample_chain(r, keys_sorted, vals_sorted, starts):
    """For each start key pick a random value among rows with that key (key-sorted arrays);
    returns (value, ok)."""
    lo = np.searchsorted(keys_sorted, starts, side="left")
    hi = np.searchsorted(keys_sorted, starts, side="right")
    ok = hi > lo
    pick = lo + (r.random(starts.size) * np.maximum(hi - lo, 1)).astype(np.int64)
    pick = np.minimum(pick, max(keys_sorted.size - 1, 0))
    return vals_sorted[pick], ok


def cfg3(seed=3, scale=1.0, batch=1 << 20) -> Workload:
    r = _rng(seed)
    n_users, n_groups = max(int(1_000_000 * scale), 32), max(int(100_000 * scale), 16)
    n_teams, n_ns = max(int(10_000 * scale), 8), max(int(100_000 * scale), 16)
    # fan-outs (80 users/group, 100 groups/team, 10 teams/namespace at full size) shrink with
    # the populations, so scaled-down graphs keep a mix of reachable and unreachable pairs
    gpt = max(2, min(100, n_groups // 100))
    tpn = max(2, min(10, n_teams // 10))
    n_gm, n_tm, n_nv = max(int(8_000_000 * scale), 128), n_teams * gpt, n_ns * tpn
    gm_g = r.integers(0, n_groups, n_gm, dtype=np.uint32)
    gm_u = r.integers(0, n_users, n_gm, dtype=np.uint32)
    tm_t = r.integers(0, n_teams, n_tm, dtype=np.uint32)
    tm_g = r.integers(0, n_groups, n_tm, dtype=np.uint32)
    nv_n = r.integers(0, n_ns, n_nv, dtype=np.uint32)
    nv_t = r.integers(0, n_teams, n_nv, dtype=np.uint32)
    groups = [
        RelGroup("group", "member", "user", gm_g, gm_u),
        RelGroup("team", "member", "group", tm_t, tm_g, srel="member"),
        RelGroup("namespace", "viewer", "team", nv_n, nv_t, srel="member"),
    ]
    nb = batch if scale >= 1 else max(int(batch * scale), 256)
    half = nb // 2
    # reachable half: namespace -> team -> group -> user along stored edges
    pick = r.integers(0, n_nv, half)
    ns, team = nv_n[pick], nv_t[pick]
    o = np.argsort(tm_t, kind="stable")
    grp, ok1 = _sample_chain(r, tm_t[o], tm_g[o], team)
    o2 = np.argsort(gm_g, kind="stable")
    usr, ok2 = _sample_chain(r, gm_g[o2], gm_u[o2], grp)
    usr = np.where(ok1 & ok2, usr, r.integers(0, n_users, half, dtype=np.uint32))
    res = np.concatenate([ns, r.integers(0, n_ns, nb - half, dtype=np.uint32)])
    sub = np.concatenate([usr, r.integers(0, n_users, nb - half, dtype=np.uint32)])
    perm = r.permutation(nb)
    c = CheckBatch("namespace", "view", "user", _u32(res[perm]), _u32(sub[perm]))
    lookups = [("namespace", "view", "user", int(u)) for u in r.integers(0, n_users, 8)]
    return Workload("cfg3", CFG3_SCHEMA, groups, [c], lookups,
                    note=f"3-hop nesting, {n_gm + n_tm + n_nv} tuples, batch {nb}")


# cfg4 with a NON-PURE folder#view: every document -> folder arrow then leads into a permission with `-`, so
# each check raises sub-queries pass after pass up the folder chain (tests of the multi-pass machinery on a
# store of the same size and shape; not a BASELINE configuration).
CFG4X_SCHEMA = CFG4_SCHEMA.replace(
    "  relation viewer: user | group#member\n  permission view = viewer + owner + parent->view\n",
    "  relation viewer: user | group#member\n  relation banned: user\n"
    "  permission view = (viewer + owner + parent->view) - banned\n")
assert CFG4X_SCHEMA != CFG4_SCHEMA


def cfg4(seed=4, scale=1.0, batch=1 << 20, nonpure_folders=False) -> Workload:
    """Doc-style schema; `scale`=1.0 is the 100M-tuple configuration."""
    r = _rng(seed)
    N = 100_000_000 * scale
    nz = lambda x, lo=8: max(int(x), lo)
    U, G, O = nz(N / 20), nz(N / 200), nz(1000 * min(1.0, scale * 100), 4)
    F, D = nz(N / 20), nz(N * 0.15)

    def ints(hi, n):
        return r.integers(0, hi, nz(n, 4), dtype=np.uint32)

    groups: List[RelGroup] = []
    gm_g, gm_u = ints(G, 0.18 * N), None
    gm_u = ints(U, gm_g.size)
    groups.append(RelGroup("group", "member", "user", gm_g, gm_u))
    # nested groups, three tiers (ids ascending by tier): tier-1 groups (25 %) include 1-2
    # tier-0 groups, tier-2 groups (5 %) include 1-2 tier-1 groups. Acyclic, depth <= 2,
    # path multiplicity <= 4: forward evaluation without result caching
    # (pkg/spicedb/spicedb.go:44-46) is exponential in the multiplicity of deeper DAGs.
    t0, t1 = int(G * 0.70), int(G * 0.95)
    par, chi = [], []
    for lo, hi, clo, chi_hi in ((t0, t1, 0, t0), (t1, G, t0, t1)):
        if hi > lo and chi_hi > clo:
            ids = np.arange(lo, hi, dtype=np.int64)
            for _rep in range(2):
                take = ids if _rep == 0 else ids[r.random(ids.size) < 0.5]
                par.append(take)
                chi.append(r.integers(clo, chi_hi, take.size))
    if par:
        groups.append(RelGroup("group", "member", "group", _u32(np.concatenate(par)), _u32(np.concatenate(chi)),
                               srel="member"))
    groups.append(RelGroup("org", "member", "user", ints(O, 0.02 * N), ints(U, nz(0.02 * N, 4))))
    groups.append(RelGroup("org", "member", "group", ints(O, 0.005 * N), ints(G, nz(0.005 * N, 4)), srel="member"))
    # folders: 6 levels, level l parents live in level l-1 (ids ascending by level)
    lvl = np.linspace(0, F, 7).astype(np.int64)
    f_child, f_parent = [], []
    for l in range(1, 6):
        ids = np.arange(lvl[l], lvl[l + 1], dtype=np.int64)
        if ids.size == 0 or lvl[l] == lvl[l - 1]:
            continue
        f_child.append(ids)
        f_parent.append(r.integers(lvl[l - 1], lvl[l], ids.size))
    if f_child:
        groups.append(RelGroup("folder", "parent", "folder", _u32(np.concatenate(f_child)), _u32(np.concatenate(f_parent))))
    fv_f, fv_u = ints(F, 0.05 * N), None
    fv_u = ints(U, fv_f.size)
    groups.append(RelGroup("folder", "viewer", "user", fv_f, fv_u))
    groups.append(RelGroup("folder", "viewer", "group", ints(F, 0.03 * N), ints(G, nz(0.03 * N, 4)), srel="member"))
    groups.append(RelGroup("folder", "owner", "user", ints(F, 0.02 * N), ints(U, nz(0.02 * N, 4))))
    d_parent = r.integers(0, F, D, dtype=np.uint32)
    groups.append(RelGroup("document", "parent", "folder", np.arange(D, dtype=np.uint32), d_parent))
    d_org = ints(D, 0.03 * N)
    groups.append(RelGroup("document", "org", "org", d_org, ints(O, d_org.size)))
    dv_d = ints(D, 0.15 * N)
    dv_u = ints(U, dv_d.size)
    groups.append(RelGroup("document", "owner", "user", ints(D, 0.15 * N), ints(U, nz(0.15 * N, 4))))
    groups.append(RelGroup("document", "viewer", "user", dv_d, dv_u))
    groups.append(RelGroup("document", "viewer", "group", ints(D, 0.05 * N), ints(G, nz(0.05 * N, 4)), srel="member"))
    groups.append(RelGroup("document", "editor", "user", ints(D, 0.05 * N), ints(U, nz(0.05 * N, 4))))
    wd = ints(D, 0.005 * N)
    groups.append(RelGroup("document", "viewer", "user", wd, np.zeros(wd.size, dtype=np.uint32), wildcard=True))
    groups.append(RelGroup("document", "banned", "user", ints(D, 0.02 * N), ints(U, nz(0.02 * N, 4))))

    nb = batch if scale >= 1 else max(int(batch * min(1.0, scale * 20)), 256)
    checks = []
    for perm, share in (("view", 0.75), ("restricted_view", 0.25)):
        n = max(int(nb * share), 64)
        a, b, c3 = n // 3, n // 3, n - 2 * (n // 3)
        # direct viewers, folder viewers of the document's parent, random pairs
        p1 = r.integers(0, dv_d.size, a)
        docs2 = r.integers(0, D, b, dtype=np.uint32)
        o = np.argsort(fv_f, kind="stable")
        u2, ok = _sample_chain(r, fv_f[o], fv_u[o], d_parent[docs2])
        u2 = np.where(ok, u2, r.integers(0, U, b, dtype=np.uint32))
        res = np.concatenate([dv_d[p1], docs2, r.integers(0, D, c3, dtype=np.uint32)])
        sub = np.concatenate([dv_u[p1], u2, r.integers(0, U, c3, dtype=np.uint32)])
        pm = r.permutation(n)
        checks.append(CheckBatch("document", perm, "user", _u32(res[pm]), _u32(sub[pm])))
    lookups = [("document", "view", "user", int(u)) for u in r.integers(0, U, 4)]
    if nonpure_folders:
        r2 = _rng(seed + 1000)
        nb_ = nz(0.005 * N, 4)
        groups.append(RelGroup("folder", "banned", "user", r2.integers(0, F, nb_, dtype=np.uint32),
                               r2.integers(0, U, nb_, dtype=np.uint32)))
        w = Workload("cfg4x", CFG4X_SCHEMA, groups, checks, lookups)
        w.note = f"cfg4 with a non-pure folder#view, {w.n_tuples()} tuples, batch {w.n_checks()}"
        return w
    w = Workload("cfg4", CFG4_SCHEMA, groups, checks, lookups)
    w.note = f"doc schema with + & - -> and user:*, {w.n_tuples()} tuples, batch {w.n_checks()}"
    return w


def object_name(type_name: str, i: int) -> str:
    """String id of dense object i in the named stores: users u%07d, pods ns%05d/p%07d (1 000 pods per namespace),
    every other type <type>%07d."""
    if type_name == "user":
        return "u%07d" % i
    if type_name == "pod":
        return "ns%05d/p%07d" % (i // 1000, i)
    return "%s%07d" % (type_name, i)


def object_counts(w: Workload) -> dict:
    """Per type: 1 + the largest object id the workload's relationships and checks name."""
    n = {}

    def see(t, ids):
        if ids.size:
            n[t] = max(n.get(t, 0), int(ids.max()) + 1)

    for g in w.groups:
        see(g.res_type, g.res)
        if not g.wildcard:
            see(g.subj_type, g.subj)
    for c in w.checks:
        see(c.res_type, c.res)
        see(c.subj_type, c.subj)
    return n


def intern_names(w: Workload, engine) -> int:
    """Gives every object of the workload its name (object_name), interned in id order BEFORE the relationships are
    loaded, so that each name's interned id is the dense id the workload uses. Returns the names interned."""
    total = 0
    for t, n in sorted(object_counts(w).items()):
        ids = engine.intern_packed(t, [object_name(t, i) for i in range(n)])
        assert ids.size == n and int(ids[0]) == 0 and int(ids[-1]) == n - 1, f"{t}: names did not intern in id order"
        total += n
    return total


def by_name(name: str, scale: float = 1.0, **kw) -> Workload:
    if name == "cfg1":
        return cfg1()
    if name == "cfg2":
        return cfg2(scale=scale, **kw)
    if name == "cfg2-zipf":
        return cfg2(scale=scale, zipf=True, **kw)
    if name == "cfg3":
        return cfg3(scale=scale, **kw)
    if name == "cfg4":
        return cfg4(scale=scale, **kw)
    raise ValueError(f"unknown workload {name}")
