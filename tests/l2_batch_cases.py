"""Shared cases for the batched two-level meet (csrc/kernels.cuh batch_l2), under the emulator and on the GPU.

mixed_case(): warps whose lanes mix range sizes 1 .. 70 (beyond kFCap = 64 the range is walked), subjects with 1 .. 24
memberships (beyond kRsetCap = 16 the meet reads them from the subject's reverse row), checks answered by their first
range before the second is met, and lanes that do not meet at all (team#member checks).

collision_cases(): object ids that collide in the batched meet's 128-bit filter (same two bits), so that "the filter
lets it through" and "it is a child of the range" can be told apart. filter_bits() must restate kernels.cuh l2_bits.
"""
from collections import defaultdict

import numpy as np

SCHEMA = """definition user {}
definition group { relation member: user }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member
  relation editor: team#member
  permission view = viewer + editor
}"""
N_TEAMS, N_GROUPS = 400, 300
SIZES = [1, 2, 3, 7, 15, 16, 17, 27, 31, 32, 33, 63, 64, 65, 70]
MEMBERSHIPS = list(range(1, 25))


def mixed_case(seed=7):
    """Returns (groups, checks): groups = [(res_type, rel, subj_type, res, subj, srel)], checks = [(res_type, perm,
    res, subj)] with user ids u = 2 * k + r holding k memberships (r = 0, 1)."""
    rng = np.random.default_rng(seed)
    tm_res, tm_subj = [], []
    for g in range(N_GROUPS):  # every group sits in 1 .. 26 teams
        for t in rng.choice(N_TEAMS, 1 + g % 26, replace=False):
            tm_res.append(t), tm_subj.append(g)
    nv_res, nv_subj, ne_res, ne_subj = [], [], [], []
    for i, nf in enumerate(SIZES):
        for t in rng.choice(N_TEAMS, nf, replace=False):
            nv_res.append(i), nv_subj.append(t)
        for t in rng.choice(N_TEAMS, 1 + (i * 5) % 20, replace=False):  # a second range: editor
            ne_res.append(i), ne_subj.append(t)
    gm_res, gm_subj = [], []
    users = []
    for k in MEMBERSHIPS:
        for r in range(2):
            u = 2 * k + r
            users.append(u)
            for g in rng.choice(N_GROUPS, k, replace=False):
                gm_res.append(g), gm_subj.append(u)
    groups = [("team", "member", "group", tm_res, tm_subj, "member"),
              ("namespace", "viewer", "team", nv_res, nv_subj, "member"),
              ("namespace", "editor", "team", ne_res, ne_subj, "member"),
              ("group", "member", "user", gm_res, gm_subj, None)]
    checks = [("namespace", "view", i, u) for i in range(len(SIZES)) for u in users]
    checks += [("team", "member", int(t), u) for t in rng.choice(N_TEAMS, 40, replace=False) for u in users[::3]]
    order = rng.permutation(len(checks))
    return groups, [checks[i] for i in order]


def load(engine, groups):
    for rt, rel, st, res, subj, srel in groups:
        engine.add_bulk(rt, rel, st, np.asarray(res, dtype=np.uint32), np.asarray(subj, dtype=np.uint32), srel=srel)


def items(target, checks, dtype):
    it = np.zeros(len(checks), dtype=dtype)
    for i, (rt, perm, res, u) in enumerate(checks):
        it["res"][i], it["subj"][i] = res, u
        it["perm"][i], it["stype"][i], it["srel"][i] = target.slot_id(rt, perm), target.type_id("user"), 0xFFFF
    return it


def over_cap_users():
    return [2 * k + r for k in MEMBERSHIPS if k > 16 for r in range(2)]


def filter_bits(obj_id: int):
    """The two bits (0 .. 127) of an object id in batch_l2's filter: must restate kernels.cuh l2_bits."""
    hv = (obj_id * 0x9E3779B1) & 0xFFFFFFFF
    return hv >> 25, (hv >> 18) & 127


def collision_cases(n_teams, max_pairs=24):
    """Team ids a != b with the same filter bits. Returns (groups, [(check, expected v1 code)]): namespace n<k> holds a
    (and a few others) but not b, namespace p<k> holds b, and user u<k> reaches only b."""
    by_key = defaultdict(list)
    for t in range(n_teams):
        by_key[tuple(sorted(filter_bits(t)))].append(t)
    pairs = [v[:2] for v in by_key.values() if len(v) > 1][:max_pairs]
    assert len(pairs) >= 8, "no colliding ids: the filter's hash changed? update filter_bits()"
    nv_res, nv_subj, tm_res, tm_subj, gm_res, gm_subj, cases = [], [], [], [], [], [], []
    for k, (a, b) in enumerate(pairs):
        others = [t for t in ((a * 7 + j * 13 + 1) % n_teams for j in range(k % 5)) if t not in (a, b)]
        for t in [a] + others:
            nv_res.append(2 * k), nv_subj.append(t)         # namespace 2k: holds a, not b
        nv_res.append(2 * k + 1), nv_subj.append(b)         # namespace 2k + 1: holds b
        tm_res.append(b), tm_subj.append(k)                 # group k is a member of team b only
        gm_res.append(k), gm_subj.append(k)                 # user k is a member of group k
        cases.append((("namespace", "view", 2 * k, k), 1))  # filter says maybe, the search says no
        cases.append((("namespace", "view", 2 * k + 1, k), 2))
    pad = list(range(n_teams))  # every team id exists (one padding relationship each)
    groups = [("team", "member", "group", pad + tm_res, [len(pairs)] * n_teams + tm_subj, "member"),
              ("namespace", "viewer", "team", nv_res, nv_subj, "member"),
              ("group", "member", "user", gm_res, gm_subj, None)]
    return groups, cases
