"""ExpandPermissionTree's kernels (csrc/expand.cuh) and Device::expand's level loop under the SIMT emulator, compared
line for line with the restatement (expand_oracle.py) in the engine's id order: the hand schemas (cfg4's view and
restricted_view, nested operators, nil, an arrow to a type without the permission, a wildcard tupleset subject),
userset and wildcard leaves, rows of 0, 1, 31, 32, 33 and 1 000 entries as leaves and as arrow fan-outs, expiring
entries straddling the 32-entry chunks at two clocks, folder chains of 50 and 51 arrow hops, a cycle, a batch mixing
failing and good requests, the output cap, and random schemas."""
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import randgen  # noqa: E402
from emu_expand import CapError, EmuEngine  # noqa: E402
from expand_oracle import DepthError, expand_tree, lines  # noqa: E402
from golden_runner import split_rel  # noqa: E402
from oracle.mini_oracle import MiniOracle  # noqa: E402
from test_expand_host import DOCS, expiring  # noqa: E402

ROWS = """definition user {}
definition group { relation member: user }
definition other { relation x: user }
definition folder {
  relation parent: folder | other | user:*
  relation viewer: user | group#member | user:*
  permission view = viewer + parent->view
}
"""


def _load(schema, rels, expires=None):
    import numpy as np

    e, m = EmuEngine(schema), MiniOracle(schema)
    for r in rels:
        m.write(r, (expires or {}).get(r, 0))
    if rels:  # ids in first-appearance order
        e.load_tuples(_tuples(e, rels), np.array([(expires or {}).get(r, 0) for r in rels], dtype=np.uint32))
    e.publish()
    return e, m


def _tuples(e, rels):
    import numpy as np

    from emu import SREL_NONE, SREL_WILDCARD, TUPLE_DTYPE

    t = np.zeros(len(rels), dtype=TUPLE_DTYPE)
    for i, r in enumerate(rels):
        rt, rid, rel, st, sid, srel = split_rel(r)
        t["rel"][i], t["stype"][i], t["res"][i] = e.slot_id(rt, rel), e.type_id(st), e._id(rt, rid, True)
        if sid == "*":
            t["srel"][i], t["subj"][i] = SREL_WILDCARD, 0
        else:
            t["srel"][i] = e.slot_id(st, srel) if srel else SREL_NONE
            t["subj"][i] = e._id(st, sid, True)
    return t


def _want(e, m, q, now):
    try:
        return lines(expand_tree(m, *q, now=now, order=lambda t, i: e._names.get((t, i), -1)))
    except DepthError:
        return "EDEPTH"


def _compare(e, m, queries, now=0, threads=64):
    got, info = e.expand(queries, now=now, threads=threads)
    for q, g in zip(queries, got):
        want = _want(e, m, q, now)
        assert (g if g == "EDEPTH" else lines(g)) == want, f"{q} now={now}\nemu={g}\nwant={want}"
    return info


def test_hand_schemas():
    rels = ["document:d#viewer@user:a", "document:d#viewer@group:g#member", "document:d#owner@user:*",
            "document:d#banned@user:b", "document:d#parent@folder:f", "document:d#org@org:o", "folder:f#viewer@user:c",
            "folder:f#parent@folder:root", "folder:root#owner@user:e", "group:g#member@user:g1", "org:o#member@user:a"]
    e, m = _load(DOCS, rels)
    _compare(e, m, [("document", x, p) for x in ("d", "nope") for p in ("view", "restricted_view", "edit", "viewer")] +
             [("folder", "f", "view"), ("org", "o", "member")])
    nest = """definition user {}
definition other { relation x: user }
definition doc {
  relation a: user
  relation b: user
  relation c: user
  relation d: user
  relation t: other | user | user:*
  permission chain = a + (b + c) + d
  permission nested = (a + b) & (c - d)
  permission excl = a - b - c
  permission none = nil
  permission arrow = t->x + t->missing
}
"""
    rels = ["doc:r#t@other:o", "doc:r#t@user:u", "doc:r#t@user:*", "other:o#x@user:v", "doc:r#a@user:u", "doc:r#d@user:v"]
    e, m = _load(nest, rels)
    _compare(e, m, [("doc", "r", p) for p in ("chain", "nested", "excl", "none", "arrow", "t")])


@pytest.mark.parametrize("size", [0, 1, 31, 32, 33, 1000])
def test_rows_around_the_warp_width(size):
    rels = [f"folder:f#viewer@user:u{i}" for i in range(size)]
    rels += [f"folder:f#viewer@group:g{i}#member" for i in range(size // 2)] + ["folder:f#viewer@user:*"] * (size > 0)
    rels += [f"folder:f#parent@folder:p{i}" for i in range(size)] + [f"folder:f#parent@other:o{i}" for i in range(size)]
    rels += [f"folder:p{i}#viewer@user:u{i}" for i in range(0, size, 3)] + ["folder:f#parent@user:*"] * (size > 0)
    e, m = _load(ROWS, rels)
    info = _compare(e, m, [("folder", "f", "view"), ("folder", "f", "viewer"), ("folder", "f", "parent"),
                           ("folder", "p0", "view"), ("folder", "none", "view")])
    assert info["levels"] == (2 if size else 1)
    _compare(e, m, [("folder", "f", "view")], threads=32)  # one warp per block


@pytest.mark.parametrize("size", [31, 33, 70, 1000])
def test_expiring_entries_straddle_the_chunks(size):
    schema = expiring(ROWS)
    rels = [f"folder:f#viewer@user:u{i}" for i in range(size)] + [f"folder:f#parent@folder:p{i}" for i in range(size)]
    rels += [f"folder:p{i}#viewer@user:u{i}" for i in range(size)]
    expires = {r: (1_500 if i % 3 == 1 else 2_500 if i % 5 == 2 else 0) for i, r in enumerate(rels)}
    e, m = _load(schema, rels, expires)
    for now in (1_000, 2_000, 3_000):
        _compare(e, m, [("folder", "f", "view"), ("folder", "f", "viewer"), ("folder", "p1", "view")], now=now)


CHAIN = "definition user {}\ndefinition folder {\n  relation parent: folder\n  relation viewer: user\n" \
        "  permission view = viewer + parent->view\n}\n"


def test_depth_cap_cycle_and_a_mixed_batch():
    rels = [f"folder:a{i}#parent@folder:a{i + 1}" for i in range(50)] + ["folder:a50#viewer@user:u"]
    rels += [f"folder:b{i}#parent@folder:b{i + 1}" for i in range(51)] + ["folder:b51#viewer@user:u"]
    rels += ["folder:c0#parent@folder:c1", "folder:c1#parent@folder:c0"]
    e, m = _load(CHAIN, rels)
    qs = [("folder", x, "view") for x in ("a0", "b0", "c0", "a1", "b1", "b0", "zz")]
    got, info = e.expand(qs)
    assert [g == "EDEPTH" for g in got] == [False, True, True, False, False, True, False]
    _compare(e, m, qs)
    assert info["levels"] == 52  # the last level holds only jobs of failed requests


def test_the_cap_then_a_call_that_fits():
    rels = [f"folder:f#viewer@user:u{i}" for i in range(40)] + [f"folder:f#parent@folder:p{i}" for i in range(40)]
    e, m = _load(ROWS, rels)
    for cap in (5, 60, 120):
        with pytest.raises(CapError):
            e.expand([("folder", "f", "view")], cap=cap)
    _compare(e, m, [("folder", "f", "view")])


@pytest.mark.parametrize("seed", range(8))
def test_random_schemas(seed):
    rng = random.Random(300 + seed)
    schema, model = randgen.random_schema(rng)
    schema = expiring(schema)
    rels = randgen.random_relationships(rng, model, n_obj=5, n_user=5)
    expires = {r: rng.choice((1_500, 2_500)) for r in rels if rng.random() < 0.3}
    e, m = _load(schema, rels, expires)
    qs = [(t, rid, name) for t in model["tnames"] for name in list(model["types"][t]["rels"]) +
          list(model["types"][t]["perms"]) for rid in ("o0", "o3", "o9")]
    for now in (1_000, 2_000):
        _compare(e, m, qs, now=now)
