"""The mention scan of zg_retire_unused_names (csrc/filter.cuh mention_scan_kernel) and its plan under the CPU kernel
emulator, against Store::mentioned over the same store: fixed and random schemas with wildcard, userset and expiring
classes, types that are never a resource or never a subject, several launches per scan, incremental merge-publishes,
and 2-4 virtual shards OR-ed as a sharded handle ORs them."""
import os
import random
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import randgen  # noqa: E402

SCHEMA = """
use expiration
definition user {}
definition lonely {}
definition group { relation member: user with expiration | group#member with expiration }
definition doc {
  relation viewer: user with expiration | user:* with expiration | group#member with expiration
  relation owner: user | user:* | group#member
  relation parent: folder
  permission view = viewer + owner + parent->view
}
definition folder { relation viewer: user | group#member  permission view = viewer }
"""


def _types(schema):
    return re.findall(r"definition\s+(\w+)", schema)


def _engine(schema, rels, expires=None):
    import emu_retire
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200._lib import split_rel

    e = emu_retire.EmuEngine(schema)
    e.write_rels(rels, split_rel)
    e.publish()
    return e


def _agree(e, schema, **kw):
    """Device bitmaps (capacity-sized) equal the host's (extent-sized) on the common words, zero beyond."""
    names = _types(schema)
    dev, launches = e.device_mentions(len(names), **kw)
    for t in range(len(names)):
        host = e.host_mentions(t)
        d = dev[t]
        assert len(d) >= len(host), names[t]
        assert np.array_equal(d[:len(host)], host), names[t]
        assert not d[len(host):].any(), names[t]
    return dev, launches


def _python_mentions(schema, rels):
    """(type, name) pairs some relationship names, from the text alone."""
    from spicedb_kubeapi_proxy_b200._lib import split_rel

    out = set()
    for r in rels:
        rt, rid, _, st, sid, _ = split_rel(r)
        out.add((rt, rid))
        if sid != "*":
            out.add((st, sid))
    return out


def test_fixed_store():
    rels = ["doc:d0#viewer@user:u0", "doc:d1#viewer@user:*", "doc:d2#owner@group:g0#member", "group:g0#member@user:u3",
            "doc:d2#parent@folder:f0", "folder:f0#viewer@user:u5", "group:g1#member@group:g0#member"]
    e = _engine(SCHEMA, rels)
    dev, launches = _agree(e, SCHEMA)
    assert launches == 1
    names = _types(SCHEMA)
    got = set()
    for t, words in enumerate(dev):
        for w, word in enumerate(words):
            for b in range(32):
                if word >> b & 1:
                    got.add((names[t], w * 32 + b))
    want = {(t, e._id(t, n, False)) for t, n in _python_mentions(SCHEMA, rels)}
    assert got == want
    # lonely is neither a resource nor a subject and holds no object: its capacity and bitmap are empty
    assert len(dev[names.index("lonely")]) == 0


@pytest.mark.parametrize("seed", range(4))
def test_random_schemas(seed):
    rng = random.Random(20300 + seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=40, n_user=40, density=0.2)
    e = _engine(schema, rels)
    for grid, max_types in ((1, 64), (3, 1), (2, 2)):
        _agree(e, schema, grid=grid, max_types=max_types)


def test_expired_and_long_rows():
    """Expired entries still mention their ids; an object with a row longer than a warp and ids past 64."""
    import emu_retire
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200._lib import split_rel

    e = emu_retire.EmuEngine(SCHEMA)
    rels = [f"group:big#member@user:u{i}" for i in range(0, 300, 3)] + ["doc:d#viewer@user:u299"]
    t = np.zeros(len(rels), dtype=emu_retire.TUPLE_DTYPE)
    for i, r in enumerate(rels):
        rt, rid, rel, st, sid, srel = split_rel(r)
        t["rel"][i], t["stype"][i], t["srel"][i] = e.slot_id(rt, rel), e.type_id(st), emu_retire.SREL_NONE
        t["res"][i], t["subj"][i] = e._id(rt, rid, True), int(sid[1:])
    e.load_tuples(t, np.array([5] * len(rels), dtype=np.uint32))  # all long expired
    e.publish()
    dev, _ = _agree(e, SCHEMA, grid=2)
    user = dev[_types(SCHEMA).index("user")]
    ids = {w * 32 + b for w, word in enumerate(user) for b in range(32) if int(word) >> b & 1}
    assert ids == set(range(0, 300, 3)) | {299}


def test_after_incremental_merges():
    rng = random.Random(20400)
    rels = ["doc:d0#viewer@user:u0", "group:g0#member@user:u1", "doc:d1#owner@group:g0#member"]
    e = _engine(SCHEMA, rels)
    for step in range(6):
        ups = np.zeros(4, dtype=np.dtype(__import__("emu").UPDATE_DTYPE))
        for i in range(4):
            ups["rel"][i], ups["stype"][i], ups["srel"][i] = e.slot_id("doc", "viewer"), e.type_id("user"), 0xFFFF
            ups["res"][i], ups["subj"][i] = rng.randrange(8), rng.randrange(8)
            ups["op"][i] = 2 if rng.random() < 0.4 else 0
        e.apply_updates(ups)
        e.merge_and_verify()
        _agree(e, SCHEMA)


@pytest.mark.parametrize("shards", [2, 3, 4])
def test_virtual_shards_ored(shards):
    rng = random.Random(20500 + shards)
    model = randgen.model_from_schema(SCHEMA)
    rels = randgen.random_relationships(rng, model, n_obj=30, n_user=30, density=0.3)
    e = _engine(SCHEMA, rels)
    names = _types(SCHEMA)
    whole, _ = e.device_mentions(len(names))
    ored = None
    for k in range(shards):
        part, _ = e.device_mentions(len(names), rank=k, count=shards)
        ored = part if ored is None else [a | b for a, b in zip(ored, part)]
    for t in range(len(names)):
        assert np.array_equal(ored[t], whole[t]), names[t]
        host = e.host_mentions(t)
        assert np.array_equal(ored[t][:len(host)], host)
