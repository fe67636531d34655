"""The collection scan (csrc/filter.cuh filter_expired_kernel) under the CPU kernel emulator, against Store::expired
and a Python statement over the same relationships: random expirations around T, `before` on an expiration exactly,
rows longer than a warp, wildcard classes, several launches per collection, the count launch against the emit launch,
and classes without CF_EXPIRY, whose rows are poisoned with expirations so that reading them would show."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import randgen  # noqa: E402

# viewer and banned may carry expirations, owner may not: its rows are never read
SCHEMA = """
use expiration
definition user {}
definition group { relation member: user with expiration | group#member with expiration }
definition doc {
  relation viewer: user with expiration | user:* with expiration | group#member with expiration
  relation owner: user | user:* | group#member
  relation banned: user with expiration
  permission view = viewer + owner - banned
}
"""


def _engine(rels, expires):
    import emu_expire
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200._lib import split_rel

    e = emu_expire.EmuEngine(SCHEMA)
    t = np.zeros(len(rels), dtype=emu_expire.TUPLE_DTYPE)
    for i, r in enumerate(rels):
        rt, rid, rel, st, sid, srel = split_rel(r)
        t["rel"][i], t["stype"][i], t["res"][i] = e.slot_id(rt, rel), e.type_id(st), e._id(rt, rid, True)
        if sid == "*":
            t["srel"][i] = emu_expire.SREL_WILDCARD
        else:
            t["srel"][i] = e.slot_id(st, srel) if srel else emu_expire.SREL_NONE
            t["subj"][i] = e._id(st, sid, True)
    e.load_tuples(t, np.array([expires.get(r, 0) for r in rels], dtype=np.uint32))
    e.publish()
    return e


def _expected(rels, expires, before):
    return sum(1 for r in rels if 0 < expires.get(r, 0) <= before)


def _agree(e, before, want_n, **kw):
    want = e.host_expired(before)
    got, info = e.device_expired(before, **kw)
    assert got == want, before
    assert info["count"] == len(want) == want_n, (before, info)
    assert info["emitted"] == (len(want) if want else 0)
    return info


def _random_rels(rng, n_obj=6, n_user=6):
    rels = randgen.random_relationships(rng, randgen.model_from_schema(SCHEMA), n_obj=n_obj, n_user=n_user, density=0.5)
    return rels + ["doc:o0#viewer@user:*", "doc:o2#owner@user:*"]


@pytest.mark.parametrize("seed", range(4))
def test_random_expirations_around_t(seed):
    """Expirations T - 2 .. T + 2 (and none) on every class that allows them; before = T - 3 .. T + 3."""
    rng = random.Random(10100 + seed)
    rels = _random_rels(rng)
    T = 1_000_000
    expires = {r: T + rng.randint(-2, 2) for r in rels if "#owner@" not in r and rng.random() < 0.7}
    e = _engine(rels, expires)
    assert any("#owner@" in r for r in rels) and expires
    for before in range(T - 3, T + 4):
        info = _agree(e, before, _expected(rels, expires, before), max_sel=1 + seed % 3)
    # the selection: every class with CF_EXPIRY (member 2, viewer 3, banned 1), none of owner's 3
    assert info["selected"] == 6


def test_before_on_an_expiration_exactly():
    rels = ["doc:a#viewer@user:u0", "doc:a#viewer@user:u1", "doc:a#viewer@user:u2", "doc:b#viewer@user:*",
            "doc:a#owner@user:u0"]
    expires = {rels[0]: 100, rels[1]: 101, rels[2]: 99, rels[3]: 100}
    e = _engine(rels, expires)
    assert _agree(e, 99, 1)
    got = e.device_expired(100)[0]
    assert len(got) == 3 and sorted(g[-1] for g in got) == [99, 100, 100]
    # the wildcard record carries subject 0 and the wildcard relation
    assert any(g[4] == 0xFFFE and g[1] == 0 for g in got)
    assert _agree(e, 101, 3 + 1)
    assert _agree(e, 1 << 31, 4)


def test_count_only_and_nothing_to_collect():
    rels = ["doc:a#viewer@user:u0", "doc:a#owner@user:u1"]
    e = _engine(rels, {rels[0]: 500})
    got, info = e.device_expired(499)
    assert got == [] and info["count"] == 0 and info["emitted"] == 0 and info["launches"] == 1
    got, info = e.device_expired(500, emit=False)
    assert got is None and info["count"] == 1 and info["launches"] == 1


def test_rows_longer_than_a_warp():
    """A group of 700 members, every third expired, and a document with 100 viewers: read by 1 and 3 emulated blocks."""
    rels = [f"group:big#member@user:u{i}" for i in range(700)] + [f"doc:d#viewer@user:u{i}" for i in range(100)]
    rels += [f"doc:d#owner@user:u{i}" for i in range(90)]
    expires = {r: (50 if i % 3 == 0 else 5000) for i, r in enumerate(rels) if "#owner@" not in r}
    e = _engine(rels, expires)
    for grid in (1, 3):
        _agree(e, 50, _expected(rels, expires, 50), grid=grid)
        _agree(e, 5000, 800, grid=grid)
        assert e.device_expired(50, grid=grid, emit=False)[1]["count"] == _expected(rels, expires, 50)


def test_classes_without_expiry_are_never_read():
    """The owner rows, poisoned with expiration 1, contribute nothing; unpoisoned the answer is the same."""
    rng = random.Random(10200)
    rels = _random_rels(rng)
    expires = {r: rng.choice([10, 20]) for r in rels if "#owner@" not in r}
    e = _engine(rels, expires)
    assert any("#owner@" in r for r in rels)
    for before in (1, 10, 20):
        a = e.device_expired(before, poison=True)[0]
        b = e.device_expired(before, poison=False)[0]
        assert a == b == e.host_expired(before)
        assert not any(g[2] == e.slot_id("doc", "owner") for g in a)


def test_schema_without_expiration_selects_nothing():
    import emu_expire
    import zgpu  # noqa: F401
    from spicedb_kubeapi_proxy_b200._lib import split_rel

    e = emu_expire.EmuEngine(randgen.FIXED_SCHEMAS["docs"])
    e.write_rels(["document:d0#viewer@user:u0", "document:d0#viewer@user:*"], split_rel)
    e.publish()
    got, info = e.device_expired(1 << 31)
    assert got == [] and info["selected"] == 0 and info["launches"] == 0
    assert e.host_expired(1 << 31) == []
