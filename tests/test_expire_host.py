"""zg_collect_expired on host-only engines (the host scan of the store): what it removes and what stays, ZG_EINVAL for a
`before` later than the engine's clock, a schema without expiration, the watch feed and the revision, and CREATE of a
collected relationship."""
import pytest

import filter_cases as cases
import randgen

EINVAL, EEXIST = -1, -2  # include/zgpu.h
TOUCH, CREATE = 0, 1


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _host(zg, schema, ups, clock):
    e = zg.Engine(schema, host_only=True)
    e.set_clock(clock)
    for i in range(0, len(ups), 1000):
        e.write_relationships(ups[i:i + 1000])
    return e


def test_counts_and_the_remaining_store(zg):
    rels = [f"doc:d{i}#viewer@user:u{i % 7}" for i in range(40)] + ["doc:d0#viewer@user:*", "group:g#member@user:u1"]
    exp = {r: (100 + i % 5) if i % 2 == 0 else 0 for i, r in enumerate(rels)}
    e = _host(zg, cases.EXP_SCHEMA, [(TOUCH, r, exp[r]) for r in rels], 50)
    assert e.num_tuples() == len(rels)
    for before in (99, 100, 102, 104, 1000):
        gone = {r for r in rels if 0 < exp[r] <= before}
        left_before = e.num_tuples()
        e.set_clock(before)
        n = e.collect_expired(before)
        assert e.num_tuples() == left_before - n
        e.set_clock(1)  # a read at clock 1 lists every relationship the store holds
        assert sorted(e.read_relationships()) == sorted(r for r in rels if r not in gone)
    e.set_clock(1000)
    assert e.num_tuples() == sum(1 for r in rels if exp[r] == 0)
    assert e.collect_expired(1000) == 0
    c = e.filter_counters()
    assert c["device_filters"] == 0 and c["host_filters"] >= 6


def test_before_later_than_the_clock(zg):
    e = _host(zg, cases.EXP_SCHEMA, [(TOUCH, "doc:a#viewer@user:u", 10)], 100)
    with pytest.raises(zg.ZgpuError) as ex:
        e.collect_expired(101)
    assert ex.value.code == EINVAL and "clock" in str(ex.value)
    assert e.num_tuples() == 1
    assert e.collect_expired(100) == 1
    # before 0 or negative: no expiration is at or before it
    e.write_relationships([(TOUCH, "doc:a#viewer@user:u", 10)])
    assert e.collect_expired(0) == 0 and e.collect_expired(-5) == 0 and e.num_tuples() == 1


def test_wall_clock_when_no_clock_is_set(zg):
    import time

    e = zg.Engine(cases.EXP_SCHEMA, host_only=True)
    e.set_clock(50)
    e.write_relationships([(TOUCH, "doc:a#viewer@user:u", 60)])
    e.set_clock(0)  # wall clock
    assert e.collect_expired(int(time.time()) - 10) == 1
    with pytest.raises(zg.ZgpuError):
        e.collect_expired(int(time.time()) + 3600)


def test_schema_without_expiration(zg):
    e = _host(zg, randgen.FIXED_SCHEMAS["docs"], [(TOUCH, "document:d#viewer@user:u", 0)], 100)
    rev = e.stats()["revision"]
    assert e.collect_expired(100) == 0
    assert e.stats()["revision"] == rev and e.num_tuples() == 1


def test_the_watch_feed_and_the_revision(zg):
    rels = ["doc:a#viewer@user:u0", "doc:a#viewer@user:u1", "group:g#member@user:u2"]
    e = _host(zg, cases.EXP_SCHEMA, [(TOUCH, rels[0], 10), (TOUCH, rels[1], 0), (TOUCH, rels[2], 20)], 5)
    feed, through = e.watch_read(0)
    rev = e.stats()["revision"]
    e.set_clock(30)
    assert e.collect_expired(5) == 0 and e.stats()["revision"] == rev  # nothing qualifies: nothing published
    assert e.collect_expired(30) == 2
    assert e.stats()["revision"] == rev + 1
    feed2, through2 = e.watch_read(0)
    assert feed2 == feed and through2 == through + 1
    assert e.watch_read(through)[0] == []
    assert e.read_relationships() == [rels[1]]


def test_create_of_a_collected_relationship(zg):
    r = "doc:a#viewer@user:u0"
    e = _host(zg, cases.EXP_SCHEMA, [(TOUCH, r, 10)], 5)
    e.set_clock(20)
    with pytest.raises(zg.ZgpuError) as ex:  # present but expired: CREATE still collides
        e.write_relationships([(CREATE, r, 0)])
    assert ex.value.code == EEXIST
    assert e.collect_expired(20) == 1
    e.write_relationships([(CREATE, r, 0)])
    assert e.read_relationships() == [r]


def test_bulk_loaded_duplicates(zg):
    """A bulk load may hold a relationship twice; the later expiration wins, as for every other read."""
    import numpy as np

    e = zg.Engine(cases.EXP_SCHEMA, host_only=True)
    e.set_clock(100)
    u, doc = e.intern("user", "u"), e.intern("doc", "a")
    t = np.zeros(3, dtype=zg.TUPLE_DTYPE)
    t["res"], t["subj"], t["rel"], t["stype"], t["srel"] = doc, u, e.slot_id("doc", "viewer"), e.type_id("user"), 0xFFFF
    t["subj"][2] = e.intern("user", "v")
    e.load_tuples(t, np.array([10, 500, 20], dtype=np.uint32))
    e.publish()
    assert e.collect_expired(100) == 1
    assert e.read_relationships() == ["doc:a#viewer@user:u"]
