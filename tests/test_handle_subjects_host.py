"""ZG_FLAG_HANDLE_SUBJECTS without a GPU: the flag is refused on an engine that is not a sharded handle, a flagged
host-only handle fails LookupSubjects as every host-only engine does, its counters are zero, and
Engine(handle_subjects=True) sets the bit, alone and beside handle_lookups."""
import pytest

import randgen
import zgpu
from spicedb_kubeapi_proxy_b200 import _lib

EINVAL, ECUDA = -1, -4  # ZG_EINVAL, ZG_ECUDA (include/zgpu.h)
FLAG_HANDLE_LOOKUPS, FLAG_HANDLE_SUBJECTS = 4, 8  # ZG_FLAG_HANDLE_LOOKUPS, ZG_FLAG_HANDLE_SUBJECTS


@pytest.mark.parametrize("kw", [dict(), dict(n_shards=1), dict(shard_rank=1, shard_count=2)])
def test_flag_needs_a_sharded_handle(kw):
    with pytest.raises(zgpu.ZgpuError, match="ZG_FLAG_HANDLE_SUBJECTS needs n_shards > 1") as ex:
        zgpu.Engine(host_only=True, handle_subjects=True, **kw)
    assert ex.value.code == EINVAL


def test_flagged_host_only_handle_fails_lookup_subjects_loudly():
    schema = randgen.FIXED_SCHEMAS["docs"]
    e = zgpu.Engine(schema, host_only=True, n_shards=3, handle_subjects=True)
    e.write_relationships([(_lib.OP_TOUCH, "document:d1#viewer@user:a", 0)])
    e.publish()
    calls = [lambda: e.lookup_subjects_ids("document", e.find("document", "d1"), "view", "user"),
             lambda: e.lookup_subjects_str("document", "d1", "view", "user"),
             lambda: e.lookup_subjects_str("document", "never-written", "view", "user")]
    for call in calls:
        with pytest.raises(zgpu.ZgpuError, match="no CPU fallback") as ex:
            call()
        assert ex.value.code == ECUDA
    assert e.handle_subjects_counters() == dict.fromkeys(_lib.Engine.HANDLE_SUBJECTS_COUNTERS, 0)
    assert e.handle_lookup_counters() == dict.fromkeys(_lib.Engine.HANDLE_LOOKUP_COUNTERS, 0)


def test_counters_are_zero_on_other_engines():
    for kw in (dict(), dict(n_shards=2), dict(n_shards=2, handle_lookups=True)):
        e = zgpu.Engine(host_only=True, **kw)
        assert e.handle_subjects_counters() == dict.fromkeys(_lib.Engine.HANDLE_SUBJECTS_COUNTERS, 0), kw


def test_python_argument_sets_the_flag(monkeypatch):
    seen = []
    real = _lib._Config

    def spy(*args):
        cfg = real(*args)
        seen.append(cfg.flags)
        return cfg

    monkeypatch.setattr(_lib, "_Config", spy)
    zgpu.Engine(host_only=True, n_shards=2, handle_subjects=True)
    zgpu.Engine(host_only=True, n_shards=2, handle_subjects=True, handle_lookups=True)
    zgpu.Engine(host_only=True, n_shards=2)
    assert seen == [1 | FLAG_HANDLE_SUBJECTS, 1 | FLAG_HANDLE_LOOKUPS | FLAG_HANDLE_SUBJECTS, 1]
