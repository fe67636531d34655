"""ZG_FLAG_HANDLE_LOOKUPS without a GPU: the flag is refused on an engine that is not a sharded handle, a flagged
host-only handle fails lookups as every host-only engine does, and Engine(handle_lookups=True) sets the bit."""
import pytest

import randgen
import zgpu
from spicedb_kubeapi_proxy_b200 import _lib

EINVAL, ECUDA = -1, -4  # ZG_EINVAL, ZG_ECUDA (include/zgpu.h)
FLAG_HANDLE_LOOKUPS = 4  # ZG_FLAG_HANDLE_LOOKUPS


@pytest.mark.parametrize("kw", [dict(), dict(n_shards=1), dict(shard_rank=1, shard_count=2)])
def test_flag_needs_a_sharded_handle(kw):
    with pytest.raises(zgpu.ZgpuError, match="ZG_FLAG_HANDLE_LOOKUPS needs n_shards > 1") as ex:
        zgpu.Engine(host_only=True, handle_lookups=True, **kw)
    assert ex.value.code == EINVAL


def test_flagged_host_only_handle_fails_lookups_loudly():
    schema = randgen.FIXED_SCHEMAS["docs"]
    e = zgpu.Engine(schema, host_only=True, n_shards=3, handle_lookups=True)
    e.write_relationships([(_lib.OP_TOUCH, "document:d1#viewer@user:a", 0)])
    e.publish()
    calls = [lambda: e.lookup_resources_ids("document", "view", "user", e.find("user", "a")),
             lambda: e.lookup_resources_str("document", "view", "user", "a"),
             lambda: e.list_prefilter(b'{"items": [{"metadata": {"name": "d1"}}]}',
                                      e.list_template("document", "view", "user", "a"))]
    for call in calls:
        with pytest.raises(zgpu.ZgpuError, match="no CPU fallback") as ex:
            call()
        assert ex.value.code == ECUDA
    assert e.handle_lookup_counters() == dict.fromkeys(_lib.Engine.HANDLE_LOOKUP_COUNTERS, 0)


def test_python_argument_sets_the_flag(monkeypatch):
    seen = []
    real = _lib._Config

    def spy(*args):
        cfg = real(*args)
        seen.append(cfg.flags)
        return cfg

    monkeypatch.setattr(_lib, "_Config", spy)
    zgpu.Engine(host_only=True, n_shards=2, handle_lookups=True)
    zgpu.Engine(host_only=True, n_shards=2)
    assert seen == [1 | FLAG_HANDLE_LOOKUPS, 1]
