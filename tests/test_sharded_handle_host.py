"""The sharded handle (zg_config.n_shards) without a GPU: its configuration is checked at create, a host-only one
refuses checks as every host-only engine does, and the host builder's per-shard arrays hold exactly the
relationships each shard owns."""
import random

import numpy as np
import pytest

import randgen
import zgpu
from spicedb_kubeapi_proxy_b200 import _lib

EINVAL, ECUDA = -1, -4  # ZG_EINVAL, ZG_ECUDA (include/zgpu.h)


@pytest.mark.parametrize("kw,msg", [
    (dict(n_shards=2, shard_count=2), "set only one of them"),
    (dict(n_shards=3, shard_rank=1, shard_count=4), "set only one of them"),
    (dict(n_shards=65), "exceeds 64"),
    (dict(n_shards=1000), "exceeds 64"),
])
def test_config_is_checked_at_create(kw, msg):
    with pytest.raises(zgpu.ZgpuError, match=msg) as ex:
        zgpu.Engine(host_only=True, **kw)
    assert ex.value.code == EINVAL


@pytest.mark.parametrize("s", [0, 1, 2, 64])
def test_valid_shard_counts_create(s):
    e = zgpu.Engine(randgen.FIXED_SCHEMAS["docs"], host_only=True, n_shards=s)
    e.publish()
    assert e.stats()["shards"] == max(s, 1)


def test_host_only_sharded_handle_refuses_checks_loudly():
    schema = randgen.FIXED_SCHEMAS["docs"]
    e = zgpu.Engine(schema, host_only=True, n_shards=3)
    rels = randgen.random_relationships(random.Random(5), randgen.model_from_schema(schema))
    e.write_relationships([(_lib.OP_TOUCH, r, 0) for r in rels])
    e.publish()
    items = np.zeros(4, dtype=zgpu.CHECK_DTYPE)
    for call in (lambda: e.check_bulk(items), lambda: e.check_bulk_str(rels[:3])):
        with pytest.raises(zgpu.ZgpuError, match="no CPU fallback") as ex:
            call()
        assert ex.value.code == ECUDA
    # the store is the whole store: reads see every shard's relationships
    assert e.num_tuples() == len(rels)


def test_shard_rows_are_refused_on_other_engines():
    e = zgpu.Engine(randgen.FIXED_SCHEMAS["docs"], host_only=True)
    e.publish()
    with pytest.raises(zgpu.ZgpuError, match="not a shard") as ex:
        e.debug_row("document", "viewer", 0, shard=0)
    assert ex.value.code == EINVAL
    h = zgpu.Engine(randgen.FIXED_SCHEMAS["docs"], host_only=True, n_shards=2)
    h.publish()
    with pytest.raises(zgpu.ZgpuError, match="not a shard"):
        h.debug_row("document", "viewer", 0, shard=2)


def _rows(e, model, n_ids, shard=None):
    """Every forward row (resource, class) and reverse row (subject, class) of every relation: {key: tuple(row)}."""
    out = {}
    for t, d in model["types"].items():
        for r, allowed in d["rels"].items():
            for k in range(len(allowed)):
                for i in range(n_ids):
                    out[(t, r, k, i, "f")] = tuple(e.debug_row(t, r, i, k, shard=shard) if shard is not None else e.debug_row(t, r, i, k))
                    out[(t, r, k, i, "r")] = tuple(e.debug_row(t, r, i, k, reverse=True, shard=shard) if shard is not None
                                                   else e.debug_row(t, r, i, k, reverse=True))
    return out


@pytest.mark.parametrize("name,S,seed", [("docs", 3, 1), ("nesting", 2, 2), ("deep_nonpure", 4, 3), ("random", 3, 4)])
def test_per_shard_arrays_hold_exactly_the_owned_relationships(name, S, seed):
    """For every shard k: the handle's host build of shard k is the whole store's build restricted to the resources
    k owns (id % S == k) -- the forward rows of those resources, the reverse rows filtered to them -- also after deletes
    and a delete-by-filter. (The GPU suite compares the same rows with engines built as shard_rank = k.)"""
    rng = random.Random(seed)
    if name == "random":
        schema, model = randgen.random_schema(rng)
    else:
        schema = randgen.FIXED_SCHEMAS[name]
        model = randgen.model_from_schema(schema)
    rels = randgen.random_relationships(rng, model, n_obj=9, n_user=7, density=0.5)
    handle, whole = zgpu.Engine(schema, host_only=True, n_shards=S), zgpu.Engine(schema, host_only=True)
    gone = rng.sample(rels, len(rels) // 4)
    first = rels[0].split("#")[0].split(":")
    for e in (handle, whole):  # the same names in the same order: ids agree on both engines
        e.write_relationships([(_lib.OP_TOUCH, r, 0) for r in rels])
        e.write_relationships([(_lib.OP_DELETE, r, 0) for r in gone])
        e.delete_relationships({"res_type": first[0], "res_id": first[1]})
        e.publish()
    n_ids = 12
    full = _rows(whole, model, n_ids)
    total = 0
    for k in range(S):
        got = _rows(handle, model, n_ids, shard=k)
        want = {key: (v if key[3] % S == k else ()) if key[4] == "f" else tuple(x for x in v if x % S == k)
                for key, v in full.items()}
        assert got == want, f"shard {k} of {S}"
        total += sum(len(v) for key, v in got.items() if key[4] == "f")
    assert total == handle.num_tuples() == whole.num_tuples() > 0
