"""Set tables of the closure index (csrc/build.cu gpu_build_closure_table) and the check kernel's signature meet that
confirms its "maybe"s in them (csrc/kernels.cuh sig_meet, kMeetSet16) on the GPU: the tables copied back against numpy
built from the index, answers against the oracle and against engines without tables (ZGPU_CLOSURE_TABLE=0: the
"maybe"s are searched in the row), generated schemas (32-bit ones keep the search), and after writes."""
import random

import numpy as np
import pytest

import randgen as R
from test_closure_set_emulation import EMPTY, M32, np_choose

pytestmark = pytest.mark.gpu


def _engine(schema, load, monkeypatch, table=True):
    import zgpu

    if not table:
        monkeypatch.setenv("ZGPU_CLOSURE_TABLE", "0")
    e = zgpu.Engine(schema, device=0)
    load(e), e.publish()
    monkeypatch.delenv("ZGPU_CLOSURE_TABLE", raising=False)
    return e


def _np_bucket(v, seed, nb):
    """closure_sig.cuh table_bucket, over arrays of entries, seeds and bucket counts."""
    h = ((v.astype(np.uint64) + ((seed.astype(np.uint64) * np.uint64(0x9E3779B9)) & np.uint64(M32)))
         * np.uint64(0x85EBCA6B)) & np.uint64(M32)
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x2C1B3C6D)) & np.uint64(M32)
    h ^= h >> np.uint64(12)
    return ((h * nb.astype(np.uint64)) >> np.uint64(32)).astype(np.int64)


def _assert_table(e, pair=0, sample=300):
    """Every entry of the index exactly once, in its own bucket; buckets ascending then 0xFFFF; headers contiguous;
    the (bucket count, seed) of `sample` rows the ones numpy's restated choice gives."""
    info = e.closure_table_info(pair)
    row_ptr, col = e.closure_index(pair)
    hdr, tab = e.closure_table(pair)
    n = row_ptr.size - 1
    assert info["built"] == 1 and info["slots"] == 4 and hdr.size == n and tab.shape[0] == info["buckets"], info
    assert info["device_bytes"] == (n + info["buckets"]) * 8, info
    off = (hdr & np.uint64(M32)).astype(np.int64)
    nb = ((hdr >> np.uint64(32)) & np.uint64(0xFFFFFF)).astype(np.int64)
    seed = (hdr >> np.uint64(56)).astype(np.int64)
    lens = np.diff(row_ptr.astype(np.int64))
    assert np.array_equal(off[1:], (off + nb)[:-1]) and off[0] == 0 and int(off[-1] + nb[-1]) == tab.shape[0]
    assert ((nb == 0) == (lens == 0)).all() and (nb >= (lens + 1) // 2).all()
    rows = np.repeat(np.arange(n), lens)
    b = off[rows] + _np_bucket(col, seed[rows], nb[rows])
    assert (tab[b] == col.astype(np.uint16)[:, None]).any(axis=1).all()  # every entry in its bucket
    used = (tab != EMPTY).sum(axis=1)
    assert int(used.sum()) == col.size and used.max(initial=0) <= 4  # ... once, and nothing else
    for s in range(1, 4):  # entries from slot 0, ascending, then empty slots
        occ = used > s
        assert (tab[occ, s] > tab[occ, s - 1]).all() and (tab[~occ, s] == EMPTY).all()
    rng = np.random.default_rng(5)
    for u in rng.choice(n, min(sample, n), replace=False):
        assert np_choose(col[row_ptr[u]:row_ptr[u + 1]].astype(np.int64)) == (int(nb[u]), int(seed[u])), u
    return info


def test_cfg3_tables_and_answers(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.1)
    e = _engine(w.schema, w.load_into, monkeypatch)
    f = _engine(w.schema, w.load_into, monkeypatch, table=False)
    info = _assert_table(e)
    print(f"cfg3 0.1 set table: {info}, {info['device_bytes'] / e.closure_index_info(0)['entries']:.2f} B per entry")
    assert f.closure_table_info(0)["built"] == 0 and f.closure_signature_info(0)["built"] == 1
    with pytest.raises(zgpu.ZgpuError):
        f.closure_table(0)
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    want = o.check_bulk(items)
    assert np.array_equal(e.check_bulk(items), want) and np.array_equal(f.check_bulk(items), want)
    # the byte model (tests/test_closure_set_emulation.py checks it exactly): the same children and signature words,
    # and one 8-byte bucket word per "maybe" instead of a search's 2-byte probes, so about as many bytes
    eb, fb = e.count_alg_bytes(items[:20000]) / 20000, f.count_alg_bytes(items[:20000]) / 20000
    print(f"cfg3 0.1 bytes per check: set tables {eb:.1f}, searches {fb:.1f}")
    for rt, perm, st, u in w.lookups[:4]:
        want = o.lookup_resources_ids(rt, perm, st, u)
        assert np.array_equal(e.lookup_resources_ids(rt, perm, st, u), want)
    c = w.checks[0]
    n_users = int(w.groups[0].subj.max()) + 1
    for res in c.res[:3]:
        ids, wild, ex = e.lookup_subjects_ids(c.res_type, int(res), c.perm, c.subj_type)
        q = np.zeros(n_users, dtype=zgpu.CHECK_DTYPE)
        q["res"], q["subj"] = int(res), np.arange(n_users)
        q["perm"], q["stype"], q["srel"] = o.slot_id(c.res_type, c.perm), o.type_id(c.subj_type), zgpu.SREL_NONE
        assert np.array_equal(ids, np.flatnonzero(o.check_bulk(q) == 2)) and not wild and ex.size == 0


def test_cfg3_full_size_against_the_oracle_and_signatures(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3()
    e = _engine(w.schema, w.load_into, monkeypatch)
    info = _assert_table(e, sample=100)
    print(f"cfg3 full-size closure set table: {info}, index {e.closure_index_info(0)}, "
          f"signatures {e.closure_signature_info(0)}")
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    got = e.check_bulk(items)
    del e
    f = _engine(w.schema, w.load_into, monkeypatch, table=False)
    assert np.array_equal(got, f.check_bulk(items))
    del f
    o = Oracle(w.schema)
    w.load_into(o)
    assert np.array_equal(got, o.check_bulk(items))


@pytest.mark.parametrize("seed,wide", [(0, False), (1, False), (3, True), (4, False), (9, True)])
def test_shaped_schemas(seed, wide, monkeypatch):
    """tests/randgen.py's generated schemas: every 16-bit pair gets a table, 32-bit pairs keep their signatures only,
    and the answers with and without tables equal the oracle's."""
    import zgpu
    from oracle.pyoracle import Oracle

    rng = random.Random(seed)
    text, plan = R.shaped_schema(rng, **({"n_pairs": seed + 1} if seed < 5 else {}))
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan, wide=wide)
    o = Oracle(text)
    R.load_shaped(o, store)
    engines = [_engine(text, lambda e: R.load_shaped(e, store), monkeypatch, table=t) for t in (True, False)]
    n_idx = min(len(plan["pairs"]), R.MAX_CLOSURE)
    for k in range(n_idx):
        if wide:
            assert engines[0].closure_table_info(k)["built"] == 0 and engines[0].closure_signature_info(k)["built"] == 1
        else:
            _assert_table(engines[0], k, sample=50)
        assert engines[1].closure_table_info(k)["built"] == 0
    queries, res, subj = R.shaped_checks(rng, store, plan, 20000)
    items = R.shaped_items(o, zgpu.CHECK_DTYPE, queries, res, subj)
    for now in ((store["now"], store["now"] + 1000) if plan["expiry"] else (store["now"],)):
        want = o.check_bulk(items, now=now)
        for e in engines:
            e.set_clock(now)
            assert np.array_equal(e.check_bulk(items), want), (seed, now)


def test_writes_rebuild_the_tables(monkeypatch):
    """5 x 1000 writes to group#member and team#member (inserts and deletes): each publish rebuilds the index and its
    table; the table is checked and the answers equal the oracle's after every publish."""
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.02)
    e, o = zgpu.Engine(w.schema, device=0), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    _assert_table(e)
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    rng = np.random.default_rng(13)
    builds = e.closure_index_counters()["builds"]
    for step in range(5):
        ups = np.zeros(1000, dtype=zgpu.UPDATE_DTYPE)
        for i in range(ups.size):
            g = w.groups[int(rng.integers(0, 2))]  # group#member@user, team#member@group#member
            ups["rel"][i], ups["stype"][i] = e.slot_id(g.res_type, g.rel), e.type_id(g.subj_type)
            ups["srel"][i] = zgpu.SREL_NONE if g.srel is None else e.slot_id(g.subj_type, g.srel)
            k = int(rng.integers(0, g.res.size))
            if rng.random() < 0.5:
                ups["res"][i], ups["subj"][i], ups["op"][i] = g.res[k], g.subj[k], 2  # DELETE
            else:
                ups["res"][i] = g.res[int(rng.integers(0, g.res.size))]
                ups["subj"][i], ups["op"][i] = g.subj[k], 0  # TOUCH of a new pairing: an insert
        key = np.stack([ups["rel"], ups["res"], ups["stype"], ups["srel"], ups["subj"]], axis=1)
        ups = ups[np.sort(np.unique(key, axis=0, return_index=True)[1])]
        e.apply_updates(ups), o.apply_updates(ups)
        e.publish()
        _assert_table(e, sample=50)
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items)), f"step {step}"
    assert e.closure_index_counters()["builds"] >= builds + 4
