"""Signatures of the closure index (csrc/build.cu gpu_build_closure_sig) and the check kernel's signature meet
(csrc/kernels.cuh sig_meet) on the GPU: the words copied back against a numpy restatement of the build, answers
against the oracle and against engines without signatures (ZGPU_CLOSURE_SIG_WORDS=0: the meet streams the rows,
closure_meet), with one word per row (ZGPU_CLOSURE_SIG_WORDS=1: nearly every test a maybe), and after writes."""
import random

import numpy as np
import pytest

import l2_batch_cases as B
import randgen as R

pytestmark = pytest.mark.gpu


def _engine(schema, load, monkeypatch, words=None):
    import zgpu

    if words is not None:
        monkeypatch.setenv("ZGPU_CLOSURE_SIG_WORDS", str(words))
    e = zgpu.Engine(schema, device=0)
    load(e), e.publish()
    monkeypatch.delenv("ZGPU_CLOSURE_SIG_WORDS", raising=False)
    return e


def _np_signature(row_ptr, col, words):
    """The build restated: entry v of row u sets three bits of word h >> (32 - lg) of the row, h = v * 0x9E3779B1."""
    lg = int(words).bit_length() - 1
    h = (col.astype(np.uint64) * 0x9E3779B1) & 0xFFFFFFFF
    word = (h >> np.uint64(32 - lg)) if lg else np.zeros_like(h)
    bits = (np.uint64(1) << (h & 63)) | (np.uint64(1) << ((h >> 6) & 63)) | (np.uint64(1) << ((h >> 12) & 63))
    rows = np.repeat(np.arange(row_ptr.size - 1), np.diff(row_ptr))
    sig = np.zeros((row_ptr.size - 1) * words, dtype=np.uint64)
    np.bitwise_or.at(sig, rows * words + word.astype(np.int64), bits)
    return sig.reshape(-1, words)


def _assert_signatures(e, pair=0, words=None):
    info = e.closure_signature_info(pair)
    row_ptr, col = e.closure_index(pair)
    n = row_ptr.size - 1
    if words is None:  # the fewest words with 64 * words >= 12 x the mean row length, at most 32
        w = 1
        while w < 32 and 64 * w * n < 12 * col.size:
            w *= 2
        words = w
    assert info["built"] == 1 and info["words"] == words and info["k"] == 3, info
    assert info["device_bytes"] == n * words * 8, info
    assert np.array_equal(e.closure_signature(pair), _np_signature(row_ptr, col, words))
    return info


def test_cfg3_signatures_and_answers(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.1)
    e = _engine(w.schema, w.load_into, monkeypatch)
    f = _engine(w.schema, w.load_into, monkeypatch, words=0)
    one = _engine(w.schema, w.load_into, monkeypatch, words=1)
    info = _assert_signatures(e)
    assert info["words"] == 16, info  # cfg3's rows hold ~80 teams
    _assert_signatures(one, words=1)
    assert f.closure_signature_info(0)["built"] == 0 and f.closure_index_counters()["indexed"] == 1
    with pytest.raises(zgpu.ZgpuError):
        f.closure_signature(0)
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    want = o.check_bulk(items)
    for x in (e, f, one):
        assert np.array_equal(x.check_bulk(items), want)
    # the byte model: ~10 tests of 12 bytes and a few searches against the row's ~80 entries streamed
    print(f"cfg3 0.1 bytes per check: signatures {e.count_alg_bytes(items[:20000]) / 20000:.1f}, "
          f"rows {f.count_alg_bytes(items[:20000]) / 20000:.1f}")
    assert e.count_alg_bytes(items[:20000]) < f.count_alg_bytes(items[:20000])
    for rt, perm, st, u in w.lookups[:4]:
        want = o.lookup_resources_ids(rt, perm, st, u)
        assert np.array_equal(e.lookup_resources_ids(rt, perm, st, u), want)
        assert np.array_equal(one.lookup_resources_ids(rt, perm, st, u), want)
    c = w.checks[0]
    n_users = int(w.groups[0].subj.max()) + 1
    for res in c.res[:3]:
        ids, wild, ex = e.lookup_subjects_ids(c.res_type, int(res), c.perm, c.subj_type)
        q = np.zeros(n_users, dtype=zgpu.CHECK_DTYPE)
        q["res"], q["subj"] = int(res), np.arange(n_users)
        q["perm"], q["stype"], q["srel"] = o.slot_id(c.res_type, c.perm), o.type_id(c.subj_type), zgpu.SREL_NONE
        assert np.array_equal(ids, np.flatnonzero(o.check_bulk(q) == 2)) and not wild and ex.size == 0


def test_cfg3_full_size_equals_the_meet_without_signatures(monkeypatch):
    import zgpu
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3()
    e = _engine(w.schema, w.load_into, monkeypatch)
    f = _engine(w.schema, w.load_into, monkeypatch, words=0)
    info = _assert_signatures(e)
    print(f"cfg3 full-size closure signatures: {info}, index {e.closure_index_info(0)}")
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    assert np.array_equal(e.check_bulk(items), f.check_bulk(items))


@pytest.mark.parametrize("words", [None, 1])
@pytest.mark.parametrize("case", ["mixed", "collisions"])
def test_two_level_meet_sweeps(case, words, monkeypatch):
    """The batched meet's sweeps (tests/l2_batch_cases.py): ranges around and past kFCap, 1 .. 24 memberships."""
    import zgpu
    from oracle.pyoracle import Oracle

    if case == "mixed":
        groups, checks = B.mixed_case()
    else:
        groups, cases = B.collision_cases(4000)
        checks = [q for q, _ in cases]
    e = _engine(B.SCHEMA, lambda x: B.load(x, groups), monkeypatch, words=words)
    _assert_signatures(e, words=words)
    o = Oracle(B.SCHEMA)
    B.load(o, groups)
    want = o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE))
    assert np.array_equal(e.check_bulk(B.items(e, checks, zgpu.CHECK_DTYPE)), want)


@pytest.mark.parametrize("seed,wide", [(0, False), (1, False), (3, True), (4, False), (9, True)])
def test_shaped_schemas(seed, wide, monkeypatch):
    """tests/randgen.py's generated schemas (1 .. 5 two-level pairs; 32-bit entries when wide): every built pair has
    signatures, and the answers with one word per row and with the chosen words equal the oracle's."""
    import zgpu
    from oracle.pyoracle import Oracle

    rng = random.Random(seed)
    text, plan = R.shaped_schema(rng, **({"n_pairs": seed + 1} if seed < 5 else {}))
    store = R.shaped_relationships(rng, R.model_from_schema(text), plan, wide=wide)
    o = Oracle(text)
    R.load_shaped(o, store)
    engines = [_engine(text, lambda e: R.load_shaped(e, store), monkeypatch, words=w) for w in (None, 1)]
    n_idx = min(len(plan["pairs"]), R.MAX_CLOSURE)
    for e, w in zip(engines, (None, 1)):
        assert e.closure_index_counters()["indexed"] == n_idx
        for k in range(n_idx):
            assert e.closure_index_info(k)["width"] == (4 if wide else 2)
            _assert_signatures(e, k, words=w)
    queries, res, subj = R.shaped_checks(rng, store, plan, 20000)
    items = R.shaped_items(o, zgpu.CHECK_DTYPE, queries, res, subj)
    for now in ((store["now"], store["now"] + 1000) if plan["expiry"] else (store["now"],)):
        want = o.check_bulk(items, now=now)
        for e in engines:
            e.set_clock(now)
            assert np.array_equal(e.check_bulk(items), want), (seed, now)


def test_writes_rebuild_the_signatures(monkeypatch):
    """5 x 1000 writes to group#member and team#member (inserts and deletes): each publish rebuilds the index and its
    signatures; the signatures equal numpy's and the answers the oracle's after every publish."""
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.02)
    e, o = zgpu.Engine(w.schema, device=0), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    items = w.check_items(e, zgpu.CHECK_DTYPE)
    rng = np.random.default_rng(12)
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
        _assert_signatures(e)
        assert np.array_equal(e.check_bulk(items), o.check_bulk(items)), f"step {step}"
    assert e.closure_index_counters()["builds"] >= builds + 4


def test_pair_without_signatures_meets_over_its_rows(monkeypatch):
    """A pair left without signatures (ZGPU_CLOSURE_SIG_WORDS=0 here; over the memory budget in use) keeps its index,
    and its steps meet through closure_meet: answers equal the oracle's."""
    import zgpu
    from oracle.pyoracle import Oracle

    groups, checks = B.mixed_case()
    e = _engine(B.SCHEMA, lambda x: B.load(x, groups), monkeypatch, words=0)
    assert e.closure_signature_info(0) == {"built": 0, "words": 0, "k": 0, "device_bytes": 0, "build_us": 0}
    assert e.closure_index_counters()["indexed"] == 1
    o = Oracle(B.SCHEMA)
    B.load(o, groups)
    want = o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE))
    assert np.array_equal(e.check_bulk(B.items(e, checks, zgpu.CHECK_DTYPE)), want)
