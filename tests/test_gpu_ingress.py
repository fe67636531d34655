"""Device ingress on the GPU: zg_resolve_checks_packed_device must be byte-identical to the host resolver
zg_resolve_checks_packed, and zg_check_bulk_packed_ingress must answer what zg_check_bulk_packed and the oracle answer:
on the emulator's hand cases, random schemas with named objects, named cfg2 / cfg3 / cfg4 stores (cfg3 at full size),
while names appear through every path, from several threads, and on a non-default stream."""
import os
import random
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import randgen  # noqa: E402
import test_ingress_emulation as hand  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def zg():
    import zgpu

    return zgpu


def _dev(buf: bytes):
    import torch

    return torch.frombuffer(bytearray(buf or b"\0"), dtype=torch.uint8).cuda()


def _resolve_dev(e, res_type, rel, subj_type, res_ids, subjects, subj_rel="", stream=None):
    """zg_resolve_checks_packed_device with the ids packed on the host and copied to the GPU."""
    import torch
    import zgpu

    blob, off = e.pack_ids(res_ids)
    n = len(res_ids)
    d_blob, d_off = _dev(blob), _dev(off.tobytes())
    out = torch.zeros(max(n, 1) * 16, dtype=torch.uint8, device="cuda")
    kw = {}
    if isinstance(subjects, (str, bytes)):
        kw["subjects"] = subjects
    else:
        sblob, soff = e.pack_ids(subjects)
        d_sblob, d_soff = _dev(sblob), _dev(soff.tobytes())
        kw["subjects"], kw["d_subj_off"] = d_sblob.data_ptr(), d_soff.data_ptr()
    st = stream.cuda_stream if stream is not None else 0
    e.resolve_checks_packed_device(res_type, rel, subj_type, d_blob.data_ptr(), d_off.data_ptr(), n, out.data_ptr(),
                                   subj_rel=subj_rel, stream=st, **kw)
    return out.cpu().numpy()[: n * 16].view(zgpu.CHECK_DTYPE)


def _same(e, res_type, rel, subj_type, res_ids, subjects, subj_rel="", stream=None):
    want = e.resolve_checks_packed(res_type, rel, subj_type, res_ids, subjects, subj_rel=subj_rel)
    got = _resolve_dev(e, res_type, rel, subj_type, res_ids, subjects, subj_rel=subj_rel, stream=stream)
    assert got.tobytes() == want.tobytes(), (res_type, rel, subj_type, np.flatnonzero(got != want)[:8])
    return got


class _GpuPair:
    """Stands in for the emulator in test_ingress_emulation's cases: one GPU engine, device resolve vs host resolve."""

    def __init__(self, zg, names):
        self.e = zg.Engine(hand.SCHEMA, device=0)
        for t, ids in names.items():
            self.e.intern_packed(t, ids)


def test_hand_cases(zg):
    rng = random.Random(11)
    ids = hand._random_ids(rng, 500)
    known = [i for i in ids if i and rng.random() < 0.6]
    e = _GpuPair(zg, {"user": known, "group": known[: len(known) // 2], "doc": known[::3]}).e
    for n in (1, 31, 33, 5000):
        res = [rng.choice(ids) for _ in range(n)]
        subj = [rng.choice(ids) if rng.random() < 0.7 else res[i] for i in range(n)]
        _same(e, "doc", "view", "user", res, subj)
        _same(e, "group", "member", "group", res, subj, subj_rel="member")
        for one in (known[0], b"never-written", b""):
            _same(e, "group", "member", "group", res, one)
    # every length (up to 4 100 bytes) at every alignment
    lens = list(range(0, 70)) + [1023, 1024, 1025, 4100]
    names = [bytes((5 * i + j) % 256 for j in range(L)) for i, L in enumerate(lens)]
    e.intern_packed("user", [x for x in names if x])
    for pad in range(8):
        res = [b"\x02" * pad] + names
        _same(e, "doc", "view", "user", res, res[::-1])
    ids = ["a/b", "a_b", "a|b", "a-b", "a=b", "a+b", "/", "_", "|", "-", "=", "+"]
    e.intern_packed("doc", ids[::2])
    _same(e, "doc", "view", "user", ids, ids[::-1])
    for args in (("nodoc", "view", "user", ""), ("doc", "nosuch", "user", ""), ("doc", "viewer", "group", "nosuch")):
        _same(e, args[0], args[1], args[2], ["d", "x"], ["u", "v"], subj_rel=args[3])
        _same(e, args[0], args[1], args[2], ["d", "x"], "u", subj_rel=args[3])


@pytest.mark.parametrize("seed", range(4))
def test_random_schemas_named(zg, seed):
    """Object ids rendered as names by randgen; the interned answers are checked against the oracle by
    test_gpu_parity, so here the three string paths must agree item for item."""
    rng = random.Random(seed)
    schema, model = randgen.random_schema(rng)
    rels = randgen.random_relationships(rng, model, n_obj=8, n_user=8)
    e = zg.Engine(schema, device=0)
    for i in range(0, len(rels), 500):
        e.write_relationships([(0, r, 0) for r in rels[i:i + 500]])
    e.publish()
    groups = {}
    for c in randgen.random_checks(rng, model, 400, n_obj=8, n_user=8):
        rt, rid, perm, st, sid, srel = zg._lib.split_rel(c)
        groups.setdefault((rt, perm, st, srel), []).append((rid, sid))
    for (rt, perm, st, srel), items in groups.items():
        res, subj = [a for a, _ in items], [b for _, b in items]
        _same(e, rt, perm, st, res, subj, subj_rel=srel)
        _same(e, rt, perm, st, res, subj[0], subj_rel=srel)
        ans = e.check_bulk_packed_ingress(rt, perm, st, res, subj, subj_rel=srel)
        assert np.array_equal(ans, e.check_bulk_packed(rt, perm, st, res, subj, subj_rel=srel))
        assert np.array_equal(ans, e.check_bulk_str([(rt, a, perm, st, b, srel) for a, b in items]))


def _named(zg, w):
    from spicedb_kubeapi_proxy_b200 import workloads

    e = zg.Engine(w.schema, device=0)
    workloads.intern_names(w, e)
    w.load_into(e)
    e.publish()
    return e


def _names(t, ids):
    from spicedb_kubeapi_proxy_b200 import workloads

    return [workloads.object_name(t, int(i)) for i in ids]


@pytest.mark.parametrize("name,scale,oracle", [("cfg2", 1.0, False), ("cfg3", 1.0, False), ("cfg4", 0.05, False),
                                               ("cfg2", 0.01, True), ("cfg3", 0.002, True), ("cfg4", 0.0005, True)])
def test_named_workloads(zg, name, scale, oracle):
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name(name, scale=scale)
    e = _named(zg, w)
    want_codes = Oracle(w.schema) if oracle else None
    if want_codes is not None:
        w.load_into(want_codes)
    for c in w.checks:
        n = min(c.res.size, 1 << 20)
        res, subj = _names(c.res_type, c.res[:n]), _names(c.subj_type, c.subj[:n])
        got = _same(e, c.res_type, c.perm, c.subj_type, res, subj)
        assert np.array_equal(got["res"], c.res[:n]) and np.array_equal(got["subj"], c.subj[:n])
        one = _same(e, c.res_type, c.perm, c.subj_type, res, subj[0])
        assert np.array_equal(one["res"], c.res[:n])
        ans = e.check_bulk_packed_ingress(c.res_type, c.perm, c.subj_type, res, subj)
        assert np.array_equal(ans, e.check_bulk_packed(c.res_type, c.perm, c.subj_type, res, subj))
        if want_codes is not None:
            assert np.array_equal(ans, want_codes.check_bulk(got))
    cnt = e.ingress_counters()
    assert cnt["names"] == sum(workloads.object_counts(w).values()) and cnt["device_bytes"] > 0


def test_sync_through_every_way_names_appear(zg):
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg2(scale=0.01)
    e = _named(zg, w)
    q_res, q_sub = _names("pod", range(0, 900, 7)), _names("user", range(0, 90))

    def check(extra_res=(), extra_sub=()):
        res = q_res + list(extra_res) + ["never/p"]
        sub = (q_sub * 20)[: len(res) - len(extra_sub) - 1] + list(extra_sub) + ["never-u"]
        _same(e, "pod", "view", "user", res, sub)
        _same(e, "pod", "view", "user", res, sub[-2])
        ans = e.check_bulk_packed_ingress("pod", "view", "user", res, sub)
        assert np.array_equal(ans, e.check_bulk_packed("pod", "view", "user", res, sub))

    check()
    base = e.ingress_counters()
    check()  # nothing new: nothing uploaded
    assert e.ingress_counters()["sync_uploads"] == base["sync_uploads"]
    new_pods, new_users = [], []
    for k in range(3):  # writes of 1 000 updates naming new objects
        pods, users = ["new%d/p%04d" % (k, i) for i in range(1000)], ["nu%d-%04d" % (k, i) for i in range(1000)]
        e.write_relationships([(0, "pod:%s#viewer@user:%s" % (p, u), 0) for p, u in zip(pods, users)])
        new_pods += pods
        new_users += users
        before = e.ingress_counters()["sync_uploads"]
        check(new_pods[-300:], new_users[-300:])
        assert e.ingress_counters()["sync_uploads"] == before + 1
    e.intern("user", "fresh-no-publish")  # interned, never published
    check(["fresh-no-publish"], ["fresh-no-publish"])
    r0 = e.ingress_counters()["rebuilds"]
    e.intern_packed("user", ["bulk-%06d" % i for i in range(40000)])  # forces table rebuilds
    check(["bulk-000001"], ["bulk-039999"])
    assert e.ingress_counters()["rebuilds"] > r0
    e._ck(e._L.zg_clear_relationships(e._h))  # names stay
    check(new_pods[:10], new_users[:10])
    w.load_into(e)
    e.publish()
    up = e.ingress_counters()["sync_uploads"]
    check(new_pods[:10], new_users[:10])
    assert e.ingress_counters()["sync_uploads"] == up  # a reload of numeric relationships names nothing new
    e.load_schema(w.schema)  # a schema load discards the mirror
    assert e.ingress_counters()["names"] == 0


def test_threads_and_streams(zg):
    import torch
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3(scale=0.01)
    e = _named(zg, w)
    c = w.checks[0]
    res, subj = _names(c.res_type, c.res), _names(c.subj_type, c.subj)
    want = e.check_bulk_packed(c.res_type, c.perm, c.subj_type, res, subj)
    errors, stop = [], threading.Event()

    def reader():
        try:
            for _ in range(10):
                got = e.check_bulk_packed_ingress(c.res_type, c.perm, c.subj_type, res, subj)
                if not np.array_equal(got, want):
                    errors.append("mismatch")
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))

    def writer():
        i = 0
        while not stop.is_set():
            e.intern_packed("user", ["writer-%07d" % (i * 100 + k) for k in range(100)])
            i += 1

    wt = threading.Thread(target=writer)
    wt.start()
    th = [threading.Thread(target=reader) for _ in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    stop.set()
    wt.join()
    assert not errors, errors[:4]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _same(e, c.res_type, c.perm, c.subj_type, res, subj, stream=s)


def test_errors_and_engine_kinds(zg):
    import torch

    e = zg.Engine(hand.SCHEMA, device=0)
    e.intern_packed("user", ["a", "b"])
    d_blob = _dev(b"abc")
    d_off = _dev(np.array([0, 2, 1, 3], dtype=np.uint32).tobytes())
    out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    with pytest.raises(zg.ZgpuError) as ex:
        e.resolve_checks_packed_device("doc", "view", "user", d_blob.data_ptr(), d_off.data_ptr(), 3, out.data_ptr(),
                                       subjects="a")
    assert ex.value.code == -1
    # nothing published yet: the call publishes the (empty) store first, as zg_check_bulk_packed does
    assert np.array_equal(e.check_bulk_packed_ingress("doc", "view", "user", ["a", "x"], "a"),
                          e.check_bulk_packed("doc", "view", "user", ["a", "x"], "a"))
    L = e._L
    for args in ((None, b"view", b"user", b"", d_blob.data_ptr(), d_off.data_ptr(), b"a", None, 1, out.data_ptr(), None),
                 (b"doc", b"view", b"user", b"", None, d_off.data_ptr(), b"a", None, 1, out.data_ptr(), None),
                 (b"doc", b"view", b"user", b"", d_blob.data_ptr(), d_off.data_ptr(), None, None, 1, out.data_ptr(), None),
                 (b"doc", b"view", b"user", b"", d_blob.data_ptr(), d_off.data_ptr(), b"a", None, 1, None, None)):
        assert L.zg_resolve_checks_packed_device(e._h, *args) == -1
    assert L.zg_check_bulk_packed_ingress(e._h, b"doc", b"view", b"user", b"", None, None, b"a", None, 1, None) == -1
    off = np.array([0, 2, 1, 3], dtype=np.uint32)
    assert L.zg_check_bulk_packed_ingress(e._h, b"doc", b"view", b"user", b"", b"abc", off.ctypes.data, b"a", None, 3,
                                          np.zeros(3, dtype=np.uint8).ctypes.data) == -1
    # a sharded engine resolves (names only) but refuses the ingress check
    s = zg.Engine(hand.SCHEMA, device=0, shard_rank=0, shard_count=2)
    s.intern_packed("user", ["a", "b", "c"])
    s.intern_packed("doc", ["d1"])
    _same(s, "doc", "view", "user", ["d1", "d2", "a"], ["a", "zz", "c"])
    with pytest.raises(zg.ZgpuError) as ex:
        s.check_bulk_packed_ingress("doc", "view", "user", ["d1"], "a")
    assert ex.value.code == -1
