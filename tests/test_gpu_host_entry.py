"""CheckBulkPermissions from HOST buffers (zg_check_bulk, csrc/device.cu check_host_multi) on the GPU, against the device
entry (zg_check_bulk_device on torch buffers) and the oracle. A call of at least 2^18 items is streamed: copied up in
chunks of 2^17 items on a copy stream while one persistent check_kernel<false, true, MEET> grid waits for each batch
to land. Smaller calls take one plain copy, and on cfg3 the lean kernel with its residual pass. Concurrent callers
are coalesced into one launch sequence: gathered chunk by chunk across request boundaries, or by helper threads for
groups of 2^20 items from 16 callers, and answered back through the pinned staging area.

Each store's batches tile and permute a pool of at most 100 000 checks that the oracle answers once. Items that name
no permission (answer 255) sit at the first and last position of chunks and of 32-item batches."""
import random
import threading
import time

import numpy as np
import pytest

import randgen as R

pytestmark = pytest.mark.gpu

STREAM_MIN, CHUNK = 1 << 18, 1 << 17  # csrc/device.h kStreamMinItems, kStreamChunkItems
INVALID = 255
COUNTERS = ("launches", "passes", "split_batches", "streamed_calls", "coalesced_launches", "coalesced_requests")


def _engine(schema, load, monkeypatch, env=(), **kw):
    import zgpu

    for k, v in env:
        monkeypatch.setenv(k, v)
    e = zgpu.Engine(schema, device=0, **kw)
    load(e), e.publish()
    for k, _ in env:
        monkeypatch.delenv(k, raising=False)
    return e


def _pool(items, o, now=0, cap=100_000):
    items = np.ascontiguousarray(items[:cap])
    return items, o.check_bulk(items, now=now)


def _edges(n):
    """First and last item of every chunk and of the 32-item batches around each chunk edge and at the end."""
    pos = {0, n - 1, n // 32 * 32, n // 32 * 32 - 1}
    for c in range(CHUNK, n, CHUNK):
        pos |= {c - 33, c - 32, c - 1, c, c + 31, c + 32}
    return np.array(sorted(p for p in pos if 0 <= p < n), dtype=np.int64)


def _batch(pool, n, seed, invalid=True):
    items, want = pool
    idx = np.random.default_rng(seed).permutation(np.resize(np.arange(items.size), n))
    b, w = items[idx], want[idx].copy()
    if invalid:
        pos = _edges(n)
        b["perm"][pos] = 0xFFF0
        w[pos] = INVALID
    return b, w


def _device(e, items):
    import torch

    import zgpu

    d_items = torch.from_numpy(np.ascontiguousarray(items, dtype=zgpu.CHECK_DTYPE).view(np.uint8).copy()).cuda()
    d_out = torch.zeros(items.size, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    e.check_bulk_device(d_items.data_ptr(), items.size, d_out.data_ptr(), s.cuda_stream)
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


def _host(e, items, pin_in=False, pin_out=False):
    """zg_check_bulk with pageable or pinned (zg_host_alloc) input and output -> (answers, counter deltas)."""
    import zgpu

    keep = []
    if pin_in:
        p = zgpu._lib.PinnedArray(items.size, zgpu.CHECK_DTYPE)
        p.array[:] = items
        keep.append(p)
        items = p.array
    out = None
    if pin_out:
        q = zgpu._lib.PinnedArray(items.size, np.uint8)
        keep.append(q)
        out = q.array
    s0 = e.stats()
    got = e.check_bulk(items, out=out)
    s1 = e.stats()
    return got.copy(), {k: s1[k] - s0[k] for k in COUNTERS}


def _three_ways(e, items, want, now=None):
    """Host entry (pageable), device entry and oracle agree item for item; -> the host call's counter deltas."""
    if now is not None:
        e.set_clock(now)
    got, d = _host(e, items)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    dev = _device(e, items)
    assert np.array_equal(dev, want), np.flatnonzero(dev != want)[:8]
    return d


# ---- threshold and chunk edges ---------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cfg3():
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg3(scale=0.02)
    e, o = zgpu.Engine(w.schema, device=0), Oracle(w.schema)
    w.load_into(e), w.load_into(o)
    e.publish()
    assert e.stats()["flat_slots"] >= 1 and e.closure_table_info(0)["built"] == 1
    yield e, _pool(w.check_items(e, zgpu.CHECK_DTYPE), o)
    e.close()


@pytest.mark.parametrize("n", [STREAM_MIN - 1, STREAM_MIN, STREAM_MIN + 1, STREAM_MIN + 33, 3 * CHUNK, 3 * CHUNK + 1,
                               (1 << 20) + 17])
def test_threshold_and_chunk_edges(cfg3, n):
    """Every buffer combination answers as the device entry and the oracle; a call is streamed exactly when it holds
    2^18 items or more."""
    e, pool = cfg3
    items, want = _batch(pool, n, n)
    dev = _device(e, items)
    assert np.array_equal(dev, want), np.flatnonzero(dev != want)[:8]
    for pin_in, pin_out in ((False, False), (True, False), (False, True), (True, True)):
        got, d = _host(e, items, pin_in, pin_out)
        assert np.array_equal(got, want), (pin_in, pin_out, np.flatnonzero(got != want)[:8])
        assert d["streamed_calls"] == int(n >= STREAM_MIN), (pin_in, pin_out, d)


# ---- every streamed instantiation --------------------------------------------------------------------------------------

def _meet_of(e, pairs):
    """The check kernel's MEET, from the snapshot's closure introspection (csrc/device.cu run_pass picks it so)."""
    c = e.closure_index_counters()
    if c["indexed"] == 0:
        return "none" if c["over_budget"] == 0 else "m32"
    info = [e.closure_index_info(k) for k in range(pairs)]
    built = [i for i in range(pairs) if info[i]["built"]]
    width = {info[i]["width"] for i in built}
    assert len(width) == 1, info
    sig = all(e.closure_signature_info(i)["built"] for i in built)
    tab = all(e.closure_table_info(i)["built"] for i in built)
    if width == {4}:
        return "sig32" if sig else "m32"
    return "set16" if sig and tab else ("sig16" if sig else "m16")


MEETS = [("none", "cfg2", ()), ("m32", "cfg3", (("ZGPU_CLOSURE_CAP", "0"),)),
         ("m16", "cfg3", (("ZGPU_CLOSURE_SIG_WORDS", "0"),)), ("sig16", "cfg3", (("ZGPU_CLOSURE_TABLE", "0"),)),
         ("sig32", "wide", ()), ("set16", "cfg3", ())]


@pytest.mark.parametrize("meet,store,env", MEETS, ids=[m[0] for m in MEETS])
def test_every_streamed_instantiation(meet, store, env, monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    now = None  # the stores without expiry keep the engine's clock
    if store == "wide":
        rng = random.Random(3)
        text, plan = R.shaped_schema(rng, n_pairs=4)
        st = R.shaped_relationships(rng, R.model_from_schema(text), plan, wide=True)
        o = Oracle(text)
        R.load_shaped(o, st)
        e = _engine(text, lambda x: R.load_shaped(x, st), monkeypatch, env)
        queries, res, subj = R.shaped_checks(rng, st, plan, 60000)
        now = st["now"]
        pool = _pool(R.shaped_items(o, zgpu.CHECK_DTYPE, queries, res, subj), o, now)
        pairs = min(len(plan["pairs"]), R.MAX_CLOSURE)
    else:
        w = workloads.cfg2(scale=0.01) if store == "cfg2" else workloads.cfg3(scale=0.02)
        o = Oracle(w.schema)
        w.load_into(o)
        e = _engine(w.schema, w.load_into, monkeypatch, env)
        pool = _pool(w.check_items(e, zgpu.CHECK_DTYPE), o)
        pairs = 1
    assert _meet_of(e, pairs) == meet
    for n in (STREAM_MIN + 33, 3 * CHUNK + 1):
        items, want = _batch(pool, n, n + len(meet))
        d = _three_ways(e, items, want, now=now)
        assert d["streamed_calls"] == 1, d


# ---- the lean / streamed crossover -------------------------------------------------------------------------------------

def test_lean_kernel_below_the_threshold_and_streamed_kernel_at_it(cfg3):
    """2^18 - 1 items: one plain copy, flat_check_kernel and its residual pass (two launches). 2^18 items: one streamed
    check_kernel<false, true, kMeetSet16> (one launch). The same items answer the same."""
    e, pool = cfg3
    items, want = _batch(pool, STREAM_MIN, 77)
    lo, dl = _host(e, items[:-1])
    hi, dh = _host(e, items)
    assert dl["launches"] == 2 and dl["streamed_calls"] == 0, dl
    assert dh["launches"] == 1 and dh["streamed_calls"] == 1, dh
    assert np.array_equal(hi, want) and np.array_equal(lo, hi[:-1])


# ---- expiry and sub-queries in a streamed call ---------------------------------------------------------------------------

PROBES = """use expiration
definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member | user with expiration | user:*
  relation reader: team#member | user:* with expiration
  permission view = viewer
  permission read = reader
}
"""


def test_expiring_probes_at_two_clocks(monkeypatch):
    import zgpu
    from oracle.pyoracle import Oracle

    rng = np.random.default_rng(41)
    nu, ng, nt, nn, t0 = 3000, 300, 60, 400, 1_000_000
    rows = []  # (res_type, rel, subj_type, srel, res, subj, expires_at)
    for g, u in {(int(a), int(b)) for a, b in zip(rng.integers(0, ng, 20000), rng.integers(0, nu, 20000))}:
        rows.append(("group", "member", "user", None, g, u, 0))
    for t, g in {(int(a), int(b)) for a, b in zip(rng.integers(0, nt, 900), rng.integers(0, ng, 900))}:
        rows.append(("team", "member", "group", "member", t, g, 0))
    for rel in ("viewer", "reader"):
        for n_, t in {(int(a), int(b)) for a, b in zip(rng.integers(0, nn, 800), rng.integers(0, nt, 800))}:
            rows.append(("namespace", rel, "team", "member", n_, t, 0))
    exps = [0, t0 - 10, t0 + 500, t0 + 5000]
    for n_, u in {(int(a), int(b)) for a, b in zip(rng.integers(0, nn, 3000), rng.integers(0, nu, 3000))}:
        rows.append(("namespace", "viewer", "user", None, n_, u, exps[int(rng.integers(0, 4))]))
    for n_ in (3, 7, 50):
        rows.append(("namespace", "viewer", "user", "*", n_, 0, 0))
    for n_, x in ((2, 0), (5, t0 + 500), (11, t0 - 10)):
        rows.append(("namespace", "reader", "user", "*", n_, 0, x))

    def updates(x):
        u = np.zeros(len(rows), dtype=zgpu.UPDATE_DTYPE)
        for i, (rt, rel, st, srel, r, sj, ex) in enumerate(rows):
            u["rel"][i], u["stype"][i], u["res"][i], u["subj"][i], u["expires_at"][i] = \
                x.slot_id(rt, rel), x.type_id(st), r, sj, ex
            u["srel"][i] = zgpu.SREL_WILDCARD if srel == "*" else (zgpu.SREL_NONE if srel is None else x.slot_id(st, srel))
        return u

    o = Oracle(PROBES)
    o.apply_updates(updates(o))
    e = _engine(PROBES, lambda x: x.apply_updates(updates(x)), monkeypatch)
    m = 50000
    q = np.zeros(m, dtype=zgpu.CHECK_DTYPE)
    q["res"], q["subj"] = rng.integers(0, nn, m), rng.integers(0, nu, m)
    dv = [(r, sj) for rt, rel, st, srel, r, sj, ex in rows if rel == "viewer" and st == "user" and srel is None]
    own = np.flatnonzero(rng.random(m) < 0.3)
    pick = rng.integers(0, len(dv), own.size)
    q["res"][own] = [dv[k][0] for k in pick]
    q["subj"][own] = [dv[k][1] for k in pick]
    q["perm"] = np.array([o.slot_id("namespace", "view"), o.slot_id("namespace", "read")], dtype=np.uint16)[
        rng.integers(0, 2, m)]
    q["stype"], q["srel"] = o.type_id("user"), zgpu.SREL_NONE
    answers = set()
    for now in (t0, t0 + 1000):
        items, want = _batch(_pool(q, o, now), STREAM_MIN + 33, now)
        d = _three_ways(e, items, want, now=now)
        assert d["streamed_calls"] == 1, d
        answers.add(want.tobytes())
    assert len(answers) == 2  # the clock changes answers


def test_sub_queries_and_splits_from_a_streamed_level_zero(monkeypatch):
    """cfg4 with a non-pure folder#view: level 0 is streamed and raises sub-queries into a small buffer, so the batch
    is split after its streamed level 0 and every half runs its passes and folds unstreamed."""
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.cfg4(scale=0.001, nonpure_folders=True)
    o = Oracle(w.schema)
    w.load_into(o)
    pool = _pool(w.check_items(o, zgpu.CHECK_DTYPE), o)
    for cap, split in ((1 << 22, False), (2048, True)):
        e = _engine(w.schema, w.load_into, monkeypatch, subquery_capacity=cap)
        items, want = _batch(pool, STREAM_MIN + 33, cap)
        d = _three_ways(e, items, want)
        assert d["streamed_calls"] == 1 and d["passes"] > 0, d
        assert (d["split_batches"] > 0) == split, d
        e.close()


# ---- coalesced groups ----------------------------------------------------------------------------------------------------

GROUPS = {
    # mixed sizes past 2^18: gathered into the staging area chunk by chunk, across request boundaries
    "mixed": ([1, 31, 40000, 32, 33, 100000, 127, CHUNK + 5, 7], None),
    # 20 callers past 2^20: gathered by the helper threads
    "parallel": ([1, 31, 33] + [62000] * 17, None),
    # pinned and pageable inputs and outputs in one group
    "pinned": ([80000, 1, 100000, 33, 90000, 31], [(True, False), (False, True), (True, True), (False, False)]),
}
BLOCKER = 1 << 22  # the call whose group the callers queue behind


@pytest.mark.parametrize("kind", list(GROUPS))
def test_coalesced_streamed_groups(cfg3, kind):
    """Callers that arrive while another call's group runs queue behind it and are answered together in the next group:
    every caller gets exactly its own answers in every round. The counters show whether the round formed one streamed
    group of all the callers; the schedule is not under the test's control, so a round that did not is run again, a
    bounded number of times."""
    import zgpu

    e, pool = cfg3
    sizes, modes = GROUPS[kind]
    k = len(sizes)
    assert sum(sizes) >= STREAM_MIN and (kind != "parallel" or (sum(sizes) >= 1 << 20 and k >= 16))
    blk_items, blk_want = _batch(pool, BLOCKER, 5)
    formed = False
    for rnd in range(10):
        ins, outs, wants, keep = [], [], [], []
        for i, n in enumerate(sizes):
            it, wt = _batch(pool, n, 1000 * rnd + i, invalid=n >= 64)
            pin_in, pin_out = modes[i % len(modes)] if modes else (False, False)
            if pin_in:
                p = zgpu._lib.PinnedArray(n, zgpu.CHECK_DTYPE)
                p.array[:] = it
                keep.append(p)
                it = p.array
            if pin_out:
                q = zgpu._lib.PinnedArray(n, np.uint8)
                keep.append(q)
                out = q.array
            else:
                out = np.empty(n, dtype=np.uint8)
            out[:] = 0xEE
            ins.append(it), outs.append(out), wants.append(wt)
        errors, blk = [], {}
        go = threading.Barrier(k)

        def caller(i):
            try:
                go.wait()
                e.check_bulk(ins[i], out=outs[i])
            except Exception as ex:  # noqa: BLE001
                errors.append((i, repr(ex)))

        def blocker():
            blk["out"] = e.check_bulk(blk_items)

        s0 = e.stats()
        tb = threading.Thread(target=blocker)
        tb.start()
        time.sleep(0.003)  # the blocker leads its own group before the callers arrive
        th = [threading.Thread(target=caller, args=(i,)) for i in range(k)]
        [t.start() for t in th]
        [t.join() for t in th]
        tb.join()
        s1 = e.stats()
        assert not errors, errors
        assert np.array_equal(blk["out"], blk_want)
        for i in range(k):
            assert np.array_equal(outs[i], wants[i]), (kind, rnd, i, sizes[i], np.flatnonzero(outs[i] != wants[i])[:8])
        d = {c: s1[c] - s0[c] for c in COUNTERS}
        print(f"{kind} round {rnd}: {d}")
        if d["coalesced_launches"] == 1 and d["coalesced_requests"] == k and d["streamed_calls"] == 2:
            formed = True
            break
    assert formed, f"no round formed one streamed group of the {k} callers"
