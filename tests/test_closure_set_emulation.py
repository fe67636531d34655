"""The check kernel's signature meet with set tables (csrc/kernels.cuh sig_meet<COUNT, true>, MEET = kMeetSet16) under
the SIMT emulator (tests/emu/): a two-level step tests its range's children against the signature of the subject's
closure row and confirms each "maybe" with one exact lookup in a hashed copy of the row, with no search.
The driver (tests/emu/emu_set.cc) builds the 16-bit closure index, its signatures and its set tables on the host in the
order a publish builds them. Answers must equal the oracle's, the tables a numpy restatement of the build, and the
COUNT bytes the meet's byte model."""
import ctypes as C
import os

import numpy as np
import pytest

from test_closure_sig_emulation import SigStore, closure_rows, edge_groups, np_sig_parts, ranges
from test_rsetless_emulation import CFG3, GRANTED, ZG_MAX_DEPTH, cfg3_groups

_TESTS = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_TESTS, "emu")
_CSRC = os.path.join(os.path.dirname(_TESTS), "spicedb-kubeapi-proxy_b200", "csrc")

K_MEET_SIG16, K_MEET_SET16 = 2 | 8, 2 | 8 | 16  # kernels.cuh kMeetSig16 / kMeetSet16
SEEDS, MAX_BUCKETS = 32, 8192  # closure_sig.cuh kTableSeeds / kTableMaxBuckets
EMPTY = 0xFFFF


@pytest.fixture(scope="module")
def emu():
    import emu as E

    so = os.path.join(_EMU, "libzgemu_set.so")
    srcs = [os.path.join(_EMU, f) for f in ("emu_set.cc", "emu_sig.cc", "emu_rset.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "closure_sig.cuh", "delta.cuh", "schema.cc", "schema.h",
                                             "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        import subprocess

        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                        os.path.join(_EMU, "emu_set.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
                        "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_create.restype = C.c_void_p
    L.emu_create.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    L.emu_destroy.argtypes = [C.c_void_p]
    L.emu_type_id.argtypes = [C.c_void_p, C.c_char_p]
    L.emu_slot_id.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    L.emu_load.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_size_t]
    L.emu_publish.argtypes = [C.c_void_p]
    L.emu_index_create.restype = C.c_void_p
    L.emu_index_create.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    L.emu_index_destroy.argtypes = [C.c_void_p]
    L.emu_index_slot_flags.restype = C.c_uint32
    L.emu_index_slot_flags.argtypes = [C.c_void_p, C.c_int]
    L.emu_index_check.restype = C.c_uint32
    L.emu_index_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    L.emu_sig_create.restype = C.c_void_p
    L.emu_sig_create.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    L.emu_sig_destroy.argtypes = [C.c_void_p]
    L.emu_sig_words.restype = C.c_uint32
    L.emu_sig_words.argtypes = [C.c_void_p, C.c_int]
    L.emu_sig_rows.restype = C.c_uint32
    L.emu_sig_rows.argtypes = [C.c_void_p, C.c_int]
    L.emu_sig_copy.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.emu_sig_check.restype = C.c_uint32
    L.emu_sig_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    L.emu_set_create.restype = C.c_void_p
    L.emu_set_create.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    L.emu_set_destroy.argtypes = [C.c_void_p]
    L.emu_set_meet.argtypes = [C.c_void_p]
    L.emu_set_built.argtypes = [C.c_void_p, C.c_int]
    L.emu_set_buckets.restype = C.c_uint64
    L.emu_set_buckets.argtypes = [C.c_void_p, C.c_int]
    L.emu_set_copy.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.emu_set_check.restype = C.c_uint32
    L.emu_set_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    return E, L


class SetStore(SigStore):
    """A SigStore with set tables for every seed budget and target capacity asked for."""

    def __init__(self, emu, schema, groups):
        super().__init__(emu, schema, groups)
        self.sets = {}

    def set(self, seeds=SEEDS, capacity=1000):
        if (seeds, capacity) not in self.sets:
            self.sets[seeds, capacity] = self.L.emu_set_create(self.sig(2, 0), seeds, capacity)
        return self.sets[seeds, capacity]

    def close(self):
        for x in self.sets.values():
            self.L.emu_set_destroy(x)
        super().close()

    def run_set(self, items, seeds=SEEDS, capacity=1000, count=False):
        out = np.zeros(items.size, dtype=np.uint8)
        nb = C.c_uint64(0)
        raw = int(not items["flags"].any())
        fl = self.L.emu_set_check(self.set(seeds, capacity), items.ctypes.data, items.size, out.ctypes.data, raw,
                                  int(count), C.byref(nb))
        assert fl & 3 == 0, fl  # no spill or sub-query overflow
        return out, nb.value

    def meet(self, seeds=SEEDS, capacity=1000):
        return self.L.emu_set_meet(self.set(seeds, capacity))

    def table(self, seeds=SEEDS, pair=0):
        t = self.set(seeds)
        assert self.L.emu_set_built(t, pair)
        hdr = np.zeros(self.rows(pair), dtype=np.uint64)
        tab = np.zeros(max(self.L.emu_set_buckets(t, pair), 1), dtype=np.uint64)
        self.L.emu_set_copy(t, pair, hdr.ctypes.data, tab.ctypes.data)
        return hdr, tab[: self.L.emu_set_buckets(t, pair)].view(np.uint16).reshape(-1, 4)


M32 = 0xFFFFFFFF


def np_bucket(v, seed, nb):
    """closure_sig.cuh table_bucket restated."""
    h = ((np.asarray(v, dtype=np.uint64) + np.uint64((seed * 0x9E3779B9) & M32)) * np.uint64(0x85EBCA6B)) & M32
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x2C1B3C6D)) & M32
    h ^= h >> np.uint64(12)
    return ((h * np.uint64(nb)) >> np.uint64(32)).astype(np.int64)


def np_choose(row, seeds=SEEDS):
    """The (bucket count, seed) a build chooses for a row: counts from ceil(len / 2), growing by about 1/8 after
    `seeds` failed seeds, until no bucket gets more than four entries. None past MAX_BUCKETS."""
    if row.size == 0:
        return 0, 0
    nb = (row.size + 1) // 2
    while nb <= MAX_BUCKETS:
        for seed in range(seeds):
            if np.bincount(np_bucket(row, seed, nb), minlength=nb).max() <= 4:
                return nb, seed
        nb += (nb + 7) // 8
    return None


def np_table(rows, seeds=SEEDS):
    """The build restated: headers (first bucket | count << 32 | seed << 56) and buckets, entries ascending per bucket."""
    hdr, tabs, off = [], [], 0
    for r in rows:
        nb, seed = np_choose(r, seeds)
        hdr.append(off | (nb << 32) | (seed << 56))
        t = np.full((nb, 4), EMPTY, dtype=np.uint16)
        fill = np.zeros(nb, dtype=np.int64)
        for v, b in zip(r.tolist(), np_bucket(r, seed, nb).tolist()):
            t[b, fill[b]] = v
            fill[b] += 1
        tabs.append(t)
        off += nb
    return np.array(hdr, dtype=np.uint64), np.concatenate(tabs) if tabs else np.zeros((0, 4), np.uint16)


def check_slots(rows, hdr, tab):
    """Every entry exactly once, in its own bucket; no other value anywhere; empty slots 0xFFFF after the entries."""
    for u, r in enumerate(rows):
        h = int(hdr[u])
        off, nb, seed = h & M32, (h >> 32) & 0xFFFFFF, h >> 56
        assert nb == (0 if r.size == 0 else nb) and (r.size == 0 or nb >= (r.size + 1) // 2)
        b = tab[off:off + nb]
        vals = b[b != EMPTY]
        assert np.array_equal(np.sort(vals), r), u  # each entry once, nothing else
        for i, v in enumerate(r.tolist()):
            k = int(np_bucket(np.array([v]), seed, nb)[0])
            assert v in b[k].tolist(), (u, v)
        used = (b != EMPTY).sum(axis=1)
        assert used.max(initial=0) <= 4
        for k in range(nb):  # entries first, ascending, then empty slots
            assert np.array_equal(b[k, :used[k]], np.sort(b[k, :used[k]])) and (b[k, used[k]:] == EMPTY).all()


@pytest.fixture(scope="module")
def cfg3(emu):
    rng = np.random.default_rng(7)
    groups, n_users, n_ns = cfg3_groups(rng)
    s = SetStore(emu, CFG3, groups)
    s.groups, s.n_users, s.n_ns = groups, n_users, n_ns
    yield s
    s.close()


@pytest.fixture(scope="module")
def edges(emu):
    groups = edge_groups()
    s = SetStore(emu, CFG3, groups)
    s.groups, s.n_users, s.n_ns = groups, 12, 10
    yield s
    s.close()


@pytest.mark.parametrize("seeds", [SEEDS, 1])
def test_cfg3_shape_answers_match_the_oracle(cfg3, seeds):
    """cfg3's shape with subjects over and at the set's cap and a range of 100 children."""
    rng = np.random.default_rng(8)
    res = np.concatenate([rng.integers(0, cfg3.n_ns, 600), np.full(64, cfg3.n_ns - 1), np.arange(cfg3.n_ns),
                          np.arange(cfg3.n_ns)]).astype(np.uint32)
    subj = np.concatenate([rng.integers(0, cfg3.n_users, 600), np.arange(64) % 8, np.zeros(cfg3.n_ns),
                           np.ones(cfg3.n_ns)]).astype(np.uint32)
    want = cfg3.oracle_answers("namespace", "view", "user", res, subj)
    assert (want == GRANTED).any() and (want != GRANTED).any()
    assert cfg3.meet(seeds) == K_MEET_SET16
    got, _ = cfg3.run_set(cfg3.items("namespace", "view", "user", res, subj), seeds)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]


@pytest.mark.parametrize("depth", [ZG_MAX_DEPTH - 3, ZG_MAX_DEPTH - 2, ZG_MAX_DEPTH - 1, ZG_MAX_DEPTH])
def test_checks_at_the_depth_limit(cfg3, depth):
    """Raised where the two-level step may no longer meet: answers (depth errors included) equal closure_meet's, and
    the oracle's where there is room."""
    rng = np.random.default_rng(9 + depth)
    res = rng.integers(0, cfg3.n_ns, 200).astype(np.uint32)
    subj = rng.integers(0, cfg3.n_users, 200).astype(np.uint32)
    items = cfg3.items("namespace", "view", "user", res, subj, depth=depth)
    got = cfg3.run_set(items)[0]
    assert np.array_equal(got, cfg3.run(items, 1)[0])
    if depth <= ZG_MAX_DEPTH - 3:
        assert np.array_equal(got, cfg3.oracle_answers("namespace", "view", "user", res, subj))


def test_cfg3_table_equals_numpy(cfg3):
    rows = closure_rows(cfg3.groups, cfg3.rows())
    hdr, tab = cfg3.table()
    want_hdr, want_tab = np_table(rows)
    assert np.array_equal(hdr, want_hdr) and np.array_equal(tab, want_tab)
    check_slots(rows, hdr, tab)


def test_tiny_seed_budget_grows_the_bucket_count(edges):
    """One seed per bucket count: the 260-entry row fails at ceil(260 / 2) buckets and is placed at a larger count."""
    rows = closure_rows(edges.groups, edges.rows())
    hdr, tab = edges.table(seeds=1)
    nb = (hdr >> np.uint64(32)) & np.uint64(0xFFFFFF)
    assert int(nb[0]) > 130 and (hdr >> np.uint64(56) == 0).all()
    assert np_choose(rows[0], 1) == (int(nb[0]), 0)
    assert np.array_equal(hdr, np_table(rows, 1)[0]) and np.array_equal(tab, np_table(rows, 1)[1])
    check_slots(rows, hdr, tab)


@pytest.mark.parametrize("seeds", [SEEDS, 1])
def test_edge_rows_and_ranges(edges, seeds):
    """Rows of 0, 1 and 260 entries, ranges of 1, 64 and 100 children, and subjects past the rows."""
    rows = closure_rows(edges.groups, edges.rows())
    assert rows[0].size == 260 and rows[1].size == 1 and rows[2].size == 0
    assert [r.size for r in ranges(edges.groups, edges.n_ns)[:3]] == [1, 64, 100]
    hdr, tab = edges.table(seeds)
    check_slots(rows, hdr, tab)
    res = np.repeat(np.arange(edges.n_ns, dtype=np.uint32), edges.n_users)
    subj = np.tile(np.arange(edges.n_users, dtype=np.uint32), edges.n_ns)  # users 10 and 11: past nsubj
    want = edges.oracle_answers("namespace", "view", "user", res, subj)
    assert (want == GRANTED).any() and (want != GRANTED).any()
    got, _ = edges.run_set(edges.items("namespace", "view", "user", res, subj), seeds)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]


def test_capacity_65536_falls_back_to_signatures(edges):
    """A target type of 65 536 objects leaves no 16-bit value to mark an empty slot: no table, and sig_meet answers."""
    assert edges.meet(capacity=65536) == K_MEET_SIG16 and edges.meet(capacity=65535) == K_MEET_SET16
    res = np.repeat(np.arange(edges.n_ns, dtype=np.uint32), edges.rows())
    subj = np.tile(np.arange(edges.rows(), dtype=np.uint32), edges.n_ns)
    got, nb = edges.run_set(edges.items("namespace", "view", "user", res, subj), capacity=65536, count=True)
    assert np.array_equal(got, edges.oracle_answers("namespace", "view", "user", res, subj))
    _, want = edges.run_sig(edges.items("namespace", "view", "user", res, subj), 2, 0, count=True)
    assert nb == want


def np_set_bytes(f, row, sig_row):
    """The meet's byte model for one lane: 12 bytes per child tested (the child, its signature word) and 8 per "maybe"
    looked up in the table (its bucket's word), rounds of 8, until the round that finds one; no probes."""
    lg = sig_row.size.bit_length() - 1
    nb, inrow = 0, set(row.tolist())
    for r in range(0, f.size, 8):
        chunk = f[r:r + 8]
        nb += 12 * chunk.size
        word, bits = np_sig_parts(chunk, lg)
        maybes = [v for v, wd, b in zip(chunk.tolist(), word.tolist(), bits.tolist()) if int(sig_row[wd]) & b == b]
        nb += 8 * len(maybes)
        if inrow.intersection(maybes):
            return nb
    return nb


@pytest.mark.parametrize("seeds", [SEEDS, 1])
def test_count_bytes_equal_the_model(edges, seeds):
    """Every check costs what a check of its namespace by user 2 (an empty row: the header, no meet) costs, plus
    the meet's bytes for its row and range as np_set_bytes models them."""
    rows, rng_ = closure_rows(edges.groups, edges.rows()), ranges(edges.groups, edges.n_ns)
    sig = edges.signature(2, 0)
    res = np.repeat(np.arange(edges.n_ns, dtype=np.uint32), edges.rows())
    subj = np.tile(np.arange(edges.rows(), dtype=np.uint32), edges.n_ns)
    base = np.full(subj.size, 2, dtype=np.uint32)
    a, got = edges.run_set(edges.items("namespace", "view", "user", res, subj), seeds, count=True)
    _, b = edges.run_set(edges.items("namespace", "view", "user", res, base), seeds, count=True)
    want = sum(np_set_bytes(rng_[n], rows[u], sig[u]) if rows[u].size else 0 for n, u in zip(res, subj))
    assert got - b == want, (got, b, want)
    assert np.array_equal(a, edges.oracle_answers("namespace", "view", "user", res, subj))
