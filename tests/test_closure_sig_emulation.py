"""The check kernel's signature meet (csrc/kernels.cuh sig_meet, MEET = kMeetSig16 / kMeetSig32) under the SIMT
emulator (tests/emu/): a two-level step tests its range's children against the signature of the subject's closure row
and searches the row only on a "maybe". The driver (tests/emu/emu_sig.cc) builds the 16-bit closure index on the host,
as tests/emu/emu_rset.cc does, and the rows' signatures as a publish does. Answers must equal the oracle's, the
signature words a numpy restatement of the build, and the COUNT bytes the meet's byte model."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_rsetless_emulation import CFG3, GRANTED, ZG_MAX_DEPTH, Store, cfg3_groups

_TESTS = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_TESTS, "emu")
_CSRC = os.path.join(os.path.dirname(_TESTS), "spicedb-kubeapi-proxy_b200", "csrc")


@pytest.fixture(scope="module")
def emu():
    import emu as E

    so = os.path.join(_EMU, "libzgemu_sig.so")
    srcs = [os.path.join(_EMU, f) for f in ("emu_sig.cc", "emu_rset.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "closure_sig.cuh", "delta.cuh", "schema.cc", "schema.h",
                                             "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        import subprocess

        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                        os.path.join(_EMU, "emu_sig.cc"), os.path.join(_CSRC, "schema.cc"), os.path.join(_CSRC, "store.cc"),
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
    return E, L


class SigStore(Store):
    """A Store (flag-on index) with signatures of every width and word count asked for."""

    def __init__(self, emu, schema, groups):
        super().__init__(emu, schema, groups)
        self.sigs = {}

    def sig(self, width, words):
        if (width, words) not in self.sigs:
            self.sigs[width, words] = self.L.emu_sig_create(self.idx[1], width, words)
        return self.sigs[width, words]

    def close(self):
        for x in self.sigs.values():
            self.L.emu_sig_destroy(x)
        super().close()

    def run_sig(self, items, width=2, words=0, count=False):
        out = np.zeros(items.size, dtype=np.uint8)
        nb = C.c_uint64(0)
        raw = int(not items["flags"].any())
        fl = self.L.emu_sig_check(self.sig(width, words), items.ctypes.data, items.size, out.ctypes.data, raw, int(count),
                                  C.byref(nb))
        assert fl & 3 == 0, fl  # no spill or sub-query overflow
        return out, nb.value

    def words(self, width=2, words=0, pair=0):
        return self.L.emu_sig_words(self.sig(width, words), pair)

    def rows(self, pair=0):
        return self.L.emu_sig_rows(self.sig(2, 0), pair)

    def signature(self, width=2, words=0, pair=0):
        w, n = self.words(width, words, pair), self.rows(pair)
        out = np.zeros(n * w, dtype=np.uint64)
        self.L.emu_sig_copy(self.sig(width, words), pair, out.ctypes.data)
        return out.reshape(n, w)


def closure_rows(groups, nsubj):
    """Row u < nsubj of the closure index: the teams user u reaches through a group, ascending and distinct."""
    gm = next(g for g in groups if g[:3] == ("group", "member", "user"))
    tm = next(g for g in groups if g[:3] == ("team", "member", "group"))
    g2t = {}
    for t, g in zip(tm[3], tm[4]):
        g2t.setdefault(int(g), set()).add(int(t))
    rows = [set() for _ in range(nsubj)]
    for g, u in zip(gm[3], gm[4]):
        rows[int(u)].update(g2t.get(int(g), ()))
    return [np.array(sorted(r), dtype=np.uint32) for r in rows]


def ranges(groups, n_ns):
    """The children of namespace n's team#member range, ascending and distinct."""
    nv = next(g for g in groups if g[:3] == ("namespace", "viewer", "team"))
    out = [set() for _ in range(n_ns)]
    for n, t in zip(nv[3], nv[4]):
        out[int(n)].add(int(t))
    return [np.array(sorted(r), dtype=np.uint32) for r in out]


def np_sig_parts(v, lg):
    h = (np.asarray(v, dtype=np.uint64) * 0x9E3779B1) & 0xFFFFFFFF
    word = (h >> np.uint64(32 - lg)) if lg else np.zeros_like(h)
    bits = (np.uint64(1) << (h & 63)) | (np.uint64(1) << ((h >> 6) & 63)) | (np.uint64(1) << ((h >> 12) & 63))
    return word.astype(np.int64), bits


def np_signature(rows, words):
    """The build restated: entry v of row u sets three bits of word h >> (32 - lg) of the row, h = v * 0x9E3779B1."""
    lg = int(words).bit_length() - 1
    sig = np.zeros((len(rows), words), dtype=np.uint64)
    for u, r in enumerate(rows):
        if r.size:
            word, bits = np_sig_parts(r, lg)
            for wd, b in zip(word.tolist(), bits.tolist()):
                sig[u, wd] |= np.uint64(b)
    return sig


def np_meet_bytes(f, row, sig_row, esize):
    """sig_meet's byte model for one lane: 12 bytes per child tested (the child, its signature word), rounds of 8, and
    sizeof(E) per probe of the binary search of each maybe, in order, until one is found."""
    lg = sig_row.size.bit_length() - 1
    nb = 0
    for r in range(0, f.size, 8):
        chunk = f[r:r + 8]
        nb += 12 * chunk.size
        word, bits = np_sig_parts(chunk, lg)
        for v, wd, b in zip(chunk.tolist(), word.tolist(), bits.tolist()):
            if int(sig_row[wd]) & b != b:
                continue
            a, z = 0, row.size
            while a < z:
                mid = a + (z - a) // 2
                nb += esize
                if row[mid] == v:
                    return nb
                if row[mid] < v:
                    a = mid + 1
                else:
                    z = mid
    return nb


@pytest.fixture(scope="module")
def cfg3(emu):
    rng = np.random.default_rng(7)
    groups, n_users, n_ns = cfg3_groups(rng)
    s = SigStore(emu, CFG3, groups)
    s.groups, s.n_users, s.n_ns = groups, n_users, n_ns
    yield s
    s.close()


@pytest.mark.parametrize("width", [2, 4])
@pytest.mark.parametrize("words", [0, 1, 32])
def test_cfg3_shape_answers_match_the_oracle(cfg3, width, words):
    """cfg3's shape with subjects over and at the set's cap and a range of 100 children; words = 1 makes most tests a
    maybe, 32 nearly none."""
    rng = np.random.default_rng(8)
    res = np.concatenate([rng.integers(0, cfg3.n_ns, 600), np.full(64, cfg3.n_ns - 1), np.arange(cfg3.n_ns),
                          np.arange(cfg3.n_ns)]).astype(np.uint32)
    subj = np.concatenate([rng.integers(0, cfg3.n_users, 600), np.arange(64) % 8, np.zeros(cfg3.n_ns),
                           np.ones(cfg3.n_ns)]).astype(np.uint32)
    want = cfg3.oracle_answers("namespace", "view", "user", res, subj)
    assert (want == GRANTED).any() and (want != GRANTED).any()
    got, _ = cfg3.run_sig(cfg3.items("namespace", "view", "user", res, subj), width, words)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]


@pytest.mark.parametrize("words", [0, 1, 4, 32])
def test_signature_words_equal_numpy(cfg3, words):
    rows = closure_rows(cfg3.groups, cfg3.rows())
    w = cfg3.words(2, words)
    if words:
        assert w == words
    else:  # the fewest words with 64 * words >= 12 x the mean row length
        mean = sum(r.size for r in rows) / len(rows)
        assert 64 * w >= 12 * mean and (w == 1 or 64 * (w // 2) < 12 * mean), (w, mean)
    assert np.array_equal(cfg3.signature(2, words), np_signature(rows, w))


@pytest.mark.parametrize("depth", [ZG_MAX_DEPTH - 3, ZG_MAX_DEPTH - 2, ZG_MAX_DEPTH - 1, ZG_MAX_DEPTH])
def test_checks_at_the_depth_limit(cfg3, depth):
    """Raised where the two-level step may no longer meet: answers (depth errors included) equal closure_meet's, and
    the oracle's where there is room."""
    rng = np.random.default_rng(9 + depth)
    res = rng.integers(0, cfg3.n_ns, 200).astype(np.uint32)
    subj = rng.integers(0, cfg3.n_users, 200).astype(np.uint32)
    items = cfg3.items("namespace", "view", "user", res, subj, depth=depth)
    got = cfg3.run_sig(items)[0]
    assert np.array_equal(got, cfg3.run(items, 1)[0])
    if depth <= ZG_MAX_DEPTH - 3:
        assert np.array_equal(got, cfg3.oracle_answers("namespace", "view", "user", res, subj))


def edge_groups():
    """Rows of 0, 1 and 260 entries and ranges of 1, 64 and 100 children: group 0 is a member of teams 0 .. 259,
    group 1 of team 300 only; user 0 is in group 0, user 1 in group 1, user 2 in group 2 (no team), users 3 .. 9 in
    random groups, and user 10 is in none (past the index's rows). Namespaces 0 / 1 / 2 list 1 / 64 / 100 teams, 3 .. 9
    random ones; nobody views a namespace directly."""
    rng = np.random.default_rng(21)
    tm_t = list(range(260)) + [300] + list(rng.integers(0, 320, 200))
    tm_g = [0] * 260 + [1] + list(rng.integers(3, 12, 200))
    gm_g = [0, 1, 2] + list(rng.integers(3, 12, 20))
    gm_u = [0, 1, 2] + list(rng.integers(3, 10, 20))
    nv = [(0, 300)] + [(1, t) for t in range(0, 320, 5)] + [(2, t) for t in range(20, 320, 3)]
    nv += [(int(n), int(t)) for n, t in zip(rng.integers(3, 10, 80), rng.integers(0, 320, 80))]
    nv = sorted(set(nv))
    pair = sorted({(int(g), int(u)) for g, u in zip(gm_g, gm_u)})
    return [("group", "member", "user", [g for g, _ in pair], [u for _, u in pair], None),
            ("team", "member", "group", tm_t, tm_g, "member"),
            ("namespace", "viewer", "team", [n for n, _ in nv], [t for _, t in nv], "member")]


@pytest.fixture(scope="module")
def edges(emu):
    groups = edge_groups()
    s = SigStore(emu, CFG3, groups)
    s.groups, s.n_users, s.n_ns = groups, 12, 10
    yield s
    s.close()


@pytest.mark.parametrize("width", [2, 4])
@pytest.mark.parametrize("words", [0, 1])
def test_edge_rows_and_ranges(edges, width, words):
    rows = closure_rows(edges.groups, edges.rows())
    assert rows[0].size == 260 and rows[1].size == 1 and rows[2].size == 0
    assert [r.size for r in ranges(edges.groups, edges.n_ns)[:3]] == [1, 64, 100]
    res = np.repeat(np.arange(edges.n_ns, dtype=np.uint32), edges.n_users)
    subj = np.tile(np.arange(edges.n_users, dtype=np.uint32), edges.n_ns)  # users 10 and 11: past nsubj
    want = edges.oracle_answers("namespace", "view", "user", res, subj)
    assert (want == GRANTED).any() and (want != GRANTED).any()
    got, _ = edges.run_sig(edges.items("namespace", "view", "user", res, subj), width, words)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]


@pytest.mark.parametrize("width", [2, 4])
@pytest.mark.parametrize("words", [0, 1])
def test_count_bytes_equal_the_model(edges, width, words):
    """Every check costs what a check of its namespace by user 2 (an empty row: the row offsets, no meet) costs, plus
    sig_meet's bytes for its row and range as np_meet_bytes models them."""
    rows, rng_ = closure_rows(edges.groups, edges.rows()), ranges(edges.groups, edges.n_ns)
    sig = edges.signature(width, words)
    res = np.repeat(np.arange(edges.n_ns, dtype=np.uint32), edges.rows())
    subj = np.tile(np.arange(edges.rows(), dtype=np.uint32), edges.n_ns)
    base = np.full(subj.size, 2, dtype=np.uint32)
    a, got = edges.run_sig(edges.items("namespace", "view", "user", res, subj), width, words, count=True)
    _, b = edges.run_sig(edges.items("namespace", "view", "user", res, base), width, words, count=True)
    want = sum(np_meet_bytes(rng_[n], rows[u], sig[u], width) if rows[u].size else 0 for n, u in zip(res, subj))
    assert got - b == want, (got, b, want)
    assert np.array_equal(a, edges.oracle_answers("namespace", "view", "user", res, subj))
