"""Streamed admission (csrc/kernels.cuh check_kernel<false, true, MEET>, wait_ready) with a real feed under the SIMT
emulator (tests/emu/emu_stream.cc). A large host call is copied up in chunks while one persistent grid already runs
(csrc/device.cu check_host_multi); here a copy thread lands the items chunk by chunk into a staging buffer full of
poison items (answer 255), each chunk only once a warp waits past what has landed. A warp that read an item before it
landed answers 255, and one that waited for more than its batch holds spins out and sets flag 32. Answers must equal the
oracle's for chunks of 1 to 4 096 items and batches that end mid-warp, with kMeet32 and with kMeetSet16 over emu_set.cc's
host-built indexes, signatures and set tables, and for a multi-pass program whose level 0 alone is streamed, split or
not; the kernels' flags word stays 0."""
import ctypes as C
import os

import numpy as np
import pytest

from test_closure_set_emulation import K_MEET_SET16, SetStore
from test_rsetless_emulation import CFG3, cfg3_groups

_TESTS = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_TESTS, "emu")
_CSRC = os.path.join(os.path.dirname(_TESTS), "spicedb-kubeapi-proxy_b200", "csrc")
INVALID = 255  # the answer to an item that names no permission (and to a poison item)
HAS = 2

# (chunk, batch): chunks around the warp's 32 items, batches that are not multiples of 32 (one below a warp)
FEEDS = [(1, 7), (1, 97), (31, 301), (32, 333), (33, 500), (100, 1001), (4096, 5000)]


@pytest.fixture(scope="module")
def emu():
    import emu as E

    so = os.path.join(_EMU, "libzgemu_stream.so")
    srcs = [os.path.join(_EMU, f) for f in ("emu_stream.cc", "emu_set.cc", "emu_sig.cc", "emu_rset.cc", "emu_main.cc",
                                             "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "closure_sig.cuh", "delta.cuh", "schema.cc", "schema.h",
                                             "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        import subprocess

        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                        os.path.join(_EMU, "emu_stream.cc"), os.path.join(_CSRC, "schema.cc"),
                        os.path.join(_CSRC, "store.cc"), "-o", so], check=True)
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
    L.emu_sig_create.restype = C.c_void_p
    L.emu_sig_create.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    L.emu_sig_destroy.argtypes = [C.c_void_p]
    L.emu_set_create.restype = C.c_void_p
    L.emu_set_create.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    L.emu_set_destroy.argtypes = [C.c_void_p]
    L.emu_set_meet.argtypes = [C.c_void_p]
    L.emu_set_check.restype = C.c_uint32
    L.emu_set_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    L.emu_stream_check.restype = C.c_uint32
    L.emu_stream_check.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(E.Opts),
                                   C.c_uint64, C.c_void_p]
    return E, L


class StreamStore(SetStore):
    def stream(self, items, chunk, meet, **opts):
        """-> (answers, flags word, passes, splits, chunks landed) of one streamed call."""
        items = np.ascontiguousarray(items, dtype=self.E.CHECK_DTYPE)
        out = np.zeros(items.size, dtype=np.uint8)
        stats = np.zeros(3, dtype=np.uint64)
        o = self.E.default_opts(**opts)
        tabled = self.set() if meet == "set16" else None
        fl = self.L.emu_stream_check(self.h, tabled, items.ctypes.data, items.size, out.ctypes.data, C.byref(o), chunk,
                                     stats.ctypes.data)
        assert fl != 0xFFFFFFFF, "the streamed check failed"
        return out, fl, int(stats[0]), int(stats[1]), int(stats[2])

    def want(self, items, now=0):
        it = items.copy()
        return np.asarray(self.oracle.check_bulk(it, now=now), dtype=np.uint8)


@pytest.fixture(scope="module")
def cfg3(emu):
    rng = np.random.default_rng(7)
    groups, n_users, n_ns = cfg3_groups(rng)
    s = StreamStore(emu, CFG3, groups)
    s.n_users, s.n_ns = n_users, n_ns
    assert s.meet() == K_MEET_SET16
    yield s
    s.close()


def cfg3_items(s, rng, n):
    res = rng.integers(0, s.n_ns, n).astype(np.uint32)
    subj = rng.integers(0, s.n_users, n).astype(np.uint32)
    return s.items("namespace", "view", "user", res, subj)


@pytest.mark.parametrize("meet", ["m32", "set16"])
@pytest.mark.parametrize("chunk,n", FEEDS)
def test_chunked_landing_matches_the_oracle(cfg3, meet, chunk, n):
    rng = np.random.default_rng(1000 * chunk + n)
    items = cfg3_items(cfg3, rng, n)
    want = cfg3.want(items)
    got, fl, _, _, landed = cfg3.stream(items, chunk, meet)
    assert fl == 0, fl
    assert landed == -(-n // chunk)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    assert not (got == INVALID).any()
    if n > 100:
        assert (got == HAS).any() and (got != HAS).any()
    if meet == "set16":
        assert np.array_equal(got, cfg3.run_set(items)[0])  # the unstreamed kMeetSet16 kernel


@pytest.mark.parametrize("meet", ["m32", "set16"])
@pytest.mark.parametrize("chunk", [31, 33])
def test_invalid_items_at_chunk_and_warp_edges(cfg3, meet, chunk):
    """Items that name no permission, at the first and last position of every chunk and of every 32-item batch: they
    answer 255 and nothing else does."""
    n = 700
    rng = np.random.default_rng(chunk)
    items = cfg3_items(cfg3, rng, n)
    edges = sorted({i for k in range(0, n, chunk) for i in (k, min(k + chunk, n) - 1)} |
                   {i for k in range(0, n, 32) for i in (k, min(k + 32, n) - 1)})
    bad = np.zeros(n, dtype=bool)
    bad[edges] = True
    items["perm"][bad] = 0xFFF0
    want = np.full(n, INVALID, dtype=np.uint8)
    want[~bad] = cfg3.want(items[~bad])
    got, fl, _, _, _ = cfg3.stream(items, chunk, meet)
    assert fl == 0, fl
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]


NONPURE = """definition user {}
definition group { relation member: user | group#member }
definition team { relation member: group#member }
definition namespace {
  relation viewer: team#member
  relation banned: user
  relation parent: namespace
  permission view = viewer
  permission allowed = viewer - banned
  permission inherited = parent->allowed + viewer
}
"""


@pytest.fixture(scope="module")
def nonpure(emu):
    rng = np.random.default_rng(21)
    nu, ng, nt, nn = 300, 60, 24, 90

    def pairs(a, b, k):
        p = np.unique(np.stack([rng.integers(0, a, k), rng.integers(0, b, k)], 1), axis=0)
        return p[:, 0], p[:, 1]

    gm, tm, nv, nb = pairs(ng, nu, 1800), pairs(nt, ng, 150), pairs(nn, nt, 220), pairs(nn, nu, 150)
    par = (np.arange(1, nn), np.array([rng.integers(0, i) for i in range(1, nn)]))  # acyclic
    groups = [("group", "member", "user", *gm, None), ("team", "member", "group", *tm, "member"),
              ("namespace", "viewer", "team", *nv, "member"), ("namespace", "banned", "user", *nb, None),
              ("namespace", "parent", "namespace", *par, None)]
    s = StreamStore(emu, NONPURE, groups)
    s.nu, s.nn = nu, nn
    assert s.meet() == K_MEET_SET16
    yield s
    s.close()


@pytest.mark.parametrize("meet", ["m32", "set16"])
@pytest.mark.parametrize("chunk,subq_cap", [(33, 1 << 16), (100, 1 << 16), (33, 24), (4096, 24)])
def test_multi_pass_program_streams_level_zero(nonpure, meet, chunk, subq_cap):
    """`inherited` raises sub-queries into `allowed`: the passes after level 0 read the sub-query buffer, not the feed,
    and the fold reads the landed items. A small sub-query buffer splits the batch after its streamed level 0; the
    halves run unstreamed over the landed items."""
    s = nonpure
    rng = np.random.default_rng(chunk + subq_cap)
    n = 801
    items = np.zeros(n, dtype=s.E.CHECK_DTYPE)
    items["res"], items["subj"] = rng.integers(0, s.nn, n), rng.integers(0, s.nu, n)
    perms = [s.slot("namespace", p) for p in ("view", "allowed", "inherited")]
    assert perms == [s.oracle.slot_id("namespace", p) for p in ("view", "allowed", "inherited")]
    items["perm"] = np.array(perms, dtype=np.uint16)[rng.integers(0, 3, n)]
    items["stype"], items["srel"] = s.type("user"), s.E.SREL_NONE
    want = s.want(items)
    got, fl, passes, splits, landed = s.stream(items, chunk, meet, subq_cap=subq_cap)
    assert fl == (2 if splits else 0), fl  # bit 1: the sub-query overflow that split the batch, and nothing else
    assert landed == -(-n // chunk)
    assert passes > 0
    assert (splits > 0) == (subq_cap < 1 << 16), splits
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    assert (got == HAS).any() and (got != HAS).any()
