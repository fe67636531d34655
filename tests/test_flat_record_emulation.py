"""The lean check kernel with range records (csrc/kernels.cuh flat_check_kernel / record_meet, csrc/closure_sig.cuh
kRecSlots) under the SIMT emulator (tests/emu/emu_flat_record.cc, which builds the records on the host as
csrc/build.cu flat_record_kernel does). Answers with records equal those without, the oracle's and the plain
check_kernel<kMeetSet16>'s, on ranges of every length around the record's 31 inline children and on the probe
schema; and the COUNT bytes equal the generic kernel's, so the byte model is unchanged."""
import ctypes as C
import os

import numpy as np
import pytest

import test_flat_check_emulation as F
from test_rsetless_emulation import CFG3, ZG_MAX_DEPTH

_TESTS = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_TESTS, "emu")
_CSRC = os.path.join(os.path.dirname(_TESTS), "spicedb-kubeapi-proxy_b200", "csrc")
LENGTHS = [0, 1, 8, 9, 16, 17, 30, 31, 32, 100]
BIG = [65534, 65533, 60001, 40000, 32768, 32767]  # team ids near the 16-bit limit


@pytest.fixture(scope="module")
def emu():
    import emu as E

    so = os.path.join(_EMU, "libzgemu_flat_record.so")
    srcs = [os.path.join(_EMU, f) for f in ("emu_flat_record.cc", "emu_flat.cc", "emu_set.cc", "emu_sig.cc",
                                             "emu_rset.cc", "emu_main.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "closure_sig.cuh", "delta.cuh", "schema.cc", "schema.h",
                                             "store.cc", "store.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        import subprocess

        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                        os.path.join(_EMU, "emu_flat_record.cc"), os.path.join(_CSRC, "schema.cc"),
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
    L.emu_set_check.restype = C.c_uint32
    L.emu_set_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint64)]
    L.emu_flat_mark.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.emu_flat_check.restype = C.c_uint32
    L.emu_flat_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                 C.c_uint32, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.emu_flat_record_check.restype = C.c_uint32
    L.emu_flat_record_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                        C.c_uint32, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                        C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
    return E, L


class RecordMixin:
    def run_rec(self, items, records=True, count=False, now=0, no_wildcards=False):
        out = np.zeros(items.size, dtype=np.uint8)
        nb, nr, nrec, nlong = C.c_uint64(0), C.c_uint64(0), C.c_uint32(0), C.c_uint64(0)
        raw = int(not items["flags"].any())
        fl = self.L.emu_flat_record_check(self.set(), items.ctypes.data, items.size, out.ctypes.data, raw, int(count),
                                          int(records), now, int(no_wildcards), C.byref(nb), C.byref(nr),
                                          C.byref(nrec), C.byref(nlong))
        assert fl & 3 == 0, fl
        return out, nb.value, nr.value, nrec.value, nlong.value


class RecStore(RecordMixin, F.FlatStore):
    pass


class RecProbeStore(RecordMixin, F.ProbeStore):
    pass


@pytest.fixture(scope="module")
def ranges(emu):
    """namespace -> team -> group -> user with namespace rows of every length in LENGTHS (cycled), over teams whose ids
    reach 65 534."""
    rng = np.random.default_rng(17)
    n_users, n_groups, n_ns = 200, 40, 3 * len(LENGTHS)
    teams = np.array(sorted(set(range(150)) | set(BIG)), dtype=np.uint32)
    gm_u = np.repeat(np.arange(n_users), 2)
    gm_g = rng.integers(0, n_groups, gm_u.size)
    tm_t = np.repeat(teams, 2)
    tm_g = rng.integers(0, n_groups, tm_t.size)
    vr_n, vr_t = [], []
    for ns in range(n_ns):
        k = LENGTHS[ns % len(LENGTHS)]
        pick = rng.choice(teams, k, replace=False)
        if k and ns % 2:
            pick[0] = BIG[ns % len(BIG)] if BIG[ns % len(BIG)] not in pick else pick[0]
        vr_n += [ns] * k
        vr_t += sorted(set(pick.tolist()))
    groups = [("group", "member", "user", gm_g, gm_u, None),
              ("team", "member", "group", tm_t, tm_g, "member"),
              ("namespace", "viewer", "team", np.array(vr_n), np.array(vr_t), "member")]
    s = RecStore(emu, CFG3, groups)
    s.n_users, s.n_ns = n_users, n_ns
    yield s
    s.close()


def all_items(s):
    res = np.repeat(np.arange(s.n_ns, dtype=np.uint32), s.n_users)
    subj = np.tile(np.arange(s.n_users, dtype=np.uint32), s.n_ns)
    return s.items("namespace", "view", "user", res, subj)


def test_records_cover_every_range_length(ranges):
    items = all_items(ranges)
    got, _, resid, nrec, nlong = ranges.run_rec(items)
    assert nrec == 1 and resid == 0
    assert nlong == sum(1 for n in range(ranges.n_ns) if LENGTHS[n % len(LENGTHS)] > 31)
    assert np.array_equal(got, ranges.run_rec(items, records=False)[0])
    assert np.array_equal(got, ranges.run_set(items)[0])
    res, subj = items["res"], items["subj"]
    want = ranges.oracle_answers("namespace", "view", "user", res, subj)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
    assert (got == F.HAS).any() and (got != F.HAS).any()


def test_records_count_bytes_equal_the_generic_kernel(ranges):
    items = all_items(ranges)[::3].copy()
    got, nb, _, _, _ = ranges.run_rec(items, count=True)
    want, wb = ranges.run_set(items, count=True)
    assert np.array_equal(got, want)
    assert nb == wb, (nb, wb)


@pytest.mark.parametrize("n", [77, 600])
def test_records_mixed_batches(emu, n):
    """cfg3's store with the residual pass's kinds of items mixed in, and subjects past the rows."""
    rng = np.random.default_rng(900 + n)
    groups, n_users, n_ns = F.cfg3_groups(rng)
    groups = [g for g in groups if not (g[0] == "namespace" and g[2] == "user")]
    s = RecStore(emu, CFG3, groups)
    s.groups, s.n_users, s.n_ns = groups, n_users, n_ns
    try:
        items, kind = F.mixed(s, rng, n)
        got, _, resid, nrec, _ = s.run_rec(items)
        assert nrec == 1 and resid >= int(np.isin(kind, [1, 2, 3, 5]).sum())
        assert np.array_equal(got, s.run_set(items)[0])
        assert np.array_equal(got, s.run_rec(items, records=False)[0])
        # (the bytes of residual items depend on which share a warp in check_kernel: compared on the lean kernel's own)
        flat = items[kind == 0].copy()
        g2, nb, _, _, _ = s.run_rec(flat, count=True)
        want, wb = s.run_set(flat, count=True)
        assert np.array_equal(g2, want) and np.array_equal(g2, got[kind == 0])
        assert nb == wb, (nb, wb)
    finally:
        s.close()


@pytest.mark.parametrize("depth", [ZG_MAX_DEPTH - 2, ZG_MAX_DEPTH - 1])
def test_records_at_the_depth_limit(ranges, depth):
    rng = np.random.default_rng(950 + depth)
    res = rng.integers(0, ranges.n_ns, 300).astype(np.uint32)
    subj = rng.integers(0, ranges.n_users, 300).astype(np.uint32)
    items = ranges.items("namespace", "view", "user", res, subj, depth=depth)
    got, _, resid, _, _ = ranges.run_rec(items)
    assert resid == (0 if depth + 2 <= ZG_MAX_DEPTH else 300)
    assert np.array_equal(got, ranges.run_set(items)[0])


@pytest.fixture(scope="module")
def probes(emu):
    rng = np.random.default_rng(31)
    groups, n_users, n_ns = F.cfg3_groups(rng)
    groups = [g + (None,) for g in groups if not (g[0] == "namespace" and g[2] == "user")]
    dv_n, dv_u = rng.integers(0, n_ns, 400), rng.integers(0, n_users, 400)
    dv_x = np.array([0, F.T0 - 10, F.T0 + 500, F.T0 + 5000], dtype=np.uint32)[rng.integers(0, 4, 400)]
    pairs = {}
    for a, u, x in zip(dv_n.tolist(), dv_u.tolist(), dv_x.tolist()):
        pairs[a, u] = x
    dv = np.array([(a, u, x) for (a, u), x in sorted(pairs.items())], dtype=np.int64)
    groups.append(("namespace", "viewer", "user", dv[:, 0], dv[:, 1], None, dv[:, 2]))
    groups.append(("namespace", "viewer", "user", [3, 7], [0, 0], "*", None))
    groups.append(("namespace", "reader", "team", rng.integers(0, n_ns, 100), rng.integers(0, 20, 100), "member", None))
    groups.append(("namespace", "reader", "user", [2, 5, 11], [0, 0, 0], "*", [0, F.T0 + 500, F.T0 - 10]))
    s = RecProbeStore(emu, F.PROBES, groups)
    s.groups, s.n_users, s.n_ns = groups, n_users, n_ns
    yield s
    s.close()


@pytest.mark.parametrize("now", [F.T0, F.T0 + 1000])
@pytest.mark.parametrize("no_wildcards", [False, True])
def test_records_with_probes(probes, now, no_wildcards):
    rng = np.random.default_rng(500 + now % 7 + no_wildcards)
    items = F.probe_items(probes, rng, 700)
    got, _, resid, nrec, _ = probes.run_rec(items, now=now, no_wildcards=no_wildcards)
    assert resid == 0 and nrec == 2  # namespace#viewer's and namespace#reader's team#member classes
    assert np.array_equal(got, probes.run_rec(items, records=False, now=now, no_wildcards=no_wildcards)[0])
    o = probes.oracle_nowild if no_wildcards else probes.oracle
    assert np.array_equal(got, F.oracle_of(probes, o, items, now))
    g2, nb, _, _, _ = probes.run_rec(items, count=True, now=now, no_wildcards=no_wildcards)
    want, wb, _, _ = probes.run_flat(items, lean=-1, count=True, now=now, no_wildcards=no_wildcards)
    assert np.array_equal(g2, want) and nb == wb, (nb, wb)
