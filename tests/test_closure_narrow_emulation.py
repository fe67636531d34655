"""The two-level meet over a 16-bit closure index (csrc/kernels.cuh closure_meet<COUNT, uint16_t>: one aligned 32-byte
sector of 16 entries per lane per round) under the SIMT emulator (tests/emu/), with the index built here in numpy:
answers and the COUNT variant's byte model (2 bytes per entry streamed) against a restatement in Python. The 32-bit
meet is covered by tests/test_closure_emulation.py; GPU twin: tests/test_gpu_closure_narrow.py."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import l2_batch_cases as B  # noqa: E402
from test_closure_emulation import filter_maybe, probes, ranges  # noqa: E402

_EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_CSRC = os.path.join(os.path.dirname(_EMU), "..", "spicedb-kubeapi-proxy_b200", "csrc")
FCAP = 64  # kernels.cuh kFCap: the largest range handed to the warp-batched meet
SECTOR = 16  # 16-bit entries per 32-byte sector


@pytest.fixture(scope="module")
def meet():
    so = os.path.join(_EMU, "libzgemu_closure_narrow.so")
    srcs = [os.path.join(_EMU, f) for f in ("emu_closure_narrow.cc", "cuda_emu.h")] + \
           [os.path.join(_CSRC, f) for f in ("kernels.cuh", "schema.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I", _EMU,
                        os.path.join(_EMU, "emu_closure_narrow.cc"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_closure_meet_narrow.argtypes = [C.c_void_p] * 3 + [C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    return L


def build_index(rows, pad_value=0):
    """rows: list of sorted distinct arrays of ids < 65 536 -> (crow, ccol) with ccol padded by 16 entries of pad_value
    (the build pads the same way; the padding must never be read as part of a row)."""
    crow = np.zeros(len(rows) + 1, dtype=np.uint32)
    crow[1:] = np.cumsum([r.size for r in rows])
    ccol = np.concatenate([np.asarray(r, dtype=np.uint16) for r in rows] + [np.full(SECTOR, pad_value, dtype=np.uint16)])
    return crow, ccol


def reference(col, crow, ccol, nsubj, lanes):
    """Per warp: (job slots answered, bytes per requesting lane when no check of the warp is answered, else None). The
    kernel counts a sector's bytes on the lane that loads it, not on the lane whose row it is: compare warp totals."""
    out = []
    for w in lanes:
        hits, nbytes = 0, np.zeros(32, dtype=np.uint64)
        for ln, (want, lo, hi, sid, js) in enumerate(w):
            if not want:
                continue
            rb = re = 0
            if sid < nsubj:
                rb, re = int(crow[sid]), int(crow[sid + 1])
                nbytes[ln] += 8
            if re <= rb:
                continue
            rng_vals, row = col[lo:hi], ccol[rb:re].astype(np.uint32)
            f0, f1 = filter_of(rng_vals)
            nbytes[ln] += 4 * (hi - lo) + 2 * (re - rb)
            for v in row:
                if filter_maybe(f0, f1, v):
                    nbytes[ln] += 4 * probes(rng_vals, v)
            if np.intersect1d(rng_vals, row).size:
                hits |= 1 << js
        out.append((hits, None if hits else nbytes))
    return out


def run(meet, col, crow, ccol, nsubj, lanes):
    lanes = np.ascontiguousarray(lanes, dtype=np.uint32)
    nw = lanes.shape[0]
    hits, nbytes = np.zeros(nw, dtype=np.uint32), np.zeros(nw * 32, dtype=np.uint64)
    col, crow = (np.ascontiguousarray(x, dtype=np.uint32) for x in (col, crow))
    # the meet loads whole aligned 32-byte sectors: give the entries the alignment cudaMalloc gives them
    buf = np.zeros(ccol.size + 32, dtype=np.uint16)
    at = (-buf.ctypes.data % 32) // 2
    aligned = buf[at: at + ccol.size]
    aligned[:] = ccol
    meet.emu_closure_meet_narrow(col.ctypes.data, crow.ctypes.data, aligned.ctypes.data, nsubj, lanes.ctypes.data, nw,
                                 hits.ctypes.data, nbytes.ctypes.data)
    return hits, nbytes.reshape(nw, 32)


def check(meet, col, crow, ccol, nsubj, lanes):
    hits, nbytes = run(meet, col, crow, ccol, nsubj, lanes)
    for w, (want_hits, want_bytes) in enumerate(reference(col, crow, ccol, nsubj, lanes)):
        assert hits[w] == want_hits, (w, hex(hits[w]), hex(want_hits))
        if want_bytes is not None:
            assert int(nbytes[w].sum()) == int(want_bytes.sum()), (w, nbytes[w], want_bytes)
    return hits


def test_mixed_warps_long_rows_and_subjects_past_nsubj(meet):
    """Lanes that meet and lanes that do not, rows of 0 .. 400 entries, empty rows, subject ids at or above nsubj, two
    lanes of one check; ids span the whole 16-bit range."""
    rng = np.random.default_rng(1)
    universe, nsubj = 65536, 200
    rows = []
    for u in range(nsubj):
        k = [0, 1, 3, 8, 15, 16, 17, 40, 80, 160, 400][u % 11]
        rows.append(np.sort(rng.choice(universe, k, replace=False)).astype(np.uint32))
    crow, ccol = build_index(rows)
    # ranges drawn partly from the rows' entries, so that some checks meet
    pool = np.unique(np.concatenate(rows + [rng.choice(universe, 3000, replace=False)]))
    col, spans = ranges(rng, 500, pool, [1, 2, 5, 10, 27, 31, 32, 33, FCAP])
    lanes = np.zeros((40, 32, 5), dtype=np.uint32)
    for w in range(40):
        for ln in range(32):
            lo, hi = spans[int(rng.integers(0, len(spans)))]
            lanes[w, ln] = (rng.random() < 0.75, lo, hi, rng.integers(0, nsubj + 8), ln if w % 2 else ln // 2)
    hits = check(meet, col, crow, ccol, nsubj, lanes)
    assert 0 < np.mean([bin(int(h)).count("1") for h in hits]) < 24


def test_byte_model_without_hits(meet):
    """No range meets any row: every entry of every row is streamed (2 bytes each) and every filter "maybe" searched."""
    rng = np.random.default_rng(2)
    rows = [np.sort(rng.choice(np.arange(0, 30000), k, replace=False)).astype(np.uint32)
            for k in [0, 1, 5, 15, 16, 17, 31, 33, 64, 100, 250]]
    crow, ccol = build_index(rows)
    col, spans = ranges(rng, 64, np.arange(30000, 65536), [1, 3, 10, 27, FCAP])
    lanes = np.zeros((6, 32, 5), dtype=np.uint32)
    for w in range(6):
        for ln in range(32):
            lo, hi = spans[int(rng.integers(0, len(spans)))]
            lanes[w, ln] = (1, lo, hi, rng.integers(0, len(rows) + 2), ln)
    hits = check(meet, col, crow, ccol, len(rows), lanes)
    assert not hits.any()


@pytest.mark.parametrize("end", range(SECTOR))
def test_rows_ending_at_every_sector_position_before_the_padding(meet, end):
    """The last rows of the index end at every entry of a 32-byte sector; the padding behind them (and the neighbouring
    rows inside their first and last sectors) hold a value every range lists: only entries inside a lane's row may
    answer."""
    rng = np.random.default_rng(10 + end)
    poison = 7
    rows = [np.array([poison], dtype=np.uint32)]  # a neighbour in the first sector of the next rows
    for k in range(1, 12):
        rows.append(np.sort(rng.choice(np.arange(100, 400), k, replace=False)).astype(np.uint32))
    tail = (SECTOR - (sum(r.size for r in rows) % SECTOR) + end) % SECTOR or SECTOR
    rows.append(np.sort(rng.choice(np.arange(100, 400), tail, replace=False)).astype(np.uint32))
    crow, ccol = build_index(rows, pad_value=poison)
    assert crow[-1] % SECTOR == end
    col, spans = [], []
    for _ in range(64):
        r = np.unique(np.concatenate([[poison], rng.choice(np.arange(100, 400), int(rng.integers(1, 20)))])).astype(np.uint32)
        spans.append((sum(c.size for c in col), sum(c.size for c in col) + r.size))
        col.append(r)
    col = np.concatenate(col)
    lanes = np.zeros((8, 32, 5), dtype=np.uint32)
    for w in range(8):
        for ln in range(32):
            lo, hi = spans[int(rng.integers(0, len(spans)))]
            lanes[w, ln] = (1, lo, hi, 1 + (ln + w) % (len(rows) - 1), ln)
    check(meet, col, crow, ccol, len(rows), lanes)
    # ranges that hold only the poison: nothing may answer, and the byte model holds
    only = np.array([poison], dtype=np.uint32)
    lanes[:, :, 1], lanes[:, :, 2] = 0, 1
    hits = check(meet, only, crow, ccol, len(rows), lanes)
    assert not hits.any()


def test_filter_collisions(meet):
    """A row holding b and a range holding a with the same two filter bits: the filter lets b through, only the search
    answers (no); the range that holds b answers yes."""
    from collections import defaultdict

    by_key = defaultdict(list)
    for t in range(4000):
        by_key[tuple(sorted(B.filter_bits(t)))].append(t)
    pairs = [v[:2] for v in by_key.values() if len(v) > 1][:31]
    assert len(pairs) >= 8
    rows = [np.array([b], dtype=np.uint32) for _, b in pairs]
    crow, ccol = build_index(rows)
    col = np.array([x for a, b in pairs for x in (a, b)], dtype=np.uint32)
    lanes = np.zeros((2, 32, 5), dtype=np.uint32)
    for k in range(len(pairs)):
        lanes[0, k] = (1, 2 * k, 2 * k + 1, k, k)          # range {a}: filter maybe, search no
        lanes[1, k] = (1, 2 * k + 1, 2 * k + 2, k, k)      # range {b}: yes
    hits, _ = run(meet, col, crow, ccol, len(rows), lanes)
    assert hits[0] == 0 and hits[1] == (1 << len(pairs)) - 1
    check(meet, col, crow, ccol, len(rows), lanes)


def test_several_maybes_in_one_sector(meet):
    """A range of kFCap children sets most filter bits, so most sectors of a row hold several entries the filter lets
    through: one is parked, the others are searched at once, and only a real member answers."""
    rng = np.random.default_rng(3)
    rng_ids = np.sort(rng.choice(30000, FCAP, replace=False)).astype(np.uint32)
    row_no = np.sort(rng.choice(np.arange(30000, 65536), 48, replace=False)).astype(np.uint32)
    maybes = sum(filter_maybe(*filter_of(rng_ids), v) for v in row_no)
    assert maybes >= 8
    rows = [row_no] + [np.sort(np.append(row_no, rng_ids[k])).astype(np.uint32) for k in (0, 31, FCAP - 1)]
    crow, ccol = build_index(rows)
    lanes = np.zeros((len(rows), 32, 5), dtype=np.uint32)
    for w in range(len(rows)):
        lanes[w, 0] = (1, 0, rng_ids.size, w, 0)
    hits = check(meet, rng_ids, crow, ccol, len(rows), lanes)
    assert hits[0] == 0 and all(hits[1:] == 1)


def filter_of(vals):
    f0 = f1 = 0
    for v in vals:
        for b in B.filter_bits(int(v)):
            if b & 64:
                f1 |= 1 << (b & 63)
            else:
                f0 |= 1 << (b & 63)
    return f0, f1


def test_empty_rows_and_no_requests(meet):
    crow, ccol = build_index([np.zeros(0, dtype=np.uint32)] * 5)
    col = np.arange(10, dtype=np.uint32)
    lanes = np.zeros((2, 32, 5), dtype=np.uint32)
    lanes[0, :, 0], lanes[0, :, 2], lanes[0, :, 3] = 1, 10, np.arange(32) % 7  # rows empty or past nsubj
    lanes[0, :, 4] = np.arange(32)
    hits = check(meet, col, crow, ccol, 5, lanes)
    assert not hits.any()
