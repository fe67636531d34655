"""The batched two-level meet (csrc/kernels.cuh batch_l2) under the SIMT emulator (tests/emu/), against the oracle and
against forward-only evaluation: mixed warps, filter collisions, and subjects with more memberships than the per-check
set holds. GPU twin: tests/test_gpu_batch_meet.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))

import l2_batch_cases as B  # noqa: E402


@pytest.fixture(scope="module")
def emu():
    import emu as E

    E.lib()
    return E


def _engine(emu, groups):
    e = emu.EmuEngine(B.SCHEMA)
    B.load(e, groups)
    e.publish()
    return e


def _oracle(groups):
    from oracle.pyoracle import Oracle

    o = Oracle(B.SCHEMA)
    B.load(o, groups)
    return o


def test_batched_meet_mixed_warps_under_the_emulator(emu):
    """Range sizes 1 .. 70, 1 .. 24 memberships, second ranges of answered checks, lanes that do not meet."""
    groups, checks = B.mixed_case()
    e, o = _engine(emu, groups), _oracle(groups)
    it = B.items(e, checks, emu.CHECK_DTYPE)
    want = o.check_bulk(B.items(o, checks, emu.CHECK_DTYPE))
    got = e.check_bulk(it)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    assert np.array_equal(e.check_bulk(it, emu.default_opts(invert=0)), want)
    assert 0.1 < (want == 2).mean() < 0.9


def test_batched_meet_filter_collisions_under_the_emulator(emu):
    """Team ids with the same two filter bits: the filter lets the subject's team through, only the search answers."""
    groups, cases = B.collision_cases(4000)
    e, o = _engine(emu, groups), _oracle(groups)
    checks = [q for q, _ in cases]
    got = e.check_bulk(B.items(e, checks, emu.CHECK_DTYPE))
    assert [int(x) for x in got] == [w for _, w in cases]
    assert np.array_equal(o.check_bulk(B.items(o, checks, emu.CHECK_DTYPE)), got)
    assert np.array_equal(e.check_bulk(B.items(e, checks, emu.CHECK_DTYPE), emu.default_opts(invert=0)), got)


def test_over_cap_subjects_meet_instead_of_walking_under_the_emulator(emu):
    """cfg3's shape (scaled): checks whose user has more than 16 memberships are answered by the meet from the
    user's reverse row instead of walking namespace -> teams -> groups: same answers as the forward walk, and far
    fewer algorithmic bytes than it."""
    import zgpu  # noqa: F401  (registers the package: the workload generators live in it)
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.01)
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(o, emu.CHECK_DTYPE)
    subj = np.concatenate([np.unique(np.stack([g.res, g.subj], 1), axis=0)[:, 1]
                           for g in w.groups if g.res_type == "group" and g.subj_type == "user"])
    per_user = np.bincount(subj)
    sel = items[per_user[np.minimum(items["subj"], per_user.size - 1)] > 16]
    assert sel.size >= 20, sel.size
    want = o.check_bulk(sel)
    e = emu.EmuEngine(w.schema)
    w.load_into(e), e.publish()
    assert np.array_equal(e.check_bulk(sel, count=True), want)
    meet_bytes = e.stat("alg_bytes")
    f = emu.EmuEngine(w.schema)
    w.load_into(f), f.publish()
    assert np.array_equal(f.check_bulk(sel, emu.default_opts(invert=0), count=True), want)
    walk_bytes = f.stat("alg_bytes")
    assert meet_bytes * 3 < walk_bytes, (meet_bytes, walk_bytes)
