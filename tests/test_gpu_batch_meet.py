"""GPU twin of tests/test_batch_meet_emulation.py: the batched two-level meet (csrc/kernels.cuh batch_l2) on the real
kernel, against the oracle and against forward-only evaluation."""
import numpy as np
import pytest

import l2_batch_cases as B

pytestmark = pytest.mark.gpu


def _engine(groups, schema=B.SCHEMA, **kw):
    import zgpu

    e = zgpu.Engine(schema, device=0, **kw)
    B.load(e, groups)
    e.publish()
    return e


def _oracle(groups):
    from oracle.pyoracle import Oracle

    o = Oracle(B.SCHEMA)
    B.load(o, groups)
    return o


def test_batched_meet_mixed_warps():
    import zgpu

    groups, checks = B.mixed_case()
    o = _oracle(groups)
    want = o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE))
    e, f = _engine(groups), _engine(groups, forward_only=True)
    assert np.array_equal(e.check_bulk(B.items(e, checks, zgpu.CHECK_DTYPE)), want)
    assert np.array_equal(f.check_bulk(B.items(f, checks, zgpu.CHECK_DTYPE)), want)
    assert 0.1 < (want == 2).mean() < 0.9


def test_batched_meet_filter_collisions():
    import zgpu

    groups, cases = B.collision_cases(4000)
    checks = [q for q, _ in cases]
    e, f = _engine(groups), _engine(groups, forward_only=True)
    got = e.check_bulk(B.items(e, checks, zgpu.CHECK_DTYPE))
    assert [int(x) for x in got] == [w for _, w in cases]
    o = _oracle(groups)
    assert np.array_equal(o.check_bulk(B.items(o, checks, zgpu.CHECK_DTYPE)), got)
    assert np.array_equal(f.check_bulk(B.items(f, checks, zgpu.CHECK_DTYPE)), got)


def test_over_cap_subjects_meet_instead_of_walking():
    import zgpu
    from oracle.pyoracle import Oracle
    from spicedb_kubeapi_proxy_b200 import workloads

    w = workloads.by_name("cfg3", 0.01)
    o = Oracle(w.schema)
    w.load_into(o)
    items = w.check_items(o, zgpu.CHECK_DTYPE)
    subj = np.concatenate([np.unique(np.stack([g.res, g.subj], 1), axis=0)[:, 1]
                           for g in w.groups if g.res_type == "group" and g.subj_type == "user"])
    per_user = np.bincount(subj)
    sel = items[per_user[np.minimum(items["subj"], per_user.size - 1)] > 16]
    assert sel.size >= 20, sel.size
    want = o.check_bulk(sel)
    e = zgpu.Engine(w.schema, device=0)
    w.load_into(e), e.publish()
    f = zgpu.Engine(w.schema, device=0, forward_only=True)
    w.load_into(f), f.publish()
    assert np.array_equal(e.check_bulk(sel), want)
    assert np.array_equal(f.check_bulk(sel), want)
    assert e.count_alg_bytes(sel) * 3 < f.count_alg_bytes(sel)
