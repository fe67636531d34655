"""tests/closure_restate.py against hand-computed stores and the emulator tests' restatements: the capacity formula at
the 16-bit boundary, capacities carried through a history, the pairs a program indexes, the rows, the budget, the
signature words and the set tables."""
import numpy as np

import closure_restate as CR
from test_closure_set_emulation import np_table
from test_closure_sig_emulation import closure_rows as emu_closure_rows
from test_closure_sig_emulation import np_signature
from test_rsetless_emulation import cfg3_groups

GM, TM, NV = ("group", "member", "user", None), ("team", "member", "group", "member"), ("namespace", "viewer", "team", "member")
STEPS = [(NV, GM, TM)]


def _cap(need):
    return need + need // 8 + 4096


def test_capacity_at_the_16_bit_boundary():
    got = [CR.next_capacity(0, n) for n in (54612, 54613, 54614, 54615)]
    assert got == [_cap(n) for n in (54612, 54613, 54614, 54615)]
    assert got == [65534, 65535, 65536, 65537]
    # narrow entries up to 65 536 objects; a set table only below it (0xFFFF marks an empty slot)
    assert [c > CR.NARROW for c in got] == [False, False, False, True]
    assert CR.next_capacity(65535, 54614) == 65535 and CR.next_capacity(65535, 65536) == _cap(65536)


def test_capacity_is_carried_through_history():
    m = CR.Model()
    m.load([("team", "member", "group", np.array([10]), np.array([3]), "member", None)])
    m.publish()
    assert m.cap["team"] == 11 + 1 + 4096 and m.cap["group"] == 4 + 0 + 4096
    m.write(0, TM, 4107, 3)  # id 4107 = capacity - 1: still fits
    m.publish()
    assert m.cap["team"] == 4108
    m.write(2, TM, 4107, 3)
    m.write(2, TM, 10, 3)
    m.publish()  # nothing left: the extent and the capacity stay
    assert m.cap["team"] == 4108 and m.n_numeric["team"] == 4108
    m.write(0, TM, 4108, 3)  # one past: grows from the new need
    m.publish()
    assert m.cap["team"] == _cap(4109)
    m.named("team", 9000)  # a name interned past the numeric extent
    m.publish()
    assert m.cap["team"] == _cap(9001)
    m.write(0, TM, 5, 3)
    m.write(0, TM, 5, 3, expires=7)  # a touch of an existing relationship is not an insert
    assert m.rels[TM] == {(4108, 3): 0, (5, 3): 7} and m.n_numeric["team"] == 4109


def _hand_model():
    """users 0..3, groups 0..2, teams 0..4: user 0 in groups 0 and 1, user 2 in group 1, user 3 in group 2 (which is in
    no team); team t has group t % 2, team 4 also group 1; namespace 0 views team 0."""
    m = CR.Model()
    m.load([("group", "member", "user", np.array([0, 1, 1, 2]), np.array([0, 0, 2, 3]), None, None),
            ("team", "member", "group", np.array([0, 1, 2, 3, 4, 4]), np.array([0, 1, 0, 1, 0, 1]), "member", None),
            ("namespace", "viewer", "team", np.array([0]), np.array([0]), "member", None)])
    m.publish()
    return m


def test_hand_computed_rows_budget_and_signatures():
    m = _hand_model()
    pl = CR.pairs(m, STEPS)
    assert pl == [(GM, TM)]
    (p,) = CR.restate(m, pl)
    n = 4 + 4096
    assert p["row_ptr"].size == n + 1 and p["width"] == 2
    rows = [p["col"][p["row_ptr"][u]:p["row_ptr"][u + 1]].tolist() for u in range(4)]
    assert rows == [[0, 1, 2, 3, 4], [], [1, 3, 4], []]
    # user 0: group 0 (teams 0, 2, 4) + group 1 (teams 1, 3, 4) = 6 before deduplication; user 2: 3
    assert p["pre"] == 9 and p["budget"] == 16 * (4 + 6) and p["built"]
    assert p["words"] == 1 and np.array_equal(p["sig"], np_signature([np.array(r, np.uint32) for r in rows] +
                                                                      [np.zeros(0, np.uint32)] * (n - 4), 1))
    hdr, tab = p["table"]
    want_hdr, want_tab = np_table([np.array(r, np.int64) for r in rows] + [np.zeros(0, np.int64)] * (n - 4))
    assert np.array_equal(hdr, want_hdr) and np.array_equal(tab, want_tab)
    assert CR.counters([p]) == {"indexed": 1, "over_budget": 0, "entries": 8}
    # a cap below the 9 entries before deduplication: no index
    (q,) = CR.restate(m, pl, cap=8)
    assert not q["built"] and CR.counters([q]) == {"indexed": 0, "over_budget": 1, "entries": 0}


def test_sig_words_follow_the_mean_row():
    assert CR.sig_words(100, 0) == 1 and CR.sig_words(100, 533) == 1 and CR.sig_words(100, 534) == 2
    assert CR.sig_words(1, 10 ** 6) == 32


def test_pairs_vanish_with_their_classes_and_cap_at_four():
    m = _hand_model()
    m.write(2, NV, 0, 0)
    assert CR.pairs(m, STEPS) == []  # the step's own class is empty
    m.write(0, NV, 0, 0)
    for r, s in [(0, 0), (1, 0), (1, 2), (2, 3)]:
        m.write(2, GM, r, s)
    assert CR.pairs(m, STEPS) == []  # the inner class is empty
    tgcs = [(f"p{i}", "member", "group", "member") for i in range(6)]
    steps = [(NV, GM, t) for t in tgcs] + [(("x", "r", "y", None), GM, tgcs[0])]
    m.write(0, GM, 0, 0)
    for i, t in enumerate(tgcs):
        if i != 1:
            m.write(0, t, 0, 0)
    # p1 is empty; the rest in step order, the first four only; a second step of p0 adds nothing
    assert [t for _, t in CR.pairs(m, steps)] == [tgcs[0], tgcs[2], tgcs[3], tgcs[4]]


def test_wide_target_has_no_table_and_width_four():
    m = _hand_model()
    m.write(0, TM, 53247, 0)  # need 53248: capacity 53248 + 6656 + 4096 = 64000
    m.publish()
    (p,) = CR.restate(m, CR.pairs(m, STEPS))
    assert m.cap["team"] == 64000 and p["width"] == 2 and p["table"] is not None
    m.write(0, TM, 54613, 0)  # need 54614, within the capacity: nothing changes
    m.publish()
    assert m.cap["team"] == 64000
    m = _hand_model()
    m.write(0, TM, 54613, 0)  # need 54614 at the first growth: capacity 65 536, still narrow, but no table
    m.publish()
    (p,) = CR.restate(m, CR.pairs(m, STEPS))
    assert m.cap["team"] == 65536 and p["width"] == 2 and p["table"] is None
    m.write(0, TM, 65536, 1)
    m.publish()
    (p,) = CR.restate(m, CR.pairs(m, STEPS))
    assert m.cap["team"] > 65536 and p["width"] == 4 and p["table"] is None
    assert 65536 in p["col"][p["row_ptr"][0]:p["row_ptr"][1]].tolist()


def test_cfg3_store_matches_the_emulator_restatements():
    rng = np.random.default_rng(7)
    groups, n_users, _ = cfg3_groups(rng)
    m = CR.Model()
    m.load([g + (None,) for g in groups])
    m.publish()
    (p,) = CR.restate(m, CR.pairs(m, STEPS))
    n = m.cap["user"]
    want = emu_closure_rows(groups, n)
    got = [p["col"][p["row_ptr"][u]:p["row_ptr"][u + 1]] for u in range(n)]
    assert all(np.array_equal(a, b) for a, b in zip(got, want)) and len(got) == len(want)
    assert np.array_equal(p["sig"], np_signature(want, p["words"]))
    hdr, tab = p["table"]
    want_hdr, want_tab = np_table([r.astype(np.int64) for r in want])
    assert np.array_equal(hdr, want_hdr) and np.array_equal(tab, want_tab)


def test_rows_past_the_table_limit_have_no_table():
    """One user whose group joins L teams: rows the bucket limit cannot place leave the pair without a table."""
    def model(L):
        m = CR.Model()
        m.load([("group", "member", "user", np.array([0]), np.array([0]), None, None),
                ("team", "member", "group", np.arange(L), np.zeros(L, np.int64), "member", None),
                ("namespace", "viewer", "team", np.array([0]), np.array([0]), "member", None)])
        m.publish()
        return CR.restate(m, CR.pairs(m, STEPS))[0]

    assert model(4000)["table"] is not None
    for L in (16383, 16384, 16385):
        p = model(L)
        assert p["built"] and p["table"] is None and p["col"].size == L
