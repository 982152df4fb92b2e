"""CPU: the id remaps of tests/id_domain_cases.py are valid, and the oracle commutes with each of them — oracle(f(x)) == f(oracle(x))
as bags for scan, BGP, hash join and fixpoint — so it is id-agnostic and can judge the device at the edges of the u32 domain."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import helpers as H
from tests import id_domain_cases as D
from tests import oracle_api as O

ROWS = D.star_store()
MAPS = D.remaps(ROWS)


@pytest.mark.parametrize("family", D.FAMILIES)
def test_remap_is_valid(family):
    f = MAPS[family]
    img = f.vals
    assert len(np.unique(img)) == len(img), "not injective"
    assert not np.any(img == D.NONE), "an id maps onto KB_ID_NONE"
    num = np.arange(D.NUM_LO, D.NUM_HI, dtype=np.uint32)
    assert np.array_equal(f(num), num), "a numeric id moved"
    assert f.id(D.NONE) == D.NONE
    if family == "identity":
        assert np.array_equal(f.keys, img)
    if family == "quoted":
        moved = img[f.keys != img]
        assert len(moved) and np.all(moved >= 0x80000000) and np.all((moved & 0x7FFFFFFF) < D.QUOTED_LIMIT)
    if family == "straddle":
        moved = img[f.keys != img]
        assert moved.min() < 0x80000000 <= moved.max()
    if family == "extremes":
        assert set(D.EXTREMES) <= set(img.tolist())


def test_remap_refuses_ids_outside_its_domain():
    with pytest.raises(AssertionError):
        MAPS["scatter"](np.array([0xFFFFFFF0], np.uint32))


def rows_of(rel, slots):
    return rel.to_numpy(slots) if rel.n_rows else np.empty((0, len(slots)), np.uint32)


def db_of(rows):
    num, isn = D.numeric_table()
    return O.Db(rows[:, 0], rows[:, 1], rows[:, 2], num, isn)


@pytest.mark.parametrize("family", D.FAMILIES)
def test_oracle_commutes_with_remap(family):
    f = MAPS[family]
    base, moved = db_of(ROWS), db_of(f(ROWS))
    # scan: every position bound in turn, a repeated variable
    some = ROWS[7]
    scans = [c.pattern(c.V(0), c.K(D.P_KNOWS), c.V(1)), c.pattern(c.K(int(some[0])), c.V(1), c.V(2)),
             c.pattern(c.V(0), c.V(1), c.K(int(some[2]))), c.pattern(c.V(0), c.K(D.P_KNOWS), c.V(0)), c.pattern(c.V(0), c.K(D.P_TAG), c.K(1))]
    for pat in scans:
        a = base.scan(pat)
        b = moved.scan(f.pattern(pat))
        assert a.n_rows == b.n_rows
        H.assert_same_bag(rows_of(b, sorted(b.slots)), f(rows_of(a, sorted(a.slots))), f"{family} scan")
    # star BGPs with a numeric FILTER, and a chain
    for name, (_, pats, filt) in D.star_queries().items():
        a = base.bgp(pats, filt)
        b = moved.bgp([f.pattern(p) for p in pats], f.filt(filt))
        assert a.n_rows > 0
        H.assert_same_bag(rows_of(b, sorted(b.slots)), f(rows_of(a, sorted(a.slots))), f"{family} {name}")
    a = base.bgp(D.bgp_chain())
    b = moved.bgp([f.pattern(p) for p in D.bgp_chain()])
    assert a.n_rows > 0
    H.assert_same_bag(rows_of(b, sorted(b.slots)), f(rows_of(a, sorted(a.slots))), f"{family} chain")
    # hash join over relations built from the store's columns
    g = np.random.default_rng(4)
    lc = [ROWS[g.integers(0, len(ROWS), 3000), 0], ROWS[g.integers(0, len(ROWS), 3000), 2]]
    rc = [ROWS[:, 0], ROWS[:, 1]]
    a = O.hash_join(O.rel_from_host([0, 1], lc), O.rel_from_host([0, 2], rc))
    b = O.hash_join(O.rel_from_host([0, 1], [f(x) for x in lc]), O.rel_from_host([0, 2], [f(x) for x in rc]))
    assert a.n_rows > 0
    H.assert_same_bag(rows_of(b, [0, 1, 2]), f(rows_of(a, [0, 1, 2])), f"{family} hash join")
    # fixpoint: facts, rounds, per-round counts and derivations
    rules = D.store_rules()
    a = base.fixpoint(rules)
    b = moved.fixpoint([f.rule(r) for r in rules])
    assert a["status"] == b["status"] == 0 and len(a["facts"]) > 0
    H.assert_same_bag(b["facts"], f(a["facts"]), f"{family} fixpoint")
    assert a["round_new"] == b["round_new"] and a["derivations"] == b["derivations"]


@pytest.mark.parametrize("hi", [0xFFFFFFFE, 0x80000000 + (1 << 19)])
@pytest.mark.parametrize("past", [False, True])
def test_threshold_builders_sit_on_their_thresholds(hi, past):
    (_, lc), (_, rc), route = D.grouped_pair(hi, past)
    assert int(rc[0].max()) == hi and int(rc[0].max()) - int(rc[0].min()) + 1 == D.GROUPED_MIN + past
    assert route == ("chained" if past else "grouped")
    for kind in ("r3", "slice", "r2"):
        tr, on = D.star_threshold(kind, hi, past)
        s = tr[:, 0].astype(np.uint64)
        n = len(np.unique(s))
        lim = {"r3": D.R3_MIN, "slice": D.slice_table_max(n), "r2": D.r2_max(n)}[kind]
        assert s.max() == hi and s.max() - s.min() + 1 == lim + past and on == (not past)
        assert len(tr) == 3 * n and len(np.unique(tr[:, [0, 1]], axis=0)) == len(tr)  # every build side single-valued
    tr, lo, top = D.directory_store(hi, past)
    assert top == hi and top - lo + 1 == D.DIRECTORY_MIN + past


@pytest.mark.parametrize("lo", [16, 0x7FF00000, 0xFFFFFFFE - (1 << 28) - 200])
def test_bitmap_store_spans_the_bitmap_edge(lo):
    tr, pats = D.bitmap_store(lo)
    # the bitmap of ?x starts at the largest of its columns' store-wide minima and ends at the smallest maximum, capped at 2^28 ids
    assert max(int(tr[:, 0].min()), int(tr[:, 2].min())) == lo
    assert min(int(tr[:, 0].max()), int(tr[:, 2].max())) >= lo + D.RED_MAX_BITS
    x_obj = set(tr[tr[:, 1] == 130, 2].tolist())
    x_subj = set(tr[tr[:, 1] == 131, 0].tolist())
    edge = {lo, lo + D.RED_MAX_BITS - 1, lo + D.RED_MAX_BITS}
    assert edge <= x_obj and edge <= x_subj
    want = db_of(tr).bgp(pats)
    got_x = set(rows_of(want, [1])[:, 0].tolist())
    assert edge <= got_x  # every edge id survives the join: a reduction that drops one is wrong
