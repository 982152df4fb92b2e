"""CPU: the exact GROUP BY reference (tests/agg_reference.py) — the CPU oracle's group_aggregate meets it on special, exact and
rounding value sets, and the checker rejects what a subtly wrong kernel would return while accepting every order's correct answer."""
import math

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import agg_cases as AC
from tests import agg_reference as R
from tests import oracle_api as O

ALL_AGGS = [(R.COUNT, 1), (R.SUM, 1), (R.MIN, 1), (R.MAX, 1), (R.AVG, 1)]


def oracle_groups(rows, num, isn, group_cols, aggs):
    db = O.Db(np.zeros(1, np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint32), num, isn)
    slots = list(range(rows.shape[1]))
    rel = O.rel_from_host(slots, [rows[:, j] for j in slots])
    return db.group(rel, group_cols, [(k, s) for k, s in aggs])


def special_table(shuffle, seed=0):
    gid, vals, codes = AC.special_rows()
    if shuffle:
        p = np.random.default_rng(seed).permutation(len(gid))
        gid, vals, codes = gid[p], vals[p], codes[p]
    ids, num, isn = AC.encode(vals, codes, base=100)
    rows = np.stack([gid.astype(np.uint32), ids], axis=1)
    return rows, num, isn


@pytest.mark.parametrize("shuffle", [False, True])
def test_oracle_group_aggregate_meets_spec_on_special_values(shuffle):
    """f64::min / f64::max ignore a NaN operand: MIN of [NaN, 5.0] is 5.0, not NaN (std::min would return whichever came first)"""
    rows, num, isn = special_table(shuffle, seed=3)
    for aggs in [ALL_AGGS] + [[a] for a in ALL_AGGS]:
        R.assert_groups_match(oracle_groups(rows, num, isn, [0], aggs), rows, num, [0], aggs, f"oracle, shuffled={shuffle}")


@pytest.mark.parametrize("vset", ["V1", "V2"])
def test_oracle_group_aggregate_meets_spec_on_exact_and_rounding_values(vset):
    rng = np.random.default_rng(11)
    gid = AC.assign_groups(rng, 20000, 65)
    vals = AC.v1_values(rng, len(gid)) if vset == "V1" else AC.v2_values(rng, gid)
    ids, num, isn = AC.encode(vals, np.zeros(len(vals), np.int8))
    rows = np.stack([gid.astype(np.uint32), ids], axis=1)
    R.assert_groups_match(oracle_groups(rows, num, isn, [0], ALL_AGGS), rows, num, [0], ALL_AGGS, vset)


# ---- the checker itself: a sequential fold with the reference's semantics, in several orders, must pass; corruptions must not


def fold(xs, kind):
    """group_and_aggregate_results for one group, rows in the given order: first value seeds, then +, f64::min, f64::max"""
    if kind == R.COUNT:
        return float(len(xs))
    acc = xs[0]
    for x in xs[1:]:
        if kind in (R.SUM, R.AVG):
            acc = acc + x
        elif kind == R.MIN:
            acc = x if math.isnan(acc) else (acc if math.isnan(x) else min(acc, x))
        else:
            acc = x if math.isnan(acc) else (acc if math.isnan(x) else max(acc, x))
    return acc / len(xs) if kind == R.AVG else acc


def one_group(values):
    """(rows, num) of one group (key 7) whose value ids index `values`"""
    values = np.asarray(values, dtype=np.float64)
    rows = np.stack([np.full(len(values), 7, np.uint32), np.arange(len(values), dtype=np.uint32)], axis=1)
    return rows, values


def got_of(rows, vals):
    return {"keys": [np.array([7], np.uint32)], "values": [np.array([v], np.float64) for v in vals],
            "counts": np.array([len(rows)], np.uint64)}


def accepts(values, kind, got):
    rows, num = one_group(values)
    try:
        R.assert_groups_match(got_of(rows, [got]), rows, num, [0], [(kind, 1)])
        return True
    except AssertionError:
        return False


@pytest.mark.parametrize("which", ["V1", "V2", "specials"])
def test_checker_accepts_every_order(which):
    rng = np.random.default_rng(5)
    if which == "V1":
        groups = [AC.v1_values(rng, n) for n in (1, 2, 33, 1000)]
    elif which == "V2":
        groups = [AC.v2_values(rng, np.zeros(n, np.int64)) for n in (1, 2, 33, 1000)]
    else:
        groups = [np.array([v if not isinstance(v, tuple) else 0.0 for v in vs]) for _, vs in AC.SPECIAL_GROUPS if len(vs)]
    for xs in groups:
        for kind in (R.COUNT, R.SUM, R.MIN, R.MAX, R.AVG):
            for order in (xs, xs[::-1], rng.permutation(xs)):
                want = fold([float(x) for x in order], kind)
                assert accepts(xs, kind, want), (which, kind, list(order)[:5], want)
            if kind in (R.SUM, R.AVG) and np.isfinite(xs).all() and not (np.signbit(xs) & (xs == 0)).all() and np.abs(xs).max() < 1e300:
                s = math.fsum(xs)  # the correctly rounded sum (fsum returns +0.0 for all -0.0, and overflows: both excluded)
                assert accepts(xs, kind, s / len(xs) if kind == R.AVG else s)


def test_checker_rejects_float32_sums():
    rng = np.random.default_rng(1)
    xs = AC.v1_values(rng, 100_000)
    acc = np.float32(0)
    for x in xs.astype(np.float32):
        acc = np.float32(acc + x)
    assert accepts(xs, R.SUM, math.fsum(xs))
    assert not accepts(xs, R.SUM, float(acc))
    assert not accepts(xs, R.AVG, float(acc) / len(xs))
    assert not accepts(xs, R.SUM, float(np.sum(xs.astype(np.float32), dtype=np.float32)))


def test_checker_rejects_a_dropped_or_doubled_value():
    rng = np.random.default_rng(2)
    xs = AC.v1_values(rng, 100_000)
    xs[xs == 0] = 1.0
    for kind in (R.SUM, R.AVG):
        d = len(xs) if kind == R.AVG else 1
        assert accepts(xs, kind, math.fsum(xs) / d)
        assert not accepts(xs, kind, math.fsum(xs[1:]) / d), "one value dropped"
        assert not accepts(xs, kind, math.fsum(np.append(xs, xs[12345])) / d), "one value counted twice"
    # a dropped row seen through the counts
    rows, num = one_group(xs)
    got = got_of(rows, [math.fsum(xs)])
    got["counts"] = np.array([len(xs) - 1], np.uint64)
    with pytest.raises(AssertionError, match="count"):
        R.assert_groups_match(got, rows, num, [0], [(R.SUM, 1)])
    got["counts"] = np.array([len(xs) + 1], np.uint64)
    with pytest.raises(AssertionError, match="count"):
        R.assert_groups_match(got, rows, num, [0], [(R.SUM, 1)])


def test_checker_rejects_wrong_special_values():
    neg0 = [-0.0] * 6
    assert accepts(neg0, R.SUM, -0.0) and accepts(neg0, R.AVG, -0.0) and accepts(neg0, R.MIN, -0.0) and accepts(neg0, R.MAX, -0.0)
    assert not accepts(neg0, R.SUM, 0.0), "+0.0 for an all-(-0.0) SUM"
    assert not accepts(neg0, R.AVG, 0.0), "+0.0 for an all-(-0.0) AVG"
    assert not accepts(neg0, R.MIN, 0.0)
    nans = [math.nan] * 4
    assert accepts(nans, R.MIN, math.nan) and accepts(nans, R.MAX, math.nan)
    assert not accepts(nans, R.MIN, math.inf), "+inf for an all-NaN MIN"
    assert not accepts(nans, R.MAX, -math.inf), "-inf for an all-NaN MAX"
    assert accepts([math.nan, 5.0], R.MIN, 5.0) and accepts([5.0, math.nan], R.MAX, 5.0)
    assert not accepts([math.nan, 5.0], R.MIN, math.nan), "NaN for MIN of [NaN, 5]"
    assert not accepts([5.0, math.nan], R.MAX, math.nan)
    assert accepts([math.nan, 5.0], R.SUM, math.nan) and not accepts([math.nan, 5.0], R.SUM, 5.0)
    assert accepts([math.inf, -math.inf], R.SUM, math.nan) and not accepts([math.inf, -math.inf], R.SUM, math.inf)
    assert accepts([math.inf, 1.0], R.AVG, math.inf) and not accepts([math.inf, 1.0], R.AVG, math.nan)
    mixed = [-0.0, 0.0]
    assert accepts(mixed, R.MIN, 0.0) and accepts(mixed, R.MIN, -0.0) and accepts(mixed, R.SUM, 0.0)
    assert not accepts(mixed, R.SUM, -0.0), "+0.0 + -0.0 is +0.0 in every order"
    big = [AC.DBL_MAX, AC.DBL_MAX]
    assert accepts(big, R.SUM, math.inf) and not accepts(big, R.SUM, AC.DBL_MAX)
    assert accepts([AC.SUBNORMAL] * 3, R.SUM, 3 * AC.SUBNORMAL) and not accepts([AC.SUBNORMAL] * 3, R.SUM, 2 * AC.SUBNORMAL)


def test_checker_rejects_sums_outside_the_rounding_bound():
    rng = np.random.default_rng(4)
    for n in (3, 100, 10_000):
        xs = AC.v2_values(rng, np.zeros(n, np.int64))
        s = math.fsum(xs)
        a = math.fsum(np.abs(xs))
        off = 4 * float(R.gamma(n - 1)) * a
        assert accepts(xs, R.SUM, s)
        assert not accepts(xs, R.SUM, s + off) and not accepts(xs, R.SUM, s - off), n
        assert not accepts(xs, R.AVG, (s + off) / n), n


def test_checker_rejects_missing_extra_and_misrouted_groups():
    rows = np.array([[1, 0], [1, 1], [2, 2]], np.uint32)
    num = np.array([1.0, 2.0, 4.0])
    ok = {"keys": [np.array([2, 1], np.uint32)], "values": [np.array([4.0, 3.0])], "counts": np.array([1, 2], np.uint64)}
    R.assert_groups_match(ok, rows, num, [0], [(R.SUM, 1)])  # order of the groups does not matter
    bad = {"keys": [np.array([1], np.uint32)], "values": [np.array([3.0])], "counts": np.array([2], np.uint64)}
    with pytest.raises(AssertionError, match="groups returned"):
        R.assert_groups_match(bad, rows, num, [0], [(R.SUM, 1)])
    bad = {"keys": [np.array([2, 3], np.uint32)], "values": [np.array([4.0, 3.0])], "counts": np.array([1, 2], np.uint64)}
    with pytest.raises(AssertionError, match="missing"):
        R.assert_groups_match(bad, rows, num, [0], [(R.SUM, 1)])
    bad = {"keys": [np.array([2, 1], np.uint32)], "values": [np.array([3.0, 4.0])], "counts": np.array([1, 2], np.uint64)}
    with pytest.raises(AssertionError, match="SUM"):
        R.assert_groups_match(bad, rows, num, [0], [(R.SUM, 1)])


def test_row_values_follow_unwrap_or_zero():
    num = np.array([1.5, -2.0, 0.0])
    ids = np.array([0, 1, 2, 3, 0x80000001, c.KB_ID_NONE], np.uint32)
    assert R.row_values(ids, num).tolist() == [1.5, -2.0, 0.0, 0.0, 0.0, 0.0]
