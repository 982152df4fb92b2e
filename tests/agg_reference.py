"""Exact reference for GROUP BY aggregates (group_and_aggregate_results, execute_query.rs:1150-1227) and the one definition of
"the device's groups agree with it" that every aggregate test uses.

The reference folds a group's rows in hash-iteration order and the device in tile-completion and atomic order, so the rules hold
for EVERY order of the rows. For one group with values x_1..x_n (x = num_or0[id]; 0.0 for ids at or above the numeric table, which
covers quoted-triple ids, and for non-numeric terms, whose num_or0 is 0.0), u = 2^-53 and gamma_k = k*u / (1 - k*u):

  COUNT  the exact row count.
  MIN    NaN iff every value is NaN; else the minimum (maximum for MAX) of the non-NaN values, bit for bit — except that when it is
  MAX    a zero and both +0.0 and -0.0 occur, either sign is accepted (f64::min / f64::max leave that case unspecified).
  SUM    NaN if any value is NaN or both infinities occur; else +-inf if that infinity occurs; else, with S the exact sum:
           if every partial sum in every order is representable (all values on a grid 2^q with sum |x_i| < 2^(q+53)), bit-identical
           to S, and -0.0 exactly when every value is -0.0;
           if S rounds past the largest double, +-inf;
           otherwise |got - S| <= gamma_{n-1} * sum |x_i|.
  AVG    the SUM rule divided by n: bit-identical to float(S / n) in the exact case, otherwise within
         gamma_{n-1} * sum |x_i| / n + u * |S / n|.

Exact sums are Python integers in units of 2^-1126 (the smallest double, 2^-1074, scaled down by the 52 bits a mantissa shift can
add), built from vectorised per-exponent partial sums, so a group of millions of rows costs one numpy pass and a short Python loop.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

COUNT, SUM, MIN, MAX, AVG = range(5)
KIND_NAMES = {COUNT: "COUNT", SUM: "SUM", MIN: "MIN", MAX: "MAX", AVG: "AVG"}

U = Fraction(1, 1 << 53)
_SCALE = 1126  # exact sums are integers times 2^-_SCALE
_NEG_ZERO_BITS = np.float64(-0.0).view(np.int64)
_DBL_MAX = int(Fraction(np.finfo(np.float64).max) * (1 << _SCALE))


def gamma(k: int) -> Fraction:
    return k * U / (1 - k * U)


def row_values(ids: np.ndarray, num_or0: np.ndarray) -> np.ndarray:
    """num_or0[id] with 0.0 for every id the table does not cover (unwrap_or(0.0), execute_query.rs:1171-1184)"""
    ids = np.asarray(ids, dtype=np.uint64)
    num_or0 = np.asarray(num_or0, dtype=np.float64)
    out = np.zeros(len(ids), dtype=np.float64)
    inside = ids < len(num_or0)
    out[inside] = num_or0[ids[inside].astype(np.int64)]
    return out


def _bits(x) -> int:
    return int(np.float64(x).view(np.int64))


def _fmt(x: float) -> str:
    return f"{float(x)!r} (0x{_bits(x) & 0xFFFFFFFFFFFFFFFF:016x})"


def _exact_group_sums(x: np.ndarray, starts: np.ndarray, n_groups: int):
    """per group: (exact sum, exact sum of |x|, q) of the FINITE values x (non-finite entries must be zeroed by the caller); sums are
    integers in units of 2^-_SCALE, q = exponent (same units) of the lowest set bit over the group's nonzero values (None: all zero)"""
    grp = np.repeat(np.arange(n_groups, dtype=np.int64), np.diff(np.append(starts, len(x))))
    m, e = np.frexp(x)
    mi = np.ldexp(m, 53).astype(np.int64)  # x = mi * 2^(e - 53), exactly (subnormals included)
    sh = e.astype(np.int64) - 53 + _SCALE   # >= 0 for every double
    nz = mi != 0
    low = np.zeros(len(x), dtype=np.int64)
    low[nz] = np.log2((mi[nz] & -mi[nz]).astype(np.float64)).astype(np.int64)  # trailing zeros of the mantissa
    q_row = np.where(nz, sh + low, np.iinfo(np.int64).max)
    q = np.minimum.reduceat(q_row, starts)  # x is sorted by group
    out = []
    for vals in (mi, np.abs(mi)):
        hi = vals >> 26
        lo = vals - (hi << 26)  # both fit 27 bits: per-(group, exponent) sums of millions of rows stay inside int64
        order = np.lexsort((sh, grp))
        g_s, sh_s = grp[order], sh[order]
        if len(order):
            brk = np.flatnonzero((np.diff(g_s) != 0) | (np.diff(sh_s) != 0)) + 1
            first = np.concatenate(([0], brk))
            shi = np.add.reduceat(hi[order], first)
            slo = np.add.reduceat(lo[order], first)
            gg, ss = g_s[first], sh_s[first]
        else:
            shi = slo = gg = ss = np.empty(0, dtype=np.int64)
        tot = [0] * n_groups
        for g, s, a, b in zip(gg.tolist(), ss.tolist(), shi.tolist(), slo.tolist()):
            tot[g] += ((a << 26) + b) << s
        out.append(tot)
    return out[0], out[1], [None if v == np.iinfo(np.int64).max else int(v) for v in q.tolist()]


class GroupTruth:
    """the exact per-group facts one aggregate column needs, computed once per (rows, column)"""

    def __init__(self, v: np.ndarray, starts: np.ndarray, n_groups: int):
        ends = np.append(starts[1:], len(v))
        self.n = (ends - starts).astype(np.int64)
        isnan = np.isnan(v)
        red = lambda f, a: f.reduceat(a, starts) if len(v) else np.zeros(0, a.dtype)  # noqa: E731
        self.n_nan = red(np.add, isnan.astype(np.int64))
        self.has_pinf = red(np.logical_or, v == np.inf)
        self.has_ninf = red(np.logical_or, v == -np.inf)
        bits = v.view(np.int64)
        self.n_negzero = red(np.add, (bits == _NEG_ZERO_BITS).astype(np.int64))
        self.has_poszero = red(np.logical_or, bits == 0)
        self.has_negzero = self.n_negzero > 0
        with np.errstate(invalid="ignore"):
            self.vmin = red(np.fmin, v)
            self.vmax = red(np.fmax, v)
        self._v, self._starts, self._n_groups = v, starts, n_groups
        self._sums = None

    def sums(self):
        """(exact sums, exact sums of |x|, q) per group, computed on first use (MIN / MAX do not need them)"""
        if self._sums is None:
            finite = np.where(np.isfinite(self._v), self._v, 0.0)
            self._sums = _exact_group_sums(finite, self._starts, self._n_groups)
        return self._sums

    def expect_minmax(self, g: int, kind: int):
        """(expected value, both zero signs occur)"""
        if self.n_nan[g] == self.n[g]:
            return float("nan"), False
        ext = self.vmin[g] if kind == MIN else self.vmax[g]
        if ext == 0.0 and self.has_poszero[g] and self.has_negzero[g]:
            return 0.0, True
        if ext == 0.0:  # only one sign occurs: that one
            return (-0.0 if self.has_negzero[g] else 0.0), False
        return float(ext), False

    def check_sum(self, g: int, got: float, kind: int):
        """None if `got` is an admissible SUM (AVG) of group g, else the rule it breaks"""
        n = int(self.n[g])
        pinf, ninf = bool(self.has_pinf[g]), bool(self.has_ninf[g])
        if self.n_nan[g] or (pinf and ninf):
            return None if np.isnan(got) else "NaN expected (a NaN, or +inf together with -inf, in the group)"
        if pinf or ninf:
            want = np.inf if pinf else -np.inf
            return None if got == want else f"{want} expected (the group holds that infinity)"
        if np.isnan(got):
            return "NaN returned for a group of finite values"
        sums, abs_sums, qs = self.sums()
        S = Fraction(sums[g], 1 << _SCALE)
        A = Fraction(abs_sums[g], 1 << _SCALE)
        div = n if kind == AVG else 1
        q = qs[g]
        # every partial sum in every order is exact: a multiple of 2^q below 2^(q+53) in magnitude, and no larger than the largest double
        if q is None or (abs_sums[g] < (1 << (q + 53)) and abs_sums[g] <= _DBL_MAX):
            if q is None:
                want = -0.0 if self.n_negzero[g] == n else 0.0
                if kind == AVG:
                    want = want / n
            else:
                want = float(S / div)
            if _bits(got) != _bits(want):
                return f"exact case: want {_fmt(want)}, got {_fmt(got)}"
            return None
        try:
            float(S)
        except OverflowError:
            want = np.inf if S > 0 else -np.inf
            return None if got == want else f"the exact sum overflows in every order: want {want}, got {_fmt(got)}"
        if np.isinf(got):
            return f"inf returned, exact sum {float(S)!r} is finite"
        err = abs(Fraction(got) - S / div)
        bound = gamma(n - 1) * A / div + (U * abs(S / div) if kind == AVG else 0)
        if err > bound:
            return f"rounding case: |got - S{'/n' if div > 1 else ''}| = {float(err):.6g} > bound {float(bound):.6g} (got {_fmt(got)}, S ~ {float(S / div)!r})"
        return None


def _group_rows(keys: np.ndarray):
    """rows sorted by group: (unique keys [g, k], order, starts)"""
    keys = np.ascontiguousarray(keys, dtype=np.uint32)
    if keys.shape[0] == 0:
        return keys, np.empty(0, np.int64), np.empty(0, np.int64)
    if keys.shape[1] <= 2:
        k64 = keys[:, 0].astype(np.uint64) << np.uint64(32)
        if keys.shape[1] == 2:
            k64 |= keys[:, 1].astype(np.uint64)
        order = np.argsort(k64, kind="stable")
        ks = k64[order]
        starts = np.concatenate(([0], np.flatnonzero(np.diff(ks) != 0) + 1))
        return keys[order][starts], order, starts
    order = np.lexsort(tuple(keys[:, c] for c in range(keys.shape[1] - 1, -1, -1)))
    ks = keys[order]
    starts = np.concatenate(([0], np.flatnonzero((np.diff(ks, axis=0) != 0).any(axis=1)) + 1))
    return ks[starts], order, starts


def assert_groups_match_slots(got: dict, rows: np.ndarray, slots, values: np.ndarray, group_slots, aggs, what: str = ""):
    """assert_groups_match for rows whose columns hold the variable slots `slots` (e.g. a relation's to_numpy(slots)), with the
    GROUP BY and the aggregates given by slot as the C ABI takes them"""
    slots = list(slots)
    aggs_c = [(k, slots.index(s) if k != COUNT else 0) for k, s in aggs]
    assert_groups_match(got, rows, values, [slots.index(s) for s in group_slots], aggs_c, what)


def assert_groups_match(got: dict, rows: np.ndarray, values: np.ndarray, group_cols, aggs, what: str = ""):
    """got: groups as the device returns them ({"keys": [col], "values": [col], "counts": col}); rows: u32 [n, c] input rows;
    values: the numeric table num_or0 (f64 per dictionary id); group_cols: columns of `rows` grouped by; aggs: [(kind, column)]
    (the column is ignored for COUNT). Groups are matched by key; keys and counts must be equal exactly, every value must meet the
    rules of this module. Raises AssertionError naming the group, the aggregate and the rule."""
    rows = np.asarray(rows, dtype=np.uint32)
    if rows.ndim == 1:
        rows = rows[:, None]
    ukeys, order, starts = _group_rows(rows[:, list(group_cols)])
    n_groups = len(starts)
    gkeys = np.stack([np.asarray(k, dtype=np.uint32) for k in got["keys"]], axis=1) if len(got["keys"]) else np.empty((0, 0), np.uint32)
    gcounts = np.asarray(got["counts"], dtype=np.uint64)
    pre = f"{what}: " if what else ""
    assert gkeys.shape == (n_groups, len(group_cols)), f"{pre}{gkeys.shape[0]} groups returned, {n_groups} expected"
    at = {tuple(k): i for i, k in enumerate(gkeys.tolist())}
    assert len(at) == n_groups, f"{pre}a group key is returned twice"
    idx = np.empty(n_groups, dtype=np.int64)
    for g, k in enumerate(ukeys.tolist()):
        i = at.get(tuple(k))
        assert i is not None, f"{pre}group {k} is missing"
        idx[g] = i
    counts = np.diff(np.append(starts, len(order))).astype(np.uint64)
    bad = np.flatnonzero(gcounts[idx] != counts)
    assert len(bad) == 0, f"{pre}group {ukeys[bad[0]].tolist()}: count {int(gcounts[idx[bad[0]]])}, expected {int(counts[bad[0]])}"
    assert len(got["values"]) == len(aggs), f"{pre}{len(got['values'])} aggregate columns returned, {len(aggs)} expected"
    if n_groups == 0:
        return
    truths = {}
    for a, (kind, col) in enumerate(aggs):
        gv = np.asarray(got["values"][a], dtype=np.float64)[idx]
        name = KIND_NAMES[kind] + ("" if kind == COUNT else f"(col {col})")
        if kind == COUNT:
            bad = np.flatnonzero(gv != counts.astype(np.float64))
            assert len(bad) == 0, f"{pre}group {ukeys[bad[0]].tolist()} {name}: {gv[bad[0]]!r}, expected {int(counts[bad[0]])}"
            continue
        if col not in truths:
            truths[col] = GroupTruth(row_values(rows[order, col], values), starts, n_groups)
        t = truths[col]
        for g in range(n_groups):
            x = float(gv[g])
            if kind in (MIN, MAX):
                want, either = t.expect_minmax(g, kind)
                if np.isnan(want):
                    ok, rule = np.isnan(x), "NaN expected: every value of the group is NaN"
                elif either:
                    ok, rule = x == 0.0, "+-0.0 expected: the extreme is a zero and both signs occur"
                else:
                    ok, rule = _bits(x) == _bits(want), f"{_fmt(want)} expected: the {'least' if kind == MIN else 'greatest'} non-NaN value"
                if not ok:
                    raise AssertionError(f"{pre}group {ukeys[g].tolist()} {name}: got {_fmt(x)}; {rule}")
            else:
                why = t.check_sum(g, x, kind)
                if why is not None:
                    raise AssertionError(f"{pre}group {ukeys[g].tolist()} {name} over {int(t.n[g])} rows: {why}")
