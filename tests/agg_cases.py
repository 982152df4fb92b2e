"""Inputs for the GROUP BY aggregate tests, with every value under the test's control: rows of (key columns, value id), the numeric
table the value ids index, and the value sets

  V1  exact: multiples of 2^-8 in (-2^20, 2^20); any group of at most 2^24 rows sums exactly in every order.
  V2  rounding: random signs, magnitudes log-uniform in [1e-290, 1e290], cancelling pairs (x, -x) and [1e16, 1, -1e16] triples.
  V3  special groups: NaN, infinities, signed zeros, DBL_MAX, subnormals, DBL_MIN, and ids whose value is 0.0 because they are not
      numeric, lie at or above the numeric table, or are quoted triples (bit 31).
"""
from __future__ import annotations

import numpy as np

NAN, INF = float("nan"), float("inf")
DBL_MAX = float(np.finfo(np.float64).max)
DBL_MIN = float(np.finfo(np.float64).tiny)
SUBNORMAL = 5e-324
QUOTED_BIT = 0x80000000

# value codes of a row: 0 = the float value, else an id whose value is 0.0 for one of these reasons
NUMERIC, NON_NUMERIC, BEYOND_TABLE, QUOTED = range(4)

# V3: (name, values); a value is a float or one of the codes above as ("id", code)
NN, BY, QT = ("id", NON_NUMERIC), ("id", BEYOND_TABLE), ("id", QUOTED)
SPECIAL_GROUPS = [
    ("all NaN", [NAN] * 40),
    ("one NaN", [NAN]),
    ("NaN first", [NAN, 5.0, -2.5, 7.0]),
    ("NaN last", [5.0, -2.5, 7.0, NAN]),
    ("+inf only", [INF, INF, INF]),
    ("-inf only", [-INF, -INF]),
    ("+inf and -inf", [INF, 1.0, -INF, 2.0]),
    ("+inf and NaN", [INF, NAN, 3.0]),
    ("-0.0 only", [-0.0] * 40),
    ("one -0.0", [-0.0]),
    ("-0.0 and +0.0", [-0.0, 0.0, -0.0, 0.0]),
    ("-0.0 and NaN", [NAN, -0.0, -0.0, NAN]),
    ("DBL_MAX twice", [DBL_MAX, DBL_MAX]),
    ("-DBL_MAX and 1", [-DBL_MAX, 1.0, -DBL_MAX]),
    ("subnormals", [SUBNORMAL] * 9),
    ("subnormals of both signs", [SUBNORMAL, -SUBNORMAL, SUBNORMAL, 3 * SUBNORMAL]),
    ("DBL_MIN", [DBL_MIN, DBL_MIN, -SUBNORMAL]),
    ("non-numeric ids with positives", [NN, 3.0, 4.5, NN]),
    ("non-numeric ids only", [NN, NN]),
    ("ids beyond the table with negatives", [BY, -1.5, -2.0]),
    ("quoted-triple ids", [QT, 8.0, QT, -0.0]),
    ("cancelling", [1e16, 1.0, -1e16]),
]


def encode(values: np.ndarray, codes: np.ndarray, base: int = 0):
    """one value id per row: row i gets id base + i with num_or0 = values[i] (codes NUMERIC), a non-numeric id, an id past the
    table or a quoted-triple id. Returns (ids u32, num_or0 f64, is_num u8); ids below `base` exist and are not numeric."""
    n = len(values)
    ids = (base + np.arange(n, dtype=np.int64)).astype(np.uint32)
    n_ids = base + n
    num = np.zeros(n_ids, dtype=np.float64)
    isn = np.zeros(n_ids, dtype=np.uint8)
    num_rows = codes == NUMERIC
    num[base:][num_rows] = values[num_rows]
    isn[base:][num_rows] = 1
    by = np.flatnonzero(codes == BEYOND_TABLE)
    ids[by] = (n_ids + np.arange(len(by))).astype(np.uint32)
    qt = np.flatnonzero(codes == QUOTED)
    ids[qt] = (QUOTED_BIT | (np.arange(len(qt)) % 1000)).astype(np.uint32)
    return ids, num, isn


def special_rows(first_group: int = 0):
    """V3: (group index per row, values, codes) of SPECIAL_GROUPS, group g of the list numbered first_group + g"""
    gid, vals, codes = [], [], []
    for g, (_, vs) in enumerate(SPECIAL_GROUPS):
        for v in vs:
            gid.append(first_group + g)
            if isinstance(v, tuple):
                vals.append(0.0)
                codes.append(v[1])
            else:
                vals.append(v)
                codes.append(NUMERIC)
    return np.array(gid, dtype=np.int64), np.array(vals, dtype=np.float64), np.array(codes, dtype=np.int8)


def v1_values(rng, n):
    return rng.integers(-(1 << 28) + 1, 1 << 28, n).astype(np.float64) / 256.0


def v2_values(rng, gid):
    """V2 for rows whose groups are `gid`: log-uniform magnitudes, random signs; a quarter of the rows cancel a neighbour of their
    group, and the first three rows of every fourth group hold [1e16, 1, -1e16]"""
    n = len(gid)
    x = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-290, 290, n)
    order = np.argsort(gid, kind="stable")
    g = gid[order]
    pair = np.flatnonzero((g[1:] == g[:-1]) & (rng.random(n - 1) < 0.25) if n > 1 else np.zeros(0, bool))
    pair = pair[np.concatenate(([True], np.diff(pair) > 1))] if len(pair) else pair  # non-overlapping
    x[order[pair + 1]] = -x[order[pair]]
    starts = np.concatenate(([0], np.flatnonzero(np.diff(g) != 0) + 1)) if n else np.zeros(0, np.int64)
    sizes = np.diff(np.append(starts, n))
    for s in starts[(sizes >= 3) & (g[starts] % 4 == 0)][:2000]:
        x[order[s:s + 3]] = (1e16, 1.0, -1e16)
    return x


def assign_groups(rng, n_rows: int, n_groups: int):
    """a group index per row: every group gets a row when n_rows >= n_groups, the rest at random, in random order"""
    if n_rows == 0:
        return np.zeros(0, dtype=np.int64)
    g = rng.integers(0, n_groups, n_rows)
    k = min(n_rows, n_groups)
    g[:k] = np.arange(k)
    return rng.permutation(g)


def group_keys(rng, n_groups: int, edge_keys=(0, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE), lo: int = 0):
    """n_groups distinct u32 keys starting with the edge ids (0, the largest dictionary id, ids with bit 31 set), then random ids"""
    keys = list(dict.fromkeys(edge_keys))[:n_groups]
    seen = set(keys)
    while len(keys) < n_groups:
        for k in rng.integers(lo, 0xFFFFFFFE, 2 * (n_groups - len(keys)) + 8).tolist():
            if k not in seen and len(keys) < n_groups:
                seen.add(k)
                keys.append(k)
    return np.array(keys, dtype=np.uint32)


def mix32(x: np.ndarray) -> np.ndarray:
    """the murmur3 finaliser of kb_device.cuh, on u32 arrays"""
    x = np.asarray(x, dtype=np.uint32).copy()
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x85EBCA6B)
    x ^= x >> np.uint32(13)
    x *= np.uint32(0xC2B2AE35)
    x ^= x >> np.uint32(16)
    return x


def warp_hash(cols) -> np.ndarray:
    """group_kernel's in-warp match value of a multi-column key: h = 0; h = mix32(h ^ k[c]) + c"""
    h = np.zeros(len(cols[0]), dtype=np.uint32)
    for c, k in enumerate(cols):
        h = mix32(h ^ np.asarray(k, dtype=np.uint32)) + np.uint32(c)
    return h


def colliding_pair(seed: int = 7):
    """two distinct 2-column keys with the same warp_hash (birthday search)"""
    rng = np.random.default_rng(seed)
    while True:
        a = rng.integers(0, 1 << 31, 1 << 18).astype(np.uint32)
        b = rng.integers(0, 1 << 31, 1 << 18).astype(np.uint32)
        h = warp_hash([a, b])
        order = np.argsort(h, kind="stable")
        hs = h[order]
        dup = np.flatnonzero(hs[1:] == hs[:-1])
        for d in dup:
            i, j = order[d], order[d + 1]
            if (a[i], b[i]) != (a[j], b[j]):
                return (int(a[i]), int(b[i])), (int(a[j]), int(b[j]))
