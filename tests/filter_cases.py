"""Edge values of f64 comparison, shared by the FILTER tests: signed zeros, infinities, NaNs of both signs, subnormals, +-DBL_MAX, the
smallest normal, a few ordinary values, and the nextafter neighbours of each on both sides."""
import numpy as np

INF = np.inf
DMIN = np.nextafter(0.0, 1.0)
DBL_MAX = 1.7976931348623157e308
NORM_MIN = 2.2250738585072014e-308
BASE = [0.0, -0.0, INF, -INF, np.nan, np.copysign(np.nan, -1.0), DMIN, -DMIN, 2 * DMIN, NORM_MIN, -NORM_MIN, np.nextafter(NORM_MIN, 0.0),
        DBL_MAX, -DBL_MAX, 1.0, -1.0, 0.5, 100000.0, 99999.5, -100000.0, 3.0]
with np.errstate(over="ignore"):  # (the neighbours of +-DBL_MAX are +-inf)
    VALUES = np.array(BASE + [np.nextafter(x, INF) for x in BASE] + [np.nextafter(x, -INF) for x in BASE], dtype=np.float64)
# constants of the index probe's rank filter tests: the edge set, and the store value 100 000 with both its neighbours
CONSTS = [0.0, -0.0, INF, -INF, np.nan, DMIN, -DMIN, 100000.0, np.nextafter(100000.0, INF), np.nextafter(100000.0, -INF), 99999.75, 2.5,
          -DBL_MAX, DBL_MAX, np.nextafter(0.0, -1.0)]


def boundary_consts(values):
    """every distinct value of `values` (NaNs and both zeros kept apart by their bits) and both of its nextafter neighbours, plus CONSTS:
    the constants at which each ordering comparison changes its answer on some stored value"""
    v = np.asarray(values, dtype=np.float64)
    with np.errstate(over="ignore"):
        allv = np.concatenate([v, np.nextafter(v, INF), np.nextafter(v, -INF), np.asarray(CONSTS, dtype=np.float64)])
    return np.unique(allv.view(np.uint64)).view(np.float64)


def numeric_table(n_ids, lit0, values=VALUES):
    """num_or0 / is_num over n_ids ids: ids lit0 .. lit0 + len(values) carry `values`, every other id is not a number"""
    num = np.zeros(n_ids, dtype=np.float64)
    isn = np.zeros(n_ids, dtype=np.uint8)
    num[lit0:lit0 + len(values)] = values
    isn[lit0:lit0 + len(values)] = 1
    return num, isn


def edge_cells(rng, n, lit0, n_plain, n_ids, relation=True):
    """ids of n cells: numeric edge values (ids lit0..), non-numeric literals (the n_plain ids after them) and ids past the numeric
    table; with relation=True also quoted-triple ids (bit 31) and KB_ID_NONE, which only a relation (never the store) holds"""
    kind = rng.integers(0, 10 if relation else 8, n)
    return np.select([kind < 6, kind == 6, kind == 7, kind == 8],
                     [lit0 + rng.integers(0, len(VALUES), n), lit0 + len(VALUES) + rng.integers(0, n_plain, n),
                      rng.integers(n_ids, n_ids + 100, n), 0x80000000 + rng.integers(0, 50, n)], 0xFFFFFFFF).astype(np.uint32)
