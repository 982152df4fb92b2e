"""GPU: the table-mode index probe's FILTER on 16-bit stored ranks when the numeric side table has more than 65535 distinct values, so
a stored rank stands for 2^shift consecutive ranks (kb_numrank.cuh: rank16). The slots whose stored rank is at an end of the FILTER's
range are decided on the value. The store mixes 140 000 distinct ordinary values with the edge values of tests/filter_cases.py, non-numeric
objects and ids past the numeric table; the constants are the values at the ends of stored ranks and their nextafter neighbours. Every
comparison is checked against the CPU oracle through the synchronous star join and a prepared plan, after the first index build,
after window slides that write the rank column in place, and through the fused GROUP BY."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import filter_cases as FC
from tests import oracle_api as O

pytestmark = pytest.mark.gpu

TITLE, VAL, NAME = 1, 2, 3
TITLES = np.array([5, 6, 7], dtype=np.uint32)
LIT0 = 10
N_PLAIN = 16
N_VALUES = 140_000  # + the edge values: V has about 140 000 values, rank_shift = 2
CMPS = [c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE]


def value_table():
    rng = np.random.default_rng(3)
    ordinary = np.unique(rng.uniform(-1e6, 1e6, N_VALUES + 1000))[:N_VALUES]
    values = np.concatenate([FC.VALUES, rng.permutation(ordinary)])
    n_ids = LIT0 + len(values) + N_PLAIN
    num = np.zeros(n_ids, dtype=np.float64)
    isn = np.zeros(n_ids, dtype=np.uint8)
    num[LIT0:LIT0 + len(values)] = values
    isn[LIT0:LIT0 + len(values)] = 1
    return values, num, isn


VALUES, NUM, ISN = value_table()
N_IDS = len(NUM)
SUBJ0 = N_IDS + 1000  # value objects may also be ids in [N_IDS, SUBJ0): past the numeric table


def constants():
    """values at both ends of stored ranks (ranks 4k - 1 and 4k of V), with their neighbours, and the edge constants"""
    w = VALUES[~np.isnan(VALUES)]
    v = np.unique(np.where(w == 0.0, 0.0, w))  # V: -0.0 folded into 0.0, NaN left out
    assert len(v) > 65535
    rng = np.random.default_rng(5)
    picks = []
    for k in rng.integers(1, len(v) // 4 - 1, 3):
        picks += [v[4 * k - 1], v[4 * k], np.nextafter(v[4 * k], np.inf), np.nextafter(v[4 * k - 1], -np.inf)]
    return picks + [0.0, np.nan, np.inf, FC.DMIN, 100000.0]


CONSTS = constants()


def segment(first_subject, n, seed):
    rng = np.random.default_rng(seed)
    subj = np.arange(first_subject, first_subject + n, dtype=np.uint32)
    kind = rng.integers(0, 20, n)
    val = np.where(kind < 18, LIT0 + rng.integers(0, len(VALUES), n),
                   np.where(kind == 18, LIT0 + len(VALUES) + rng.integers(0, N_PLAIN, n), rng.integers(N_IDS, SUBJ0, n))).astype(np.uint32)
    s = np.repeat(subj, 3)
    p = np.tile(np.array([TITLE, VAL, NAME], dtype=np.uint32), n)
    o = np.empty(3 * n, dtype=np.uint32)
    o[0::3] = TITLES[rng.integers(0, 3, n)]
    o[1::3] = val
    o[2::3] = subj
    return s, p, o


def query(cmp, const):
    e, t, v, nm = 0, 1, 2, 3
    pats = [c.pattern(c.V(e), c.K(TITLE), c.V(t)), c.pattern(c.V(e), c.K(VAL), c.V(v)), c.pattern(c.V(e), c.K(NAME), c.V(nm))]
    return e, pats, [c.fop(c.F_CMP_NUM, slot=v, cmp=cmp, value=float(const))]


def rows(rel):
    return datagen.canonical_rows(rel.to_numpy(sorted(rel.slots)))


class Store:
    def __init__(self):
        self.ctx = c.Context(0)
        self.segs = {}
        self.ctx.dict_numeric_load(NUM, ISN)

    def append(self, tag, first_subject, n, seed):
        s, p, o = segment(first_subject, n, seed)
        self.ctx.store_append(s, p, o, tag)
        self.segs[tag] = (s, p, o)

    def evict(self, tag):
        self.ctx.store_evict(tag)
        del self.segs[tag]

    def oracle(self):
        s, p, o = (np.concatenate([seg[k] for seg in self.segs.values()]) for k in range(3))
        return O.Db(s, p, o, NUM, ISN)


def check(st, consts=CONSTS, plan=True):
    db = st.oracle()
    n0 = st.ctx.get_stats()["index_joins"]
    for cmp in CMPS:
        for const in consts:
            js, pats, filt = query(cmp, const)
            want = rows(db.bgp(pats, filt))
            got = st.ctx.star_join(js, pats, filt)
            assert np.array_equal(rows(got), want), (cmp, const, "star join")
            got.free()
            if plan:
                pl = st.ctx.prepare_star_join(js, pats, filt, ring=2)
                r = pl.collect_rows(pl.submit())
                assert np.array_equal(rows(r), want), (cmp, const, "prepared plan")
                r.free()
                pl.free()
    assert st.ctx.get_stats()["index_joins"] >= n0 + len(CMPS) * len(consts) * (2 if plan else 1), "the index probe did not run"


@pytest.fixture
def store(monkeypatch):
    monkeypatch.setenv("KOLIBRIE_PROBE_TABLE", "1")
    st = Store()
    yield st
    st.ctx.close()


def test_first_build(store):
    store.append(1, SUBJ0, 150_000, seed=1)
    store.ctx.build_index()
    check(store)


def test_window_slides(store):
    E = 40_000
    for k in range(2):
        store.append(k + 1, SUBJ0 + k * E, E, seed=10 + k)
    store.ctx.build_index()
    for k in range(2, 4):  # the new segment's ranks are written into the rank column in place, the oldest segment leaves
        store.append(k + 1, SUBJ0 + k * E, E, seed=10 + k)
        store.evict(k - 1)
        check(store, consts=CONSTS[:8])


def test_fused_group_by(store):
    store.append(1, SUBJ0, 150_000, seed=30)
    store.ctx.build_index()
    db = store.oracle()
    for cmp in CMPS:
        for const in CONSTS[:8]:
            js, pats, filt = query(cmp, const)
            want = db.bgp(pats, filt).to_numpy([1])
            keys, counts = np.unique(want[:, 0], return_counts=True)
            groups, n_rows = store.ctx.star_join_aggregate(js, pats, filt, [1], [(c.AGG_COUNT, 0)])
            assert n_rows == len(want), (cmp, const)
            order = np.argsort(groups["keys"][0])
            assert np.array_equal(groups["keys"][0][order], keys) and np.array_equal(groups["counts"][order], counts), (cmp, const)
