"""GPU: FILTER(?v <cmp> c) on the probe pattern of an index-resident star join, where the table-mode probe filters on the rank of the
value in the numeric side table's value order (kb_numrank.cuh) instead of on the value. The store's numeric objects are edge values
(signed zeros, infinities, NaNs of both signs, subnormals, nextafter neighbours of the constants), plus non-numeric objects and ids past
the numeric table; every comparison is checked against the CPU oracle through the synchronous star join and a prepared plan, on the
first index build and after a numeric reload, window slides with the index maintained, an append that rebuilds the subject table, and
through the fused GROUP BY."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import filter_cases as FC
from tests import oracle_api as O

pytestmark = pytest.mark.gpu

TITLE, VAL, NAME = 1, 2, 3
TITLES = np.array([5, 6, 7], dtype=np.uint32)
LIT0 = 10        # literal ids LIT0 .. LIT0 + len(values) carry the edge values
N_PLAIN = 16     # then this many non-numeric literals
SUBJ0 = 1000     # subjects; the value objects may also be ids in [N_IDS, SUBJ0): past the numeric table (num_of = 0.0)
E = 2000         # employees per segment
# subjects this far above the first segment's fall outside its subject tables (E + 2 E + 65 536 slots), yet the ids stay dense enough
# (range <= 4 rows + 65 536) for the tables to be rebuilt rather than dropped
REBUILD_GAP = 72_000

VALUES, CONSTS = FC.VALUES, FC.CONSTS
N_IDS = LIT0 + len(VALUES) + N_PLAIN
CMPS = [c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE]


def numeric_table(values):
    num = np.zeros(N_IDS, dtype=np.float64)
    isn = np.zeros(N_IDS, dtype=np.uint8)
    num[LIT0:LIT0 + len(values)] = values
    isn[LIT0:LIT0 + len(values)] = 1
    return num, isn


def segment(first_subject, n, seed):
    """n employees: (e title t), (e value v), (e name e); v is an edge-value literal, a non-numeric literal or an id past the table"""
    rng = np.random.default_rng(seed)
    subj = np.arange(first_subject, first_subject + n, dtype=np.uint32)
    kind = rng.integers(0, 10, n)
    val = np.where(kind < 8, LIT0 + rng.integers(0, len(VALUES), n),
                   np.where(kind == 8, LIT0 + len(VALUES) + rng.integers(0, N_PLAIN, n), rng.integers(N_IDS, SUBJ0, n))).astype(np.uint32)
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
    """the device context and the host copy of its triples (what the oracle runs on)"""

    def __init__(self, values):
        self.ctx = c.Context(0)
        self.segs = {}
        self.num, self.isn = numeric_table(values)
        self.ctx.dict_numeric_load(self.num, self.isn)

    def append(self, tag, first_subject, n, seed):
        s, p, o = segment(first_subject, n, seed)
        self.ctx.store_append(s, p, o, tag)
        self.segs[tag] = (s, p, o)

    def evict(self, tag):
        self.ctx.store_evict(tag)
        del self.segs[tag]

    def reload(self, values):
        self.num, self.isn = numeric_table(values)
        self.ctx.dict_numeric_load(self.num, self.isn)

    def oracle(self):
        s, p, o = (np.concatenate([seg[k] for seg in self.segs.values()]) for k in range(3))
        return O.Db(s, p, o, self.num, self.isn)


def check(st, consts=CONSTS, cmps=CMPS, plan=True):
    db = st.oracle()
    n_nonempty = 0
    for cmp in cmps:
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
            n_nonempty += len(want) > 0
    assert n_nonempty > 0


@pytest.fixture
def store():
    st = Store(VALUES)
    yield st
    st.ctx.close()


def test_first_build(store):
    store.append(1, SUBJ0, E, seed=1)
    store.ctx.build_index()
    n0 = store.ctx.get_stats()["index_joins"]
    check(store)
    assert store.ctx.get_stats()["index_joins"] >= n0 + 2 * len(CMPS) * len(CONSTS), "the index probe did not run"


def test_only_zero_and_nan_values(store):
    """V = {0.0}: every value is 0.0, -0.0 or NaN"""
    store.reload(np.array([0.0, -0.0, np.nan, np.copysign(np.nan, -1.0)] * (len(VALUES) // 4) + [0.0] * (len(VALUES) % 4)))
    store.append(1, SUBJ0, E, seed=2)
    store.ctx.build_index()
    check(store)


def test_numeric_reload_then_build_index(store):
    store.append(1, SUBJ0, E, seed=3)
    store.ctx.build_index()
    check(store, consts=CONSTS[:4], plan=False)
    flipped = -VALUES[::-1].copy()  # other values on the same ids: every rank moves
    store.reload(flipped)
    check(store, consts=CONSTS[:4], plan=False)  # the index's rank column is stale until the next build
    store.ctx.build_index()
    check(store)


def test_window_slides(store):
    for k in range(3):
        store.append(k + 1, SUBJ0 + k * E, E, seed=10 + k)
    store.ctx.build_index()
    check(store, consts=CONSTS[:8])
    for k in range(3, 7):  # slide: the new segment's subjects are inserted into the tables in place, the oldest segment leaves
        store.append(k + 1, SUBJ0 + k * E, E, seed=10 + k)
        store.evict(k - 2)
        check(store, consts=CONSTS[:8])


def test_append_rebuilds_subject_table(store):
    store.append(1, SUBJ0, E, seed=20)
    store.ctx.build_index()
    check(store, consts=CONSTS[:4], plan=False)
    store.append(2, SUBJ0 + REBUILD_GAP, 200, seed=21)
    check(store)


def test_fused_group_by_with_probe_filter(store):
    store.append(1, SUBJ0, E, seed=30)
    store.ctx.build_index()
    db = store.oracle()
    for cmp in CMPS:
        for const in CONSTS:
            js, pats, filt = query(cmp, const)
            want = db.bgp(pats, filt).to_numpy([1])
            keys, counts = np.unique(want[:, 0], return_counts=True) if len(want) else (np.empty(0, np.uint32), np.empty(0, np.int64))
            groups, n_rows = store.ctx.star_join_aggregate(js, pats, filt, [1], [(c.AGG_COUNT, 0)])
            assert n_rows == len(want), (cmp, const)
            order = np.argsort(groups["keys"][0])
            assert np.array_equal(groups["keys"][0][order], keys) and np.array_equal(groups["counts"][order], counts), (cmp, const)
            pl = store.ctx.prepare_star_join(js, pats, filt, group_slots=[1], aggs=[(c.AGG_COUNT, 0)], ring=2)
            g, n_plan = pl.collect_groups(pl.submit())
            assert n_plan == len(want), (cmp, const, "plan")
            order = np.argsort(g["keys"][0])
            assert np.array_equal(g["keys"][0][order], keys) and np.array_equal(g["counts"][order], counts), (cmp, const, "plan")
            pl.free()
