"""GPU: the index probe's one-byte subject codes (PredSlice::xcode). kb_store_build_index codes a subject table whose slots hold at most
255 distinct objects; the index probe then reads one byte a slot and decodes it through the table's dictionary. The star is
?e TITLE ?t . ?e VAL ?v . ?e NAME ?n with FILTER(?v > c) on the probe pattern: TITLE is coded, VAL and NAME (thousands of distinct
objects) are not. Subjects are every other id, the ids between them are NAME literals, and some subjects have no TITLE. Every result
is checked as a bag against the CPU oracle through the synchronous star join and a prepared plan. The build uploads nothing but the
dictionaries, so its host-to-device bytes say which tables it coded; a store mutation drops the codes, and results after one must
still equal the oracle for subjects and titles the dictionary never saw."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import helpers as H
from tests import oracle_api as O

pytestmark = pytest.mark.gpu

TITLE, VAL, NAME = 1, 2, 3
EXTRA = list(range(4, 14))  # predicates that push a segment past KB_MAX_PATTERNS: it is indexed by the batched scan path
LIT0, NV = 10, 2000         # numeric literals
TITLE0 = 3000               # title ids
N_IDS = 4000
S0 = 100_000                # subjects S0 + 2i; NAME objects S0 + 2i + 1
EDGE_TITLES = np.array([0, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE], dtype=np.uint32)
E, T, V, N = 0, 1, 2, 3


def numeric_table():
    num = np.zeros(N_IDS, dtype=np.float64)
    isn = np.zeros(N_IDS, dtype=np.uint8)
    num[LIT0:LIT0 + NV] = np.random.default_rng(1).permutation(NV).astype(np.float64)
    isn[LIT0:LIT0 + NV] = 1
    return num, isn


NUM, ISN = numeric_table()


def titles(k):
    return np.arange(TITLE0, TITLE0 + k, dtype=np.uint32)


def star(subjects, tvals, seed, missing=0.1, extra=False):
    rng = np.random.default_rng(seed)
    subjects = np.asarray(subjects, dtype=np.uint32)
    n = len(subjects)
    has_t = rng.random(n) >= missing
    parts = [(subjects[has_t], TITLE, tvals[rng.integers(0, len(tvals), n)][has_t]),
             (subjects, VAL, (LIT0 + rng.integers(0, NV, n)).astype(np.uint32)),
             (subjects, NAME, subjects + 1)]
    if extra:
        parts += [(subjects[:5], p, subjects[:5] + 1) for p in EXTRA]
    s = np.concatenate([q[0] for q in parts]).astype(np.uint32)
    p = np.concatenate([np.full(len(q[0]), q[1], dtype=np.uint32) for q in parts])
    o = np.concatenate([q[2] for q in parts]).astype(np.uint32)
    order = rng.permutation(len(s))
    return s[order], p[order], o[order]


def subj(first, n):
    return S0 + 2 * np.arange(first, first + n, dtype=np.uint64)


def query(const=float(NV // 3), title_filter=None):
    pats = [c.pattern(c.V(E), c.K(TITLE), c.V(T)), c.pattern(c.V(E), c.K(VAL), c.V(V)), c.pattern(c.V(E), c.K(NAME), c.V(N))]
    filt = [c.fop(c.F_CMP_NUM, slot=V, cmp=c.CMP_GT, value=const)]
    if title_filter is not None:  # a FILTER on the coded column, evaluated on the joined row
        filt += [c.fop(c.F_NE_ID, slot=T, id=int(title_filter)), c.fop(c.F_AND)]
    return E, pats, filt


def rows(rel, slots=(E, T, V, N)):
    return rel.to_numpy(list(slots))


class Store:
    def __init__(self, monkeypatch, table=True, ordered=False):
        monkeypatch.setenv("KOLIBRIE_PROBE_TABLE", "1" if table else "0")
        monkeypatch.setenv("KOLIBRIE_ORDERED", "1" if ordered else "0")
        self.ctx = c.Context(0)
        self.ctx.dict_numeric_load(NUM, ISN)
        self.segs = {}

    def append(self, tag, trip):
        self.ctx.store_append(*trip, tag)
        self.segs[tag] = trip

    def triples(self):
        return tuple(np.concatenate([seg[k] for seg in self.segs.values()]).astype(np.uint32) for k in range(3))

    def build(self):
        """kb_store_build_index; returns its kernel launches and host-to-device bytes (4 per dictionary entry)"""
        s0 = self.ctx.get_stats()
        self.ctx.build_index()
        s1 = self.ctx.get_stats()
        return s1["kernel_launches"] - s0["kernel_launches"], s1["h2d_bytes"] - s0["h2d_bytes"]

    def check(self, filters=(None,), plan=True):
        db = O.Db(*self.triples(), NUM, ISN)
        n0 = self.ctx.get_stats()["index_joins"]
        for tf in filters:
            js, pats, filt = query(title_filter=tf)
            want = rows(db.bgp(pats, filt))
            got = self.ctx.star_join(js, pats, filt)
            H.assert_same_bag(rows(got), want, f"star join, title filter {tf}")
            got.free()
            if plan:
                pl = self.ctx.prepare_star_join(js, pats, filt, ring=2)
                r = pl.collect_rows(pl.submit())
                H.assert_same_bag(rows(r), want, f"prepared plan, title filter {tf}")
                r.free()
                pl.free()
        assert self.ctx.get_stats()["index_joins"] >= n0 + len(filters) * (2 if plan else 1), "the index probe did not run"


def dictionary_bytes(st):
    """what a build uploads: 4 bytes per object of every subject table (unique, dense subjects) with at most 255 distinct objects"""
    s, p, o = st.triples()
    total = 0
    for pred in np.unique(p).tolist():
        ss, oo = s[p == pred], o[p == pred]
        if len(np.unique(ss)) == len(ss) and len(np.unique(oo)) <= 255:
            total += 4 * len(np.unique(oo))
    return total


@pytest.mark.parametrize("k", [1, 3, 255, 256])
@pytest.mark.parametrize("table", [True, False])
def test_threshold(monkeypatch, k, table):
    st = Store(monkeypatch, table=table)
    st.append(1, star(subj(0, 6000), titles(k), seed=k))
    _, h2d = st.build()
    assert h2d == (4 * k if k <= 255 else 0), (k, h2d)  # only TITLE is coded, and only up to 255 objects
    st.check(filters=(None, TITLE0, TITLE0 + k - 1))
    st.ctx.close()


def test_255_codes_256_does_not(monkeypatch):
    launches = {}
    for k in (255, 256):
        st = Store(monkeypatch)
        st.append(1, star(subj(0, 6000), titles(k), seed=7))
        launches[k], _ = st.build()
        st.ctx.close()
    assert launches[255] == launches[256] + 1, launches  # the code pass


@pytest.mark.parametrize("table", [True, False])
def test_edge_ids(monkeypatch, table):
    st = Store(monkeypatch, table=table)
    st.append(1, star(subj(0, 5000), np.concatenate([EDGE_TITLES, titles(3)]), seed=11, missing=0.3))
    _, h2d = st.build()
    assert h2d == 4 * 7
    st.check(filters=[None] + EDGE_TITLES.tolist())
    st.ctx.close()


def test_ordered_sequence_equals_uncoded(monkeypatch):
    """KOLIBRIE_ORDERED=1: store order. An empty append is a store mutation that leaves store and index as they were and drops the
    codes: the row sequence with and without them must be the same."""
    st = Store(monkeypatch, ordered=True)
    st.append(1, star(subj(0, 4000), titles(3), seed=21))
    st.append(2, star(subj(4000, 4000), titles(3), seed=22))
    assert st.build()[1] == 4 * 3
    js, pats, filt = query(title_filter=TITLE0)
    coded = rows(st.ctx.star_join(js, pats, filt))
    e = np.zeros(0, dtype=np.uint32)
    st.ctx.store_append(e, e, e, 3)
    plain = rows(st.ctx.star_join(js, pats, filt))
    assert len(coded) > 0 and np.array_equal(coded, plain)
    st.check(filters=(None, TITLE0))
    st.ctx.close()


@pytest.mark.parametrize("plan", [False, True])
def test_fused_group_by_on_coded_column(monkeypatch, plan):
    st = Store(monkeypatch)
    st.append(1, star(subj(0, 8000), np.concatenate([EDGE_TITLES, titles(20)]), seed=31))
    assert st.build()[1] == 4 * 24
    js, pats, filt = query()
    want = O.Db(*st.triples(), NUM, ISN).bgp(pats, filt).to_numpy([T])
    keys, counts = np.unique(want[:, 0], return_counts=True)
    if plan:
        pl = st.ctx.prepare_star_join(js, pats, filt, group_slots=[T], aggs=[(c.AGG_COUNT, 0)], ring=2)
        groups, n_rows = pl.collect_groups(pl.submit())
        pl.free()
    else:
        groups, n_rows = st.ctx.star_join_aggregate(js, pats, filt, [T], [(c.AGG_COUNT, 0)])
    assert n_rows == len(want)
    order = np.argsort(groups["keys"][0])
    assert np.array_equal(groups["keys"][0][order], keys) and np.array_equal(groups["counts"][order], counts)
    st.ctx.close()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_subject_compaction(monkeypatch, world):
    rank = 1
    cand = subj(0, 20000)
    mine = np.array([x for x in cand.tolist() if c.lib().kb_shard_of(x, world) == rank], dtype=np.uint64)
    assert len(mine) > 2000
    st = Store(monkeypatch)
    st.ctx.set_sharding(rank, world)
    st.append(1, star(mine, titles(3), seed=41))
    assert st.build()[1] == 4 * 3
    st.check(filters=(None, TITLE0))
    st.ctx.close()


def test_mutations_drop_codes_and_a_build_restores_them(monkeypatch):
    """after each mutation the codes are gone (a new title or a new subject would be missed, an evicted one kept, if they were read)
    and the result equals the oracle; the next build codes the table again, its dictionary grown by the new titles"""
    st = Store(monkeypatch)
    st.append(1, star(subj(0, 4000), titles(3), seed=51))
    st.append(2, star(subj(4000, 4000), titles(3), seed=52))
    assert st.build()[1] == 4 * 3
    st.check(filters=(None, TITLE0))
    steps = [
        ("append, split path", lambda: st.append(3, star(subj(8000, 2000), titles(5), seed=53))),
        ("append, scan path", lambda: st.append(4, star(subj(10000, 2000), titles(7), seed=54, extra=True))),
        ("evict", lambda: (st.ctx.store_evict(1), st.segs.pop(1))),
    ]
    for name, step in steps:
        step()
        st.check(filters=(None, TITLE0))
        assert st.build()[1] == dictionary_bytes(st), name
        st.check(filters=(None, TITLE0))
    # kb_store_insert: a TITLE for subjects that had none, with a title no dictionary holds
    s, p, o = st.triples()
    has = set(s[p == TITLE].tolist())
    bare = np.array([x for x in np.unique(s).tolist() if x not in has][:50], dtype=np.uint32)
    assert len(bare) > 0
    ins = (bare, np.full(len(bare), TITLE, dtype=np.uint32), np.full(len(bare), TITLE0 + 100, dtype=np.uint32))
    assert st.ctx.store_insert(*ins, tag=5).all()
    st.segs[5] = ins
    st.check(filters=(None, TITLE0 + 100))
    assert st.build()[1] == dictionary_bytes(st)
    # kb_store_remove: the TITLE of some subjects goes
    sel = np.flatnonzero(p == TITLE)[:300]
    rem = (s[sel], p[sel], o[sel])
    assert st.ctx.store_remove(*rem).all()
    gone = set(zip(*(x.tolist() for x in rem)))
    for tag, (a, b, d) in list(st.segs.items()):
        keep = np.array([(x, y, z) not in gone for x, y, z in zip(a.tolist(), b.tolist(), d.tolist())], dtype=bool)
        st.segs[tag] = (a[keep], b[keep], d[keep])
    st.check(filters=(None, TITLE0))
    assert st.build()[1] == dictionary_bytes(st)
    st.check(filters=(None, TITLE0))
    st.ctx.close()
