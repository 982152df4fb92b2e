"""CPU: the restatement of DatabaseStats::gather_stats_fast (tests/stats_reference.py) on hand-worked cases, its numpy twin, the
host path of SparqlDatabase.get_or_build_stats and planner.DatabaseStats.from_counts."""
import numpy as np
import pytest

from kolibrie_b200 import engine as E
from kolibrie_b200 import planner as P
from tests import stats_reference as R
from tests.oracle_ctx import OracleCtx


def closed_form(T):
    """T triples whose (s, p, o) order is their index i: (i // 6, 100 + (i % 6) // 3, i % 3)"""
    i = np.arange(T, dtype=np.int64)
    return np.stack([i // 6, 100 + (i % 6) // 3, i % 3], axis=1).astype(np.uint32)


def as_set(rows):
    return {tuple(int(x) for x in r) for r in rows}


def test_empty_store():
    st = R.gather_stats_fast(set(), quoted_count=3)
    assert (st.total_triples, st.quoted_triple_count, st.take, st.step) == (0, 3, 0, 1)
    assert st.maps() == ({}, {}, {})


def test_one_triple():
    st = R.gather_stats_fast({(5, 6, 7)})
    assert (st.total_triples, st.take, st.step) == (1, 1, 1)
    assert st.maps() == ({5: 1}, {6: 1}, {7: 1})


def test_seven_triples():
    t = {(1, 10, 5), (1, 10, 6), (1, 11, 5), (2, 10, 5), (3, 12, 9), (3, 12, 8), (4, 10, 6)}
    st = R.gather_stats_fast(t)
    assert (st.total_triples, st.take, st.step) == (7, 7, 1)
    assert st.subject == {1: 3, 2: 1, 3: 2, 4: 1}
    assert st.predicate == {10: 4, 11: 1, 12: 2}
    assert st.object == {5: 3, 6: 2, 8: 1, 9: 1}


def test_small_max_sample_steps():
    """T = 7 with max_sample 3: step 2, positions 0, 2, 4 of the sorted set; with max_sample 2: step 3, positions 0 and 3"""
    t = sorted({(1, 10, 5), (1, 10, 6), (1, 11, 5), (2, 10, 5), (3, 12, 8), (3, 12, 9), (4, 10, 6)})
    st = R.gather_stats_fast(t, max_sample=3)
    assert (st.take, st.step) == (3, 2)
    assert st.subject == {1: 4, 3: 2}  # positions 0 (1,10,5), 2 (1,11,5), 4 (3,12,8)
    assert st.predicate == {10: 2, 11: 2, 12: 2}
    st = R.gather_stats_fast(t, max_sample=2)
    assert (st.take, st.step) == (2, 3)
    assert st.subject == {1: 3, 2: 3} and st.object == {5: 6}  # positions 0 and 3; 6 never sampled
    st = R.gather_stats_fast(t, max_sample=1)
    assert (st.take, st.step) == (1, 7) and st.subject == {1: 7}


def test_repeats_collapse():
    st = R.gather_stats_fast([(1, 2, 3), (1, 2, 3), (1, 2, 4), (1, 2, 3)])
    assert st.total_triples == 2 and st.subject == {1: 2} and st.object == {3: 1, 4: 1}


def test_edge_ids():
    ids = (0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE)
    t = {(a, b, c) for a in ids for b in ids[:2] for c in ids[::2]}
    st = R.gather_stats_fast(t, quoted_count=1)
    assert st.subject == {a: 6 for a in ids} and st.predicate == {0: 15, 1: 15} and st.object == {c: 10 for c in ids[::2]}


# the full-size cases on the closed-form store: s = i // 6 holds positions 6s .. 6s + 5, p is 100 for i % 6 < 3, o = i % 3
FULL_100K = ({**{s: 6 for s in range(16666)}, 16666: 4}, {100: 50001, 101: 49999}, {0: 33334, 1: 33333, 2: 33333})
FULL_STEP2 = ({**{s: 6 for s in range(33333)}, 33333: 2}, {100: 133334, 101: 66666}, {0: 66668, 1: 66666, 2: 66666})


@pytest.mark.parametrize("T,take,step,maps", [
    (100_000, 100_000, 1, FULL_100K),
    (100_001, 100_000, 1, FULL_100K),   # step 1: the last triple (16666, 101, 1) is in no map
    (199_999, 100_000, 1, FULL_100K),   # the first 100 000 only
    (200_000, 100_000, 2, FULL_STEP2),  # every other triple, each count doubled
    (250_001, 100_000, 2, FULL_STEP2),  # positions past 199 998 are never sampled
])
def test_closed_form_sizes(T, take, step, maps):
    rows = closed_form(T)
    st = R.gather_stats_fast(as_set(rows))
    assert (st.total_triples, st.take, st.step) == (T, take, step)
    assert st.maps() == maps
    assert all(sum(m.values()) == take * step for m in st.maps())
    got = R.gather_stats_numpy(rows)
    assert (got["total_triples"], got["take"], got["step"]) == (T, take, step)
    for name, m in zip(("subject", "predicate", "object"), maps):
        assert all(np.array_equal(a, b) for a, b in zip(got[name], R.as_arrays(m)))


def test_max_sample_zero_is_the_planner_count():
    g = np.random.default_rng(1)
    rows = g.integers(0, 50, size=(3000, 3))
    t = as_set(rows)
    st = R.gather_stats_fast(t, quoted_count=4, max_sample=0)
    ds = P.DatabaseStats(t)
    assert (st.take, st.step) == (len(t), 1)
    assert st.total_triples == ds.total_triples
    assert (st.subject, st.predicate, st.object) == (ds.subject_card, ds.predicate_card, ds.object_card)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("max_sample", [0, 1, 2, 3, 7, 1000, 100_000])
def test_numpy_equals_literal(seed, max_sample):
    g = np.random.default_rng(seed)
    n = int(g.integers(1, 4000))
    rows = g.integers(0, [40, 6, 300], size=(n, 3)).astype(np.uint32)
    rows = np.concatenate([rows, rows[: n // 3]])  # repeats
    rows[g.integers(0, len(rows), 5)] = [0xFFFFFFFE, 0x80000000, 0x7FFFFFFF]
    lit = R.gather_stats_fast(as_set(rows), 2, max_sample)
    vec = R.gather_stats_numpy(rows, 2, max_sample)
    assert (vec["total_triples"], vec["take"], vec["step"]) == (lit.total_triples, lit.take, lit.step)
    for name, m in zip(("subject", "predicate", "object"), lit.maps()):
        assert all(np.array_equal(a, b) for a, b in zip(vec[name], R.as_arrays(m)))


def test_from_counts_quoted_count_defaults_to_zero():
    st = P.DatabaseStats.from_counts(10, {1: 10}, {2: 10}, {3: 10})
    assert st.quoted_triple_count == 0 and st.total_triples == 10
    st = P.DatabaseStats.from_counts(10, {1: 10}, quoted_triple_count=7)
    assert st.quoted_triple_count == 7 and st.subject_card == {}


def test_host_get_or_build_stats_caches_until_invalidated():
    """without kb_store_gather_stats (the oracle context) the database gathers on the host; the cache is kept across a write"""
    db = E.SparqlDatabase(ctx=OracleCtx())
    rows = closed_form(250_001)
    db.triples = as_set(rows)
    db.quoted_triple_store.encode(1, 100, 2)
    st = db.get_or_build_stats()
    ref = R.gather_stats_fast(db.triples, quoted_count=1)
    assert st.total_triples == 250_001 and st.quoted_triple_count == 1
    assert (st.subject_card, st.predicate_card, st.object_card) == ref.maps()
    db.add_triple((999_999, 5, 5))
    assert db.get_or_build_stats() is st and 999_999 not in st.subject_card
    db.invalidate_stats_cache()
    st2 = db.get_or_build_stats()
    assert st2 is not st and st2.total_triples == 250_002
