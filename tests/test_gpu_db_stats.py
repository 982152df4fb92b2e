"""GPU: kb_store_gather_stats against the restatement of DatabaseStats::gather_stats_fast (tests/stats_reference.py), map for map and
count for count: seeded stores with repeats inside and across segments, the store after every kind of mutation and after a fixpoint
(index on and off), ids at the edges of the u32 domain, the sizes around the sampling thresholds, small sample sizes, the empty store,
the quoted-triple count, the refusals; that the store and its index are left as they were; the cache of get_or_build_stats; the plans
Streamertail picks from device statistics; cfg2's 10 M-triple store and the 100 M-triple bench store."""
import ctypes as C

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200 import engine as E
from kolibrie_b200 import planner as P
from tests import id_domain_cases as D
from tests import stats_reference as R

pytestmark = pytest.mark.gpu

SAMPLES = [R.FAST, 0, 1, 2, 3, 7]


@pytest.fixture(scope="module")
def module_ctx():
    x = c.Context(0)
    yield x
    x.close()


@pytest.fixture
def ctx(module_ctx):
    """the module's context with no quoted-triple table: a test that loads one clears it again here"""
    module_ctx.quoted_load([], [], [], [])
    return module_ctx


def cols(rows):
    a = np.asarray(rows, dtype=np.uint32).reshape(-1, 3)
    return a[:, 0].copy(), a[:, 1].copy(), a[:, 2].copy()


def stored(ctx):
    return np.stack(ctx.store_download(), axis=1)


def check(ctx, max_sample, quoted=0, rows=None, literal=False):
    """the device's statistics equal the restatement over the store's rows (downloaded unless given)"""
    rows = stored(ctx) if rows is None else rows
    got = ctx.store_gather_stats(max_sample)
    if literal:
        lit = R.gather_stats_fast({tuple(int(x) for x in r) for r in rows}, quoted, max_sample)
        want = {"total_triples": lit.total_triples, "quoted_triple_count": quoted, "take": lit.take, "step": lit.step,
                **{k: R.as_arrays(m) for k, m in zip(("subject", "predicate", "object"), lit.maps())}}
    else:
        want = R.gather_stats_numpy(rows, quoted, max_sample)
    for k in ("total_triples", "quoted_triple_count", "take", "step"):
        assert got[k] == want[k], (k, got[k], want[k])
    for j, k in enumerate(("subject", "predicate", "object")):
        assert got[k][0].dtype == np.uint32 and got[k][1].dtype == np.uint64
        assert np.array_equal(got[k][0], want[k][0]), k
        assert np.array_equal(got[k][1], want[k][1]), k
        assert got["n_ids"][j] == len(want[k][0])
    return got


def seeded(seed, n=5000):
    g = np.random.default_rng(seed)
    rows = g.integers(0, [300, 8, 2000], size=(n, 3)).astype(np.uint32)
    return np.concatenate([rows, rows[g.integers(0, n, n // 4)]])  # repeats inside the segment


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("max_sample", SAMPLES)
def test_seeded_segments_with_repeats(ctx, seed, max_sample):
    rows = seeded(seed)
    ctx.store_load(*cols(rows))
    ctx.store_append(*cols(rows[::3]), 7)  # repeats across segments
    ctx.store_append(*cols(seeded(seed + 10, 700)), 8)
    check(ctx, max_sample, literal=max_sample in (0, 7))


@pytest.mark.parametrize("indexed", [False, True])
def test_after_every_mutation(ctx, indexed):
    ctx.dict_strings_load([f"t{i}" for i in range(50100)])  # remove_template needs a string for every template cell
    rows = seeded(5)
    ctx.store_load(*cols(rows))
    if indexed:
        ctx.build_index()

    def both():
        for ms in (R.FAST, 0, 3):
            check(ctx, ms)

    ctx.store_append(*cols(seeded(6, 1500)), 1)
    both()
    ctx.store_append(*cols(seeded(7, 1500)), 2)
    ctx.store_evict(1)
    both()
    ctx.store_delete(*cols(rows[:400]))
    both()
    ctx.store_insert(*cols(np.concatenate([seeded(8, 300), rows[400:500]])), 3)
    both()
    ctx.store_remove(*cols(rows[500:900]))
    both()
    keep = rows[1000:1100]
    rel = ctx.rel_from_host([0, 1], [keep[:, 0].copy(), keep[:, 2].copy()])
    ctx.store_remove_template(rel, [c.pattern(c.V(0), c.K(int(keep[0, 1])), c.V(1))])
    rel.free()
    both()
    link = 20
    chain = np.array([(i, link, i + 1) for i in range(50000, 50040)], dtype=np.uint32)
    ctx.store_append(*cols(chain), 4)
    rules = [{"premise": [c.pattern(c.V(0), c.K(link), c.V(1))], "conclusion": [c.pattern(c.V(0), c.K(21), c.V(1))], "filters": []},
             {"premise": [c.pattern(c.V(0), c.K(21), c.V(1)), c.pattern(c.V(1), c.K(link), c.V(2))],
              "conclusion": [c.pattern(c.V(0), c.K(21), c.V(2))], "filters": []}]
    rel, _ = ctx.datalog_fixpoint(rules)
    rel.free()
    assert (stored(ctx)[:, 1] == 21).sum() == 40 * 41 // 2  # the inferred segment is in the store
    both()


@pytest.mark.parametrize("family", D.FAMILIES)
def test_id_domain_remaps(ctx, family):
    rows = D.star_store(seed=2)
    f = D.remaps(rows, seed=2)[family]
    r = f(rows)
    ctx.store_load(*cols(r[: len(r) // 2]))
    ctx.store_append(*cols(r[len(r) // 3:]), 9)
    for ms in (R.FAST, 0, 7):
        check(ctx, ms)


def closed_form(T):
    i = np.arange(T, dtype=np.int64)
    return np.stack([i // 6, 100 + (i % 6) // 3, i % 3], axis=1).astype(np.uint32)


@pytest.mark.parametrize("T", [99_999, 100_000, 100_001, 199_999, 200_000, 200_001])
@pytest.mark.parametrize("max_sample", [R.FAST, 0])
def test_sampling_thresholds(ctx, T, max_sample):
    rows = closed_form(T)
    g = np.random.default_rng(T)
    perm = rows[g.permutation(T)]
    ctx.store_load(*cols(perm[: T // 2]))
    ctx.store_append(*cols(perm[T // 3:]), 5)  # a sixth of the triples twice
    got = check(ctx, max_sample, rows=rows)
    take, step = R.sample_plan(T, max_sample)
    assert (got["take"], got["step"]) == (take, step)
    for k in ("subject", "predicate", "object"):  # the triples past (take - 1) * step are in no map
        assert int(got[k][1].sum()) == take * step


def test_empty_store(ctx):
    ctx.store_clear()
    ctx.quoted_load([0x80000000, 0x80000005], [1, 2], [3, 4], [5, 6])
    for ms in (R.FAST, 0, 1):
        got = ctx.store_gather_stats(ms)
        assert (got["total_triples"], got["quoted_triple_count"], got["take"], got["step"]) == (0, 2, 0, 1)
        assert all(len(got[k][0]) == 0 for k in ("subject", "predicate", "object"))
    ctx.quoted_load([], [], [], [])


def test_quoted_count_after_load_and_triple_bind(ctx):
    q = [0x80000000, 0x80000002, 0x80000003]  # a hole at index 1
    ctx.quoted_load(q, [1, 2, 3], [10, 10, 10], [4, 5, 6])
    rows = np.array([(0x80000000, 10, 7), (1, 10, 0x80000002), (2, 11, 3)], dtype=np.uint32)
    ctx.store_load(*cols(rows))
    check(ctx, R.FAST, quoted=3, literal=True)
    rel = ctx.rel_from_host([0, 1, 2], [np.array([1, 1, 9, 1], np.uint32), np.array([10, 10, 11, 12], np.uint32),
                                        np.array([4, 4, 8, 8], np.uint32)])
    res, info = ctx.bind(rel, c.BIND_TRIPLE, [c.V(0), c.V(1), c.V(2)], 3, 0x80000004)
    assert info["quoted_new"] == 2  # (1, 10, 4) is entry 0x80000000; (9, 11, 8) and (1, 12, 8) are new
    res.free()
    rel.free()
    check(ctx, 0, quoted=5, literal=True)
    ctx.quoted_load([], [], [], [])
    check(ctx, 0, quoted=0, literal=True)


def test_refusals(ctx):
    ctx.store_load(*cols(seeded(1, 100)))
    h, info = C.c_void_p(), c.KbDbStatsInfo()
    assert c.lib().kb_store_gather_stats(ctx.h, 10, None, C.byref(info)) == c.KB_E_INVALID
    assert c.lib().kb_store_gather_stats(None, 10, C.byref(h), C.byref(info)) == c.KB_E_INVALID
    assert c.lib().kb_store_gather_stats(ctx.h, 10, C.byref(h), None) == c.KB_OK  # info is optional
    ids, counts, n = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint64)(), C.c_uint64()
    assert c.lib().kb_db_stats_counts(h, 3, C.byref(ids), C.byref(counts), C.byref(n)) == c.KB_E_INVALID
    assert c.lib().kb_db_stats_counts(None, 0, C.byref(ids), C.byref(counts), C.byref(n)) == c.KB_E_INVALID
    assert c.lib().kb_db_stats_counts(h, 0, None, C.byref(counts), C.byref(n)) == c.KB_E_INVALID
    assert c.lib().kb_db_stats_counts(h, 0, C.byref(ids), None, C.byref(n)) == c.KB_E_INVALID
    assert c.lib().kb_db_stats_counts(h, 0, C.byref(ids), C.byref(counts), None) == c.KB_E_INVALID
    assert c.lib().kb_db_stats_counts(h, 2, C.byref(ids), C.byref(counts), C.byref(n)) == c.KB_OK and n.value > 0
    c.lib().kb_db_stats_free(h)
    c.lib().kb_db_stats_free(None)


def test_store_and_index_untouched(ctx):
    d = datagen.employee_dataset(20000)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    before = stored(ctx)
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    n0 = ctx.get_stats()["index_joins"]
    want = ctx.star_join(js, pats, filt).to_numpy()
    n1 = ctx.get_stats()["index_joins"]
    assert n1 > n0, "the star join does not take the index route before the call"
    check(ctx, R.FAST, rows=before)
    check(ctx, 0, rows=before)
    assert np.array_equal(stored(ctx), before)
    got = ctx.star_join(js, pats, filt).to_numpy()
    assert ctx.get_stats()["index_joins"] > n1, "the star join left the index route"
    assert np.array_equal(datagen.canonical_rows(got), datagen.canonical_rows(want))


def test_get_or_build_stats_keeps_a_stale_cache(ctx):
    db = E.SparqlDatabase(ctx=ctx)
    for i in range(300):
        db.add_statement(f"http://e/{i % 40}", f"http://p/{i % 3}", f"v{i}")
    db.add_statement(("http://e/1", "http://p/0", "v0"), "http://p/said", "v1")
    st = db.get_or_build_stats()
    ref = R.gather_stats_fast(db.triples, len(db.quoted_triple_store))
    assert (st.total_triples, st.quoted_triple_count) == (ref.total_triples, 1)
    assert (st.subject_card, st.predicate_card, st.object_card) == ref.maps()
    db.insert_triples([(0, 1, 2), (5, 5, 5)])
    assert db.get_or_build_stats() is st  # a write does not refresh the cache
    db.invalidate_stats_cache()
    st2 = db.get_or_build_stats()
    ref2 = R.gather_stats_fast(db.triples, 1)
    assert st2 is not st and (st2.subject_card, st2.predicate_card, st2.object_card) == ref2.maps()
    assert st2.total_triples == len(db.triples)


@pytest.mark.parametrize("n_employees", [3000, 40000])
def test_streamertail_plans_from_device_statistics(ctx, n_employees):
    """cfg1/2/3: the plans chosen from the device's statistics are those chosen from the restatement's"""
    from tests.test_planner import cfg_patterns

    d = datagen.employee_dataset(n_employees)
    ctx.quoted_load([], [], [], [])
    ctx.store_load(d.s, d.p, d.o)
    rows = np.stack([d.s, d.p, d.o], axis=1)
    for ms in (R.FAST, 0):
        g = ctx.store_gather_stats(ms)
        dev = P.DatabaseStats.from_counts(g["total_triples"], dict(zip(g["predicate"][0].tolist(), g["predicate"][1].tolist())),
                                          dict(zip(g["subject"][0].tolist(), g["subject"][1].tolist())),
                                          dict(zip(g["object"][0].tolist(), g["object"][1].tolist())), quoted_triple_count=g["quoted_triple_count"])
        lit = R.gather_stats_fast({tuple(int(x) for x in r) for r in rows}, 0, ms)
        host = P.DatabaseStats.from_counts(lit.total_triples, lit.predicate, lit.subject, lit.object)
        for name, (pats, cond, vars_) in cfg_patterns(d).items():
            for gpu in (True, False):
                a = P.Streamertail(dev, gpu=gpu).find_best_plan(P.build_logical_plan(pats, cond, vars_))
                b = P.Streamertail(host, gpu=gpu).find_best_plan(P.build_logical_plan(pats, cond, vars_))
                assert a == b, (name, gpu)


@pytest.mark.parametrize("n_employees", [1_666_667, 16_666_667], ids=["cfg2_10M", "bench_100M"])
def test_full_size_stores(ctx, n_employees):
    d = datagen.employee_dataset(n_employees)
    ctx.store_load(d.s, d.p, d.o)
    rows = R.distinct_sorted(np.stack([d.s, d.p, d.o], axis=1))
    del d
    for ms in (R.FAST, 0):
        check(ctx, ms, rows=rows)
    ctx.store_clear()
