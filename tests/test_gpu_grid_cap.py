"""GPU (-m gpu): the persistent tile kernels with a capped grid, so that every CTA runs many tiles through its two-stage TMA ring.

Each persistent kernel starts per_sm x n_sms CTAs, and each CTA takes tiles from a global ticket. On a full H100 grid, an input of a few
thousand rows gives every CTA one tile at most, and the code that only runs from a CTA's second tile onward never runs: the stage handed
back to TMA after the first compaction barrier, the mbarrier phase flip, one stage's tile count and next ticket rewritten while the other
stage is read, the fused GROUP BY's 64-entry shared table filling over several tiles, the ordered look-back over tiles of CTAs that are
themselves mid-ring. KOLIBRIE_SMS=<n> caps a context's n_sms, so inputs of 10^4..10^5 rows give each CTA tens of tiles.

Every case runs on a full-grid context and on contexts capped to 1, 2 and 3 SMs, and checks three things:
  - the result equals the oracle (or the exact reference the suite uses for that operator), as a multiset on u32 ids; groups through
    tests/agg_reference.py;
  - the kb_stats fingerprint (every integer counter's change across the call, device time excluded) is the same under every cap: n_sms
    selects no route. Cases taken at their own size from a ROUTES table assert the recorded literal itself;
  - with KOLIBRIE_ORDERED=1 the output is row for row the full-grid output (tile order does not depend on the grid).
Input sizes sit at k*TILE - 1, k*TILE, k*TILE + 1 and at row counts that are 1, 2, 3 (mod 4), for each kernel's tile; multi-segment
stores cross segment boundaries within a CTA's run of tickets, with one segment emptied by kb_store_remove.
"""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import agg_reference as R
from tests import helpers as H
from tests import oracle_api as O
from tests import rsp_join_reference as J
from tests import test_gpu_aggregate as GA
from tests import test_gpu_datalog_routes as DR
from tests import test_gpu_group_routes as GR
from tests import test_gpu_join_routes as JR
from tests import test_gpu_probe_codes as PC
from tests import test_gpu_probe_rank16 as PR16
from tests import test_gpu_probe_rank_filter as PRF
from tests import test_gpu_star_routes as SR
from tests import watdiv_cases as W

pytestmark = pytest.mark.gpu

FIELDS = SR.FIELDS
DEFAULT_ENV = {**SR.DEFAULT_ENV, "KOLIBRIE_DERIVE_PART": "1", "KOLIBRIE_DERIVE_SLICE": str(32 << 20), "KOLIBRIE_DERIVE_MIN_ROWS": str(1 << 20),
               "KOLIBRIE_DERIVE_SLACK": "8192", "KOLIBRIE_FIX_STATE": "1"}
CAPS = ("full", "1", "2", "3")
ORDERED = {"unordered": {}, "ordered": {"KOLIBRIE_ORDERED": "1"}}
SCAN_TILE = 2048   # scan_kernel, scan_star_kernel
PROBE_TILE = 1024  # probe_index_kernel, probe_fast_kernel, probe_direct_kernel, probe_grouped_kernel, quoted_match_kernel
PROBEC_TILE = 512  # probe_chained_kernel

# kernel -> the tests here that run it on a capped grid (tests/test_grid_cap_cpu.py: every tiled kernel of csrc must be listed)
KERNELS = {
    "scan_kernel": ["test_scan", "test_scan_segments", "test_bgp_execute"],
    "scan_star_kernel": ["test_star_scaled", "test_star_route_literal", "test_probe_codes_segments"],
    "probe_index_kernel": ["test_star_scaled", "test_star_route_literal", "test_probe_codes_segments", "test_probe_rank_filter",
                           "test_star_aggregate", "test_coded_aggregate", "test_store_insert_remove"],
    "probe_fast_kernel": ["test_star_scaled", "test_star_route_literal"],
    "probe_direct_kernel": ["test_filter", "test_star_scaled"],
    "probe_chained_kernel": ["test_hash_join", "test_hash_join_literal"],
    "probe_grouped_kernel": ["test_hash_join", "test_hash_join_literal"],
    "quoted_match_kernel": ["test_quoted"],
    "shuffle_scatter_kernel": ["test_shuffle"],
    "part_count_kernel": ["test_shuffle"],
    "part_scatter_kernel": ["test_shuffle"],
    "derive_partition_kernel": ["test_datalog_partitioned"],
    "derive_probe_kernel": ["test_datalog_partitioned"],
    "derive_kernel": ["test_datalog_partitioned"],
    "group_kernel": ["test_group_aggregate"],
    "group1_kernel": ["test_group_aggregate"],
}


@pytest.fixture
def make_ctx(monkeypatch):
    """make(cap, **env): a fresh context created after the switches are set; cap 'full' leaves KOLIBRIE_SMS unset"""
    made = []

    def make(cap, **env):
        for k, v in {**DEFAULT_ENV, **env}.items():
            monkeypatch.setenv(k, v)
        if cap == "full":
            monkeypatch.delenv("KOLIBRIE_SMS", raising=False)
        else:
            monkeypatch.setenv("KOLIBRIE_SMS", cap)
        cx = c.Context(0)
        made.append(cx)
        return cx

    yield make
    for cx in made:
        cx.close()


def stats_delta(a, b):
    return {f: b[f] - a[f] for f in FIELDS if b[f] != a[f]}


def fingerprint(cx, call):
    a = cx.get_stats()
    out = call()
    return out, stats_delta(a, cx.get_stats())


def across_caps(make_ctx, env, run):
    """run(cx, cap) -> (output, fingerprint) on a context of each cap; the fingerprints must all be the full grid's. Returns the outputs."""
    outs, fps = {}, {}
    for cap in CAPS:
        cx = make_ctx(cap, **env)
        outs[cap], fps[cap] = run(cx, cap)
        cx.close()
    for cap in CAPS[1:]:
        assert fps[cap] == fps["full"], f"KOLIBRIE_SMS={cap} took another route: {fps[cap]!r}, full grid {fps['full']!r}"
    return outs


def same_order(outs, what=""):
    """ordered mode: every capped run's rows are the full-grid run's, row for row"""
    for cap in CAPS[1:]:
        a, b = outs[cap], outs["full"]
        assert a.shape == b.shape and np.array_equal(a, b), f"{what} KOLIBRIE_SMS={cap}: row order differs from the full grid"


def u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def rng(seed):
    return np.random.default_rng(seed)


def boundary(tile, k, which):
    """row counts at a tile boundary (k*tile - 1, k*tile, k*tile + 1) and ≡ 2 (mod 4)"""
    return {"m1": k * tile - 1, "0": k * tile, "p1": k * tile + 1, "p2": k * tile + 2}[which]


# ---- kb_scan with the index off: scan_kernel<K>
N_LIT = 3000  # object ids below N_LIT; the even ones are numeric


def scan_numeric():
    num = np.zeros(N_LIT, np.float64)
    isn = np.zeros(N_LIT, np.uint8)
    num[0::2] = np.arange(0, N_LIT, 2) * 0.5 - 300.0
    isn[0::2] = 1
    return num, isn


def scan_triples(n, seed):
    """n triples over P100..P103 and ids 0..7 (so constants and repeated variables match)"""
    g = rng(seed)
    tr = np.stack([g.integers(0, max(n // 4, 8), n), 100 + g.integers(0, 4, n), g.integers(0, N_LIT, n)], axis=1)
    small = g.random(n) < 0.05
    tr[small] = g.integers(0, 8, (int(small.sum()), 3))
    return u32(tr)


P, V, K = c.pattern, c.V, c.K
SCAN_PATS = [P(V(0), K(100), V(1)), P(V(0), K(101), V(2)), P(V(3), V(4), K(7)), P(K(5), V(1), V(2))]


def scan_filter():
    return [c.fop(c.F_CMP_NUM, slot=1, cmp=c.CMP_GT, value=100.0)]


def run_scan(make_ctx, env, segments, pats, filtered, remove=None):
    """kb_scan of pats over a store appended as `segments` (then `remove` taken out) under every cap; each pattern's rows against
    the oracle, and in ordered mode row for row against the full grid and (unfiltered) against store order"""
    num, isn = scan_numeric()
    tr = np.concatenate(segments)
    if remove is not None:
        gone = set(map(tuple, remove.tolist()))
        tr = tr[np.array([tuple(t) not in gone for t in tr.tolist()], dtype=bool)]
    db = O.Db(tr[:, 0], tr[:, 1], tr[:, 2], num, isn)
    pushdown = [scan_filter() if (filtered and k == 0) else None for k in range(len(pats))]
    wants = [db.bgp([p], pd or None) for p, pd in zip(pats, pushdown)]
    ordered = env.get("KOLIBRIE_ORDERED") == "1"

    def run(cx, cap):
        cx.dict_numeric_load(num, isn)
        for t, seg in enumerate(segments):
            cx.store_append(seg[:, 0], seg[:, 1], seg[:, 2], t)
        if remove is not None:
            assert cx.store_remove(remove[:, 0], remove[:, 1], remove[:, 2]).all()
        got, fp = fingerprint(cx, lambda: cx.scan(pats, pushdown if filtered else None))
        out = []
        for k, (rel, want) in enumerate(zip(got, wants)):
            sl = sorted(want.slots)
            assert sorted(rel.slots) == sl, (cap, k)
            rows = rel.to_numpy(sl) if rel.n_rows else np.empty((0, len(sl)), np.uint32)
            H.assert_same_bag(rows, want.to_numpy(sl), f"KOLIBRIE_SMS={cap} pattern {k}")
            if ordered and remove is None and pushdown[k] is None and k < 2:  # (?s P ?o): store order is the order of tr
                m = tr[:, 1] == pats[k].p.value
                assert np.array_equal(rows, tr[m][:, [0, 2]]), f"KOLIBRIE_SMS={cap} pattern {k}: not in store order"
            out.append(rows)
        return np.concatenate([o.reshape(-1) for o in out]), fp

    outs = across_caps(make_ctx, {"KOLIBRIE_USE_INDEX": "0", **env}, run)
    if ordered:
        same_order(outs, "scan")


@pytest.mark.parametrize("mode", list(ORDERED))
@pytest.mark.parametrize("filtered", [False, True], ids=["plain", "filter"])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_scan(make_ctx, k, filtered, mode):
    """scan_kernel<K>: 40 tiles of 2048 triples (about 10 per CTA under cap 1), total rows at a tile boundary or ≡ 2 (mod 4)"""
    n = boundary(SCAN_TILE, 40, ["m1", "0", "p1", "p2"][(k + filtered) % 4])
    run_scan(make_ctx, ORDERED[mode], [scan_triples(n, seed=k)], SCAN_PATS[:k], filtered)


SEG_SIZES = (SCAN_TILE - 1, 1, SCAN_TILE + 1, 5, 3 * SCAN_TILE, 30 * SCAN_TILE + 3)


@pytest.mark.parametrize("mode", list(ORDERED))
def test_scan_segments(make_ctx, mode):
    """segments of TILE-1, 1, TILE+1, 5, 3*TILE and 30*TILE+3 triples, the 5-triple one emptied by kb_store_remove: consecutive
    tickets cross segment boundaries, and a segment's first tile skips the empty one"""
    segs = [scan_triples(n, seed=50 + i) for i, n in enumerate(SEG_SIZES)]
    segs[3] = u32(np.stack([np.arange(900_000, 900_005), np.full(5, 100), np.arange(5)], axis=1))
    run_scan(make_ctx, ORDERED[mode], segs, SCAN_PATS[:2], False, remove=segs[3])


# ---- star joins: the route table's cases at their own size, and the same shapes over 40 000 employees
@pytest.mark.parametrize("name", list(SR.STAR_CASES))
def test_star_route_literal(make_ctx, name):
    """every case of test_gpu_star_routes.STAR_CASES under every cap: the oracle, and the recorded fingerprints themselves"""
    env, load, query = SR.STAR_CASES[name]

    def run(cx, cap):
        db = load(cx)
        js, pats, filt = query()
        want = db.bgp(pats, filt)
        want_rows = want.to_numpy(sorted(want.slots))

        def check(got, what):
            assert sorted(got.slots) == sorted(want.slots), what
            H.assert_same_bag(got.to_numpy(sorted(got.slots)), want_rows, f"KOLIBRIE_SMS={cap} {what}")
        SR.twice(cx, name, lambda: cx.star_join(js, pats, filt), check)
        out = cx.star_join(js, pats, filt)
        return out.to_numpy(sorted(out.slots)), {}

    outs = across_caps(make_ctx, env, run)
    if env.get("KOLIBRIE_ORDERED") == "1":
        same_order(outs, name)


N_EMP = 40_000
_BIG = {}


def big_employees():
    if "emp" not in _BIG:
        d = datagen.employee_dataset(N_EMP)
        _BIG["emp"] = (d, O.Db(d.s, d.p, d.o, d.num_or0, d.is_num))
    return _BIG["emp"]


def big_query(name):
    d, _ = big_employees()
    q = datagen.employee_queries(d)
    if name == "prefilter":
        return 0, q["cfg2"][1], [c.fop(c.F_EQ_ID, slot=1, id=d.ids["Manager"])]
    if name == "six":
        preds = ["foaf:name", "foaf:title", "foaf:workplaceHomepage", "ds:full_or_part_time", "ds:salary_or_hourly", "ds:annual_salary"]
        return 0, [c.pattern(c.V(0), c.K(d.ids[p]), c.V(i + 1)) for i, p in enumerate(preds)], []
    return q[name]


# name -> (switches, index built, query); R1 one-kernel index join, R2 index + direct builds, R3 fused scan + build, R4 scan + batches
BIG_STAR = {
    "r1_cfg2": ({}, True, "cfg2"),
    "r1_cfg3": ({}, True, "cfg3"),
    "r1_star3": ({}, True, "star3"),
    "r1_cfg1": ({}, True, "cfg1"),
    "r1_prefilter": ({}, True, "prefilter"),
    "r1_cfg2_streamed": ({"KOLIBRIE_PROBE_TABLE": "0"}, True, "cfg2"),
    "r1_cfg3_streamed": ({"KOLIBRIE_PROBE_TABLE": "0"}, True, "cfg3"),
    "r1_cfg2_ordered": ({"KOLIBRIE_ORDERED": "1"}, True, "cfg2"),
    "r1_cfg2_streamed_ordered": ({"KOLIBRIE_PROBE_TABLE": "0", "KOLIBRIE_ORDERED": "1"}, True, "cfg2"),
    "r2_cfg2": ({"KOLIBRIE_INDEX_KERNEL": "0"}, True, "cfg2"),
    "r2_cfg2_ordered": ({"KOLIBRIE_INDEX_KERNEL": "0", "KOLIBRIE_ORDERED": "1"}, True, "cfg2"),
    "r3_cfg2": ({}, False, "cfg2"),
    "r3_cfg3": ({}, False, "cfg3"),
    "r3_cfg2_ordered": ({"KOLIBRIE_ORDERED": "1"}, False, "cfg2"),
    "r4_six": ({}, False, "six"),
    "r4_six_ordered": ({"KOLIBRIE_ORDERED": "1"}, False, "six"),
}


@pytest.mark.parametrize("name", list(BIG_STAR))
def test_star_scaled(make_ctx, name):
    """40 000 employees: 240 000 triples (about 30 scan tiles per CTA under cap 1) and 40 probe tiles of 1 024 rows; index build
    (scan_star_kernel), probe_index_kernel with T = 1..3, with and without its FILTER prefilter, table and slice mode, probe_fast_kernel
    after the direct builds, and the generic probe of R4's second batch"""
    env, index, qname = BIG_STAR[name]
    d, db = big_employees()
    js, pats, filt = big_query(qname)
    want = db.bgp(pats, filt)
    sl = sorted(want.slots)
    want_rows = want.to_numpy(sl)

    def run(cx, cap):
        cx.store_load(d.s, d.p, d.o)
        cx.dict_numeric_load(d.num_or0, d.is_num)
        if index:
            cx.build_index()
        got, fp = fingerprint(cx, lambda: cx.star_join(js, pats, filt))
        assert sorted(got.slots) == sl
        rows = got.to_numpy(sl)
        H.assert_same_bag(rows, want_rows, f"{name} KOLIBRIE_SMS={cap}")
        return rows, fp

    outs = across_caps(make_ctx, env, run)
    if env.get("KOLIBRIE_ORDERED") == "1":
        same_order(outs, name)


# ---- the index probe over coded subject tables, on a store of segments at the probe tile's boundaries
PC_SEGS = (PROBE_TILE - 1, 1, PROBE_TILE + 1, 5, 3 * PROBE_TILE, 30 * PROBE_TILE + 2)


@pytest.mark.parametrize("mode", list(ORDERED))
@pytest.mark.parametrize("table", [True, False], ids=["table", "slice"])
def test_probe_codes_segments(make_ctx, table, mode):
    """test_gpu_probe_codes' star (TITLE coded, FILTER on VAL) over segments of TILE-1, 1, TILE+1, 5, 3*TILE and 30*TILE+2 subjects
    (the VAL slice of a segment has one row per subject), the 5-subject segment emptied by kb_store_remove before the index is built"""
    segs, first = [], 0
    for i, n in enumerate(PC_SEGS):
        segs.append(PC.star(PC.subj(first, n), PC.titles(3), seed=70 + i, missing=0.0 if i == 3 else 0.1))
        first += n
    gone = segs[3]
    keep = [seg for i, seg in enumerate(segs) if i != 3]
    trip = tuple(np.concatenate([seg[k] for seg in keep]).astype(np.uint32) for k in range(3))
    db = O.Db(*trip, PC.NUM, PC.ISN)
    env = {"KOLIBRIE_PROBE_TABLE": "1" if table else "0", **ORDERED[mode]}
    queries = [PC.query(), PC.query(title_filter=PC.TITLE0)]

    def run(cx, cap):
        cx.dict_numeric_load(PC.NUM, PC.ISN)
        for t, seg in enumerate(segs):
            cx.store_append(*seg, t)
        assert cx.store_remove(*gone).all()
        cx.build_index()
        out, fps = [], []
        for js, pats, filt in queries:
            got, fp = fingerprint(cx, lambda: cx.star_join(js, pats, filt))
            assert fp.get("index_joins") == 1, fp
            rows = PC.rows(got)
            H.assert_same_bag(rows, PC.rows(db.bgp(pats, filt)), f"KOLIBRIE_SMS={cap}")
            out.append(rows)
            fps.append(fp)
        return np.concatenate(out), fps

    outs = across_caps(make_ctx, env, run)
    if mode == "ordered":
        same_order(outs, "coded probe")


@pytest.mark.parametrize("store", ["rank16", "rank_filter"])
def test_probe_rank_filter(make_ctx, store):
    """the table-mode probe's FILTER on stored ranks (16-bit ranks with a rank shift; the edge-value store), 60 000 subjects"""
    mod = PR16 if store == "rank16" else PRF
    s, p, o = mod.segment(mod.SUBJ0, 60_000, 1)
    num, isn = (PR16.NUM, PR16.ISN) if store == "rank16" else PRF.numeric_table(PRF.VALUES)
    db = O.Db(s, p, o, num, isn)
    consts = list(mod.CONSTS[:4]) + [0.0, float("nan")]
    cases = [(cmp, const) for cmp in mod.CMPS for const in consts]
    wants = [datagen.canonical_rows(db.bgp(*mod.query(cmp, const)[1:]).to_numpy([0, 1, 2, 3])) for cmp, const in cases]

    def run(cx, cap):
        cx.dict_numeric_load(num, isn)
        cx.store_load(s, p, o)
        cx.build_index()
        fps = []
        for (cmp, const), want in zip(cases, wants):
            js, pats, filt = mod.query(cmp, const)
            got, fp = fingerprint(cx, lambda: cx.star_join(js, pats, filt))
            assert np.array_equal(datagen.canonical_rows(got.to_numpy([0, 1, 2, 3])), want), (cap, cmp, const)
            got.free()
            fps.append(fp)
        return None, fps

    across_caps(make_ctx, {"KOLIBRIE_PROBE_TABLE": "1"}, run)


# ---- the GROUP BY folded into the index probe
@pytest.mark.parametrize("order", ["key probes", "value probes"])
@pytest.mark.parametrize("groups", [63, 64, 65, 4096, 4097])
def test_star_aggregate(make_ctx, groups, order):
    """60 001 joined rows: under cap 1 one CTA's 64-entry shared table sees every group over tens of tiles and, past 64 groups,
    overflows into the global table; 4 097 groups is past the fused table (join, then group)"""
    rows, num, isn = GA.make_rows(groups + 3, 60_001, groups, "V3")
    aggs = [(R.SUM, GA.V)]

    def run(cx, cap):
        GA.load_star(cx, rows, num, isn)
        (g, n_joined), fp = fingerprint(cx, lambda: cx.star_join_aggregate(GA.E, GA.ORDERS[order], None, [GA.K], aggs))
        assert n_joined == len(rows), cap
        R.assert_groups_match(g, rows[:, :2], num, [0], [(R.SUM, 1)], f"KOLIBRIE_SMS={cap}")
        return None, fp

    across_caps(make_ctx, {}, run)


@pytest.mark.parametrize("plan", [False, True])
def test_coded_aggregate(make_ctx, plan):
    """the fused GROUP BY on a coded column (test_gpu_probe_codes), 60 000 subjects"""
    trip = PC.star(PC.subj(0, 60_000), np.concatenate([PC.EDGE_TITLES, PC.titles(20)]), seed=31)
    js, pats, filt = PC.query()
    want = O.Db(*trip, PC.NUM, PC.ISN).bgp(pats, filt).to_numpy([PC.T])
    keys, counts = np.unique(want[:, 0], return_counts=True)

    def call(cx):
        if plan:
            pl = cx.prepare_star_join(js, pats, filt, group_slots=[PC.T], aggs=[(c.AGG_COUNT, 0)], ring=2)
            out = pl.collect_groups(pl.submit())
            pl.free()
            return out
        return cx.star_join_aggregate(js, pats, filt, [PC.T], [(c.AGG_COUNT, 0)])

    def run(cx, cap):
        cx.dict_numeric_load(PC.NUM, PC.ISN)
        cx.store_append(*trip, 1)
        cx.build_index()
        (groups, n_rows), fp = fingerprint(cx, lambda: call(cx))
        assert n_rows == len(want), cap
        order = np.argsort(groups["keys"][0])
        assert np.array_equal(groups["keys"][0][order], keys) and np.array_equal(groups["counts"][order], counts), cap
        return None, fp

    across_caps(make_ctx, {}, run)


# ---- kb_hash_join and kb_filter
# name -> (switches, sides): test_gpu_join_routes.HASH_CASES at 5..10 times their probe side
BIG_HASH = {
    "grouped": ({}, lambda: JR.two_sides(2, 100_001, 4000, [0, 1], [0, 2], JR.one_key(0, 5000))),
    "grouped_heavy": ({}, lambda: JR.two_sides(3, 90_002, 120, [0, 1], [0, 2], JR.skewed_key)),
    "chained_fits": ({}, lambda: JR.two_sides(4, 100_003, 5000, [0, 1, 2], [1, 0, 3], JR.keys_of(2000, 5))),
    "chained_resize": ({}, lambda: JR.two_sides(6, 40 * PROBEC_TILE - 1, 5000, [0, 1, 2], [0, 1, 3], JR.keys_of(200, 2))),
    "chained_csr_off": ({"KOLIBRIE_CSR_JOIN": "0"}, lambda: JR.two_sides(2, 100 * PROBEC_TILE + 1, 4000, [0, 1], [0, 2], JR.one_key(0, 5000))),
    "sparse_keys": ({}, lambda: JR.two_sides(7, 100 * PROBE_TILE, 3000, [0, 1], [0, 2], JR.sparse_key)),
    "multi_column_keys": ({}, lambda: JR.two_sides(8, 100_002, 6000, [0, 1, 2, 5], [2, 3, 1, 0], JR.keys_of(40, 3, 30))),
}


@pytest.mark.parametrize("mode", list(ORDERED))
@pytest.mark.parametrize("case", list(BIG_HASH))
def test_hash_join(make_ctx, case, mode):
    """probe_grouped_kernel (light, and heavy tiles spread by its second launch) and probe_chained_kernel (fitting its output, or the
    exact count of a second pass) over 20 000..100 000 probe rows"""
    env, sides = BIG_HASH[case]
    (ls, lc), (rs, rc) = sides()
    want = O.hash_join(O.rel_from_host(ls, lc), O.rel_from_host(rs, rc))
    sl = sorted(want.slots)
    want_rows = want.to_numpy(sl)

    def run(cx, cap):
        left, right = cx.rel_from_host(ls, lc), cx.rel_from_host(rs, rc)
        got, fp = fingerprint(cx, lambda: cx.hash_join(left, right))
        rows = got.to_numpy(sl)
        H.assert_same_bag(rows, want_rows, f"{case} KOLIBRIE_SMS={cap}")
        return got.to_numpy(ls), fp

    outs = across_caps(make_ctx, {**env, **ORDERED[mode]}, run)
    if mode == "ordered":  # probe-row order; the matches of one probe row come in build-insertion order, which is not defined
        same_order(outs, case)


@pytest.mark.parametrize("mode", list(ORDERED))
@pytest.mark.parametrize("case", list(JR.HASH_CASES))
def test_hash_join_literal(make_ctx, case, mode):
    """test_gpu_join_routes.HASH_CASES at their own size under every cap: the recorded fingerprints themselves"""
    env, sides = JR.HASH_CASES[case]
    (ls, lc), (rs, rc) = sides()
    want = O.hash_join(O.rel_from_host(ls, lc), O.rel_from_host(rs, rc))
    sl = sorted(want.slots)

    def run(cx, cap):
        left, right = cx.rel_from_host(ls, lc), cx.rel_from_host(rs, rc)
        JR.twice(cx, case + ("_ordered" if mode == "ordered" else ""), lambda: cx.hash_join(left, right), JR.same_bag(want.to_numpy(sl), sl))
        return None, {}

    across_caps(make_ctx, {**env, **ORDERED[mode]}, run)


@pytest.mark.parametrize("mode", list(ORDERED))
@pytest.mark.parametrize("n", [boundary(PROBE_TILE, 150, w) for w in ("m1", "0", "p1", "p2")])
def test_filter(make_ctx, n, mode):
    """kb_filter: probe_direct_kernel with zero tables over 150 tiles"""
    g = rng(n)
    cols = [u32(g.integers(0, 10, n)), u32(g.integers(0, 1000, n))]
    prog = [c.fop(c.F_NE_ID, slot=1, id=3), c.fop(c.F_EQ_ID, slot=2, id=7), c.fop(c.F_OR)]
    keep = (cols[0] != 3) | (cols[1] == 7)
    want = np.stack([cols[0][keep], cols[1][keep]], axis=1)

    def run(cx, cap):
        rel = cx.rel_from_host([1, 2], cols)
        got, fp = fingerprint(cx, lambda: cx.filter(rel, prog))
        rows = got.to_numpy([1, 2])
        if mode == "ordered":
            assert np.array_equal(rows, want), f"KOLIBRIE_SMS={cap}: not in input order"
        else:
            H.assert_same_bag(rows, want, f"KOLIBRIE_SMS={cap}")
        return rows, fp

    across_caps(make_ctx, ORDERED[mode], run)


# ---- GROUP BY: the grid-stride group kernels, whose per-CTA tables now take many rows each
@pytest.mark.parametrize("name", [n for n in GR.GROUP_CASES if n != "group_empty"])
def test_group_aggregate(make_ctx, name):
    """test_gpu_group_routes.GROUP_CASES at 10 times their rows"""
    seed, n_rows, n_groups, n_keys, aggs = GR.GROUP_CASES[name]
    rows, num, isn = GA.make_rows(seed, 10 * n_rows + 3, n_groups, "V3", n_key_cols=n_keys)
    slots = list(range(n_keys + 1))
    aggs = [(k, n_keys if s == "v" else s) for k, s in aggs]
    gcols = list(range(n_keys))

    def run(cx, cap):
        cx.dict_numeric_load(num, isn)
        rel = cx.rel_from_host(slots, [rows[:, j] for j in slots])
        g, fp = fingerprint(cx, lambda: cx.group_aggregate(rel, gcols, aggs))
        R.assert_groups_match(g, rows, num, gcols, aggs, f"{name} KOLIBRIE_SMS={cap}")
        return None, fp

    across_caps(make_ctx, {}, run)


# ---- RDF-star: quoted_match_kernel over a quoted table of 50 000 entries
@pytest.mark.parametrize("mode", list(ORDERED))
@pytest.mark.parametrize("index", [True, False], ids=["index", "scan"])
@pytest.mark.parametrize("n", [50 * PROBE_TILE - 1, 50 * PROBE_TILE + 2])
def test_quoted(make_ctx, n, index, mode):
    """<< ?1 P200 ?2 >> P300 ?3 (test_gpu_join_routes' quoted route): the match pass over 50 tiles, then the bind join"""
    g = rng(41 + n)
    ids = u32(0x80000000 + np.arange(n))
    qp_ = u32(np.where(g.random(n) < 0.7, 200, 201))
    qs, qo = u32(g.integers(0, 500, n)), u32(g.integers(0, 500, n))
    annotated = g.random(n) < 0.8
    s3 = ids[annotated]
    o3 = u32(9000 + g.integers(0, 30, len(s3)))
    inner = c.pattern(c.V(1), c.K(200), c.V(2))
    qpat = c.KbQuotedPattern(c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.K(300), c.V(3)), inner, c.pattern(c.V(0), c.V(0), c.V(0)))
    hit = annotated & (qp_ == 200)
    want = np.stack([qs[hit], qo[hit], o3[hit[annotated]]], axis=1)

    def run(cx, cap):
        cx.quoted_load(ids, qs, qp_, qo)
        cx.store_load(s3, u32(np.full(len(s3), 300)), o3)
        if index:
            cx.build_index()
        else:
            cx.set_use_index(False)
        got, fp = fingerprint(cx, lambda: cx.scan_quoted(qpat))
        rows = got.to_numpy([1, 2, 3])
        H.assert_same_bag(rows, want, f"KOLIBRIE_SMS={cap}")
        return rows, fp

    outs = across_caps(make_ctx, ORDERED[mode], run)
    if mode == "ordered" and not index:  # the index route binds the match pass's rows, which come in completion order
        same_order(outs, "quoted")


# ---- kb_partition, kb_shuffle_scatter and kb_shuffle_push in a world of one
@pytest.mark.parametrize("n", [200_003, 100_001])
def test_shuffle(make_ctx, n):
    """the fused partition + transfer kernel, both reservation modes, every destination buffer on this GPU (test_gpu_plan's shuffle test)"""
    import torch

    n_parts, n_cols = 8, 2
    g = rng(n)
    cols = [u32(g.integers(0, 1 << 22, n)) for _ in range(n_cols)]
    slots = [10, 11]
    dest = datagen.shard_of_np(cols[1], n_parts)
    counts = np.bincount(dest, minlength=n_parts)
    full = np.stack(cols, axis=1)
    cap_rows = int(counts.max()) + 64

    def run(cx, cap):
        dev = torch.device("cuda", cx.device)
        rel = cx.rel_from_host(slots, cols)
        got_counts, fp0 = fingerprint(cx, lambda: cx.partition_counts(rel, 11, n_parts))
        assert got_counts == [int(x) for x in counts], cap
        parts, fp1 = fingerprint(cx, lambda: cx.partition(rel, 11, n_parts))
        fps = [fp0, fp1]
        for mode in ("planned", "push"):
            bufs = torch.full((n_parts, n_cols, cap_rows), -1, dtype=torch.int32, device=dev)
            cursors = torch.zeros(n_parts, 64, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            peer_cols = [bufs[d_, c_].data_ptr() for d_ in range(n_parts) for c_ in range(n_cols)]
            if mode == "planned":
                _, fp = fingerprint(cx, lambda: cx.shuffle_scatter(rel, 11, n_parts, peer_cols, [0] * n_parts, cap_rows))
                got = counts
            else:
                _, fp = fingerprint(cx, lambda: cx.shuffle_push(rel, 11, n_parts, peer_cols, [cursors[d_].data_ptr() for d_ in range(n_parts)], cap_rows))
                got = cursors[:, 0].cpu().numpy()
                assert np.array_equal(got, counts), cap
            fps.append(fp)
            host = bufs.cpu().numpy().astype(np.uint32)
            for d_ in range(n_parts):
                m = int(got[d_])
                H.assert_same_bag(host[d_, :, :m].T, full[dest == d_], f"KOLIBRIE_SMS={cap} {mode} destination {d_}")
                assert (host[d_, :, m:] == 0xFFFFFFFF).all(), "nothing written past the reserved range"
        rel.free()
        return parts, fps

    outs = across_caps(make_ctx, {}, run)
    for cap in CAPS:
        assert outs[cap] is not None


# ---- Datalog: the radix-partitioned dedup forced onto a small store
@pytest.mark.parametrize("strategy", ["semi_naive", "naive"])
def test_datalog_partitioned(make_ctx, strategy):
    """a taxonomy closure with KOLIBRIE_DERIVE_MIN_ROWS=16 and 2 KB slices: derive_kernel, derive_partition_kernel (4 096-candidate
    tiles) and derive_probe_kernel over rounds of tens of thousands of candidates; the facts, the predicate-block layout and every
    returned statistic are the same under every cap"""
    t = datagen.taxonomy_dataset(fanout=3, depth=5, n_instances=40_000)
    rules = datagen.taxonomy_rules(t)
    s = DR.STRATEGIES[strategy]
    want = O.Db(t.s, t.p, t.o).fixpoint(rules, s)
    env = {"KOLIBRIE_DERIVE_PART": "1", "KOLIBRIE_DERIVE_SLICE": "2048", "KOLIBRIE_DERIVE_MIN_ROWS": "16"}

    def run(cx, cap):
        cx.store_load(t.s, t.p, t.o)
        a = cx.get_stats()
        rel, st = cx.datalog_fixpoint(rules, s)
        fp = (stats_delta(a, cx.get_stats()), DR.returned(st))
        got = DR.rel_rows(rel)
        H.assert_same_bag(got, want["facts"], f"KOLIBRIE_SMS={cap}")
        DR.assert_blocks(got[:, 1], f"KOLIBRIE_SMS={cap}")
        assert [int(x) for x in st.round_new[: st.rounds]] == [int(x) for x in want["round_new"]]
        assert st.derivations == want["derivations"]
        return None, fp

    across_caps(make_ctx, env, run)


# ---- end to end through the grid-stride paths
def test_store_insert_remove(make_ctx):
    """kb_store_insert / kb_store_remove with the index maintained (the inserted salaries make that predicate multi-valued), then a
    star join over the maintained index"""
    d, _ = big_employees()
    g = rng(91)
    sal = d.ids["ds:annual_salary"]
    subj = np.unique(d.s)
    new_s = u32(subj[g.choice(len(subj), 3000, replace=False)])
    ins = (new_s, u32(np.full(3000, sal)), u32(d.o[d.p == sal][g.integers(0, int((d.p == sal).sum()), 3000)]))
    ti = set(zip(d.s.tolist(), d.p.tolist(), d.o.tolist()))
    fresh = np.array([(x, y, z) not in ti for x, y, z in zip(*(a.tolist() for a in ins))])
    sel = np.flatnonzero(d.p == d.ids["foaf:title"])[g.choice(int((d.p == d.ids["foaf:title"]).sum()), 2000, replace=False)]
    rem = (d.s[sel], d.p[sel], d.o[sel])
    keep = np.ones(len(d.s), bool)
    keep[sel] = False
    ss, pp, oo = (np.concatenate([x[keep], y[fresh]]) for x, y in zip((d.s, d.p, d.o), ins))
    db = O.Db(u32(ss), u32(pp), u32(oo), d.num_or0, d.is_num)
    js, pats, filt = big_query("cfg2")
    want = db.bgp(pats, filt)
    sl = sorted(want.slots)

    def run(cx, cap):
        cx.store_load(d.s, d.p, d.o)
        cx.dict_numeric_load(d.num_or0, d.is_num)
        cx.build_index()
        added, fp0 = fingerprint(cx, lambda: cx.store_insert(*ins, tag=5))
        assert np.array_equal(np.asarray(added, bool), fresh), cap
        removed, fp1 = fingerprint(cx, lambda: cx.store_remove(*rem))
        assert np.asarray(removed, bool).all(), cap
        got, fp2 = fingerprint(cx, lambda: cx.star_join(js, pats, filt))
        H.assert_same_bag(got.to_numpy(sl), want.to_numpy(sl), f"KOLIBRIE_SMS={cap}")
        return None, [fp0, fp1, fp2]

    across_caps(make_ctx, {}, run)


@pytest.fixture(scope="module")
def watdiv_100k():
    d = datagen.watdiv(100_000)
    return d, O.Db(d.s, d.p, d.o)


@pytest.mark.parametrize("indexed", [False, True], ids=["scan", "index"])
def test_bgp_execute(make_ctx, watdiv_100k, indexed):
    """kb_bgp_execute's component route (semi-join domain reduction, join-tree order) on WatDiv 100 000, every query that is not a star"""
    from tests import bgp_cases as B

    d, db = watdiv_100k
    queries = [q for q in W.QUERIES if q["name"] not in W.STAR]
    wants = []
    for q in queries:
        pats, project = W.compile_query(d, q)
        want, _ = B.oracle(db, pats, None, project, max_rows=1 << 40)
        wants.append((pats, project, want))

    def run(cx, cap):
        cx.store_load(d.s, d.p, d.o)
        if indexed:
            cx.build_index()
        fps = []
        for q, (pats, project, want) in zip(queries, wants):
            got, fp = fingerprint(cx, lambda: cx.bgp_execute(pats, None, project))
            assert got.n_rows == want.n_rows, (q["name"], cap)
            if want.n_rows <= 2_000_000:
                H.assert_same_bag(got.to_numpy(project), want.to_numpy(project), f"{q['name']} KOLIBRIE_SMS={cap}")
            got.free()
            fps.append(fp)
        return None, fps

    across_caps(make_ctx, {}, run)


@pytest.mark.parametrize("limit", [0, 10, 150_000])
@pytest.mark.parametrize("desc", [False, True])
def test_order_by(make_ctx, desc, limit):
    """kb_order_by on 200 001 rows of numeric keys with long runs of ties: the stable sort (limit 0, or a large limit) and top-k"""
    n = 200_001
    strings = [str(v) for v in range(-2000, 2000)]
    vals = np.arange(-2000, 2000, dtype=np.float64)
    g = rng(7 + desc)
    ids = u32(g.integers(0, len(strings), n))
    other = u32(np.arange(n))
    key = -vals[ids] if desc else vals[ids]
    want = np.argsort(key, kind="stable")
    if limit:
        want = want[:limit]
    expect = np.stack([ids[want], other[want]], axis=1)

    def run(cx, cap):
        cx.dict_strings_load(strings)
        cx.dict_numeric_derive(c.NUMERIC_F64, 0)
        rel = cx.rel_from_host([3, 5], [ids, other])
        (out, info), fp = fingerprint(cx, lambda: cx.order_by(rel, [(3, desc)], limit))
        got = out.to_numpy([3, 5])
        assert got.shape == expect.shape and np.array_equal(got, expect), (cap, info)
        return got, (fp, info["route"])

    outs = across_caps(make_ctx, {}, run)
    same_order(outs, "order by")


@pytest.mark.parametrize("unbound", [False, True])
def test_natural_join(make_ctx, unbound):
    """kb_natural_join over 3 000 x 2 000 rows: kb_hash_join when no shared cell is unbound; else check, mask, partition, sub-joins"""
    g = rng(61 + unbound)
    ls, rs = [10, 11, 20], [30, 11, 10]

    def side(n, slots, unb):
        a = g.integers(0, 60, (n, len(slots))).astype(np.uint32)
        for j, s in enumerate(slots):
            if s in unb:
                a[g.random(n) < 0.3, j] = c.KB_ID_NONE
        return a

    la = side(3000, ls, {10} if unbound else set())
    ra = side(2000, rs, {11} if unbound else set())
    ref = J.natural_join([{s: v for s, v in zip(ls, r) if v != c.KB_ID_NONE} for r in la.tolist()],
                         [{s: v for s, v in zip(rs, r) if v != c.KB_ID_NONE} for r in ra.tolist()])
    out_slots = [10, 11, 20, 30]
    want = np.array([[r.get(s, c.KB_ID_NONE) for s in out_slots] for r in ref], dtype=np.uint32).reshape(-1, 4)

    def run(cx, cap):
        left = cx.rel_from_host(ls, [u32(la[:, j]) for j in range(3)])
        right = cx.rel_from_host(rs, [u32(ra[:, j]) for j in range(3)])
        got, fp = fingerprint(cx, lambda: cx.natural_join(left, right))
        H.assert_same_bag(got.to_numpy(out_slots), want, f"KOLIBRIE_SMS={cap}")
        return None, fp

    across_caps(make_ctx, {}, run)
