"""GPU (-m gpu): which route the star-join planner takes for each query shape, pinned by what it costs.

Every case runs its query twice on a context of its own (the second call sees the multi-/single-valued caches the first one
filled) and checks, for each call, the result against the oracle and the *fingerprint* against a literal: the change of every
integer counter of kb_stats across the call (launches per family, kernel launches, rows scanned / built / probed, bytes copied,
fused scan builds, index joins). d2h_bytes counts whole control-arena reads, so it also pins the number of host synchronisations.
Counters that did not move are left out of the literals.

The planner's routes:
  R1  one-kernel index join (probe_index_kernel): every build side is a persistent table of the store index; fused GROUP BY
  R2  index join that builds direct tables from predicate slices, then the register-staged probe
  R3  fused scan + build: the scan fills the direct tables, then the register-staged probe
  R4  scan, then batches of at most MAXT direct builds (first batch: register-staged probe; later ones: generic probe)
  R5  chained natural joins (multi-valued keys, a shared non-join variable, a sparse key range)
What tells them apart: R1 and R2 count an index join, but R1 reads back one word (d2h_bytes 4) where R2 reads a whole control
arena; R3 counts a fused scan build; R4 and R5 scan without one, and R5 alone unpairs its inputs (other_launches).
"""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import helpers as H
from tests import oracle_api as O

pytestmark = pytest.mark.gpu

FIELDS = ("scan_launches", "build_launches", "probe_launches", "filter_launches", "group_launches", "other_launches", "kernel_launches",
          "rows_scanned", "rows_built", "rows_probed", "h2d_bytes", "d2h_bytes", "fused_scan_builds", "index_joins")
# switches that select routes: pinned to their defaults, so that the literals hold whatever the caller's environment says
DEFAULT_ENV = {"KOLIBRIE_ORDERED": "0", "KOLIBRIE_USE_INDEX": "1", "KOLIBRIE_INDEX_KERNEL": "1", "KOLIBRIE_PROBE_TABLE": "1",
               "KOLIBRIE_CSR_JOIN": "1", "KOLIBRIE_INDEX_MAINTAIN": "1"}

# name -> fingerprints of the first and the second call (recorded on an H100)
ROUTES = {
    "r1_cfg2": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r1_cfg3": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r1_cfg2_streamed_probe": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r1_cfg3_streamed_probe": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r1_general_prefilter": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r1_long_probe_filter": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r1_object_star": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 3000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r1_missing_predicate": [{}] * 2,
    "r1_cfg2_ordered": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "r2_cfg2": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 32768, "index_joins": 1}] * 2,
    "r2_cfg3": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 32768, "index_joins": 1}] * 2,
    "r2_cfg2_ordered": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 32768, "index_joins": 1}] * 2,
    "r2_multivalued_index": [{"scan_launches": 1, "build_launches": 5, "probe_launches": 5, "other_launches": 3, "kernel_launches": 23, "rows_scanned": 3889, "rows_built": 5110, "rows_probed": 5487, "d2h_bytes": 196608, "index_joins": 1},
                               {"scan_launches": 1, "build_launches": 4, "probe_launches": 4, "other_launches": 3, "kernel_launches": 20, "rows_scanned": 3889, "rows_built": 2555, "rows_probed": 4153, "d2h_bytes": 163840}],
    "r3_cfg2": [{"scan_launches": 1, "build_launches": 2, "probe_launches": 1, "kernel_launches": 4, "rows_scanned": 36000, "rows_built": 8515, "rows_probed": 6000, "d2h_bytes": 65536, "fused_scan_builds": 1},
                  {"scan_launches": 1, "build_launches": 2, "probe_launches": 1, "kernel_launches": 3, "rows_scanned": 36000, "rows_built": 8515, "rows_probed": 6000, "d2h_bytes": 65536, "fused_scan_builds": 1}],
    "r3_cfg2_ordered": [{"scan_launches": 1, "build_launches": 3, "probe_launches": 1, "kernel_launches": 4, "rows_scanned": 36000, "rows_built": 8515, "rows_probed": 6000, "d2h_bytes": 65536, "fused_scan_builds": 1},
                          {"scan_launches": 1, "build_launches": 3, "probe_launches": 1, "kernel_launches": 3, "rows_scanned": 36000, "rows_built": 8515, "rows_probed": 6000, "d2h_bytes": 65536, "fused_scan_builds": 1}],
    "r3_multivalued": [{"scan_launches": 2, "build_launches": 6, "probe_launches": 5, "other_launches": 3, "kernel_launches": 24, "rows_scanned": 7778, "rows_built": 5110, "rows_probed": 5487, "d2h_bytes": 229376, "fused_scan_builds": 1},
                         {"scan_launches": 1, "build_launches": 4, "probe_launches": 4, "other_launches": 3, "kernel_launches": 20, "rows_scanned": 3889, "rows_built": 2555, "rows_probed": 4153, "d2h_bytes": 163840}],
    "r4_six_patterns": [{"scan_launches": 1, "build_launches": 2, "probe_launches": 2, "kernel_launches": 8, "rows_scanned": 36000, "rows_built": 30000, "rows_probed": 12000, "d2h_bytes": 98304}] * 2,
    "r4_six_patterns_ordered": [{"scan_launches": 1, "build_launches": 2, "probe_launches": 2, "kernel_launches": 8, "rows_scanned": 36000, "rows_built": 30000, "rows_probed": 12000, "d2h_bytes": 98304}] * 2,
    "r4_constant_object": [{"scan_launches": 1, "build_launches": 1, "probe_launches": 1, "kernel_launches": 4, "rows_scanned": 36000, "rows_built": 8009, "rows_probed": 6000, "d2h_bytes": 65536}] * 2,
    "r4_single_pattern_filter": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 36000, "d2h_bytes": 32768}] * 2,
    "r4_multivalued_second_batch": [{"scan_launches": 1, "build_launches": 4, "probe_launches": 4, "other_launches": 6, "kernel_launches": 22, "rows_scanned": 22000, "rows_built": 20000, "rows_probed": 12000, "d2h_bytes": 163840},
                                      {"scan_launches": 1, "build_launches": 10, "probe_launches": 10, "other_launches": 6, "kernel_launches": 47, "rows_scanned": 22000, "rows_built": 10000, "rows_probed": 20000, "d2h_bytes": 360448}],
    "r5_shared_variable": [{"scan_launches": 1, "build_launches": 1, "probe_launches": 1, "other_launches": 2, "kernel_launches": 5, "rows_scanned": 3889, "rows_built": 1270, "rows_probed": 1285, "d2h_bytes": 65536}] * 2,
    "r5_sparse_keys": [{"scan_launches": 1, "build_launches": 2, "probe_launches": 1, "other_launches": 2, "kernel_launches": 6, "rows_scanned": 4000, "rows_built": 2000, "rows_probed": 2000, "d2h_bytes": 98304}] * 2,
    "duplicating_append": [{"scan_launches": 2, "build_launches": 7, "probe_launches": 6, "other_launches": 3, "kernel_launches": 27, "rows_scanned": 72012, "rows_built": 22062, "rows_probed": 24004, "d2h_bytes": 262144, "fused_scan_builds": 1},
                             {"scan_launches": 1, "build_launches": 4, "probe_launches": 4, "other_launches": 3, "kernel_launches": 20, "rows_scanned": 36006, "rows_built": 5030, "rows_probed": 12002, "d2h_bytes": 163840}],
    "host_cfg2": [{"scan_launches": 1, "build_launches": 1, "probe_launches": 1, "kernel_launches": 7, "rows_scanned": 36000, "rows_built": 8515, "rows_probed": 6000, "h2d_bytes": 432000, "d2h_bytes": 105776}] * 2,
    "agg_by_title_fused": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 409600, "index_joins": 1}] * 2,
    "agg_by_salary_join_then_group": [{"probe_launches": 2, "group_launches": 2, "kernel_launches": 6, "rows_probed": 12000, "d2h_bytes": 6127620, "index_joins": 2}] * 2,
    "plan_rows": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 6000, "d2h_bytes": 40244, "index_joins": 1}] * 2,
    "plan_groups": [{"probe_launches": 1, "group_launches": 2, "kernel_launches": 3, "rows_probed": 6000, "d2h_bytes": 284, "index_joins": 1}] * 2,
    "refuse_missing_predicate": [{}] * 2,
    "refuse_build_side_not_persistent": [{}] * 2,
    "refuse_no_index": [{}] * 2,
    "refuse_group_variable_unbound": [{}] * 2,
}

_DATA = {}


def employees():
    """6 000 employees, 6 single-valued predicates; salaries take more than 4 096 distinct values"""
    if "emp" not in _DATA:
        d = datagen.employee_dataset(6000)
        _DATA["emp"] = (d, O.Db(d.s, d.p, d.o, d.num_or0, d.is_num))
    return _DATA["emp"]


def multivalued():
    """1:N predicates 100..102 over 600 subjects (the store of the parity suite's chained-fallback test)"""
    if "mv" not in _DATA:
        rng = np.random.default_rng(3)
        n = 4000
        tr = np.unique(np.stack([rng.integers(0, 600, n), rng.integers(100, 103, n), rng.integers(1000, 1040, n)], axis=1).astype(np.uint32), axis=0)
        _DATA["mv"] = (tr, O.Db(tr[:, 0], tr[:, 1], tr[:, 2]))
    return _DATA["mv"]


def inverse_functional():
    """P101 maps 3 000 subjects to distinct, dense objects (its object column has a persistent table); P100 to 64 shared ones"""
    if "inv" not in _DATA:
        rng = np.random.default_rng(11)
        n = 3000
        subj = np.arange(50, 50 + n, dtype=np.uint32)
        uniq = 50 + n + 64 + rng.permutation(n).astype(np.uint32)
        vals = (50 + n + rng.integers(0, 64, n)).astype(np.uint32)
        tr = np.concatenate([np.stack([subj, np.full(n, 100, np.uint32), vals], axis=1), np.stack([subj, np.full(n, 101, np.uint32), uniq], axis=1)])
        tr = tr[rng.permutation(len(tr))]
        _DATA["inv"] = (tr, O.Db(tr[:, 0], tr[:, 1], tr[:, 2]))
    return _DATA["inv"]


def sparse_keys():
    """two single-valued predicates over 2 000 subjects spread across 50 M ids: no direct table is dense enough"""
    if "sparse" not in _DATA:
        rng = np.random.default_rng(13)
        subj = np.sort(rng.choice(50_000_000, 2000, replace=False)).astype(np.uint32)
        tr = np.concatenate([np.stack([subj, np.full(2000, p, np.uint32), rng.integers(0, 500, 2000).astype(np.uint32)], axis=1) for p in (100, 101)])
        _DATA["sparse"] = (tr, O.Db(tr[:, 0], tr[:, 1], tr[:, 2]))
    return _DATA["sparse"]


def six_with_multivalued_fifth_build():
    """six predicates over 4 000 subjects; P105 has two objects for each of 1 000 subjects: a multi-valued build side smaller
    than the probe side, the fifth build side in pattern order (the second batch of direct builds)"""
    if "six" not in _DATA:
        rng = np.random.default_rng(17)
        n = 4000
        subj = np.arange(n, dtype=np.uint32)
        parts = [np.stack([subj, np.full(n, 100 + p, np.uint32), (10_000 + rng.integers(0, 200, n)).astype(np.uint32)], axis=1) for p in range(5)]
        few = np.repeat(subj[rng.choice(n, 1000, replace=False)], 2)
        parts.append(np.stack([few, np.full(len(few), 105, np.uint32), np.arange(20_000, 20_000 + len(few), dtype=np.uint32)], axis=1))
        tr = np.concatenate(parts)
        _DATA["six"] = (tr, O.Db(tr[:, 0], tr[:, 1], tr[:, 2]))
    return _DATA["six"]


@pytest.fixture
def make_ctx(monkeypatch):
    """a fresh context, created after the route switches are set (they are read when a context is created)"""
    made = []

    def make(**env):
        for k, v in {**DEFAULT_ENV, **env}.items():
            monkeypatch.setenv(k, v)
        cx = c.Context(0)
        made.append(cx)
        return cx

    yield make
    for cx in made:
        cx.close()


def load_employees(cx, index):
    d, db = employees()
    cx.store_load(d.s, d.p, d.o)
    cx.dict_numeric_load(d.num_or0, d.is_num)
    if index:
        cx.build_index()
    return d, db


def load_triples(cx, data, index):
    tr, db = data
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    if index:
        cx.build_index()
    return db


def fingerprint(cx, call):
    a = cx.get_stats()
    out = call()
    b = cx.get_stats()
    return out, {f: b[f] - a[f] for f in FIELDS if b[f] != a[f]}


def twice(cx, name, call, check):
    fps = []
    for rep in range(2):
        out, fp = fingerprint(cx, call)
        check(out, f"{name} call {rep + 1}")
        fps.append(fp)
    assert fps == ROUTES.get(name), f"{name}: {fps!r}"


def gt(slot, v):
    return [c.fop(c.F_CMP_NUM, slot=slot, cmp=c.CMP_GT, value=v)]


def emp_query(q):
    d, _ = employees()
    return datagen.employee_queries(d)[q]


def emp_pattern(pred, var, slot=0):
    d, _ = employees()
    return c.pattern(c.V(slot), c.K(d.ids[pred]), c.V(var))


def emp_six():
    preds = ["foaf:name", "foaf:title", "foaf:workplaceHomepage", "ds:full_or_part_time", "ds:salary_or_hourly", "ds:annual_salary"]
    return 0, [emp_pattern(p, i + 1) for i, p in enumerate(preds)], []


def mv_star():
    return 0, [c.pattern(c.V(0), c.K(100 + i), c.V(i + 1)) for i in range(3)], []


# name -> (context switches, store loader(cx) -> oracle, query () -> (join slot, patterns, filter))
STAR_CASES = {
    "r1_cfg2": ({}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg2")),
    "r1_cfg3": ({}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg3")),
    "r1_cfg2_streamed_probe": ({"KOLIBRIE_PROBE_TABLE": "0"}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg2")),
    "r1_cfg3_streamed_probe": ({"KOLIBRIE_PROBE_TABLE": "0"}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg3")),
    "r1_general_prefilter": ({}, lambda cx: load_employees(cx, True)[1],
                             lambda: (0, emp_query("cfg2")[1], [c.fop(c.F_EQ_ID, slot=1, id=employees()[0].ids["Manager"])])),
    "r1_long_probe_filter": ({}, lambda cx: load_employees(cx, True)[1],
                             lambda: (0, [emp_pattern("ds:annual_salary", 2), emp_pattern("foaf:title", 1), emp_pattern("foaf:name", 3)],
                                      gt(2, 40000.0) + gt(2, 50000.0) + [c.fop(c.F_AND)] + gt(2, 60000.0) + [c.fop(c.F_AND)] + gt(2, 70000.0) +
                                      [c.fop(c.F_AND)] + gt(2, 80000.0) + [c.fop(c.F_AND)])),
    "r1_object_star": ({}, lambda cx: load_triples(cx, inverse_functional(), True),
                       lambda: (0, [c.pattern(c.V(1), c.K(101), c.V(0)), c.pattern(c.V(2), c.K(101), c.V(0))], [])),
    "r1_missing_predicate": ({}, lambda cx: load_employees(cx, True)[1],
                             lambda: (0, [emp_pattern("foaf:title", 1), c.pattern(c.V(0), c.K(999_999), c.V(2))], [])),
    "r1_cfg2_ordered": ({"KOLIBRIE_ORDERED": "1"}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg2")),
    "r2_cfg2": ({"KOLIBRIE_INDEX_KERNEL": "0"}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg2")),
    "r2_cfg3": ({"KOLIBRIE_INDEX_KERNEL": "0"}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg3")),
    "r2_cfg2_ordered": ({"KOLIBRIE_INDEX_KERNEL": "0", "KOLIBRIE_ORDERED": "1"}, lambda cx: load_employees(cx, True)[1], lambda: emp_query("cfg2")),
    "r2_multivalued_index": ({}, lambda cx: load_triples(cx, multivalued(), True), mv_star),
    "r3_cfg2": ({}, lambda cx: load_employees(cx, False)[1], lambda: emp_query("cfg2")),
    "r3_cfg2_ordered": ({"KOLIBRIE_ORDERED": "1"}, lambda cx: load_employees(cx, False)[1], lambda: emp_query("cfg2")),
    "r3_multivalued": ({}, lambda cx: load_triples(cx, multivalued(), False), mv_star),
    "r4_six_patterns": ({}, lambda cx: load_employees(cx, False)[1], emp_six),
    "r4_six_patterns_ordered": ({"KOLIBRIE_ORDERED": "1"}, lambda cx: load_employees(cx, False)[1], emp_six),
    "r4_constant_object": ({}, lambda cx: load_employees(cx, False)[1],
                           lambda: (0, [c.pattern(c.V(0), c.K(employees()[0].ids["foaf:title"]), c.K(employees()[0].ids["Manager"])),
                                        emp_pattern("ds:annual_salary", 2), emp_pattern("foaf:name", 3)], [])),
    "r4_single_pattern_filter": ({}, lambda cx: load_employees(cx, False)[1], lambda: (0, [emp_pattern("ds:annual_salary", 2)], gt(2, 100000.0))),
    "r4_multivalued_second_batch": ({}, lambda cx: load_triples(cx, six_with_multivalued_fifth_build(), False),
                                    lambda: (0, [c.pattern(c.V(0), c.K(100 + i), c.V(i + 1)) for i in range(6)], [])),
    "r5_shared_variable": ({}, lambda cx: load_triples(cx, multivalued(), False),
                           lambda: (0, [c.pattern(c.V(0), c.K(100), c.V(1)), c.pattern(c.V(0), c.K(101), c.V(1))], [])),
    "r5_sparse_keys": ({}, lambda cx: load_triples(cx, sparse_keys(), False),
                       lambda: (0, [c.pattern(c.V(0), c.K(100), c.V(1)), c.pattern(c.V(0), c.K(101), c.V(2))], [])),
}


@pytest.mark.parametrize("name", list(STAR_CASES))
def test_star_join_route(make_ctx, name):
    env, load, query = STAR_CASES[name]
    cx = make_ctx(**env)
    db = load(cx)
    js, pats, filt = query()
    want = db.bgp(pats, filt)
    want_rows = want.to_numpy(sorted(want.slots))

    def check(got, what):
        assert sorted(got.slots) == sorted(want.slots), what
        H.assert_same_bag(got.to_numpy(sorted(got.slots)), want_rows, what)

    twice(cx, name, lambda: cx.star_join(js, pats, filt), check)


def test_star_join_route_after_duplicating_append(make_ctx):
    """an append that repeats subjects makes the predicates multi-valued: the index keeps its slices, loses their tables"""
    cx = make_ctx()
    d, _ = load_employees(cx, True)
    cx.store_append(d.s[:6], d.p[:6], d.o[:6], tag=77)
    db = O.Db(np.concatenate([d.s, d.s[:6]]), np.concatenate([d.p, d.p[:6]]), np.concatenate([d.o, d.o[:6]]), d.num_or0, d.is_num)
    js, pats, filt = emp_query("cfg2")
    want = db.bgp(pats, filt)
    want_rows = want.to_numpy(sorted(want.slots))
    twice(cx, "duplicating_append", lambda: cx.star_join(js, pats, filt),
          lambda got, what: H.assert_same_bag(got.to_numpy(sorted(got.slots)), want_rows, what))


def test_star_join_host_route(make_ctx):
    """the one-shot host call: its upload statistics arrive with the scan, so the fused scan + build cannot size its tables"""
    cx = make_ctx()
    d, db = employees()
    cx.dict_numeric_load(d.num_or0, d.is_num)
    js, pats, filt = emp_query("cfg2")
    want = db.bgp(pats, filt)
    want_rows = want.to_numpy(sorted(want.slots))

    def check(got, what):
        rows, slots = got
        H.assert_same_bag(rows[:, [slots.index(s) for s in sorted(slots)]], want_rows, what)

    twice(cx, "host_cfg2", lambda: cx.star_join_host(d.s, d.p, d.o, js, pats, filt), check)


def group_table(g):
    keys = np.stack(g["keys"], axis=1)
    order = np.lexsort(tuple(keys[:, k] for k in range(keys.shape[1] - 1, -1, -1)))
    return keys[order], g["counts"][order]


@pytest.mark.parametrize("name,gslot", [("agg_by_title_fused", 1), ("agg_by_salary_join_then_group", 2)])
def test_star_join_aggregate_route(make_ctx, name, gslot):
    """GROUP BY folded into the index probe (3 titles), and past its 4 096-slot table (salaries): join, then group"""
    cx = make_ctx()
    _, db = load_employees(cx, True)
    js, pats, _ = emp_query("cfg3")
    aggs = [(c.AGG_COUNT, 0)]
    orel = db.bgp(pats)
    wk, wc = group_table(db.group(orel, [gslot], aggs))

    def check(got, what):
        g, n_rows = got
        gk, gc = group_table(g)
        assert n_rows == orel.n_rows, what
        assert np.array_equal(gk, wk) and np.array_equal(gc, wc), what

    twice(cx, name, lambda: cx.star_join_aggregate(js, pats, None, [gslot], aggs), check)


@pytest.mark.parametrize("grouped", [False, True])
def test_prepared_plan_route(make_ctx, grouped):
    """prepare, submit, collect: the plan resolves the one-kernel index join once"""
    cx = make_ctx()
    _, db = load_employees(cx, True)
    js, pats, filt = emp_query("cfg3" if grouped else "cfg2")
    want = db.bgp(pats, filt)
    aggs = [(c.AGG_COUNT, 0)]

    def run():
        plan = cx.prepare_star_join(js, pats, filt, group_slots=[1] if grouped else [], aggs=aggs if grouped else [], ring=2)
        t = plan.submit()
        if grouped:
            out = plan.collect_groups(t)
        else:
            r = plan.collect_rows(t)
            out = (r.to_numpy(sorted(r.slots)), r.n_rows)
        plan.free()
        return out

    def check(got, what):
        if grouped:
            g, n_rows = got
            assert n_rows == want.n_rows, what
            gk, gc = group_table(g)
            wk, wc = group_table(db.group(want, [1], aggs))
            assert np.array_equal(gk, wk) and np.array_equal(gc, wc), what
        else:
            H.assert_same_bag(got[0], want.to_numpy(sorted(want.slots)), what)

    twice(cx, "plan_groups" if grouped else "plan_rows", run, check)


# name -> (store loader(cx), query () -> (join slot, patterns, group slots))
REFUSALS = {
    "refuse_missing_predicate": (lambda cx: load_employees(cx, True),
                                 lambda: (0, [emp_pattern("foaf:title", 1), c.pattern(c.V(0), c.K(999_999), c.V(2))], [])),
    "refuse_build_side_not_persistent": (lambda cx: load_triples(cx, multivalued(), True), lambda: mv_star()[:2] + ([],)),
    "refuse_no_index": (lambda cx: load_employees(cx, False), lambda: emp_query("cfg2")[:2] + ([],)),
    "refuse_group_variable_unbound": (lambda cx: load_employees(cx, True), lambda: emp_query("cfg2")[:2] + ([9],)),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_prepare_refusal_route(make_ctx, name):
    load, query = REFUSALS[name]
    cx = make_ctx()
    load(cx)
    js, pats, gslots = query()

    def run():
        with pytest.raises(c.KolibrieError) as e:
            cx.prepare_star_join(js, pats, None, group_slots=gslots, aggs=[(c.AGG_COUNT, 0)] if gslots else [], ring=2)
        return e.value.status

    def check(status, what):
        assert status == c.KB_E_UNSUPPORTED, what

    twice(cx, name, run, check)
