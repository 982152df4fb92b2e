"""GPU (-m gpu): what every GROUP BY entry point costs, pinned for each shape it takes.

Like test_gpu_star_routes.py: every case runs twice on a context of its own and checks, for each call, the result and the
*fingerprint* against a literal: the change of every integer counter of kb_stats across the call (launches per family, kernel
launches, rows, bytes copied, index joins). d2h_bytes counts whole control-arena reads and whole group-table downloads, so it also
pins the number of host synchronisations and the size of every table read back. Results are checked against agg_reference as a
multiset of groups (group order is hash-table slot order). Counters that did not move are left out of the literals.

The shapes:
  kb_group_aggregate      group1_kernel<0> (one key, COUNT), group1_kernel<AGG>, group_kernel (2..4 keys, five aggregates), the
                          4096-slot first try overflowing into the 16x retry, an empty relation
  kb_star_join_aggregate  fused into the one-kernel index join; fused try overflowing into join + kb_group_aggregate; not fusable
                          (two group variables, a store without an index)
  prepared grouped plan   submit / collect over a ring of 4; more groups than its table (KB_E_LIMIT at collect); attached as a world
                          of one (barrier, init, peer merge, compaction)
  kb_groups_merge         three partials one of which is empty; every partial empty
and the status code of each invalid call at each entry point.
"""
import ctypes as C

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import agg_reference as R
from tests.test_gpu_aggregate import E, K, ORDERS, V, load_star, make_rows

pytestmark = pytest.mark.gpu

FIELDS = ("scan_launches", "build_launches", "probe_launches", "filter_launches", "group_launches", "other_launches", "kernel_launches",
          "rows_scanned", "rows_built", "rows_probed", "h2d_bytes", "d2h_bytes", "fused_scan_builds", "index_joins")
DEFAULT_ENV = {"KOLIBRIE_ORDERED": "0", "KOLIBRIE_USE_INDEX": "1", "KOLIBRIE_INDEX_KERNEL": "1", "KOLIBRIE_PROBE_TABLE": "1",
               "KOLIBRIE_CSR_JOIN": "1", "KOLIBRIE_INDEX_MAINTAIN": "1"}

# name -> fingerprints of the first and the second call (recorded on an H100)
ROUTES = {
    "group1_count": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group1_sum": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group1_avg": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group1_min": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group1_max": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group_two_keys": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group_three_keys": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group_four_keys": [{"group_launches": 1, "kernel_launches": 2, "d2h_bytes": 409600}] * 2,
    "group_overflow_retry": [{"group_launches": 2, "kernel_launches": 4, "d2h_bytes": 6094848}] * 2,
    "group_empty": [{}] * 2,
    "star_fused": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 4000, "d2h_bytes": 409600, "index_joins": 1}] * 2,
    "star_fused_overflow": [{"probe_launches": 2, "group_launches": 2, "kernel_launches": 6, "rows_probed": 65552, "d2h_bytes": 6127620, "index_joins": 2}] * 2,
    "star_two_group_vars": [{"probe_launches": 1, "group_launches": 1, "kernel_launches": 3, "rows_probed": 4000, "d2h_bytes": 409604, "index_joins": 1}] * 2,
    "star_no_index": [{"scan_launches": 1, "build_launches": 2, "probe_launches": 1, "group_launches": 1, "kernel_launches": 5, "rows_scanned": 12000, "rows_built": 4000, "rows_probed": 4000, "d2h_bytes": 475136, "fused_scan_builds": 1},
                      {"scan_launches": 1, "build_launches": 1, "probe_launches": 1, "group_launches": 1, "kernel_launches": 4, "rows_scanned": 12000, "rows_built": 4000, "rows_probed": 4000, "d2h_bytes": 475136, "fused_scan_builds": 1}],
    "plan_ring4": [{"probe_launches": 6, "group_launches": 12, "kernel_launches": 18, "rows_probed": 48000, "d2h_bytes": 158520, "index_joins": 6}] * 2,
    "plan_world_of_one": [{"probe_launches": 6, "group_launches": 12, "kernel_launches": 36, "rows_probed": 48000, "d2h_bytes": 158520, "index_joins": 6}] * 2,
    "plan_limit": [{"probe_launches": 1, "group_launches": 2, "kernel_launches": 3, "rows_probed": 40000, "d2h_bytes": 360468, "index_joins": 1}] * 2,
    "merge_three_one_empty": [{"group_launches": 1, "kernel_launches": 1, "h2d_bytes": 52360, "d2h_bytes": 221184}] * 2,
    "merge_all_empty": [{}] * 2,
    "group_no_group": [{}] * 2,
    "group_five_groups": [{}] * 2,
    "group_nine_aggs": [{}] * 2,
    "group_unknown_kind": [{}] * 2,
    "group_slot_not_column": [{}] * 2,
    "group_agg_slot_not_column": [{}] * 2,
    "star_no_group": [{}] * 2,
    "star_five_groups": [{}] * 2,
    "star_nine_aggs": [{}] * 2,
    "star_unknown_kind": [{}] * 2,
    "star_slot_not_column": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 4000, "d2h_bytes": 4, "index_joins": 1}] * 2,
    "prepare_aggs_without_group": [{}] * 2,
    "prepare_five_groups": [{}] * 2,
    "prepare_nine_aggs": [{}] * 2,
    "prepare_unknown_kind": [{}] * 2,
    "prepare_slot_not_column": [{}] * 2,
    "prepare_two_group_vars": [{}] * 2,
    "merge_different_group_by": [{}] * 2,
    "merge_truncated": [{}] * 2,
}
# kb_plan_peer_scratch_bytes of a grouped plan, by ring depth
PEER_SCRATCH_BYTES = {2: 754432, 4: 1508608}


@pytest.fixture
def make_ctx(monkeypatch):
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


def groups_check(rows, num, gcols, aggs):
    return lambda g, what: R.assert_groups_match(g, rows, num, gcols, aggs, what)


FIVE = [(R.COUNT, 0), (R.SUM, "v"), (R.MIN, "v"), (R.MAX, "v"), (R.AVG, "v")]

# name -> (seed, rows, groups, key columns, aggregates [(kind, value column or "v")])
GROUP_CASES = {
    "group1_count": (1, 20_000, 65, 1, [(R.COUNT, 0)]),
    "group1_sum": (2, 20_000, 65, 1, [(R.SUM, "v")]),
    "group1_avg": (3, 20_000, 65, 1, [(R.AVG, "v")]),
    "group1_min": (4, 20_000, 65, 1, [(R.MIN, "v")]),
    "group1_max": (5, 20_000, 65, 1, [(R.MAX, "v")]),
    "group_two_keys": (6, 20_000, 300, 2, FIVE),
    "group_three_keys": (7, 20_000, 300, 3, FIVE),
    "group_four_keys": (8, 20_000, 300, 4, FIVE),
    "group_overflow_retry": (9, 40_000, 5000, 1, [(R.SUM, "v")]),
    "group_empty": (10, 0, 1, 2, FIVE),
}


@pytest.mark.parametrize("name", list(GROUP_CASES))
def test_group_aggregate_route(make_ctx, name):
    seed, n_rows, n_groups, n_keys, aggs = GROUP_CASES[name]
    cx = make_ctx()
    rows, num, isn = make_rows(seed, n_rows, n_groups, "V3" if n_rows else "V1", n_key_cols=n_keys)
    cx.dict_numeric_load(num, isn)
    slots = list(range(n_keys + 1))
    rel = cx.rel_from_host(slots, [rows[:, j] for j in slots])
    aggs = [(k, n_keys if s == "v" else s) for k, s in aggs]
    gcols = list(range(n_keys))
    twice(cx, name, lambda: cx.group_aggregate(rel, gcols, aggs), groups_check(rows, num, gcols, aggs))
    rel.free()


# name -> (groups, index built, group variables, aggregates)
STAR_CASES = {
    "star_fused": (65, True, [K], [(R.SUM, V)]),
    "star_fused_overflow": (4097, True, [K], [(R.SUM, V)]),
    "star_two_group_vars": (65, True, [K, V], [(R.COUNT, 0)]),
    "star_no_index": (65, False, [K], [(R.SUM, V)]),
}


@pytest.mark.parametrize("name", list(STAR_CASES))
def test_star_join_aggregate_route(make_ctx, name):
    n_groups, index, gslots, aggs = STAR_CASES[name]
    cx = make_ctx()
    rows, num, isn = make_rows(n_groups + 17, max(8 * n_groups, 4000), n_groups, "V3")
    load_star(cx, rows, num, isn, index=index)
    col = {K: 0, V: 1}
    check_groups = groups_check(rows[:, :2], num, [col[s] for s in gslots], [(k, col[s] if k != R.COUNT else 0) for k, s in aggs])

    def check(got, what):
        g, n_joined = got
        assert n_joined == len(rows), what
        check_groups(g, what)

    twice(cx, name, lambda: cx.star_join_aggregate(E, ORDERS["key probes"], None, gslots, aggs), check)


def plan_run(cx, ring, n_submits, attach=False):
    """prepare a grouped plan, submit n_submits queries keeping at most `ring` in flight, collect them all, free: [(groups, rows)]"""
    plan = cx.prepare_star_join(E, ORDERS["value probes"], None, group_slots=[K], aggs=[(R.AVG, V)], ring=ring)
    if attach:
        import torch

        scratch = torch.zeros((plan.peer_scratch_bytes() + 3) // 4, dtype=torch.int32, device=torch.device("cuda", cx.device))
        torch.cuda.synchronize()
        plan.attach_peers(0, 1, [scratch.data_ptr()], keep=scratch)
    out, tickets = [], []
    for _ in range(n_submits):
        tickets.append(plan.submit())
        if len(tickets) == ring:
            out.append(plan.collect_groups(tickets.pop(0)))
    out += [plan.collect_groups(t) for t in tickets]
    plan.free()
    return out


@pytest.mark.parametrize("name,ring,attach", [("plan_ring4", 4, False), ("plan_world_of_one", 2, True)])
def test_prepared_group_plan_route(make_ctx, name, ring, attach):
    cx = make_ctx()
    rows, num, isn = make_rows(31, 8000, 300, "V3")
    load_star(cx, rows, num, isn)
    check_groups = groups_check(rows[:, :2], num, [0], [(R.AVG, 1)])

    def check(got, what):
        assert len(got) == 6, what
        for i, (g, n_joined) in enumerate(got):
            assert n_joined == len(rows), f"{what} query {i}"
            check_groups(g, f"{what} query {i}")

    twice(cx, name, lambda: plan_run(cx, ring, 6, attach), check)


def test_prepared_group_plan_limit_route(make_ctx):
    cx = make_ctx()
    rows, num, isn = make_rows(4097, 40_000, 4097, "V3")
    load_star(cx, rows, num, isn)

    def run():
        plan = cx.prepare_star_join(E, ORDERS["key probes"], None, group_slots=[K], aggs=[(R.SUM, V)], ring=2)
        t = plan.submit()
        with pytest.raises(c.KolibrieError) as e:
            plan.collect_groups(t)
        plan.free()
        return e.value.status

    twice(cx, "plan_limit", run, lambda status, what: (assert_status(status, c.KB_E_LIMIT, what)))


def test_peer_scratch_bytes(make_ctx):
    cx = make_ctx()
    rows, num, isn = make_rows(5, 4000, 65, "V1")
    load_star(cx, rows, num, isn)
    got = {}
    for ring in (2, 4):
        plan = cx.prepare_star_join(E, ORDERS["key probes"], None, group_slots=[K], aggs=[(R.SUM, V)], ring=ring)
        got[ring] = plan.peer_scratch_bytes()
        plan.free()
    assert got == PEER_SCRATCH_BYTES, f"{got!r}"


def assert_status(status, want, what):
    assert status == want, f"{what}: status {status}, expected {want}"


def packed(cx, rel, gcols, aggs):
    gs = (C.c_uint32 * len(gcols))(*gcols)
    ag = (c.KbAgg * max(len(aggs), 1))(*[c.KbAgg(k, s) for k, s in aggs])
    g = C.c_void_p()
    cx._check(c.lib().kb_group_aggregate(cx.h, rel.h, gs, len(gcols), ag, len(aggs), C.byref(g)))
    try:
        return cx._groups_pack(g)
    finally:
        c.lib().kb_groups_free(g)


def no_groups(part):
    """a partial of the same GROUP BY that holds no group: the header of `part` with n_groups = 0"""
    out = part[:56].copy()
    out[8:16] = 0
    return out


@pytest.mark.parametrize("name", ["merge_three_one_empty", "merge_all_empty"])
def test_groups_merge_route(make_ctx, name):
    cx = make_ctx()
    rows, num, isn = make_rows(41, 9000, 300, "V3", n_key_cols=2)
    cx.dict_numeric_load(num, isn)
    aggs = [(k, 2 if s == "v" else s) for k, s in FIVE]
    parts = []
    for a, b in ((0, 4000), (4000, 9000)):
        rel = cx.rel_from_host([0, 1, 2], [rows[a:b, j] for j in range(3)])
        parts.append(packed(cx, rel, [0, 1], aggs))
        rel.free()
    if name == "merge_three_one_empty":
        parts.insert(1, no_groups(parts[0]))
        merged = rows
    else:
        parts = [no_groups(parts[0])] * 3
        merged = rows[:0]
    twice(cx, name, lambda: cx.groups_merge(parts), groups_check(merged, num, [0, 1], aggs))


def call_status(call):
    with pytest.raises(c.KolibrieError) as e:
        call()
    return e.value.status


def refusal_calls(cx, rel):
    """entry point / invalid argument -> a call that must be refused"""
    bad_kind = [(7, 1)]
    nine = [(R.SUM, 1)] * 9
    pats = ORDERS["key probes"]
    ga = lambda gs, aggs: lambda: cx.group_aggregate(rel, gs, aggs)  # noqa: E731
    sja = lambda gs, aggs: lambda: cx.star_join_aggregate(E, pats, None, gs, aggs)  # noqa: E731
    prep = lambda gs, aggs: lambda: cx.prepare_star_join(E, pats, None, group_slots=gs, aggs=aggs, ring=2)  # noqa: E731
    return {
        "group_no_group": ga([], [(R.COUNT, 0)]),
        "group_five_groups": ga([0, 0, 0, 0, 0], [(R.COUNT, 0)]),
        "group_nine_aggs": ga([0], nine),
        "group_unknown_kind": ga([0], bad_kind),
        "group_slot_not_column": ga([9], [(R.COUNT, 0)]),
        "group_agg_slot_not_column": ga([0], [(R.SUM, 9)]),
        "star_no_group": sja([], [(R.COUNT, 0)]),
        "star_five_groups": sja([K] * 5, [(R.COUNT, 0)]),
        "star_nine_aggs": sja([K], [(R.SUM, V)] * 9),
        "star_unknown_kind": sja([K], [(7, V)]),
        "star_slot_not_column": sja([9], [(R.COUNT, 0)]),
        "prepare_aggs_without_group": prep([], [(R.COUNT, 0)]),
        "prepare_five_groups": prep([K] * 5, [(R.COUNT, 0)]),
        "prepare_nine_aggs": prep([K], [(R.SUM, V)] * 9),
        "prepare_unknown_kind": prep([K], [(7, V)]),
        "prepare_slot_not_column": prep([9], [(R.COUNT, 0)]),
        "prepare_two_group_vars": prep([K, V], [(R.COUNT, 0)]),
    }


REFUSALS = {
    "group_no_group": c.KB_E_LIMIT,
    "group_five_groups": c.KB_E_LIMIT,
    "group_nine_aggs": c.KB_E_LIMIT,
    "group_unknown_kind": c.KB_E_INVALID,
    "group_slot_not_column": c.KB_E_INVALID,
    "group_agg_slot_not_column": c.KB_E_INVALID,
    "star_no_group": c.KB_E_LIMIT,
    "star_five_groups": c.KB_E_LIMIT,
    "star_nine_aggs": c.KB_E_LIMIT,
    "star_unknown_kind": c.KB_E_INVALID,
    "star_slot_not_column": c.KB_E_INVALID,
    "prepare_aggs_without_group": c.KB_E_INVALID,
    "prepare_five_groups": c.KB_E_UNSUPPORTED,
    "prepare_nine_aggs": c.KB_E_UNSUPPORTED,
    "prepare_unknown_kind": c.KB_E_INVALID,
    "prepare_slot_not_column": c.KB_E_UNSUPPORTED,
    "prepare_two_group_vars": c.KB_E_UNSUPPORTED,
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_refusal_route(make_ctx, name):
    cx = make_ctx()
    rows, num, isn = make_rows(3, 4000, 65, "V1")
    load_star(cx, rows, num, isn)
    rel = cx.rel_from_host([0, 1], [rows[:, 0], rows[:, 1]])
    call = refusal_calls(cx, rel)[name]
    twice(cx, name, lambda: call_status(call), lambda status, what: assert_status(status, REFUSALS[name], what))
    rel.free()


@pytest.mark.parametrize("name", ["merge_different_group_by", "merge_truncated"])
def test_merge_refusal_route(make_ctx, name):
    cx = make_ctx()
    rows, num, isn = make_rows(43, 4000, 65, "V1", n_key_cols=2)
    cx.dict_numeric_load(num, isn)
    rel = cx.rel_from_host([0, 1, 2], [rows[:, j] for j in range(3)])
    a = packed(cx, rel, [0, 1], [(R.SUM, 2)])
    b = packed(cx, rel, [0], [(R.SUM, 2)]) if name == "merge_different_group_by" else a[:-1]
    rel.free()
    twice(cx, name, lambda: call_status(lambda: cx.groups_merge([a, b])), lambda status, what: assert_status(status, c.KB_E_INVALID, what))
