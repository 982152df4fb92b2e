"""GPU (-m gpu): kb_bgp_execute's component route — connected components, domain reduction, join-tree order — against an oracle that
plans nothing of its own (tests/bgp_cases.py: ko_scan + ko_hash_join in a BFS order of the test, then ko_filter / ko_project).
  * the 20 WatDiv-shaped queries at ~100 K triples, index off and on: the bag, the route kb_bgp_last_plan reports, and no join
    output above the query's unprojected result (the reduction makes these tree-shaped components globally consistent);
  * random BGPs of 2-16 patterns with fixed seeds: the bag and the column order, and a decline only where a cross join between
    components passes 2^28 rows;
  * the 20 queries at 10 M triples: answered, and equal to the oracle (whole bags up to 10 M rows, (count, sum, xor) of a 64-bit row
    hash beyond)."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import bgp_cases as B
from tests import helpers as H
from tests import oracle_api as O
from tests import watdiv_cases as W

pytestmark = pytest.mark.gpu

TALLY = {"ran": 0, "declined": 0}


def check_watdiv(ctx, d, db, q, bag_limit=10_000_000):
    pats, project = W.compile_query(d, q)
    want, sizes = B.oracle(db, pats, None, project, max_rows=1 << 40)
    got = ctx.bgp_execute(pats, None, project)
    plan = ctx.bgp_last_plan()
    try:
        assert got.slots == project, (q["name"], got.slots)
        assert got.n_rows == want.n_rows, (q["name"], got.n_rows, want.n_rows)
        if want.n_rows <= bag_limit:
            H.assert_same_bag(got.to_numpy(project), want.to_numpy(project), q["name"])
        else:
            assert digest(got.to_numpy(project)) == digest(want.to_numpy(project)), q["name"]
    finally:
        got.free()
    assert plan["route"] == (c.BGP_STAR if q["name"] in W.STAR else c.BGP_COMPONENTS), (q["name"], plan)
    if plan["route"] == c.BGP_COMPONENTS:
        assert plan["n_components"] == 1 and plan["acyclic"] == [1], (q["name"], plan)
        assert plan["max_intermediate"] <= plan["rows_unprojected"], (q["name"], plan)
        assert plan["rows_unprojected"] == sizes[0]
    return plan


def is_star(pats):
    pv = [set(B.pattern_vars(p)) for p in pats]
    return len(pats) <= 8 and bool(set.intersection(*pv))


def digest(rows):
    """(count, sum, xor) of a 64-bit mix of every row — a bag digest"""
    h = np.zeros(len(rows), np.uint64)
    with np.errstate(over="ignore"):
        for j in range(rows.shape[1]):
            h = datagen.splitmix64_at(0, h ^ rows[:, j].astype(np.uint64))
    return len(rows), int(h.sum(dtype=np.uint64)), int(np.bitwise_xor.reduce(h)) if len(h) else 0


@pytest.fixture(scope="module")
def watdiv_small(ctx):
    d = datagen.watdiv(100_000)
    return d, O.Db(d.s, d.p, d.o)


@pytest.mark.parametrize("indexed", [False, True])
@pytest.mark.parametrize("q", W.QUERIES, ids=[q["name"] for q in W.QUERIES])
def test_watdiv_100k(ctx, watdiv_small, q, indexed):
    d, db = watdiv_small
    ctx.store_load(d.s, d.p, d.o)
    if indexed:
        ctx.build_index()
    plan = check_watdiv(ctx, d, db, q)
    if plan["route"] == c.BGP_COMPONENTS and len(q["patterns"]) >= 3:
        assert plan["reduce_rounds"][0] >= 1, plan


@pytest.mark.parametrize("seed", range(60))
def test_random_bgp_components(ctx, seed):
    tr, num, isn, pats, filt, project = B.random_bgp(seed)
    ctx.dict_numeric_load(num, isn)
    ctx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    db = O.Db(tr[:, 0], tr[:, 1], tr[:, 2], num, isn)
    want, why = B.oracle(db, pats, filt, project)
    if want is None and why == "big":
        pytest.skip("the oracle's result is too large for a test")
    cols = B.columns(pats, project)
    outcome = []
    for indexed in (False, True):
        if indexed:
            ctx.build_index()
        try:
            got = ctx.bgp_execute(pats, filt, project)
        except c.KolibrieError as e:
            outcome.append(e.status)
            TALLY["declined"] += 1
            if is_star(pats):  # the star route declines what it declined before (tests/test_gpu_fuzz.py)
                assert e.status in (c.KB_E_UNSUPPORTED, c.KB_E_LIMIT), (seed, str(e))
            else:  # the component route declines only a cross join above 2^28 rows
                assert e.status == c.KB_E_LIMIT and why == "cross", (seed, indexed, str(e))
            continue
        outcome.append("ok")
        assert why != "cross", (seed, "a cross join above 2^28 rows was answered")
        assert got.slots == cols, (seed, indexed, got.slots, cols)
        H.assert_same_bag(got.to_numpy(cols), want.to_numpy(cols), f"seed {seed} indexed={indexed}")
        plan = ctx.bgp_last_plan()
        if plan["route"] == c.BGP_COMPONENTS and min(plan["rows_reduced"]) > 0:  # (an empty pattern ends the call before any join)
            assert plan["n_patterns"] == len(pats) and sorted(plan["join_order"]) == list(range(len(pats))), plan
        got.free()
        TALLY["ran"] += 1
    assert outcome[0] == outcome[1], (seed, outcome)


def test_random_bgp_mostly_executes():
    """runs after the cases above: the fuzzer is only worth something if the device answers most of them"""
    total = TALLY["ran"] + TALLY["declined"]
    assert total == 0 or TALLY["declined"] <= total // 5, TALLY


def test_more_than_16_patterns_is_a_limit(ctx):
    ctx.store_load(np.array([1], np.uint32), np.array([2], np.uint32), np.array([3], np.uint32))
    pats = [c.pattern(c.V(k), c.K(2), c.V(k + 1)) for k in range(17)]
    with pytest.raises(c.KolibrieError) as e:
        ctx.bgp_execute(pats)
    assert e.value.status == c.KB_E_LIMIT


@pytest.fixture(scope="module")
def watdiv_full(ctx):
    d = datagen.watdiv(10_000_000)
    ctx.store_load(d.s, d.p, d.o)  # (no test of this module loads another store after these)
    ctx.build_index()
    return d, O.Db(d.s, d.p, d.o)


@pytest.mark.parametrize("q", W.QUERIES, ids=[q["name"] for q in W.QUERIES])
def test_watdiv_10m(ctx, watdiv_full, q):
    d, db = watdiv_full
    check_watdiv(ctx, d, db, q)
