"""GPU (-m gpu): FILTER at every place the device evaluates it, against the exact restatement of tests/filter_reference.py.

The store's values are the edge values of tests/filter_cases.py (signed zeros, infinities, NaNs of both signs, subnormals, +-DBL_MAX and
their nextafter neighbours), non-numeric literals and ids past the numeric table; a relation built on the host also holds quoted-triple
ids and KB_ID_NONE (unbound) cells. The constants of the single comparisons are every stored value and both of its neighbours, so the
boundary of each comparison is hit exactly. The expected rows are the restatement applied to the unfiltered result (the oracle's BGP
without a filter, or the input relation): the oracle's own FILTER is never the authority.

Each case runs on a context created with its route switches set, and asserts a kb_stats counter (or the BGP plan) that proves the
site it is meant for ran: a planner change that moves a case elsewhere fails it instead of silently testing another site.
KOLIBRIE_ORDERED is left to the environment except where a case sets it, so the whole file also runs with KOLIBRIE_ORDERED=1."""
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import engine as E
from tests import filter_cases as FC
from tests import filter_reference as R
from tests import helpers as H
from tests import oracle_api as O

pytestmark = pytest.mark.gpu

NONE = R.KB_ID_NONE
TITLE, VAL, NAME, VAL2, MV1, MV2, SMALL1, SMALL2, CH_A, CH_B, CH_C, DER1, DER2 = range(1, 14)
TITLES = np.array([5, 6, 7], dtype=np.uint32)
LIT0 = 20
N_PLAIN = 16
N_IDS = LIT0 + len(FC.VALUES) + N_PLAIN
SUBJ0 = 1000
N_SUBJ = 2000
CMPS = [c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE]
ALL_CONSTS = FC.boundary_consts(FC.VALUES)
FEW_CONSTS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, FC.DMIN, -FC.DMIN, 1.0, np.nextafter(1.0, 2.0), 100000.0, 99999.5,
                       np.nextafter(100000.0, 0.0), FC.DBL_MAX, -FC.DBL_MAX, FC.NORM_MIN, 2.5])
# switches that select routes, pinned to their defaults (KOLIBRIE_ORDERED is left to the caller)
DEFAULT_ENV = {"KOLIBRIE_USE_INDEX": "1", "KOLIBRIE_INDEX_KERNEL": "1", "KOLIBRIE_PROBE_TABLE": "1", "KOLIBRIE_CSR_JOIN": "1",
               "KOLIBRIE_INDEX_MAINTAIN": "1"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# nextafter(1, +inf) * nextafter(1, -inf) = 1 + 2^-53 - 2^-105 rounds to exactly 1.0, so ?a * ?b - 1 is 0.0 (false); a fused multiply-add
# keeps 2^-53 - 2^-105 (true). Every store and relation below holds rows that pair the two, so the contraction case is decided.
ONE_UP, ONE_DOWN = LIT0 + 21 + 14, LIT0 + 42 + 14
assert FC.VALUES[ONE_UP - LIT0] == np.nextafter(1.0, 2.0) and FC.VALUES[ONE_DOWN - LIT0] == np.nextafter(1.0, 0.0)


def contraction_rows(rows, slots, a, b, terms=None):
    """rows whose ?a * ?b rounds to exactly 1.0 while the exact product does not equal 1: they tell a contracted ?a * ?b - 1 apart"""
    terms = terms or TERMS
    _, x, xn = terms.number(rows[:, slots.index(a)])
    _, y, yn = terms.number(rows[:, slots.index(b)])
    with np.errstate(all="ignore"):
        near = np.flatnonzero(xn & yn & (x * y == 1.0))
    return sum(1 for i in near if Fraction(float(x[i])) * Fraction(float(y[i])) != 1)


# ---- programs
def cmp(slot, k, v):
    return c.fop(c.F_CMP_NUM, slot=slot, cmp=k, value=float(v))


def f(code, **kw):
    return c.fop(code, **kw)


def single_comparisons(slot, consts):
    """FILTER(?x <cmp> c) and its NOT, at every constant"""
    for k in CMPS:
        for v in consts:
            yield [cmp(slot, k, v)]
            yield [cmp(slot, k, v), f(c.F_NOT)]


def deep_program(a, b):
    """depth 10 (the deepest the API accepts): ten comparisons pushed, then nine ANDs / ORs"""
    ops = [cmp(a if i % 2 else b, CMPS[i % 4], [0.0, -1.0, 1.0, np.inf, 99999.5][i % 5]) for i in range(10)]
    return ops + [f(c.F_OR if i % 3 else c.F_AND) for i in range(9)]


def long_program(a, b):
    """32 ops (the longest the API accepts), stack depth 2"""
    ops = [cmp(a, c.CMP_GE, -FC.DBL_MAX)]
    for i in range(9):
        ops += [cmp(b, CMPS[i % 4], [0.0, 1.0, -0.0, FC.DMIN][i % 4]), f(c.F_NOT), f(c.F_OR)]
    return ops + [cmp(a, c.CMP_LT, np.inf), f(c.F_AND), f(c.F_NOT), f(c.F_NOT)]


def mixed_programs(a, b, ids):
    """NOT / AND / OR mixes, id (in)equality, arithmetic, isTRIPLE and the longest and deepest accepted programs over slots a, b"""
    T = f(c.F_TRUTHY)
    progs = [
        [cmp(a, c.CMP_GT, 0.0), cmp(b, c.CMP_LE, 1.0), f(c.F_NOT), f(c.F_AND)],
        [cmp(a, c.CMP_GE, -0.0), cmp(b, c.CMP_LT, FC.DMIN), f(c.F_OR)],
        [cmp(a, c.CMP_LT, np.inf), f(c.F_NOT), cmp(b, c.CMP_GT, -np.inf), f(c.F_NOT), f(c.F_OR), f(c.F_NOT)],
        [f(c.F_PUSH_VAR, slot=a), f(c.F_PUSH_VAR, slot=b), f(c.F_SUB), T],                  # inf - inf is NaN: truthy
        [f(c.F_PUSH_VAR, slot=a), f(c.F_PUSH_VAR, slot=b), f(c.F_MUL), f(c.F_PUSH_CONST, value=1.0), f(c.F_SUB), T],  # no contraction
        [f(c.F_PUSH_VAR, slot=a), f(c.F_PUSH_VAR, slot=b), f(c.F_DIV), T],                  # a zero divisor of either sign: invalid
        [f(c.F_PUSH_VAR, slot=a), f(c.F_PUSH_CONST, value=-0.0), f(c.F_DIV), T, f(c.F_NOT)],
        [f(c.F_PUSH_VAR, slot=a), f(c.F_PUSH_CONST, value=10.0), f(c.F_MUL), T],            # DBL_MAX * 10 = inf: truthy
        [f(c.F_PUSH_VAR, slot=a), f(c.F_PUSH_CONST, value=1.0), f(c.F_ADD), T, f(c.F_NOT)],
        [f(c.F_IS_TRIPLE, slot=a)],
        [f(c.F_IS_TRIPLE, slot=b), f(c.F_NOT)],
        deep_program(a, b),
        long_program(a, b),
    ]
    for i in ids:
        progs += [[f(c.F_EQ_ID, slot=a, id=int(i))], [f(c.F_NE_ID, slot=b, id=int(i))], [f(c.F_NE_ID, slot=a, id=int(i)), f(c.F_NOT)]]
    return progs


def programs(a, b, consts, ids):
    return list(single_comparisons(a, consts)) + mixed_programs(a, b, ids)


def test_program_shapes():
    a, b = deep_program(0, 1), long_program(0, 1)
    assert R.stack_shape(a) == (19, 10) and R.stack_shape(b) == (32, 2)


# ---- the store
def store_triples(seed=1):
    """per subject e: (e TITLE t), (e VAL v), (e VAL2 w), (e NAME e); 1..3 objects of MV1 / MV2 for a third of them; a 60-row SMALL1 /
    SMALL2 pair for the cartesian product; a chain CH_A -> CH_B -> CH_C whose join keys are literals"""
    rng = np.random.default_rng(seed)
    subj = np.arange(SUBJ0, SUBJ0 + N_SUBJ, dtype=np.uint32)
    cells = lambda n: FC.edge_cells(rng, n, LIT0, N_PLAIN, N_IDS, relation=False)  # noqa: E731
    val, val2 = cells(N_SUBJ), cells(N_SUBJ)
    val[:16], val2[:16] = [ONE_UP, ONE_DOWN] * 8, [ONE_DOWN, ONE_UP] * 8  # the contraction pair (both orders)
    parts = [np.stack([subj, np.full(N_SUBJ, TITLE), TITLES[rng.integers(0, 3, N_SUBJ)]], 1),
             np.stack([subj, np.full(N_SUBJ, VAL), val], 1),
             np.stack([subj, np.full(N_SUBJ, VAL2), val2], 1),
             np.stack([subj, np.full(N_SUBJ, NAME), subj], 1)]
    for p in (MV1, MV2):
        few = np.repeat(subj[rng.choice(N_SUBJ, N_SUBJ // 3, replace=False)], rng.integers(1, 4, N_SUBJ // 3))
        parts.append(np.stack([few, np.full(len(few), p), cells(len(few))], 1))
    for p in (SMALL1, SMALL2):
        parts.append(np.stack([subj[:60] + (p - SMALL1) * 60, np.full(60, p), cells(60)], 1))
    lit = LIT0 + np.arange(len(FC.VALUES) + N_PLAIN)
    for p in (CH_A, CH_B, CH_C):  # subjects: employees for CH_A, literals for the next links (ids are ids)
        src = subj[:300] if p == CH_A else lit
        n = len(src) * 2
        parts.append(np.stack([np.repeat(src, 2), np.full(n, p), rng.choice(lit, n)], 1))
    tr = np.unique(np.concatenate(parts).astype(np.uint32), axis=0)
    return tr[rng.permutation(len(tr))]


TRIPLES = store_triples()
NUM, ISN = FC.numeric_table(N_IDS, LIT0)
TERMS = R.Terms(NUM, ISN)
_DB = {}


def oracle():
    if "db" not in _DB:
        _DB["db"] = O.Db(TRIPLES[:, 0], TRIPLES[:, 1], TRIPLES[:, 2], NUM, ISN)
    return _DB["db"]


def stored_ids(pred, n=3):
    """a few objects of `pred`, and KB_ID_NONE as a literal missing from the dictionary"""
    o = np.unique(TRIPLES[TRIPLES[:, 1] == pred, 2])
    return list(o[:: max(1, len(o) // n)][:n]) + [NONE]


def load_ctx(index):
    cx = c.Context(0)
    cx.store_load(TRIPLES[:, 0], TRIPLES[:, 1], TRIPLES[:, 2])
    cx.dict_numeric_load(NUM, ISN)
    if index:
        cx.build_index()
    return cx


@pytest.fixture
def make_ctx(monkeypatch):
    """a fresh context on the edge-value store, created after the route switches are set (they are read when a context is created)"""
    made = []

    def make(index=False, **env):
        for k, v in {**DEFAULT_ENV, **env}.items():
            monkeypatch.setenv(k, v)
        cx = load_ctx(index)
        made.append(cx)
        return cx

    yield make
    for cx in made:
        cx.close()


def delta(cx, call):
    a = cx.get_stats()
    out = call()
    b = cx.get_stats()
    return out, {k: b[k] - a[k] for k in b if isinstance(b[k], int)}


def rows_of(rel, slots):
    return rel.to_numpy(slots) if rel.n_rows else np.empty((0, len(slots)), np.uint32)


def unfiltered(pats):
    """the oracle's BGP without a filter: (rows over sorted slots, slots)"""
    r = oracle().bgp(pats)
    slots = sorted(r.slots)
    return rows_of(r, slots), slots


def check_rows(got, want, what):
    H.assert_same_bag(got, want, what)


def describe(prog):
    return [(o.op, o.slot, o.cmp, o.id, o.value) for o in prog]


# ---- kb_filter over relations
def host_relation(cx, seed, n=3000):
    rng = np.random.default_rng(seed)
    cols = [FC.edge_cells(rng, n, LIT0, N_PLAIN, N_IDS) for _ in range(3)]
    cols[0][:8], cols[1][:8] = ONE_UP, ONE_DOWN  # the contraction pair
    return cx.rel_from_host([0, 1, 2], cols), np.stack(cols, axis=1)


def test_kb_filter_host_relation(make_ctx):
    cx = make_ctx()
    rel, rows = host_relation(cx, 3)
    assert contraction_rows(rows, [0, 1, 2], 0, 1) >= 8
    progs = programs(0, 1, FEW_CONSTS, [LIT0 + 4, LIT0 + len(FC.VALUES) + 1, 0x80000003, NONE])
    for prog in progs:
        got, d = delta(cx, lambda: cx.filter(rel, prog))
        check_rows(rows_of(got, [0, 1, 2]), R.filter_rows(rows, [0, 1, 2], prog, TERMS), describe(prog))
        assert d["filter_launches"] >= 1, "kb_filter did not launch its kernel"
        got.free()


def test_kb_filter_unbound_cells(make_ctx):
    """KB_ID_NONE is a variable the row leaves unbound: every comparison over it is false, != and isTRIPLE included, and NOT is true"""
    cx = make_ctx()
    vals = np.array([NONE, LIT0 + 14, NONE, 0x80000001, LIT0 + len(FC.VALUES), NONE, N_IDS + 3], dtype=np.uint32)  # 1.0 at LIT0 + 14
    assert FC.VALUES[14] == 1.0
    rel = cx.rel_from_host([0], [vals])
    bound = vals[vals != NONE][:, None]
    cases = {"ne_id": ([f(c.F_NE_ID, slot=0, id=LIT0 + 14)], np.array([[0x80000001], [LIT0 + len(FC.VALUES)], [N_IDS + 3]])),
             "ne_missing_literal": ([f(c.F_NE_ID, slot=0, id=NONE)], bound),
             "cmp_num_fast": ([cmp(0, c.CMP_GT, -1.0)], bound),
             "cmp_num_general": ([cmp(0, c.CMP_GT, -1.0), cmp(0, c.CMP_LT, 5.0), f(c.F_AND)], bound),
             "not_cmp_num": ([cmp(0, c.CMP_GT, -1.0), f(c.F_NOT)], vals[vals == NONE][:, None]),
             "is_triple": ([f(c.F_IS_TRIPLE, slot=0)], np.array([[0x80000001]])),
             "arith": ([f(c.F_PUSH_VAR, slot=0), f(c.F_PUSH_CONST, value=0.0), f(c.F_SUB), f(c.F_TRUTHY), f(c.F_NOT)], vals[vals != LIT0 + 14][:, None])}
    for name, (prog, want) in cases.items():
        np.testing.assert_array_equal(R.filter_rows(vals[:, None], [0], prog, TERMS), np.asarray(want, np.uint32).reshape(-1, 1), name)
        got, d = delta(cx, lambda: cx.filter(rel, prog))
        check_rows(rows_of(got, [0]), want, name)
        assert d["filter_launches"] >= 1


def test_kb_filter_over_bind_output(make_ctx):
    """SUBJECT(?t) leaves the rows whose ?t is not a quoted triple unbound; FILTER over that column then drops them"""
    cx = make_ctx()
    qb = E.QUOTED_TRIPLE_ID_BIT
    k = 40
    qids = np.arange(qb, qb + k, dtype=np.uint32)
    cx.quoted_load(qids, LIT0 + np.arange(k, dtype=np.uint32), np.full(k, VAL, np.uint32), LIT0 + np.arange(k, dtype=np.uint32))
    rng = np.random.default_rng(9)
    t = np.where(rng.random(500) < 0.5, rng.choice(qids, 500), rng.integers(SUBJ0, SUBJ0 + N_SUBJ, 500)).astype(np.uint32)
    rel = cx.rel_from_host([0], [t])
    out, info = cx.bind(rel, c.BIND_SUBJECT, [c.V(0)], 1)
    rows = rows_of(out, [0, 1])
    assert info["n_unbound"] == int((t < qb).sum()) > 0 and (rows[:, 1] == NONE).sum() == info["n_unbound"]
    progs = programs(1, 0, FEW_CONSTS, [LIT0 + 3, NONE])
    for prog in progs:
        got, d = delta(cx, lambda: cx.filter(out, prog))
        check_rows(rows_of(got, [0, 1]), R.filter_rows(rows, [0, 1], prog, TERMS), describe(prog))
        assert d["filter_launches"] >= 1
        got.free()


# ---- scans with a pushed-down filter
@pytest.mark.parametrize("where", ["o", "s", "p"])
def test_scan_pushdown(make_ctx, where):
    """kb_scan with a pushed-down program: one CMP_NUM takes scan_kernel's gather-then-compare path, the others the stack machine"""
    cx = make_ctx()
    if where == "o":
        pat, slot = c.pattern(c.V(0), c.K(VAL), c.V(2)), 2
        sel = TRIPLES[TRIPLES[:, 1] == VAL]
        rows, slots = sel[:, [0, 2]], [0, 2]
    else:  # all triples of the chain predicates (literal subjects) and TITLE, filtered on the subject or the predicate
        pat, slot = c.pattern(c.V(0), c.V(1), c.V(2)), (0 if where == "s" else 1)
        rows, slots = TRIPLES, [0, 1, 2]
    consts = ALL_CONSTS if where == "o" else FEW_CONSTS
    for prog in programs(slot, 2 if slot != 2 else 0, consts, stored_ids(VAL)):
        got, d = delta(cx, lambda: cx.scan([pat], [prog])[0])
        check_rows(rows_of(got, slots), R.filter_rows(rows, slots, prog, TERMS), (where, describe(prog)))
        assert d["scan_launches"] >= 1 and d["fused_scan_builds"] == 0 and d["index_joins"] == 0
        got.free()


# ---- star joins
def star():
    e, t, v, nm, w = 0, 1, 2, 3, 4
    pats = [c.pattern(c.V(e), c.K(TITLE), c.V(t)), c.pattern(c.V(e), c.K(VAL), c.V(v)), c.pattern(c.V(e), c.K(NAME), c.V(nm)),
            c.pattern(c.V(e), c.K(VAL2), c.V(w))]
    return e, pats


# name -> (switches, index built, the counters that prove the route)
#   fused_star_scan: without an index the scan fills the direct tables (R3). Four patterns with constant predicates and at most one
#     CMP_NUM each on s or o: scan_is_star holds, so scan_star_kernel runs, with its strict -> non-strict rewrite of > and <. Both scan
#     kernels count a fused scan build; scan_star_off below runs the same cases on scan_kernel.
#   fused_scan_ordered: store-order output takes scan_kernel (scan_is_star refuses ordered scans).
#   index_table_mode / index_slice_mode: R1 (probe_index_kernel, one word read back), the probe stream over the subject table or the
#     predicate slice (the typed column's pre-filter).
#   index_staged_probe: KOLIBRIE_INDEX_KERNEL=0 takes R2 over the persistent tables: no build (every side has a table), the filtered
#     pattern probes with probe_fast_kernel's pre-filter and the other filters run as its post-filter. The filtered build of R2 is
#     test_filtered_build_side.
STAR_ROUTES = {
    "fused_star_scan": ({}, False, lambda d: d["fused_scan_builds"] >= 1 and d["index_joins"] == 0),
    "fused_scan_ordered": ({"KOLIBRIE_ORDERED": "1"}, False, lambda d: d["fused_scan_builds"] >= 1 and d["index_joins"] == 0),
    "index_table_mode": ({}, True, lambda d: d["index_joins"] >= 1 and d["d2h_bytes"] == 4),
    "index_slice_mode": ({"KOLIBRIE_PROBE_TABLE": "0"}, True, lambda d: d["index_joins"] >= 1 and d["d2h_bytes"] == 4),
    "index_staged_probe": ({"KOLIBRIE_INDEX_KERNEL": "0"}, True, lambda d: d["index_joins"] >= 1 and d["d2h_bytes"] > 4 and d["rows_built"] == 0),
    # the star scan switched off (read once per process: run in a process of its own by test_star_scan_switched_off)
    "scan_star_off": ({"KOLIBRIE_SCAN_STAR": "0"}, False, lambda d: d["fused_scan_builds"] >= 1 and d["index_joins"] == 0),
}


def star_cases(route):
    """(patterns, programs): a filter on ?v (the probe pattern or a build side), on ?w, and one spanning both"""
    js, pats = star()
    out = []
    single = ALL_CONSTS if route in ("fused_star_scan", "fused_scan_ordered", "index_slice_mode", "scan_star_off") else FEW_CONSTS
    out += [(js, pats, p) for p in single_comparisons(2, single)]
    out += [(js, pats, p) for p in single_comparisons(4, FEW_CONSTS)]
    out += [(js, pats, p) for p in mixed_programs(2, 4, stored_ids(VAL))]
    out += [(js, pats, p) for p in mixed_programs(4, 4, stored_ids(VAL2))]
    out += [(js, pats[1:2] + pats[:1], p) for p in single_comparisons(2, FEW_CONSTS)]  # ?v on the first (probe) pattern
    out += [(js, pats[3:4] + pats[:3], p) for p in mixed_programs(2, 4, [NONE])]
    return out


def run_star_route(cx, route):
    proof = STAR_ROUTES[route][2]
    base = {}
    for js, pats, prog in star_cases(route):
        key = tuple((p.s.is_var, p.s.value, p.p.value, p.o.value) for p in pats)
        if key not in base:
            base[key] = unfiltered(pats)
            if 2 in base[key][1] and 4 in base[key][1]:
                assert contraction_rows(base[key][0], base[key][1], 2, 4) >= 16
        rows, slots = base[key]
        got, d = delta(cx, lambda: cx.star_join(js, pats, prog))
        check_rows(rows_of(got, slots), R.filter_rows(rows, slots, prog, TERMS), (route, describe(prog)))
        assert proof(d), (route, d)
        got.free()


@pytest.mark.parametrize("route", [r for r in STAR_ROUTES if r != "scan_star_off"])
def test_star_join_sites(make_ctx, route):
    env, index, _ = STAR_ROUTES[route]
    run_star_route(make_ctx(index=index, **env), route)


def star_route_in_process(route):
    """one STAR_ROUTES case with its switches set in this process's environment (for a switch read once per process)"""
    env, index, _ = STAR_ROUTES[route]
    os.environ.update({**DEFAULT_ENV, **env})
    cx = load_ctx(index)
    try:
        run_star_route(cx, route)
    finally:
        cx.close()


def test_star_scan_switched_off():
    """KOLIBRIE_SCAN_STAR=0: the star shape of fused_star_scan on scan_kernel. The switch is read once per process, so the case runs in
    a process of its own."""
    env = {**os.environ, **DEFAULT_ENV, **STAR_ROUTES["scan_star_off"][0]}
    r = subprocess.run([sys.executable, "-c", "from tests import test_gpu_filter_sites as T; T.star_route_in_process('scan_star_off')"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]


# ---- R2: filtered build sides
SPARSE0, SPARSE_N, SPARSE_GAP = 10_000, 30_000, 7


def sparse_star_store(seed=5):
    """three single-valued predicates over 30 000 subjects 7 ids apart. The subject range (about 210 000) is too sparse for the index to
    keep a persistent table of any of them (more than 4 n + 65 536 ids), yet dense enough (at most 8 n) for R2 to build direct tables
    from the predicate slices: the sides that do not probe are built by build_pairs_filtered_kernel, with their own filters."""
    rng = np.random.default_rng(seed)
    subj = (SPARSE0 + SPARSE_GAP * np.arange(SPARSE_N)).astype(np.uint32)
    v, w = (FC.edge_cells(rng, SPARSE_N, LIT0, N_PLAIN, N_IDS, relation=False) for _ in range(2))
    v[:16], w[:16] = [ONE_UP, ONE_DOWN] * 8, [ONE_DOWN, ONE_UP] * 8
    tr = np.concatenate([np.stack([subj, np.full(SPARSE_N, p), o], 1) for p, o in ((VAL, v), (VAL2, w), (NAME, subj))]).astype(np.uint32)
    return tr[rng.permutation(len(tr))]


def test_filtered_build_side(make_ctx):
    cx = make_ctx(index=True)
    tr = sparse_star_store()
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    cx.build_index()
    db = O.Db(tr[:, 0], tr[:, 1], tr[:, 2], NUM, ISN)
    pats = [c.pattern(c.V(0), c.K(VAL), c.V(2)), c.pattern(c.V(0), c.K(VAL2), c.V(4)), c.pattern(c.V(0), c.K(NAME), c.V(3))]
    r = db.bgp(pats)
    slots = sorted(r.slots)
    rows = rows_of(r, slots)
    assert len(rows) == SPARSE_N and contraction_rows(rows, slots, 2, 4) >= 16
    # a filter on ?v alone or on ?w alone is pushed into that side's build; one over both runs on the joined row
    progs = (list(single_comparisons(2, ALL_CONSTS)) + list(single_comparisons(4, FEW_CONSTS)) + mixed_programs(2, 2, stored_ids(VAL)) +
             mixed_programs(4, 4, [NONE]) + mixed_programs(2, 4, [NONE]))
    for prog in progs:
        got, d = delta(cx, lambda: cx.star_join(0, pats, prog))
        check_rows(rows_of(got, slots), R.filter_rows(rows, slots, prog, TERMS), describe(prog))
        assert d["index_joins"] >= 1 and d["rows_built"] >= SPARSE_N and d["fused_scan_builds"] == 0, d  # R2 built a side from its slice
        got.free()


def test_index_slice_mode_after_numeric_reload(make_ctx):
    """a dict_numeric_load after the index build makes the typed value column stale: the probe must not filter on it"""
    cx = make_ctx(index=True, KOLIBRIE_PROBE_TABLE="0")
    flipped = -FC.VALUES[::-1].copy()
    num, isn = FC.numeric_table(N_IDS, LIT0, flipped)
    cx.dict_numeric_load(num, isn)
    terms = R.Terms(num, isn)
    js, pats = star()
    rows, slots = unfiltered(pats)
    for prog in list(single_comparisons(2, FEW_CONSTS)) + mixed_programs(2, 4, [NONE]):
        got, d = delta(cx, lambda: cx.star_join(js, pats, prog))
        check_rows(rows_of(got, slots), R.filter_rows(rows, slots, prog, terms), describe(prog))
        assert d["index_joins"] >= 1
        got.free()


@pytest.mark.parametrize("mode", ["1", "0"])
def test_prepared_plans(make_ctx, mode):
    cx = make_ctx(index=True, KOLIBRIE_PROBE_TABLE=mode)
    js, pats = star()
    rows, slots = unfiltered(pats)
    for prog in list(single_comparisons(2, FEW_CONSTS[::2])) + mixed_programs(2, 4, [NONE]):
        def run():
            pl = cx.prepare_star_join(js, pats, prog, ring=2)
            r = pl.collect_rows(pl.submit())
            out = rows_of(r, slots)
            r.free()
            pl.free()
            return out
        got, d = delta(cx, run)
        check_rows(got, R.filter_rows(rows, slots, prog, TERMS), (mode, describe(prog)))
        assert d["index_joins"] >= 1


@pytest.mark.parametrize("csr", ["1", "0"])
def test_chained_join_filter(make_ctx, csr):
    """multi-valued build sides: chained natural joins (R5), with a filter over both sides evaluated after the join"""
    cx = make_ctx(KOLIBRIE_CSR_JOIN=csr)
    pats = [c.pattern(c.V(0), c.K(MV1), c.V(1)), c.pattern(c.V(0), c.K(MV2), c.V(2))]
    rows, slots = unfiltered(pats)
    assert len(rows) > 100
    joined = 0
    for prog in list(single_comparisons(1, FEW_CONSTS)) + mixed_programs(1, 2, stored_ids(MV1)):
        got, d = delta(cx, lambda: cx.bgp_execute(pats, prog))
        want = R.filter_rows(rows, slots, prog, TERMS)
        check_rows(rows_of(got, slots), want, (csr, describe(prog)))
        assert d["index_joins"] == 0, d
        if len(want):  # (a pushed-down filter that empties a side ends the query before any join)
            assert d["other_launches"] >= 1, d  # the chained joins unpair their inputs
            joined += 1
        got.free()
    assert joined >= 50


def test_cartesian_product_filter(make_ctx):
    cx = make_ctx()
    pats = [c.pattern(c.V(0), c.K(SMALL1), c.V(1)), c.pattern(c.V(2), c.K(SMALL2), c.V(3))]
    rows, slots = unfiltered(pats)
    assert len(rows) == 3600
    for prog in list(single_comparisons(1, FEW_CONSTS)) + mixed_programs(1, 3, [NONE]):
        got = cx.bgp_execute(pats, prog)
        check_rows(rows_of(got, slots), R.filter_rows(rows, slots, prog, TERMS), describe(prog))
        plan = cx.bgp_last_plan()
        assert plan["route"] == c.BGP_COMPONENTS and plan["n_components"] == 2, plan  # two components: their cross join
        got.free()


def test_component_route_post_filter(make_ctx):
    """a chain of three patterns (not a star): the component route, with filters over one link and across links"""
    cx = make_ctx()
    pats = [c.pattern(c.V(0), c.K(CH_A), c.V(1)), c.pattern(c.V(1), c.K(CH_B), c.V(2)), c.pattern(c.V(2), c.K(CH_C), c.V(3))]
    rows, slots = unfiltered(pats)
    assert len(rows) > 100
    for prog in list(single_comparisons(3, FEW_CONSTS)) + mixed_programs(1, 3, [NONE]) + mixed_programs(2, 3, [LIT0 + 5]):
        got = cx.bgp_execute(pats, prog)
        check_rows(rows_of(got, slots), R.filter_rows(rows, slots, prog, TERMS), describe(prog))
        assert cx.bgp_last_plan()["route"] == c.BGP_COMPONENTS
        got.free()


# ---- FILTER limits at every entry point
def test_filter_limits_at_every_entry_point(make_ctx):
    cx = make_ctx(index=True)
    too_deep = [cmp(2, c.CMP_GT, float(i)) for i in range(11)] + [f(c.F_AND)] * 10  # depth 11, 21 ops
    too_long = long_program(2, 2) + [f(c.F_NOT)]  # 33 ops
    assert R.stack_shape(too_deep) == (21, 11) and len(too_long) == 33
    js, pats = star()
    rel, _ = host_relation(cx, 4, 10)
    calls = {"filter": lambda p: cx.filter(rel, p), "scan": lambda p: cx.scan([pats[1]], [p]), "star_join": lambda p: cx.star_join(js, pats, p),
             "bgp_execute": lambda p: cx.bgp_execute(pats, p), "prepare": lambda p: cx.prepare_star_join(js, pats, p),
             "aggregate": lambda p: cx.star_join_aggregate(js, pats, p, [1], [(c.AGG_COUNT, 0)])}
    for name, call in calls.items():
        for prog in (too_deep, too_long):
            with pytest.raises(c.KolibrieError) as e:
                call(prog)
            assert e.value.status == c.KB_E_LIMIT, (name, len(prog))
        for prog in (deep_program(2, 2), long_program(2, 2)):  # the limits themselves are accepted
            r = call(prog)
            if hasattr(r, "free"):
                r.free()


# ---- Datalog rule filters
def rule_filter(k, v):
    return c.KbRuleFilter(0, k, 0, 0, float(v))


RULE_FILTERS = [(k, v) for k in (c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE, c.CMP_EQ, c.CMP_NE)
                for v in (1.0, 0.0, -0.0, np.inf, np.nan, 100000.0, FC.DMIN, -FC.DBL_MAX)]


def rules_for(k1, v1, k2, v2):
    """?x VAL ?v, FILTER(?v k1 v1) -> ?x DER1 ?v; ?x DER1 ?v, FILTER(?v k2 v2) -> ?x DER2 ?v"""
    return [{"premise": [c.pattern(c.V(1), c.K(VAL), c.V(0))], "filters": [rule_filter(k1, v1)], "conclusion": [c.pattern(c.V(1), c.K(DER1), c.V(0))]},
            {"premise": [c.pattern(c.V(1), c.K(DER1), c.V(0))], "filters": [rule_filter(k2, v2)], "conclusion": [c.pattern(c.V(1), c.K(DER2), c.V(0))]}]


def closure(base, k1, v1, k2, v2, terms=TERMS, filtered=True):
    """the facts the two rules add to `base`, with the rule filters restated from rules.rs (filtered=False: KB_SEMI_NAIVE_PARALLEL,
    which evaluates no rule filter, as semi_naive_parallel.rs:11-176 does not)"""
    src = base[base[:, 1] == VAL]
    d1 = src[R.rule_filter_pass(rule_filter(k1, v1), src[:, 2], None, terms)] if filtered else src
    d2 = d1[R.rule_filter_pass(rule_filter(k2, v2), d1[:, 2], None, terms)] if filtered else d1
    new = np.concatenate([np.stack([d1[:, 0], np.full(len(d1), DER1), d1[:, 2]], 1), np.stack([d2[:, 0], np.full(len(d2), DER2), d2[:, 2]], 1)])
    return {tuple(int(x) for x in r) for r in new.astype(np.uint32)}


def fact_set(rel):
    return {tuple(int(x) for x in r) for r in rows_of(rel, [0, 1, 2])}


@pytest.mark.parametrize("partitioned", [False, True])
@pytest.mark.parametrize("strategy", [c.SEMI_NAIVE, c.NAIVE, c.SEMI_NAIVE_PARALLEL, c.SEMI_NAIVE_OLD_DELTA])
def test_datalog_rule_filters(make_ctx, strategy, partitioned):
    env = {"KOLIBRIE_DERIVE_PART": "1", "KOLIBRIE_DERIVE_SLICE": "2048", "KOLIBRIE_DERIVE_MIN_ROWS": "16"} if partitioned else {}
    cx = make_ctx(**env)
    base = TRIPLES[np.isin(TRIPLES[:, 1], [VAL, TITLE])]
    base_set = {tuple(int(x) for x in r) for r in base}
    rng = np.random.default_rng(strategy)
    for k1, v1 in RULE_FILTERS:
        k2, v2 = RULE_FILTERS[int(rng.integers(0, len(RULE_FILTERS)))]
        cx.store_load(base[:, 0], base[:, 1], base[:, 2])
        (rel, st), d = delta(cx, lambda: cx.datalog_fixpoint(rules_for(k1, v1, k2, v2), strategy))
        want = closure(base, k1, v1, k2, v2, filtered=strategy != c.SEMI_NAIVE_PARALLEL)
        assert fact_set(rel) - base_set == want, (strategy, k1, v1, k2, v2)
        assert st.rounds >= 1 and d["kernel_launches"] >= 1
        if partitioned and len(want) >= 64:
            assert d["rows_built"] > 0, "the partitioned dedup did not run"


def test_datalog_maintain_rule_filters(make_ctx):
    """two window slides under filtered rules: the inferred facts after each equal the restated closure of the live segments"""
    cx = make_ctx()
    base = TRIPLES[TRIPLES[:, 1] == VAL]
    segs = {t: base[t::4] for t in range(4)}
    for k1, v1, k2, v2 in [(c.CMP_GE, 0.0, c.CMP_EQ, 1.0), (c.CMP_NE, 1.0, c.CMP_LT, np.inf), (c.CMP_EQ, np.nan, c.CMP_GT, -0.0)]:
        cx.store_clear()
        cx.dict_numeric_load(NUM, ISN)
        live = {}
        for t in (0, 1):
            cx.store_append(segs[t][:, 0], segs[t][:, 1], segs[t][:, 2], t + 1)
            live[t] = segs[t]
        rules = rules_for(k1, v1, k2, v2)
        rel, _ = cx.datalog_fixpoint(rules)
        inferred = fact_set(rel) - {tuple(int(x) for x in r) for r in np.concatenate(list(live.values()))}
        assert inferred == closure(np.concatenate(list(live.values())), k1, v1, k2, v2)
        for old, new in ((0, 2), (1, 3)):
            gone, added, _ = cx.datalog_maintain(rules, [old + 1], segs[new], new + 1)
            del live[old]
            live[new] = segs[new]
            want = closure(np.concatenate(list(live.values())), k1, v1, k2, v2)
            assert fact_set(gone) == inferred - want and fact_set(added) == want - inferred, (k1, v1, k2, v2, new)
            inferred = want


# ---- end to end from strings
STRINGS = ["NaN", "-0", "inf", "-infinity", "4.9e-324", "1e309", "2.2250738585072011e-308", "+1", "1.", ".5", "1_0", " 1", "-inf",
           "1.7976931348623157e308", "-1.7976931348623157e308", "0", "1", "100000", "nan", "infinity", "abc", "", "+0.0", "1e-400", "-5e-324"]


def test_end_to_end_from_strings(make_ctx):
    """dictionary strings Rust parses to edge values (and some it does not), the numeric table derived on the device, a filtered star
    join: against the restatement over rust_parse_f64 of the same strings"""
    cx = make_ctx()
    n_str = 64
    strings = (STRINGS + [f"name{i}" for i in range(n_str)])[:n_str]
    assert len(strings) == n_str and all(s in strings for s in STRINGS)
    parsed = [E.rust_parse_f64(s) for s in strings]
    assert parsed[0] != parsed[0] and parsed[5] == np.inf and parsed[8] == 1.0 and parsed[9] == 0.5 and parsed[10] is None and parsed[11] is None
    num = np.array([0.0 if p is None else p for p in parsed], dtype=np.float64)
    isn = np.array([p is not None for p in parsed], dtype=np.uint8)
    terms = R.Terms(num, isn)
    rng = np.random.default_rng(21)
    subj = np.arange(100, 100 + 1500, dtype=np.uint32)  # subjects and predicates past the string table: not numbers
    obj = rng.integers(0, n_str, len(subj)).astype(np.uint32)
    tr = np.concatenate([np.stack([subj, np.full(len(subj), 70), obj], 1), np.stack([subj, np.full(len(subj), 71), subj], 1)]).astype(np.uint32)
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    cx.dict_strings_load(strings)
    cx.dict_numeric_derive(c.NUMERIC_F64, 0)
    dnum, disn = cx.dict_numeric_download(0, n_str)
    np.testing.assert_array_equal(disn, isn)
    np.testing.assert_array_equal(dnum.view(np.uint64)[isn == 1], num.view(np.uint64)[isn == 1])
    pats = [c.pattern(c.V(0), c.K(70), c.V(1)), c.pattern(c.V(0), c.K(71), c.V(2))]
    rows = np.stack([subj, obj, subj], 1)
    consts = FC.boundary_consts(num[isn == 1])
    for prog in list(single_comparisons(1, consts)) + mixed_programs(1, 1, [3, NONE]):
        got, d = delta(cx, lambda: cx.star_join(0, pats, prog))
        check_rows(rows_of(got, [0, 1, 2]), R.filter_rows(rows, [0, 1, 2], prog, terms), describe(prog))
        assert d["fused_scan_builds"] >= 1
        got.free()
