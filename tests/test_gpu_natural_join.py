"""GPU (-m gpu): kb_natural_join against the restatement of natural_join (tests/rsp_join_reference.py), compared as bags, and
engine.WindowJoin (multi-window and static-data emits through R2S) against the restated emit path, emit by emit."""
import ctypes as C
import random
from collections import Counter

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200.engine import Bind, Constant, SimpleR2R, SlotMap, SparqlDatabase, TableScan, Variable, WindowJoin
from tests import rsp_join_reference as J
from tests.r2s_reference import Relation2Stream

pytestmark = pytest.mark.gpu
NONE = c.KB_ID_NONE


def rel_of(ctx, slots, rows):
    a = np.asarray(rows, dtype=np.uint32).reshape(-1, len(slots))
    return ctx.rel_from_host(list(slots), [np.ascontiguousarray(a[:, j]) for j in range(len(slots))])


def dict_rows(slots, rows):
    return [{s: v for s, v in zip(slots, r) if v != NONE} for r in rows]


def device_bag(rel):
    n, slots = rel.info()
    a = rel.to_numpy(slots) if n else np.zeros((0, len(slots)), dtype=np.uint32)
    return Counter(tuple(sorted((s, int(v)) for s, v in zip(slots, r) if v != NONE)) for r in a.tolist()), slots


def ref_bag(ls, lrows, rs, rrows):
    return Counter(tuple(sorted(r.items())) for r in J.natural_join(dict_rows(ls, lrows), dict_rows(rs, rrows)))


def check(ctx, ls, lrows, rs, rrows):
    got, slots = device_bag(ctx.natural_join(rel_of(ctx, ls, lrows), rel_of(ctx, rs, rrows)))
    assert slots == list(ls) + [s for s in rs if s not in ls]
    assert got == ref_bag(ls, lrows, rs, rrows)
    return got


def random_side(rng, n, slots, unbound_slots, domain=4, p_none=0.3):
    return [tuple(NONE if s in unbound_slots and rng.random() < p_none else rng.randrange(domain) for s in slots) for _ in range(n)]


@pytest.mark.parametrize("n_u", [0, 1, 2, 3, 4])
def test_seeded_relations_by_unbound_shared_slots(ctx, n_u):
    rng = random.Random(100 + n_u)
    for trial in range(6):
        shared = [10, 11, 12, 13][: max(n_u, 1 + trial % 3)]
        ls, rs = shared + [20, 21], [30] + shared[::-1]  # the right side lists the shared slots in another order
        U = set(shared[:n_u])
        lrows = random_side(rng, rng.randrange(1, 300), ls, U)
        rrows = random_side(rng, rng.randrange(1, 300), rs, U)
        ctx.get_stats(reset=True)
        check(ctx, ls, lrows, rs, rrows)
        st = ctx.get_stats()
        if not any(NONE in r for r in lrows + rrows):
            assert st["other_launches"] == 1, st  # fast route: the check pass, then kb_hash_join's own launches
        else:
            assert st["other_launches"] >= 4, st  # check, mask, partition, coalesce


def test_one_side_wholly_unbound_in_a_shared_slot(ctx):
    rng = random.Random(3)
    lrows = [(rng.randrange(5), NONE, rng.randrange(9)) for _ in range(200)]
    rrows = [(rng.randrange(5), rng.randrange(4)) for _ in range(150)]
    got = check(ctx, [1, 2, 3], lrows, [1, 2], rrows)
    assert sum(got.values()) == sum(1 for a in lrows for b in rrows if a[0] == b[0])


def test_a_slot_unbound_on_both_sides_stays_unbound(ctx):
    got = check(ctx, [1, 2], [(1, NONE), (2, NONE)], [2, 3], [(NONE, 7), (5, 8)])
    assert got == Counter({((1, 1), (3, 7)): 1, ((1, 2), (3, 7)): 1, ((1, 1), (2, 5), (3, 8)): 1, ((1, 2), (2, 5), (3, 8)): 1})


def test_disjoint_slots_give_the_cartesian_product(ctx):
    got = check(ctx, [1, 2], [(1, 2), (3, NONE), (1, 2)], [5], [(7,), (8,)])
    assert sum(got.values()) == 6


def test_duplicate_rows_multiply(ctx):
    got = check(ctx, [1, 2], [(1, 2)] * 3 + [(1, NONE)] * 2, [1, 3], [(1, 9)] * 4)
    assert sum(got.values()) == 5 * 4


def test_empty_sides(ctx):
    for lrows, rrows in (([], [(1, 2)]), ([(1, NONE)], []), ([], [])):
        rel = ctx.natural_join(rel_of(ctx, [1, 2], lrows), rel_of(ctx, [2, 3], rrows))
        assert rel.info() == (0, [1, 2, 3])


def call_raw(ctx, left, right):
    """kb_natural_join with an output pointer that must stay as it was when the call is refused"""
    out = C.c_void_p(0x1234)
    st = c.lib().kb_natural_join(ctx.h, left.h, right.h, C.byref(out))
    return st, out.value


def test_limits_leave_the_output_untouched(ctx):
    shared = [1, 2, 3, 4, 5]
    row = lambda k: tuple(NONE if j == k else j for j in range(5))
    left = rel_of(ctx, shared, [row(k) for k in range(5)])
    right = rel_of(ctx, shared, [tuple(range(5))])
    assert call_raw(ctx, left, right) == (c.KB_E_LIMIT, 0x1234)  # |U| = 5
    big_l = ctx.rel_from_host([1], [np.arange(1 << 14, dtype=np.uint32)])
    big_r = ctx.rel_from_host([2], [np.arange((1 << 14) + 1, dtype=np.uint32)])
    assert call_raw(ctx, big_l, big_r) == (c.KB_E_LIMIT, 0x1234)  # cartesian product over 2^28 rows
    check(ctx, [1, 2], [(1, NONE)], [2], [(3,)])  # the context still works


# ------------------------------------------------------------------ WindowJoin: multi-window and static-data emits
TYPE = "http://www.w3.org/1999/02/22-rdf-syntax-ns#type"


def host_query(triples, kind):
    """the window queries on the host over string triples: 'sensor' = ?sensor a Sensor; 'room' = ?room a Room; 'subj' =
    ?q a Reading BIND(SUBJECT(?q) AS ?sensor) — ?q is not a quoted triple id here, so ?sensor stays unbound"""
    if kind == "sensor":
        return [{"sensor": s} for s, p, o in triples if p == TYPE and o == "Sensor"]
    if kind == "room":
        return [{"room": s} for s, p, o in triples if p == TYPE and o == "Room"]
    return [{"q": s} for s, p, o in triples if p == TYPE and o == "Reading"]


def plan_of(kind, d):
    if kind == "sensor":
        return TableScan((Variable("sensor"), Constant(d.encode(TYPE)), Constant(d.encode("Sensor"))))
    if kind == "room":
        return TableScan((Variable("room"), Constant(d.encode(TYPE)), Constant(d.encode("Room"))))
    return Bind(TableScan((Variable("q"), Constant(d.encode(TYPE)), Constant(d.encode("Reading")))), "SUBJECT", ["?q"], "sensor")


SCRIPT = [  # (window, ts, window content) per firing; None = the emitter drains here
    ("w1", 2, [("s0", TYPE, "Sensor"), ("s1", TYPE, "Sensor"), ("q0", TYPE, "Reading")]), None,
    ("w2", 3, [("r0", TYPE, "Room")]), None,
    ("w1", 4, [("s1", TYPE, "Sensor"), ("s2", TYPE, "Sensor"), ("q0", TYPE, "Reading"), ("q1", TYPE, "Reading")]),
    ("w2", 5, [("r0", TYPE, "Room"), ("r1", TYPE, "Room")]), None,
    ("w1", 6, [("s2", TYPE, "Sensor"), ("q2", TYPE, "Reading")]), None,
    ("w2", 7, []), None,
    ("w1", 8, [("s0", TYPE, "Sensor"), ("s3", TYPE, "Sensor")]), ("w2", 9, [("r1", TYPE, "Room")]), None,
]
STATIC = [("s0", "locatedIn", "r0"), ("s1", "locatedIn", "r1"), ("s2", "locatedIn", "r1")]


@pytest.mark.parametrize("policy", ["wait", "steal"])
@pytest.mark.parametrize("stream", ["RSTREAM", "ISTREAM", "DSTREAM"])
@pytest.mark.parametrize("queries", [("sensor", "room"), ("subj", "room")], ids=["two_windows", "bind_unbound"])
def test_window_join_replay(stream, policy, queries):
    """two windows over ONE store (the reference's windows share the R2R store, rsp_engine.rs:92-109) joined with static data
    (?sensor locatedIn ?room), through the single-thread rule, every emit compared with the restatement"""
    ctx, sctx = c.Context(0), c.Context(0)
    try:
        r2r = SimpleR2R(ctx)
        d = r2r.item.dictionary
        static_db = SparqlDatabase(sctx)
        static_db.dictionary = d  # one dictionary for the windows and the static store (rsp_engine.rs:238-243)
        for t in STATIC:
            static_db.add_triple_parts(*t)
        slots = SlotMap()
        plans = {"w1": plan_of(queries[0], d), "w2": plan_of(queries[1], d)}
        static_plan = TableScan((Variable("sensor"), Constant(d.encode("locatedIn")), Variable("room")))
        wj = WindowJoin(ctx, ["w1", "w2"], slots, stream, policy, static_db, static_plan)
        static_rows = [{"sensor": s, "room": o} for s, p, o in STATIC]
        r2s = Relation2Stream(stream)
        ref = J.SingleThreadEmitter(["w1", "w2"], policy, lambda last, ts: J.emit_results(last, static_rows, r2s, ["w1", "w2"]))
        kind = {"w1": queries[0], "w2": queries[1]}
        prev = {"w1": [], "w2": []}
        store = set()
        n_emits = 0
        for step in SCRIPT:
            if step is None:
                got, want = wj.process_single_thread(), ref.process()
                assert (got is None) == (want is None)
                if got is not None:
                    assert Counter(map(tuple, got)) == Counter(want)  # bags: the join's row order is unspecified
                    n_emits += 1
                continue
            w, ts, content = step
            for t in prev[w]:  # evict the window's previous firing, add the current one (rsp_engine.rs:94-104)
                r2r.remove(tuple(d.encode(x) for x in t))
                store.discard(t)
            for t in content:
                r2r.add(tuple(d.encode(x) for x in t))
                store.add(t)
            prev[w] = content
            r2r.materialize()
            rel = r2r.execute_query_rel(plans[w], slots)
            wj.put(w, rel, ts)
            ref.send(w, host_query(sorted(store), kind[w]), ts)
        assert n_emits == (4 if policy == "wait" else 5)
        # static triples are invisible to the window queries (rsp_engine_test.rs:533-580)
        r = r2r.execute_query_rel(TableScan((Variable("x"), Constant(d.encode("locatedIn")), Variable("y"))), slots)
        assert r.n_rows == 0
        wj.free()
    finally:
        ctx.close()
        sctx.close()


# ------------------------------------------------------------------ full size: cfg2's star split across two windows on ?e
def test_full_size_two_windows_and_static():
    ctx = c.Context(0)
    try:
        d = datagen.employee_dataset(166_667 * 10)
        ctx.store_load(d.s, d.p, d.o)
        ctx.dict_numeric_load(d.num_or0, d.is_num)
        ctx.build_index()
        js, pats, filt = datagen.employee_queries(d)["cfg2"]
        a = ctx.star_join(js, pats[:2], filt)  # e, t, s   (title, salary > 100000)
        b = ctx.star_join(js, pats[1:], filt)  # e, s, n   (salary > 100000, name)
        n_rich = int(np.count_nonzero(d.salary_of_employee > 100000))
        assert a.n_rows == b.n_rows == n_rich
        A, B = a.to_numpy([0, 1, 2]), b.to_numpy([0, 2, 3])
        titles = np.unique(A[:, 1])
        static = ctx.rel_from_host([1, 9], [titles, titles + 1_000_000])  # one static row per title: ?t -> ?x
        ab = ctx.natural_join(a, b)
        full = ctx.natural_join(ab, static)
        assert full.n_rows == n_rich  # every rich employee once: e is unique on both sides, one static row per title
        got = datagen.canonical_rows(full.to_numpy([0, 1, 2, 3, 9]))
        # numpy sort-merge join on e, then the title map
        A, B = A[np.argsort(A[:, 0], kind="stable")], B[np.argsort(B[:, 0], kind="stable")]
        assert np.array_equal(A[:, 0], B[:, 0]) and np.array_equal(A[:, 2], B[:, 1])  # same employees, same salaries
        want = datagen.canonical_rows(np.column_stack([A[:, 0], A[:, 1], A[:, 2], B[:, 2], A[:, 1] + 1_000_000]).astype(np.uint32))
        assert np.array_equal(got, want)
        # the unbound route on the same data: 1 % of b's salaries unbound -> the left value fills them, same answer
        Bm = b.to_numpy([0, 2, 3])
        rng = np.random.default_rng(5)
        Bm[rng.random(len(Bm)) < 0.01, 1] = NONE
        bu = ctx.rel_from_host([0, 2, 3], [Bm[:, 0].copy(), Bm[:, 1].copy(), Bm[:, 2].copy()])
        ctx.get_stats(reset=True)
        abu = ctx.natural_join(a, bu)
        assert ctx.get_stats()["other_launches"] >= 4
        assert np.array_equal(datagen.canonical_rows(abu.to_numpy([0, 1, 2, 3])), datagen.canonical_rows(ab.to_numpy([0, 1, 2, 3])))
        # a 1 % subject slice, row by row against the restatement (per employee: ?e is bound in every row of both windows, so the join
        # of the slice is the union of the per-employee joins)
        es = np.unique(A[:, 0])[::100]
        rows_of = lambda M, sl_: {int(r[0]): [{k: int(v) for k, v in zip(sl_, r) if v != NONE}] for r in M[np.isin(M[:, 0], es)].tolist()}
        a_rows, b_rows = rows_of(A, [0, 1, 2]), rows_of(Bm, [0, 2, 3])
        static_rows = [{1: int(t), 9: int(t) + 1_000_000} for t in titles]
        ref = [r for e in a_rows for r in J.natural_join(J.natural_join(a_rows[e], b_rows.get(e, [])), static_rows)]
        G = full.to_numpy([0, 1, 2, 3, 9])
        got_slice = Counter(map(tuple, G[np.isin(G[:, 0], es)].tolist()))
        assert got_slice == Counter(tuple(r[k] for k in (0, 1, 2, 3, 9)) for r in ref)
    finally:
        ctx.close()


# ------------------------------------------------------------------ the reference's multi-window tests, replayed emit by emit
def fixture_cases():
    from tests.rsp_multi_window_cases import CASES

    return CASES


def device_replay(case, stream):
    ctx, sctx = c.Context(0), c.Context(0)
    try:
        r2r = SimpleR2R(ctx)
        d = r2r.item.dictionary
        term = lambda q: Variable(q[1:]) if q.startswith("?") else Constant(d.encode(q))
        static_db = static_plan = None
        if case["static_pattern"]:
            static_db = SparqlDatabase(sctx)
            static_db.dictionary = d
            for t in case["static_triples"]:
                static_db.add_triple_parts(*t)
            static_plan = TableScan(tuple(term(q) for q in case["static_pattern"]))
        slots = SlotMap()
        order = [w["iri"] for w in case["windows"]]
        plans = {w["iri"]: TableScan(tuple(term(q) for q in w["pattern"])) for w in case["windows"]}
        policy = ("timeout", 0.1, "steal") if case["policy"] == "timeout" else case["policy"]
        wj = WindowJoin(ctx, order, slots, stream, policy, static_db, static_plan)
        prev = {w: [] for w in order}
        emits = []
        for step in case["steps"]:
            if step == "drain":
                got = wj.process_single_thread()
                if got is not None:
                    emits.append(got)
                continue
            w = step["window"]
            for t in prev[w]:
                r2r.remove(tuple(d.encode(x) for x in t))
            for t in step["content"]:
                r2r.add(tuple(d.encode(x) for x in t))
            prev[w] = step["content"]
            r2r.materialize()
            rel = r2r.execute_query_rel(plans[w], slots)
            if case["mode"] == "single_thread":
                wj.put(w, rel, step["ts"])
            else:
                emits.extend(wj.receive([(w, rel, step["ts"])], 0.0))
        wj.free()
        return emits
    finally:
        ctx.close()
        sctx.close()


@pytest.mark.parametrize("stream", ["RSTREAM", "ISTREAM", "DSTREAM"])
@pytest.mark.parametrize("case", fixture_cases(), ids=lambda c_: c_["name"])
def test_reference_multi_window_tests_replayed(case, stream):
    from tests.test_rsp_join_cpu import check_expect

    got = device_replay(case, stream)
    want = J.replay_case(case, stream, Relation2Stream)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert Counter(map(tuple, g)) == Counter(w), k
    if stream == "RSTREAM":
        check_expect(case, [tuple(r) for em in got for r in em])


def test_window_query_before_any_triple_arrived():
    """a window that fires before its store ever held a triple (a window of the second stream closing first, as in the single-thread
    multi-window replay) scans a context whose store was never loaded: 0 rows, not a fault"""
    ctx = c.Context(0)
    try:
        rel = ctx.scan([c.pattern(c.V(0), c.K(1), c.V(1))])[0]
        assert rel.info() == (0, [0, 1])
    finally:
        ctx.close()
