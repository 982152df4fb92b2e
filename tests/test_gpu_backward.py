"""GPU (-m gpu): kb_datalog_query (backward chaining on the device) against the restatements of tests/bc_reference.py — the reference's
bc_* tests, seeded programs against the bounded closure, the depth bound, refusals, and a store that stays exactly as it was."""
import random

import numpy as np
import pytest

import tests.bc_reference as B
from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200.engine import Constant, Reasoner, Rule, Variable
from tests import oracle_api as O
from tests.test_backward_cpu import build_case, check_assertions, load_fixture, random_program, random_query

pytestmark = pytest.mark.gpu


def to_kb(rules, query):
    """bc_reference rules / query -> kb_rule dicts and a kb_pattern (variables numbered per rule; the query's by first appearance)"""
    out = []
    for prem, conc in rules:
        slot = {}

        def t(x):
            return c.V(slot.setdefault(x.name, len(slot))) if isinstance(x, Variable) else c.K(x.id)
        out.append({"premise": [c.pattern(*map(t, p)) for p in prem], "conclusion": [c.pattern(*map(t, p)) for p in conc]})
    qs = {}

    def qt(x):
        return c.V(qs.setdefault(x.name, 100 + len(qs))) if isinstance(x, Variable) else c.K(x.id)
    return out, c.pattern(*map(qt, query))


def run(cx, facts, rules, query, depth=B.MAX_DEPTH):
    kr, kq = to_kb(rules, query)
    rel, st = cx.datalog_query(kr, kq, depth)
    n, slots = rel.info()
    names = B.query_vars(query)
    assert slots == [100 + i for i in range(len(names))]
    rows = rel.to_numpy() if slots else np.zeros((n, 0), np.uint32)
    got = [tuple(int(x) for x in r) for r in rows]
    assert len(got) == len(set(got)), "rows must be distinct"
    assert st.answers == n
    return set(got), st


def load(cx, facts, segments=1):
    a = np.array(facts, np.uint32).reshape(-1, 3)
    cx.store_load(a[:, 0], a[:, 1], a[:, 2])
    for k in range(1, segments):  # the same triples again: stored duplicates across segments
        cx.store_append(a[:, 0], a[:, 1], a[:, 2], k)


@pytest.mark.parametrize("cs", load_fixture()["cases"], ids=lambda cs: cs["name"])
def test_reference_bc_tests(ctx, cs):
    facts, rules, query, ids = build_case(cs)
    load(ctx, facts)
    got, _ = run(ctx, facts, rules, query)
    check_assertions(cs, ids, got, query)
    assert got == B.device_answers(facts, rules, query)


@pytest.mark.parametrize("cs", load_fixture()["cases"], ids=lambda cs: cs["name"])
def test_reasoner_backward_chaining(ctx, cs):
    r = Reasoner(ctx)
    for f in cs["facts"]:
        r.add_abox_triple(*f)
    ids = {x: r.dictionary.encode(x) for x in [y for f in cs["facts"] for y in f] + cs["encode"]}

    def tm(x):
        return Variable(x[1:]) if x.startswith("?") else Constant(ids[x])
    for pr, cc in cs["rules"]:
        r.add_rule(Rule([tuple(tm(x) for x in p) for p in pr], [tuple(tm(x) for x in p) for p in cc]))
    res = r.backward_chaining(tuple(tm(x) for x in cs["query"]))
    for var, val in cs["has"]:
        assert any(b.get(var) == Constant(ids[val]) for b in res), (cs["name"], var, val)
    if cs["empty"] is not None:
        assert (len(res) == 0) == cs["empty"]


def random_device_program(rng):
    facts, rules = random_program(rng, n_facts=rng.randint(4, 30), n_ent=6)
    for prem, heads in rules:  # up to 6 premises
        while len(prem) < rng.choice([1, 2, 3, 6]) and len(prem) < 6:
            prem.append((Variable(rng.choice("XYZW")), Constant(rng.choice((100, 101, 102))), Variable(rng.choice("XYZW"))))
            if prem[-1][0] == prem[-1][2]:
                prem.pop()
                break
    return facts, rules


@pytest.mark.parametrize("index", [False, True])
def test_seeded_programs_equal_the_bounded_closure(ctx, index):
    rng = random.Random(7 + index)
    for it in range(120):
        facts, rules = random_device_program(rng)
        q = random_query(rng, n_ent=6)
        depth = rng.randint(0, 10)
        load(ctx, facts, segments=1 + it % 3)
        if index:
            ctx.build_index()
        a = np.array(facts, np.uint32).reshape(-1, 3)
        want = B.answers(B.bounded_closure([tuple(map(int, r)) for r in a], rules, depth)[0], q)
        got, st = run(ctx, facts, rules, q, depth)
        assert got == want, (facts, rules, q, depth)
        assert st.rounds <= depth


def two_hop(n):
    """n (a p y_i) + n (y_i q z_i) and (X p Z), (Z s X) :- (X p Y), (Y q Z): the query (a p ?Z) restricts p to subject a, which keeps
    every p fact, and demands nothing of s"""
    a, P, Q, S = 0, 500, 501, 502
    facts = [(a, P, 10 + i) for i in range(n)] + [(10 + i, Q, 10 + n + i) for i in range(n)]
    X, Y, Z = Variable("X"), Variable("Y"), Variable("Z")
    rules = [([(X, Constant(P), Y), (Y, Constant(Q), Z)], [(X, Constant(P), Z), (Z, Constant(S), X)])]
    return facts, rules, (Constant(a), Constant(P), Variable("W"))


@pytest.mark.parametrize("n", [1000, 5000])
def test_restricted_relation_that_keeps_most_of_its_facts_grows(ctx, n):
    """a restricted head predicate that keeps a quarter of the store or more: the derived rows (n, far more than any allocation slack)
    must land in a relation that grew to hold them"""
    facts, rules, q = two_hop(n)
    load(ctx, facts)
    got, st = run(ctx, facts, rules, q)
    assert got == B.answers(B.bounded_closure(facts, rules, B.MAX_DEPTH)[0], q)
    assert len(got) == 2 * n and st.derived == n and st.restricted_predicates >= 1


def test_partitioned_dedup_route(monkeypatch):
    """the demand test on the radix-partitioned dedup, forced onto small inputs: the same query with the direct dedup and with the
    partitioned one. The undemanded head (s) is dropped on both routes, so both derive exactly the n demanded p facts; the partitioned
    route alone counts its candidates in rows_built, so the forced context counts more"""
    facts, rules, q = two_hop(4000)
    want = B.answers(B.bounded_closure(facts, rules, B.MAX_DEPTH)[0], q)
    built, derivations = {}, {}
    for part in ("0", "1"):
        monkeypatch.setenv("KOLIBRIE_DERIVE_PART", part)
        monkeypatch.setenv("KOLIBRIE_DERIVE_SLICE", "2048")
        monkeypatch.setenv("KOLIBRIE_DERIVE_MIN_ROWS", "16")
        cx = c.Context(0)
        try:
            load(cx, facts)
            cx.get_stats(reset=True)
            got, st = run(cx, facts, rules, q)
            built[part] = cx.get_stats()["rows_built"]
            derivations[part] = st.derivations
            assert got == want
            assert st.derived == 4000
        finally:
            cx.close()
    assert derivations["0"] == derivations["1"]
    assert built["1"] >= built["0"] + 2 * 4000, built


def anc_rules(doubling):
    parent, anc = Constant(200), Constant(201)
    X, Y, Z = Variable("X"), Variable("Y"), Variable("Z")
    step = [(X, anc, Y), (Y, anc, Z)] if doubling else [(X, parent, Y), (Y, anc, Z)]
    return [([(X, parent, Y)], [(X, anc, Y)]), (step, [(X, anc, Z)])]


@pytest.mark.parametrize("doubling", [False, True])
@pytest.mark.parametrize("length", [9, 10, 11, 12])
def test_the_depth_bound(ctx, length, doubling):
    facts = [(i, 200, i + 1) for i in range(length)]
    rules = anc_rules(doubling)
    load(ctx, facts)
    for depth in (1, 3, 10):
        q = (Constant(0), Constant(201), Variable("A"))
        got, st = run(ctx, facts, rules, q, depth)
        assert got == B.device_answers(facts, rules, q, depth)
    q = (Constant(0), Constant(201), Variable("A"))
    got, _ = run(ctx, facts, rules, q, 10)
    if not doubling:
        assert got == {(k,) for k in range(1, min(length, 10) + 1)}


def test_ground_query_stops_early(ctx):
    facts = [(i, 200, i + 1) for i in range(30)]
    rules = anc_rules(False)
    load(ctx, facts)
    got, st = run(ctx, facts, rules, (Constant(0), Constant(201), Constant(3)), 10)
    assert got == {()} and st.stopped_early and st.rounds == 3
    got, st = run(ctx, facts, rules, (Constant(0), Constant(201), Constant(25)), 10)
    assert got == set() and not st.stopped_early and st.rounds == 10
    got, st = run(ctx, facts, rules, (Constant(0), Constant(200), Constant(1)), 10)  # no rule derives `parent`: none runs
    assert got == {()} and st.relevant_rules == 0 and st.derivations == 0


def test_irrelevant_rule_runs_no_derivation(ctx):
    """a rule whose head no demand pattern reaches does not run, however large its closure"""
    n = 3000
    facts = [(i, 300, i + 1) for i in range(n)] + [(0, 200, 1)]
    T, R = Constant(300), Constant(301)
    X, Y, Z = Variable("X"), Variable("Y"), Variable("Z")
    rules = [([(X, T, Y)], [(X, R, Y)]), ([(X, R, Y), (Y, R, Z)], [(X, R, Z)]), ([(X, Constant(200), Y)], [(X, Constant(201), Y)])]
    load(ctx, facts)
    got, st = run(ctx, facts, rules, (Variable("Q"), Constant(201), Variable("W")))
    assert got == {(0, 1)}
    assert st.relevant_rules == 1 and st.derivations == 1


def test_refusals_change_nothing(ctx):
    facts = [(0, 200, 1), (1, 200, 2)]
    load(ctx, facts)
    before = ctx.store_download()
    v = ctx.store_size()
    X, Y = c.V(0), c.V(1)
    ok_rule = {"premise": [c.pattern(X, c.K(200), Y)], "conclusion": [c.pattern(X, c.K(201), Y)]}
    q = c.pattern(c.K(0), c.K(201), c.V(5))
    cases = [
        ([ok_rule], q, 65, c.KB_E_LIMIT),
        ([{"premise": [], "conclusion": [c.pattern(c.K(0), c.K(201), c.K(1))]}], q, 10, c.KB_E_UNSUPPORTED),
        ([{"premise": [c.pattern(X, c.V(2), Y)], "conclusion": [c.pattern(X, c.K(201), Y)]}], q, 10, c.KB_E_UNSUPPORTED),
        ([{"premise": [c.pattern(X, c.K(200), Y)], "conclusion": [c.pattern(X, c.K(201), c.V(7))]}], q, 10, c.KB_E_UNSUPPORTED),
        ([{"premise": [c.pattern(X, c.K(200), Y)], "conclusion": [c.pattern(X, c.V(1), Y)]}], q, 10, c.KB_E_UNSUPPORTED),
        ([{"premise": [c.pattern(X, c.K(200), X)], "conclusion": [c.pattern(X, c.K(201), X)]}], q, 10, c.KB_E_UNSUPPORTED),
        ([ok_rule], c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.K(201), c.V(5)), 10, c.KB_E_UNSUPPORTED),
        ([{"premise": [c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.K(200), Y)], "conclusion": [c.pattern(Y, c.K(201), Y)]}], q, 10, c.KB_E_UNSUPPORTED),
    ]
    for rules, qq, depth, code in cases:
        with pytest.raises(c.KolibrieError) as e:
            ctx.datalog_query(rules, qq, depth)
        assert e.value.status == code, (rules, depth)
    assert ctx.store_size() == v
    assert all(np.array_equal(a, b) for a, b in zip(ctx.store_download(), before))
    rel, st = ctx.datalog_query([ok_rule], q, 64)
    assert rel.to_numpy().tolist() == [[1]]


def test_the_store_is_left_as_it_was(ctx):
    """size and contents, a plan prepared before the query, and kb_datalog_maintain's precondition all survive a query"""
    d = datagen.employee_dataset(5000)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    plan = ctx.prepare_star_join(js, pats, filt, ring=2)
    want = plan.collect_rows(plan.submit()).to_numpy(sorted(pats_slots(pats)))
    size, before = ctx.store_size(), ctx.store_download()
    title = int(pats[0].p.value)
    rule = {"premise": [c.pattern(c.V(0), c.K(title), c.V(1)), c.pattern(c.V(0), c.K(title), c.V(2))],
            "conclusion": [c.pattern(c.V(1), c.K(0xABCDE), c.V(2))]}
    rel, st = ctx.datalog_query([rule], c.pattern(c.V(7), c.K(0xABCDE), c.V(8)))
    assert st.answers > 0 and st.derived > 0
    assert ctx.store_size() == size
    assert all(np.array_equal(a, b) for a, b in zip(ctx.store_download(), before))
    got = plan.collect_rows(plan.submit()).to_numpy(sorted(pats_slots(pats)))
    assert np.array_equal(datagen.canonical_rows(got), datagen.canonical_rows(want))
    plan.free()
    # a closed store stays closed: kb_datalog_maintain accepts it after a query
    t = datagen.taxonomy_dataset(fanout=3, depth=4, n_instances=2000)
    rules = datagen.taxonomy_rules(t)
    ctx.store_load(t.s, t.p, t.o)
    ctx.datalog_fixpoint(rules)
    ctx.datalog_query(rules, c.pattern(c.K(int(t.s[-1])), c.K(t.ids["rdf:type"]), c.V(9)))
    add = np.array([[int(t.s[-1]) + 1, t.ids["rdf:type"], 3]], np.uint32)
    gone, new, mst = ctx.datalog_maintain(rules, [], add, 77)
    assert new.n_rows > 0


def pats_slots(pats):
    return {int(t.value) for p in pats for t in (p.s, p.p, p.o) if t.is_var}


def test_variable_predicate_query_over_duplicate_segments(ctx):
    facts = [(0, 200, 1), (1, 200, 2), (2, 300, 0)]
    rules = anc_rules(True)
    load(ctx, facts, segments=3)
    for q in [(Variable("S"), Variable("P"), Variable("O")), (Constant(0), Variable("P"), Variable("O")), (Variable("S"), Variable("P"), Variable("S"))]:
        got, _ = run(ctx, facts, rules, q)
        assert got == B.device_answers(facts, rules, q), q


def cfg4_query_vs_fixpoint(n_instances, js):
    t = datagen.taxonomy_dataset(n_instances=n_instances)
    rules = datagen.taxonomy_rules(t)
    ty = t.ids["rdf:type"]
    a = c.Context(0)
    b = c.Context(0)
    try:
        a.store_load(t.s, t.p, t.o)
        b.store_load(t.s, t.p, t.o)
        b.datalog_fixpoint(rules)
        X0 = 2 + t.n_classes
        for j in js:
            x = X0 + j
            rel, st = a.datalog_query(rules, c.pattern(c.K(x), c.K(ty), c.V(9)))
            got = sorted(rel.to_numpy().ravel().tolist())
            want = sorted(set(b.scan([c.pattern(c.K(x), c.K(ty), c.V(9))])[0].to_numpy().ravel().tolist()))
            assert got == want and len(got) >= 1, j
            assert st.restricted_predicates >= 1 and st.base_facts < len(t.s)
        return t
    finally:
        a.close()
        b.close()


def test_cfg4_small_scale():
    cfg4_query_vs_fixpoint(488_889, [0, 1, 17, 488_888])


def test_cfg4_full_size():
    cfg4_query_vs_fixpoint(48_888_890, list(np.random.default_rng(5).integers(0, 48_888_890, 4)))


def test_cpp_host_mirror(tmp_path):
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "kolibrie_b200")
    exe = os.path.join(str(tmp_path), "bc_tests")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(root, "tests", "cpp", "bc_tests.cpp"), f"-L{libdir}",
           "-lkolibrie_b200", f"-Wl,-rpath,{libdir}"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
