"""GPU (-m gpu): kb_datalog_query_repairs against the IAR restatement of tests/repairs_reference.py — the reference's examples, seeded
programs with and without the index, duplicate segments, an inferred segment, evicted and deleted facts, ids at the edges of the u32
domain, both minimality routes, the refusals, the mirrors, and the taxonomy shape of the benchmark. After every call the store is
checked to be as it was."""
import os
import random
import subprocess

import numpy as np
import pytest

import tests.repairs_reference as R
from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200.engine import Constant, Reasoner, Rule, Variable
from tests import id_domain_cases as D
from tests.test_repairs_cpu import build_case, load_fixture, random_program, random_query

pytestmark = pytest.mark.gpu


def to_kb(constraints, query):
    """restatement constraints / query -> kb_rule dicts and a kb_pattern (variables numbered per constraint; the query's from 100)"""
    out = []
    for prem in constraints:
        slot = {}
        t = lambda x: c.V(slot.setdefault(x, len(slot))) if R.is_var(x) else c.K(x)  # noqa: E731
        out.append({"premise": [c.pattern(*map(t, p)) for p in prem]})
    qs = {}
    qt = lambda x: c.V(qs.setdefault(x, 100 + len(qs))) if R.is_var(x) else c.K(x)  # noqa: E731
    return out, c.pattern(*map(qt, query))


def snapshot(cx):
    return cx.store_size(), [a.copy() for a in cx.store_download()]


def assert_untouched(cx, snap):
    size, cols = snap
    assert cx.store_size() == size
    assert all(np.array_equal(a, b) for a, b in zip(cx.store_download(), cols))


def run(cx, constraints, query):
    snap = snapshot(cx)
    kc, kq = to_kb(constraints, query)
    rel, st = cx.datalog_query_repairs(kc, kq)
    n, slots = rel.info()
    names = R.query_vars(query)
    assert slots == [100 + i for i in range(len(names))]
    rows = rel.to_numpy() if slots else np.zeros((n, 0), np.uint32)
    got = [tuple(int(x) for x in r) for r in rows]
    assert len(got) == len(set(got)), "rows must be distinct"
    assert st.answers == n
    assert_untouched(cx, snap)
    return set(got), st


def load(cx, facts, segments=1):
    a = np.array(facts, np.uint32).reshape(-1, 3)
    cx.store_load(a[:, 0], a[:, 1], a[:, 2])
    for k in range(1, segments):  # the same triples again: stored duplicates across segments
        cx.store_append(a[:, 0], a[:, 1], a[:, 2], k)


def check(cx, facts, constraints, query):
    got, st = run(cx, constraints, query)
    assert got == R.iar(facts, constraints, query), (facts, constraints, query)
    s = R.stats(facts, constraints)
    assert {k: getattr(st, k) for k in s} == s
    return st


@pytest.mark.parametrize("cs", load_fixture()["cases"], ids=lambda cs: cs["name"])
def test_reference_examples(ctx, cs):
    facts, constraints, query, ids = build_case(cs)
    load(ctx, facts)
    check(ctx, facts, constraints, query)


@pytest.mark.parametrize("index", [False, True], ids=["scan", "index"])
@pytest.mark.parametrize("segments", [1, 3])
def test_seeded_programs(ctx, index, segments):
    rng = random.Random(7 + segments)
    for _ in range(25):
        facts, constraints = random_program(rng)
        load(ctx, facts, segments)
        ctx.set_use_index(index)
        if index:
            ctx.build_index()
        for _ in range(3):
            check(ctx, facts, constraints, random_query(rng, facts))
    ctx.set_use_index(True)


def test_both_minimality_routes(ctx):
    x, y, z, w = (1, 10, 2), (1, 11, 3), (2, 12, 3), (4, 10, 4)
    big = [("?A", 10, "?B"), ("?A", 11, "?C"), ("?D", 12, "?C")]
    load(ctx, [x, y, z, w])
    q = ("?S", "?P", "?O")
    st = check(ctx, [x, y, z, w], [big], q)  # one size: every conflict is minimal, no probe
    assert st.subsets_probed == 0 and st.minimal_conflicts == 1 and st.conflicted_facts == 3
    st = check(ctx, [x, y, z, w], [big, [("?A", 11, 3)]], q)  # a size-1 conflict {y} makes {x, y, z} non-minimal
    assert st.subsets_probed == 1 and st.minimal_conflicts == 1 and st.conflicted_facts == 1
    got, _ = run(ctx, [big, [("?A", 11, 3)]], q)
    assert got == {x, z, w}


def test_premises_binding_one_fact_and_constant_only_premises(ctx):
    facts = [(1, 10, 2), (1, 11, 2), (3, 10, 3)]
    load(ctx, facts)
    for cons in ([[("?A", 10, "?B"), ("?A", "?P", 2)]], [[(1, 10, 2), (1, 11, 2)]], [[(1, 10, 2)], [(3, 10, 3), (1, 10, 2)]],
                 [[("?A", 10, "?A")]], [[("?A", "?P", "?B"), ("?B", "?P", "?A")]]):
        for q in [("?S", "?P", "?O"), ("?S", 10, "?S"), (1, "?P", 2)]:
            check(ctx, facts, cons, q)


def test_no_constraints_and_constraints_that_never_match(ctx):
    facts = [(1, 10, 2), (1, 11, 2), (3, 10, 3)]
    load(ctx, facts, segments=2)
    q = ("?S", 10, "?O")
    want = {tuple(int(v) for v in r) for r in ctx.scan([c.pattern(c.V(100), c.K(10), c.V(101))])[0].to_numpy()}
    for cons in ([], [[]], [[("?A", 99, "?B")]], [[("?A", 10, "?B"), ("?B", 11, "?C")]]):
        got, st = run(ctx, cons, q)
        assert got == want == R.iar(facts, cons, q)
        assert st.minimal_conflicts == 0 and st.conflicted_facts == 0


def test_ground_queries(ctx):
    facts = [(1, 10, 2), (1, 11, 2), (3, 10, 3)]
    cons = [[("?A", 10, "?B"), ("?A", 11, "?B")]]
    load(ctx, facts)
    for q in [(1, 10, 2), (3, 10, 3), (9, 10, 9)]:
        got, _ = run(ctx, cons, q)
        assert got == R.iar(facts, cons, q) == ({()} if q == (3, 10, 3) else set())


def test_after_fixpoint_the_inferred_segment_takes_part(ctx):
    t = datagen.taxonomy_dataset(fanout=3, depth=3, n_instances=200)
    ctx.store_load(t.s, t.p, t.o)
    rel, _ = ctx.datalog_fixpoint(datagen.taxonomy_rules(t))
    facts = [tuple(int(v) for v in r) for r in np.stack(ctx.store_download(), 1)]
    ty = t.ids["rdf:type"]
    cons = [[("?X", ty, 3), ("?X", ty, 4)], [("?X", ty, 5), ("?X", ty, 8)]]  # level-1 classes 3, 4, 5 are only inferred types
    for q in [("?X", ty, "?C"), ("?X", ty, 3), (int(t.s[-1]), ty, "?C")]:
        check(ctx, facts, cons, q)


def test_after_evict_and_delete(ctx):
    a = [(1, 10, 2), (1, 11, 2), (3, 10, 3)]
    b = [(1, 12, 2), (3, 11, 3)]
    cons = [[("?A", 10, "?B"), ("?A", "?P", "?B"), ("?A", 11, "?B")], [("?A", 12, "?B")]]
    load(ctx, a)
    x = np.array(b, np.uint32)
    ctx.store_append(x[:, 0], x[:, 1], x[:, 2], 5)
    q = ("?S", "?P", "?O")
    check(ctx, a + b, cons, q)
    ctx.store_evict(5)
    check(ctx, a, cons, q)
    ctx.store_delete(np.array([1], np.uint32), np.array([11], np.uint32), np.array([2], np.uint32))
    check(ctx, [a[0], a[2]], cons, q)


@pytest.mark.parametrize("family", D.FAMILIES)
def test_ids_at_the_edges_of_the_u32_domain(ctx, family):
    rng = random.Random(31)
    for k in range(8):
        facts, constraints = random_program(rng)
        qs = [random_query(rng, facts) for _ in range(2)]
        dom = {v for f in facts for v in f} | {t for cs in constraints for p in cs for t in p if not R.is_var(t)}
        dom |= {t for q in qs for t in q if not R.is_var(t)}
        m = D.Remap(family, sorted(dom), seed=k)
        f = lambda v: v if R.is_var(v) else int(m(np.array([v], np.uint32))[0])  # noqa: E731
        facts = [tuple(map(f, t)) for t in facts]
        constraints = [[tuple(map(f, p)) for p in cs] for cs in constraints]
        load(ctx, facts)
        for q in qs:
            check(ctx, facts, constraints, tuple(map(f, q)))


def test_refusals_change_nothing(ctx):
    facts = [(1, 10, 2), (1, 11, 2)]
    load(ctx, facts)
    snap = snapshot(ctx)
    X, Y = c.V(0), c.V(1)
    ok = {"premise": [c.pattern(X, c.K(10), Y)]}
    q = c.pattern(c.V(100), c.K(10), c.V(101))
    Q = c.KbTerm(c.KB_TERM_QUOTED, 0)
    cases = [
        ([ok], c.pattern(Q, c.K(10), c.V(101)), c.KB_E_UNSUPPORTED),
        ([{"premise": [c.pattern(X, c.K(10), Q)]}], q, c.KB_E_UNSUPPORTED),
        ([ok], c.pattern(c.V(100), c.K(0xFFFFFFFF), c.V(101)), c.KB_E_INVALID),
        ([{"premise": [c.pattern(X, c.K(0xFFFFFFFF), Y)]}], q, c.KB_E_INVALID),
        ([{"premise": [c.pattern(X, c.K(10), Y)] * 7}], q, c.KB_E_LIMIT),
        ([{"premise": [c.pattern(c.V(3 * i), c.V(3 * i + 1), c.V(3 * i + 2)) for i in range(6)]}], q, c.KB_E_LIMIT),  # 18 variables
    ]
    for cons, qq, code in cases:
        with pytest.raises(c.KolibrieError) as e:
            ctx.datalog_query_repairs(cons, qq)
        assert e.value.status == code, cons
        assert_untouched(ctx, snap)
    ctx.set_sharding(0, 2)
    with pytest.raises(c.KolibrieError) as e:
        ctx.datalog_query_repairs([ok], q)
    assert e.value.status == c.KB_E_UNSUPPORTED
    ctx.set_sharding(0, 1)
    rel, st = ctx.datalog_query_repairs([ok], c.pattern(c.V(100), c.V(101), c.K(2)))  # (1 10 2) is a conflict of its own
    assert st.answers == 1 and st.conflicted_facts == 1


def test_the_store_is_left_as_it_was(ctx):
    """size and contents, the index, a plan prepared before the query, and kb_datalog_maintain's precondition all survive a query"""
    d = datagen.employee_dataset(5000)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    plan = ctx.prepare_star_join(js, pats, filt, ring=2)
    want = plan.collect_rows(plan.submit()).to_numpy(sorted(pats_slots(pats)))
    snap = snapshot(ctx)
    title = int(pats[0].p.value)
    cons = [{"premise": [c.pattern(c.V(0), c.K(title), c.V(1)), c.pattern(c.V(0), c.K(title), c.V(2))]}]  # every title fact conflicts
    rel, st = ctx.datalog_query_repairs(cons, c.pattern(c.V(7), c.K(title), c.V(8)))
    assert st.conflicts > 0 and st.answers == 0
    assert_untouched(ctx, snap)
    n0 = ctx.get_stats()["index_joins"]
    got = plan.collect_rows(plan.submit()).to_numpy(sorted(pats_slots(pats)))
    assert np.array_equal(datagen.canonical_rows(got), datagen.canonical_rows(want))
    ctx.star_join(js, pats, filt)
    assert ctx.get_stats()["index_joins"] > n0, "the index is still valid"
    plan.free()
    t = datagen.taxonomy_dataset(fanout=3, depth=4, n_instances=2000)
    rules = datagen.taxonomy_rules(t)
    ctx.store_load(t.s, t.p, t.o)
    ctx.datalog_fixpoint(rules)
    ty = t.ids["rdf:type"]
    ctx.datalog_query_repairs([{"premise": [c.pattern(c.V(0), c.K(ty), c.K(3)), c.pattern(c.V(0), c.K(ty), c.K(4))]}],
                              c.pattern(c.V(5), c.K(ty), c.V(6)))
    add = np.array([[int(t.s[-1]) + 1, ty, 3]], np.uint32)
    gone, new, mst = ctx.datalog_maintain(rules, [], add, 77)
    assert new.n_rows > 0, "a closed store stays closed"


def pats_slots(pats):
    return {int(t.value) for p in pats for t in (p.s, p.p, p.o) if t.is_var}


def test_reasoner_mirror(ctx):
    for cs in load_fixture()["cases"]:
        r = Reasoner(ctx)
        for f in cs["facts"]:
            r.add_abox_triple(*f)
        enc = r.dictionary.encode
        tm = lambda x: Variable(x[1:]) if x.startswith("?") else Constant(enc(x))  # noqa: E731
        for prem in cs["constraints"]:
            r.add_constraint(Rule(premise=[tuple(map(tm, p)) for p in prem], filters=[], conclusion=[(Constant(0), Constant(0), Constant(0))]))
        assert r.query_with_repairs(tuple(map(tm, cs["query"]))) == []
        r.add_abox_triple("mary", "isA", "student")
        got = r.query_with_repairs((Variable("X"), Constant(enc("isA")), Variable("Y")))
        assert got == [{"X": enc("mary"), "Y": enc("student")}]
        assert r.last_stats.minimal_conflicts == 1


def test_cpp_host_mirror(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "kolibrie_b200")
    exe = os.path.join(str(tmp_path), "repair_tests")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(root, "tests", "cpp", "repair_tests.cpp"), f"-L{libdir}",
           "-lkolibrie_b200", f"-Wl,-rpath,{libdir}"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout


# ---- the benchmark's shape: taxonomy_dataset + a second leaf type for 1 % of the instances, closed, + disjointWith between level-1 classes
FANOUT, DEPTH = 10, 6


def level1(cls):
    """the level-1 ancestor of each class index (0 for the root)"""
    a = np.asarray(cls, np.int64).copy()
    while (a > FANOUT).any():
        a = np.where(a > FANOUT, (a - 1) // FANOUT, a)
    return a


def ancestors(cls):
    out = [cls]
    while cls > 0:
        cls = (cls - 1) // FANOUT
        out.append(cls)
    return out


def taxonomy_iar_reference(t, extra, k):
    """numpy IAR for (i) (?x type ?a), (?x type ?b), (?a disjointWith ?b) and (ii) (i) plus (?x type C_k): per instance its base
    classes (one or two), their level-1 ancestors, and the counts kb_repair_stats reports"""
    X0 = 2 + t.n_classes
    n = t.n_instances
    base1 = t.o[t.p == t.ids["rdf:type"]].astype(np.int64) - 2
    l1a = level1(base1)
    l1b = l1a.copy()
    s2, o2 = extra[0][extra[1] == t.ids["rdf:type"]].astype(np.int64) - X0, extra[2][extra[1] == t.ids["rdf:type"]].astype(np.int64) - 2
    l1b[s2] = level1(o2)
    second = {int(a): int(b) for a, b in zip(s2, o2)}
    bad = (l1a != l1b) & (l1a > 0) & (l1b > 0)
    kk = k - 2  # class index of C_k
    under_k = (l1a == kk) | (l1b == kk)
    pairs_i = {frozenset((int(a), int(b))) for a, b in zip(l1a[bad], l1b[bad])}  # each gives (a dw b) and (b dw a)
    rest = bad & ~under_k
    pairs_ii = {frozenset((int(a), int(b))) for a, b in zip(l1a[rest], l1b[rest])}
    nb, nk, nr = int(bad.sum()), int(under_k.sum()), int(rest.sum())
    return {
        "i": {"conflicts": 2 * nb, "minimal_conflicts": 2 * nb, "conflicted_facts": 2 * nb + 2 * len(pairs_i), "subsets_probed": 0},
        "ii": {"conflicts": 2 * nb + nk, "minimal_conflicts": 2 * nr + nk, "conflicted_facts": nk + 2 * nr + 2 * len(pairs_ii), "subsets_probed": 1},
        "bad": bad, "base1": base1, "second": second, "l1a": l1a, "l1b": l1b, "under_k": under_k,
    }


def types_of(ref, j):
    cls = set(ancestors(int(ref["base1"][j])))
    if j in ref["second"]:
        cls |= set(ancestors(ref["second"][j]))
    return {c_ + 2 for c_ in cls}


def cfg4_repairs(n_instances, n_queries):
    t = datagen.taxonomy_dataset(n_instances=n_instances)
    extra, dw, lv1 = datagen.taxonomy_conflicts(t)
    ty = t.ids["rdf:type"]
    k = int(lv1[3])
    ref = taxonomy_iar_reference(t, extra, k)
    cx = c.Context(0)
    try:
        cx.store_load(np.concatenate([t.s, extra[0]]), np.concatenate([t.p, extra[1]]), np.concatenate([t.o, extra[2]]))
        cx.datalog_fixpoint(datagen.taxonomy_rules(t))
        cx.build_index()
        body = {"premise": [c.pattern(c.V(0), c.K(ty), c.V(1)), c.pattern(c.V(0), c.K(ty), c.V(2)), c.pattern(c.V(1), c.K(dw), c.V(2))]}
        only_k = {"premise": [c.pattern(c.V(0), c.K(ty), c.K(k))]}
        X0 = 2 + t.n_classes
        bad = np.flatnonzero(ref["bad"])
        free = np.flatnonzero(~ref["bad"])
        js = list(bad[:n_queries]) + list(free[:n_queries])
        for run_name, cons in (("i", [body]), ("ii", [body, only_k])):
            size = cx.store_size()
            for j in js:
                rel, st = cx.datalog_query_repairs(cons, c.pattern(c.K(X0 + int(j)), c.K(ty), c.V(9)))
                got = set(rel.to_numpy().ravel().tolist())
                want = types_of(ref, int(j))
                if ref["bad"][j] and (run_name == "i" or not ref["under_k"][j]):
                    want -= {int(ref["l1a"][j]) + 2, int(ref["l1b"][j]) + 2}
                if run_name == "ii" and ref["under_k"][j]:
                    want -= {k}
                assert got == want, (run_name, j)
                assert {n: getattr(st, n) for n in ref[run_name] if n in ("conflicts", "minimal_conflicts", "conflicted_facts", "subsets_probed")} == ref[run_name]
            rel, st = cx.datalog_query_repairs(cons, c.pattern(c.V(9), c.K(ty), c.K(k)))
            n_k = int(ref["under_k"].sum())
            assert st.answers == (0 if run_name == "ii" else n_k - int((ref["bad"] & ((ref["l1a"] == k - 2) | (ref["l1b"] == k - 2))).sum()))
            assert cx.store_size() == size
    finally:
        cx.close()


def test_cfg4_small_scale():
    cfg4_repairs(488_889, 3)


def test_cfg4_full_size():
    cfg4_repairs(48_888_890, 2)
