"""The backward-chaining restatements (tests/bc_reference.py) against the reference's own tests and against each other, and
engine.Reasoner.backward_chaining over a CPU stand-in of the device call. No GPU needed."""
import importlib.util
import json
import os
import random

import numpy as np
import pytest

import tests.bc_reference as B
from kolibrie_b200 import capi as c
from kolibrie_b200.engine import Constant, Reasoner, Rule, Variable
from tests.oracle_ctx import OracleCtx

HERE = os.path.dirname(os.path.abspath(__file__))
FIX = os.path.join(HERE, "golden", "backward")


def load_fixture():
    with open(os.path.join(FIX, "bc.json")) as f:
        return json.load(f)


def term(x, ids):
    return Variable(x[1:]) if x.startswith("?") else Constant(ids[x])


def build_case(cs):
    """(facts, rules, query, ids) of a fixture case, ids given in the reasoner's encode order"""
    ids = {}
    for f in cs["facts"]:
        for x in f:
            ids.setdefault(x, len(ids))
    for x in cs["encode"]:
        ids.setdefault(x, len(ids))
    facts = [tuple(ids[x] for x in f) for f in cs["facts"]]
    rules = [([tuple(term(x, ids) for x in p) for p in r[0]], [tuple(term(x, ids) for x in p) for p in r[1]]) for r in cs["rules"]]
    query = tuple(term(x, ids) for x in cs["query"])
    return facts, rules, query, ids


def check_assertions(cs, ids, got, query):
    names = B.query_vars(query)
    for var, val in cs["has"]:
        assert any(row[names.index(var)] == ids[val] for row in got), (cs["name"], var, val)
    if cs["empty"] is not None:
        assert (len(got) == 0) == cs["empty"], cs["name"]


def test_fixture_is_its_generators_output():
    spec = importlib.util.spec_from_file_location("bc_make_fixture", os.path.join(FIX, "make_fixture.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    assert json.loads(json.dumps(m.doc)) == load_fixture()


def test_fixture_cites_lines_that_exist():
    with open(os.path.join(HERE, "golden", "kolibrie_sources.tsv")) as f:
        n_lines = dict(line.rstrip("\n").split("\t") for line in f if "\t" in line)
    n = int(n_lines["datalog/tests/reasoning_tests.rs"])
    doc = load_fixture()
    assert len(doc["cases"]) == 10
    for cs in doc["cases"]:
        assert 22 < cs["line"] <= n and cs["name"].startswith("bc_")


@pytest.mark.parametrize("cs", load_fixture()["cases"], ids=lambda cs: cs["name"])
def test_restatements_pass_the_reference_tests(cs):
    facts, rules, query, ids = build_case(cs)
    sld = B.project_sld(B.sld(facts, rules, query, B.MAX_DEPTH), query)
    dev = B.device_answers(facts, rules, query)
    check_assertions(cs, ids, sld, query)
    check_assertions(cs, ids, dev, query)
    assert sld == dev


def random_program(rng, n_facts=8, n_ent=5, preds=(100, 101, 102)):
    ent = list(range(n_ent))
    facts = sorted({(rng.choice(ent), rng.choice(preds[:2]), rng.choice(ent)) for _ in range(n_facts)})
    vs = ["X", "Y", "Z", "W"]

    def tm(pool_vars):
        return Variable(rng.choice(pool_vars)) if rng.random() < 0.8 else Constant(rng.choice(ent))

    rules = []
    for _ in range(rng.randint(1, 3)):
        prem = []
        for _ in range(rng.randint(1, 3)):
            s, o = tm(vs), tm(vs)
            while isinstance(s, Variable) and isinstance(o, Variable) and s == o:
                o = tm(vs)
            prem.append((s, Constant(rng.choice(preds)), o))
        bound = sorted({t.name for p in prem for t in (p[0], p[2]) if isinstance(t, Variable)})
        heads = []
        for _ in range(rng.randint(1, 2)):
            hs = Variable(rng.choice(bound)) if bound and rng.random() < 0.85 else Constant(rng.choice(ent))
            ho = Variable(rng.choice(bound)) if bound and rng.random() < 0.85 else Constant(rng.choice(ent))
            heads.append((hs, Constant(rng.choice(preds)), ho))
        rules.append((prem, heads))
    return facts, rules


def random_query(rng, n_ent=5, preds=(100, 101, 102)):
    shape = rng.choice(["cvv", "vcv", "vvc", "cc", "vv", "rep", "vpred", "ground"])
    e = lambda: Constant(rng.randrange(n_ent))  # noqa: E731
    p = Constant(rng.choice(preds))
    return {"cvv": (e(), p, Variable("Q")), "vcv": (Variable("Q"), p, e()), "vvc": (Variable("Q"), p, Variable("R")),
            "cc": (e(), p, e()), "vv": (Variable("Q"), p, Variable("R")), "rep": (Variable("Q"), p, Variable("Q")),
            "vpred": (Variable("Q"), Variable("P"), Variable("R")) if rng.random() < 0.5 else (e(), Variable("P"), Variable("R")),
            "ground": (e(), p, e())}[shape]


def test_sld_equals_bounded_closure_on_seeded_programs():
    rng = random.Random(1234)
    checked = 0
    for _ in range(300):
        facts, rules = random_program(rng)
        q = random_query(rng)
        depth = rng.randint(0, 3)
        try:
            sld = B.project_sld(B.sld(facts, rules, q, depth, budget=20_000), q)
        except B.BudgetExceeded:
            continue
        assert sld == B.answers(B.bounded_closure(facts, rules, depth)[0], q), (facts, rules, q, depth)
        checked += 1
    assert checked >= 150


def test_bounded_closure_equals_demand_restricted_on_seeded_programs():
    rng = random.Random(99)
    restricted = 0
    for _ in range(400):
        facts, rules = random_program(rng, n_facts=12)
        q = random_query(rng)
        depth = rng.randint(0, 6)
        full, _ = B.bounded_closure(facts, rules, depth)
        part, _ = B.restricted_closure(facts, rules, q, depth)
        assert B.answers(full, q) == B.answers(part, q), (facts, rules, q, depth)
        restricted += len(part) < len(full)
    assert restricted > 50


def chain(n, parent=200):
    return [(i, parent, i + 1) for i in range(n)]


def test_the_depth_bound_binds_on_a_long_chain():
    parent, anc = Constant(200), Constant(201)
    X, Y, Z = Variable("X"), Variable("Y"), Variable("Z")
    rules = [([(X, parent, Y)], [(X, anc, Y)]), ([(X, parent, Y), (Y, anc, Z)], [(X, anc, Z)])]
    q = (Constant(0), anc, Variable("A"))
    facts = chain(14)
    got = B.device_answers(facts, rules, q, 10)
    assert got == {(k,) for k in range(1, 11)}
    assert B.project_sld(B.sld(facts, rules, q, 10, budget=2_000_000), q) == got
    assert B.device_answers(facts, rules, q, 14) == {(k,) for k in range(1, 15)}


def test_query_variable_named_like_a_renamed_rule_variable_is_a_documented_divergence():
    """quirk Q12: the reference renames rule variables to v0, v1, ... in the same namespace as the query's; a query variable `?v0`
    then aliases a rule variable. Here the rule's `?Y` becomes v0, the head (v1 child v0) unifies with (v0 child W) by chaining
    v1 -> v0 -> W, so the premise asks for (W parent W) and the reference finds nothing. The device answers (B, A)."""
    A, Bc, parent, child = 0, 1, 200, 202
    rules = [([(Variable("Y"), Constant(parent), Variable("X"))], [(Variable("X"), Constant(child), Variable("Y"))])]
    facts = [(A, parent, Bc)]
    q = (Variable("v0"), Constant(child), Variable("W"))
    assert B.project_sld(B.sld(facts, rules, q), q) == set()
    assert B.device_answers(facts, rules, q) == {(Bc, A)}
    q2 = (Variable("C"), Constant(child), Variable("W"))
    assert B.project_sld(B.sld(facts, rules, q2), q2) == {(Bc, A)}


class BcOracleCtx(OracleCtx):
    """OracleCtx plus kb_datalog_query restated by tests/bc_reference.py"""

    def datalog_query(self, rules, query, max_depth=c.BC_MAX_DEPTH):
        def t(k):
            return Variable(str(k.value)) if k.is_var else Constant(int(k.value))

        def pat(p):
            return (t(p.s), t(p.p), t(p.o))
        rs = [([pat(p) for p in r["premise"]], [pat(p) for p in r["conclusion"]]) for r in rules]
        q = pat(query)
        facts = [tuple(int(x) for x in row) for row in self._rows()]
        got = sorted(B.device_answers(facts, rs, q, max_depth))
        names = B.query_vars(q)
        slots = [int(n) for n in names]
        cols = [np.array([row[j] for row in got], np.uint32) for j in range(len(names))]
        if not names:
            return _Ground(len(got)), None
        return self.rel_from_host(slots, cols), None


class _Ground:
    """a relation without columns: what kb_datalog_query returns for a ground query"""

    def __init__(self, n):
        self.n = n

    def info(self):
        return self.n, []


@pytest.mark.parametrize("cs", load_fixture()["cases"], ids=lambda cs: cs["name"])
def test_reasoner_backward_chaining_over_the_stand_in(cs):
    r = Reasoner(ctx=BcOracleCtx())
    for f in cs["facts"]:
        r.add_abox_triple(*f)
    ids = {x: r.dictionary.encode(x) for x in cs["encode"]}
    for f in cs["facts"]:
        for x in f:
            ids[x] = r.dictionary.encode(x)

    def tm(x):
        return Variable(x[1:]) if x.startswith("?") else Constant(ids[x])
    for pr, cc in cs["rules"]:
        r.add_rule(Rule([tuple(tm(x) for x in p) for p in pr], [tuple(tm(x) for x in p) for p in cc]))
    res = r.backward_chaining(tuple(tm(x) for x in cs["query"]))
    for var, val in cs["has"]:
        assert any(b.get(var) == Constant(ids[val]) for b in res), (cs["name"], var, val)
    if cs["empty"] is not None:
        assert (len(res) == 0) == cs["empty"]
    names = B.query_vars(tuple(tm(x) for x in cs["query"]))
    assert all(set(b) == set(names) for b in res)
    assert len({tuple(sorted((k, v.id) for k, v in b.items())) for b in res}) == len(res)
