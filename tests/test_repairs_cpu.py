"""The restatements of query_with_repairs (tests/repairs_reference.py) against each other, against the reference's examples and against
the documented divergence Q13. No GPU needed."""
import importlib.util
import json
import os
import random

import pytest

import tests.repairs_reference as R

HERE = os.path.dirname(os.path.abspath(__file__))
FIX = os.path.join(HERE, "golden", "repairs")

S, P, O = [1, 2, 3, 4], [10, 11, 12], [1, 2, 3, 20]  # subjects and objects share ids, so a variable can join them
VARS = ["?X", "?Y", "?Z", "?W"]


def load_fixture():
    with open(os.path.join(FIX, "repairs.json")) as f:
        return json.load(f)


def build_case(cs):
    """(facts, constraints, query, ids) of a fixture case, ids in the reasoner's encode order"""
    ids = {}
    for f in cs["facts"]:
        for x in f:
            ids.setdefault(x, len(ids))
    t = lambda x: x if x.startswith("?") else ids.setdefault(x, len(ids))  # noqa: E731
    facts = [tuple(ids[x] for x in f) for f in cs["facts"]]
    constraints = [[tuple(t(x) for x in p) for p in c] for c in cs["constraints"]]
    return facts, constraints, tuple(t(x) for x in cs["query"]), ids


def random_facts(rng, n):
    facts = set()
    while len(facts) < n:
        facts.add((rng.choice(S), rng.choice(P), rng.choice(O)))
    return sorted(facts)


def random_premise(rng, facts):
    """a premise with constants, repeated variables, a variable predicate or none at all; often a fact with some terms replaced"""
    base = rng.choice(facts) if rng.random() < 0.7 else (rng.choice(S), rng.choice(P), rng.choice(O))
    out = []
    for k, v in enumerate(base):
        r = rng.random()
        if k == 1:
            out.append(rng.choice(VARS) if r < 0.15 else v)
        else:
            out.append(rng.choice(VARS[:3]) if r < 0.6 else v)
    return tuple(out)


def random_program(rng, max_facts=12):
    facts = random_facts(rng, rng.randint(1, max_facts))
    constraints = [[random_premise(rng, facts) for _ in range(rng.randint(1, 4))] for _ in range(rng.randint(1, 4))]
    if rng.random() < 0.1:
        constraints.append([])  # never fires
    return facts, constraints


def random_query(rng, facts):
    f = rng.choice(facts)
    q = [rng.choice(["?A", "?B"]) if rng.random() < 0.5 else v for v in f]
    if rng.random() < 0.2:
        q = ["?A", "?B", "?C"]
    return tuple(q)


def test_fixture_is_its_generators_output():
    spec = importlib.util.spec_from_file_location("repairs_make_fixture", os.path.join(FIX, "make_fixture.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    assert json.loads(json.dumps(m.doc)) == load_fixture()


@pytest.mark.parametrize("cs", load_fixture()["cases"], ids=lambda cs: cs["name"])
def test_fixture_cases(cs):
    facts, constraints, query, ids = build_case(cs)
    want = R.iar(facts, constraints, query)
    assert want == R.brute_force(facts, constraints, query)
    # john is both professor and student: both facts are in the one minimal conflict, so no isA fact is certain
    assert want == set()
    assert R.conflicted_facts(facts, constraints) == {(ids["john"], ids["isA"], ids["professor"]), (ids["john"], ids["isA"], ids["student"])}
    for seed in range(4):
        order = list(facts)
        random.Random(seed).shuffle(order)
        got, kept = R.transcribe(facts, constraints, query, order)
        assert got <= want


@pytest.mark.parametrize("seed", range(60))
def test_polynomial_rule_equals_brute_force(seed):
    rng = random.Random(seed)
    facts, constraints = random_program(rng)
    for _ in range(3):
        q = random_query(rng, facts)
        assert R.iar(facts, constraints, q) == R.brute_force(facts, constraints, q), (facts, constraints, q)


@pytest.mark.parametrize("seed", range(25))
def test_transcription_keeps_every_maximal_repair_and_answers_a_subset(seed):
    rng = random.Random(1000 + seed)
    facts, constraints = random_program(rng, max_facts=7)
    maximal = set(R.maximal_repairs(facts, constraints))
    for k in range(3):
        order = list(facts)
        rng.shuffle(order)
        q = random_query(rng, facts)
        got, kept = R.transcribe(facts, constraints, q, order)
        assert maximal <= set(kept), "compute_repairs must reach every maximal repair"
        assert got <= R.iar(facts, constraints, q)


@pytest.mark.parametrize("seed", range(20))
def test_transcription_equals_iar_on_a_consistent_store(seed):
    rng = random.Random(2000 + seed)
    facts, constraints = random_program(rng, max_facts=8)
    facts = sorted(set(facts) - R.conflicted_facts(facts, constraints))  # no minimal conflict left: consistent
    if not facts:
        return
    assert not R.violates(constraints, facts)
    order = list(facts)
    rng.shuffle(order)
    q = random_query(rng, facts)
    got, kept = R.transcribe(facts, constraints, q, order)
    assert kept == [frozenset(facts)]
    assert got == R.iar(facts, constraints, q) == R.answer(q, facts)


def test_q13_a_non_maximal_kept_set_drops_a_free_fact():
    a, b, c = (1, 10, 1), (1, 10, 2), (1, 10, 3)
    constraints = [[(1, 10, 1), (1, 10, 2)]]  # one conflict {a, b}; c is in every maximal repair
    q = ("?S", "?P", "?O")
    assert R.iar([a, b, c], constraints, q) == {a, b, c} - {a, b} == {c}
    # iteration order (a, b, c): {a, b} is pushed last, so it is popped first and {a} and {b} are kept before {a, c} and {b, c}
    got, kept = R.transcribe([a, b, c], constraints, q, [a, b, c])
    assert kept[:2] == [frozenset({a}), frozenset({b})]
    assert got == set(), "the reference's answer is a strict subset (quirk Q13)"
    # order (c, a, b) pops {c, a} first: only maximal repairs are kept and the answers agree
    got, kept = R.transcribe([a, b, c], constraints, q, [c, a, b])
    assert set(kept) == {frozenset({a, c}), frozenset({b, c})} and got == {c}


def test_conflict_sizes_and_minimality():
    x, y, z = (1, 10, 2), (1, 11, 3), (2, 12, 3)
    big = [("?A", 10, "?B"), ("?A", 11, "?C"), ("?D", 12, "?C")]  # size 3: {x, y, z}
    small = [("?A", 11, 3)]                                        # size 1: {y}
    s = R.stats([x, y, z], [big, small])
    assert s == {"constraints": 2, "conflicts": 2, "minimal_conflicts": 1, "conflicted_facts": 1, "subsets_probed": 1}
    assert R.conflicted_facts([x, y, z], [big, small]) == {y}
    # two premises that bind the same fact: a conflict of one fact
    same = [("?A", 10, "?B"), ("?A", "?P", 2)]
    assert R.conflicts([x], [same]) == {frozenset({x})}
