"""CPU: the restatement of generate_ntriples / generate_turtle (tests/serialize_reference.py) against the assertions of the reference's
own serializer tests (tests/golden/serialize/serialize.json, rdf_star_test.rs:406-462) and against hand-worked texts (tests/serialize_cases.py);
and SparqlDatabase.generate_ntriples / generate_turtle on the oracle context (the host path of kolibrie_b200/engine.py) against the
restatement."""
import json
import os
import random
import shutil
import subprocess
import sys

import pytest

from kolibrie_b200 import engine as E
from tests import serialize_reference as R
from tests.oracle_ctx import OracleCtx
from tests.serialize_cases import CASES, Q

FIXTURE_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "serialize")
with open(os.path.join(FIXTURE_DIR, "serialize.json")) as _f:
    GOLDEN = json.load(_f)


def test_fixture_is_what_its_generator_writes(tmp_path):
    shutil.copy(os.path.join(FIXTURE_DIR, "make_fixture.py"), tmp_path / "make_fixture.py")
    r = subprocess.run([sys.executable, str(tmp_path / "make_fixture.py")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert json.load(open(tmp_path / "serialize.json")) == GOLDEN


def data_term(t):
    return tuple(data_term(x) for x in t) if isinstance(t, list) else t


def golden_db(case):
    db = E.SparqlDatabase(ctx=OracleCtx())
    for s, p, o in case["data"]:
        db.add_statement(data_term(s), data_term(p), data_term(o))
    return db


def restate(db, fmt):
    qt = db.quoted_triple_store.id_to_components
    if fmt == "ntriples":
        return R.generate_ntriples(db.triples, db.dictionary.id_to_string, qt)
    return R.generate_turtle(db.triples, db.dictionary.id_to_string, qt, db.prefixes)


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=lambda c: c["name"])
def test_reference_assertions(case):
    db = golden_db(case)
    for out in (restate(db, case["format"]), db.generate_ntriples() if case["format"] == "ntriples" else db.generate_turtle()):
        for x in case.get("contains", []):
            assert x in out, (x, out)
        for x, n in case.get("count", {}).items():
            assert out.count(x) == n, (x, out)
        if "ends_with" in case:
            assert out.endswith(case["ends_with"])


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_hand_worked_texts(case):
    assert R.generate_ntriples(case["triples"], case["strings"], case["quoted"]) == case["nt"]
    assert R.generate_turtle(case["triples"], case["strings"], case["quoted"], case["prefixes"]) == case["ttl"]


def case_db(case):
    db = E.SparqlDatabase(ctx=OracleCtx())
    db.dictionary.id_to_string = list(case["strings"])
    db.dictionary.string_to_id = {s: i for i, s in enumerate(case["strings"])}
    for i, comp in case["quoted"].items():
        db.quoted_triple_store.id_to_components[i] = comp
    for t in case["triples"]:
        db.add_triple(t)
    db.set_prefixes(case["prefixes"])
    return db


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_engine_mirror_on_the_oracle(case):
    db = case_db(case)
    assert db.generate_ntriples() == case["nt"]
    assert db.generate_turtle() == case["ttl"]


def random_store(seed, n=400):
    """ids from a small dictionary (some past it), quoted ids (some nested, some missing) and repeated triples"""
    rng = random.Random(seed)
    words = ["http://x/" + w for w in ("a", "ab", "b", "é", "z")] + ["https://y/1", "lit", "", "<< a b c >>", "ü", "a b"]
    quoted = {Q: (0, 1, 2), Q + 1: (Q, 3, 4), Q + 2: (0, 99, 2), Q + 3: (Q + 1, 0, Q)}
    pool = list(range(len(words))) + [50, 51] + [Q, Q + 1, Q + 2, Q + 3, Q + 9]
    triples = [tuple(rng.choice(pool) for _ in range(3)) for _ in range(n)]
    return words, quoted, triples + triples[: n // 4]


@pytest.mark.parametrize("seed", range(4))
def test_engine_mirror_equals_the_restatement_on_random_stores(seed):
    words, quoted, triples = random_store(seed)
    case = dict(strings=words, quoted=quoted, triples=triples, prefixes=[("x", "http://x/")])
    db = case_db(case)
    assert db.generate_ntriples() == R.generate_ntriples(triples, words, quoted)
    assert db.generate_turtle() == R.generate_turtle(triples, words, quoted, [("x", "http://x/")])
