"""CPU: the WatDiv-shaped generator (datagen.watdiv) — deterministic per seed, rows per predicate equal to the closed form, ids in
first-seen order — and every one of the 20 queries of tests/golden/watdiv/queries.json answered with rows by the oracle at ~100 K
triples."""
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from kolibrie_b200 import datagen
from tests import bgp_cases as B
from tests import oracle_api as O
from tests import watdiv_cases as W
from tests.test_golden_provenance import reference_sources

FIXTURE_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "watdiv")


def test_fixture_is_what_its_generator_writes(tmp_path):
    shutil.copy(os.path.join(FIXTURE_DIR, "make_queries.py"), tmp_path / "make_queries.py")
    r = subprocess.run([sys.executable, str(tmp_path / "make_queries.py")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert sorted(f for f in os.listdir(tmp_path) if f.endswith(".json")) == ["queries.json"]
    assert json.load(open(tmp_path / "queries.json")) == json.load(open(os.path.join(FIXTURE_DIR, "queries.json")))


def test_fixture_cites_existing_reference_lines():
    doc = json.load(open(os.path.join(FIXTURE_DIR, "queries.json")))
    path, a, b = re.fullmatch(r"([\w/\.\-]+\.rs):(\d+)-(\d+)", doc["source"]).groups()
    n = reference_sources()[path]
    assert 1 <= int(a) <= int(b) <= n
    assert len(doc["queries"]) == 20
    for q in doc["queries"]:  # each query's cited line lies inside the cited range, in harness order
        assert int(a) <= q["line"] <= int(b), q["name"]
    assert [q["line"] for q in doc["queries"]] == sorted(q["line"] for q in doc["queries"])


def test_deterministic_and_closed_form_counts():
    a, b, other = datagen.watdiv(100_000, seed=3), datagen.watdiv(100_000, seed=3), datagen.watdiv(100_000, seed=4)
    assert all(np.array_equal(getattr(a, x), getattr(b, x)) for x in "spo") and a.ids == b.ids
    assert not np.array_equal(a.o, other.o)
    want = datagen.watdiv_predicate_counts(100_000)
    assert sum(want.values()) == len(a.s) and 90_000 <= len(a.s) <= 110_000
    for iri, n in want.items():
        assert int((a.p == a.ids[iri]).sum()) == n, iri


def test_ids_are_first_seen_order():
    d = datagen.watdiv(5_000)
    seq = np.stack([d.s, d.p, d.o], axis=1).reshape(-1)
    _, first = np.unique(seq, return_index=True)
    assert np.array_equal(seq[np.sort(first)], np.arange(d.n_ids, dtype=np.uint32))


@pytest.mark.parametrize("q", W.QUERIES, ids=[q["name"] for q in W.QUERIES])
def test_every_query_has_answers_at_100k(q):
    d = datagen.watdiv(100_000)
    pats, project = W.compile_query(d, q)
    rel, sizes = B.oracle(O.Db(d.s, d.p, d.o), pats, None, project)
    assert rel is not None and rel.n_rows > 0, (q["name"], sizes)
