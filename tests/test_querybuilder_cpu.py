"""CPU: the QueryBuilder transcription (tests/qb_reference.py) against the answers the reference's own tests assert
(kolibrie/tests/integration_test.rs:131-299) and the hand-worked cases of tests/golden/querybuilder/querybuilder.json; then the engine's QueryBuilder
on its host restatement (a context without the device query) against the same answers, and the ref / engine agreement on closures."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

from kolibrie_b200 import engine as E
from tests import helpers as H
from tests import qb_reference as R
from tests.test_golden_provenance import reference_sources

FIXTURE_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "querybuilder")
FX = H.load(os.path.join("querybuilder", "querybuilder.json"))
INT, HAND = FX["integration"], FX["hand"]


def test_fixture_is_what_its_generator_writes(tmp_path):
    shutil.copy(os.path.join(FIXTURE_DIR, "make_fixture.py"), tmp_path / "make_fixture.py")
    r = subprocess.run([sys.executable, str(tmp_path / "make_fixture.py")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert json.load(open(tmp_path / "querybuilder.json")) == FX


def test_fixture_citations_exist():
    ref = reference_sources()
    cited = 0
    for path, spans in re.findall(r"(\b(?:kolibrie|shared|datalog)/[\w/\.\-]+\.(?:rs|cu)):([\d\-,: ]+)", FX["source"]):
        assert path in ref, path
        for a in re.findall(r"\d+", spans):
            assert 1 <= int(a) <= ref[path], (path, a)
            cited += 1
    assert cited >= 4


def _int_db():
    db = E.SparqlDatabase(ctx=_NoDevice())
    for t in INT["terms"]:
        db.dictionary.encode(t)
    for t in INT["triples"]:
        db.add_triple(tuple(t))
    return db


class _NoDevice:
    """a context without kb_qb_triples: the engine takes its host restatement"""


def _hand_db(rows):
    db = E.SparqlDatabase(ctx=_NoDevice())
    for s in HAND["strings"]:
        db.dictionary.encode(s)
    for t in rows:
        db.add_triple(tuple(t))
    return db


def _right(q, left):
    return {None: None, "R": HAND["right"], "self": left, "empty": []}[q["right"]]


@pytest.mark.parametrize("case", INT["queries"], ids=lambda c: c["name"])
def test_integration_answers_on_the_transcription(case):
    all_rows = [list(t) for t in R.Ref(INT["triples"], INT["terms"]).get_triples()]
    R.assert_expect(lambda: R.ref_query(INT["triples"], INT["terms"], case["query"]), case["expect"], all_rows)


@pytest.mark.parametrize("case", INT["queries"], ids=lambda c: c["name"])
def test_integration_answers_on_the_engine_host_path(case):
    db = _int_db()
    all_rows = [list(t) for t in sorted(db.query().get_triples())]
    R.assert_expect(lambda: R.engine_query(db, case["query"]), case["expect"], all_rows)
    assert db.query().last_path is None


def test_second_email_after_adding_a_triple():
    se = INT["second_email"]
    strings = list(INT["terms"])
    ids = []
    for t in se["add"]:
        if t not in strings:
            strings.append(t)
        ids.append(strings.index(t))
    rows = list(map(tuple, INT["triples"])) + [tuple(ids)]
    R.assert_expect(lambda: R.ref_query(rows, strings, se["query"]), se["expect"])
    db = _int_db()
    db.add_statement(*se["add"])
    R.assert_expect(lambda: R.engine_query(db, se["query"]), se["expect"])


@pytest.mark.parametrize("case", HAND["cases"], ids=lambda c: c["name"])
def test_hand_worked_cases_on_the_transcription(case):
    q = case["query"]
    right = _right(q, HAND["store"])
    R.assert_expect(lambda: R.ref_query(HAND["store"], HAND["strings"], q, right), case["expect"])


@pytest.mark.parametrize("case", HAND["cases"], ids=lambda c: c["name"])
def test_hand_worked_cases_on_the_engine_host_path(case):
    q = case["query"]
    db = _hand_db(HAND["store"])
    right = _right(q, HAND["store"])
    right_db = None if right is None else db if q["right"] == "self" else _hand_db(right)
    R.assert_expect(lambda: R.engine_query(db, q, right_db), case["expect"])


def test_closures_run_on_the_host_and_agree_with_the_transcription():
    db = _hand_db(HAND["store"])
    ref = R.Ref(HAND["store"], HAND["strings"], HAND["right"])
    ref.custom_filter = lambda t: t[0] != 6
    b = db.query().filter(lambda t: t[0] != 6)
    assert sorted(b.get_triples()) == ref.get_triples()
    assert b.last_path == "host"
    ref = R.Ref(HAND["store"], HAND["strings"], HAND["right"])
    ref.join_conditions = [lambda l, r: l[2] == r[2] or l[0] == r[0]]
    b = db.query().join(_hand_db(HAND["right"])).join_with(lambda l, r: l[2] == r[2] or l[0] == r[0])
    assert sorted(b.get_triples()) == ref.get_triples()
    ref = R.Ref(HAND["store"], HAND["strings"])
    ref.object_filter = ("Custom", lambda v: len(v) == 3)
    b = db.query()
    b.object_filter = ("Custom", lambda v: len(v) == 3)
    assert sorted(b.get_triples()) == ref.get_triples() == [(3, 7, 5), (6, 7, 0), (HAND["Q"], 7, 8)]


def test_group_by_runs_the_key_on_the_host_in_key_order():
    db = _int_db()
    strings = INT["terms"]
    groups = db.query().group_by(lambda t: strings[t[1]])
    assert len(groups["ex:name"]) == 3 and len(groups["ex:age"]) == 2  # integration_test.rs:250-258
    assert list(groups) == sorted(groups)
