"""The restatement of the reference's writes (tests/update_reference.py) on the reference's own update tests
(kolibrie/tests/rdf_star_test.rs:332-405, 465-491) and on hand-worked cases; the engine's host encode_term_star pieces against it."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

from kolibrie_b200 import engine
from tests.test_golden_provenance import reference_sources
from tests.update_reference import RefDb, batch_insert, batch_remove, clean_term, run_fixture_case, split_quoted_triple_content

A, B, C, D = "<http://example.org/a>", "<http://example.org/b>", "<http://example.org/c>", "<http://example.org/d>"
ALICE, KNOWS, BOB = "<http://example.org/alice>", "<http://example.org/knows>", "<http://example.org/bob>"


def test_insert_normal_and_quoted_triple():  # test_insert_normal_triple, test_insert_quoted_triple, test_handle_update_insert*
    db = RefDb()
    assert db.handle_update("INSERT", [(ALICE, KNOWS, BOB)]) == "Update Successful"
    assert len(db.triples) == 1
    db = RefDb()
    assert db.handle_update("INSERT", [(f"<< {A} {B} {C} >>", "<http://example.org/src>", D)]) == "Update Successful"
    assert len(db.triples) == 1 and len(db.qt_to_id) == 1
    (s, p, o), = db.triples
    assert db.id_to_qt[s] == (db.string_to_id["http://example.org/a"], db.string_to_id["http://example.org/b"], db.string_to_id["http://example.org/c"])


def test_delete_basic_and_quoted():  # test_delete_basic, test_delete_quoted_triple, test_handle_update_delete
    db = RefDb()
    db.handle_update("INSERT", [(ALICE, KNOWS, BOB), (ALICE, "<http://example.org/name>", '"Alice"')])
    assert db.handle_update("DELETE", [(ALICE, KNOWS, BOB)]) == "Update Successful"
    assert len(db.triples) == 1
    db = RefDb()
    q = f"<< {ALICE} {KNOWS} {BOB} >>"
    db.handle_update("INSERT", [(q, "<http://example.org/source>", "<http://example.org/doc1>")])
    db.handle_update("DELETE", [(q, "<http://example.org/source>", "<http://example.org/doc1>")])
    assert len(db.triples) == 0


def test_delete_where_removes_every_match():  # test_delete_where
    db = RefDb()
    db.handle_update("INSERT", [(ALICE, KNOWS, BOB), (ALICE, KNOWS, "<http://example.org/carol>"), (ALICE, "<http://example.org/name>", '"Alice"')])
    rows = [{"?s": "http://example.org/alice", "?o": "http://example.org/bob"}, {"?s": "http://example.org/alice", "?o": "http://example.org/carol"}]
    db.delete_where([("?s", KNOWS, "?o")], rows)
    assert len(db.triples) == 1


def test_unknown_kind_fails():
    assert RefDb().handle_update("LOAD", [(A, B, C)]) == "Update Failed"


def test_repeats_inside_a_batch_resolve_in_batch_order():
    st = {(1, 2, 3)}
    assert batch_insert(st, [(1, 2, 3), (4, 5, 6), (4, 5, 6), (7, 8, 9)]) == [False, True, False, True]
    assert batch_remove(st, [(4, 5, 6), (4, 5, 6), (0, 0, 0), (1, 2, 3)]) == [True, False, False, True]
    assert st == {(7, 8, 9)}


def test_delete_then_insert_of_the_same_triple():
    db = RefDb()
    db.handle_update("INSERT", [(A, B, C)])
    db.handle_update("DELETE", [(A, B, C)])
    db.handle_update("INSERT", [(A, B, C)])
    assert len(db.triples) == 1


def test_quirk_delete_of_unknown_terms_adds_them_to_the_dictionary():
    db = RefDb()
    db.handle_update("DELETE", [(A, B, "<http://example.org/never>")])
    assert "http://example.org/never" in db.string_to_id and not db.triples


def test_quirk_insert_template_is_inserted_literally():
    db = RefDb()
    db.handle_update("INSERT", [(A, B, C)])
    db.delete_where([("?s", B, "?o")], [{"?s": "http://example.org/a", "?o": "http://example.org/c"}], insert_template=[("?s", B, D)])
    (s, p, o), = db.triples
    assert db.id_to_string[s] == "?s"


def test_nested_quoted_terms_encode_components_first():
    db = RefDb()
    inner = f"<< {A} {B} {C} >>"
    db.handle_update("INSERT", [(f"<< {inner} {B} \"x y\" >>", B, D)])
    assert db.id_to_string[:3] == ["http://example.org/a", "http://example.org/b", "http://example.org/c"]
    assert len(db.qt_to_id) == 2
    outer_id = next(iter(db.triples))[0]
    s, p, o = db.id_to_qt[outer_id]
    assert s == db.qt_to_id[(0, 1, 2)] and db.id_to_string[o] == "x y"


SPLITS = [  # content -> the three parts split_quoted_triple_content returns (sparql_database.rs:125-190), worked by hand
    ("<a> <b> <c>", ("<a>", "<b>", "<c>")),
    ('<a> <b> "lit with spaces"', ("<a>", "<b>", '"lit with spaces"')),
    ("<< <a> <b> <c> >> <p> <o>", ("<< <a> <b> <c> >>", "<p>", "<o>")),
    ("<s> <p> << <a> << <x> <y> <z> >> <c> >>", ("<s>", "<p>", "<< <a> << <x> <y> <z> >> <c> >>")),
    ('<s> <p> "esc \\" quote"', ("<s>", "<p>", '"esc \\" quote"')),
    ("<s> <p>", ("<s>", "<p>", "")),
    ("a b c d e", ("a", "b", "c d e")),
    ("", ("", "", "")),
]
CLEANS = [  # a trimmed plain term -> what encode_term_star hands to Dictionary::encode (sparql_database.rs:96-106), worked by hand
    ("<http://x>", "http://x"), ('"lit"', "lit"), ('"lit"@en', "lit"), ('"a"b"', "a"), ('"open', "open"), ("plain", "plain"),
    ("<<odd", "<<odd"), ("<>", ""), ('""', ""),
]


@pytest.mark.parametrize("content,parts", SPLITS)
def test_split_quoted_content_by_hand(content, parts):
    assert engine._split_quoted_content(content) == parts
    assert split_quoted_triple_content(content) == parts


@pytest.mark.parametrize("term,cleaned", CLEANS)
def test_clean_term_by_hand(term, cleaned):
    assert engine._clean_term(term) == cleaned
    assert clean_term(term) == cleaned


FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "update")


def test_update_fixture_is_what_its_generator_writes(tmp_path):
    shutil.copy(os.path.join(FIXTURE, "make_fixture.py"), tmp_path / "make_fixture.py")
    r = subprocess.run([sys.executable, str(tmp_path / "make_fixture.py")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert sorted(f for f in os.listdir(tmp_path) if f.endswith(".json")) == ["update.json"]
    assert json.load(open(tmp_path / "update.json")) == json.load(open(os.path.join(FIXTURE, "update.json")))


def test_update_fixture_cites_existing_reference_lines():
    ref = reference_sources()
    doc = json.load(open(os.path.join(FIXTURE, "update.json")))
    cited = re.findall(r"(\b(?:kolibrie|shared|datalog)/[\w/\.\-]+\.rs):([\d\-,: ]+)", doc["source"])
    assert len(cited) >= 3
    for path, spans in cited:
        assert path in ref
        assert all(1 <= int(a) <= ref[path] for a in re.findall(r"\d+", spans))
    for case in doc["cases"]:
        assert 1 <= case["line"] <= ref["kolibrie/tests/rdf_star_test.rs"]


@pytest.mark.parametrize("case", json.load(open(os.path.join(FIXTURE, "update.json")))["cases"], ids=lambda c: c["name"])
def test_restatement_passes_the_reference_update_tests(case):
    db = RefDb()
    db.load(case["data"])
    run_fixture_case(db, case)
