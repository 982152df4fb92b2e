"""Writes update.json in this directory: a hand transcription of the INPUTS and ASSERTIONS of the reference's own SPARQL Update tests
(the "source" field cites them, by path inside the Kolibrie checkout). No reference output is captured: the fixture pins the
restatement of the writes (tests/update_reference.py), which then pins the device store and the engine (tests/test_gpu_update.py).
Run: python tests/golden/update/make_fixture.py"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
EX = "http://example.org/"


def iri(x):
    return "<" + EX + x + ">"


def dump(name, doc):
    with open(os.path.join(HERE, name), "w") as f:
        json.dump(doc, f, indent=1)


Q_AKB = "<< " + iri("alice") + " " + iri("knows") + " " + iri("bob") + " >>"
dump("update.json", {
    "source": "kolibrie/tests/rdf_star_test.rs:332-405 (test_insert_quoted_triple, test_insert_normal_triple, test_delete_basic, "
              "test_delete_quoted_triple, test_delete_where) and kolibrie/tests/rdf_star_test.rs:465-491 (test_handle_update_insert, _delete, "
              "_insert_quoted_triple); handle_update is kolibrie/src/sparql_database.rs:3091-3117, DELETE WHERE kolibrie/src/execute_query.rs:354-413",
    "note": "data = the triples parse_ntriples_and_add stores for the test's input (IRIs without brackets, literals without quotes; a nested "
            "[s, p, o] list is a quoted triple << s p o >>); a step is handle_update (kind INSERT / DELETE, the term strings parse_insert / "
            "parse_delete yield) or a DELETE { template } WHERE { where } query; result, triples and quoted_nonempty are the test's assertions",
    "cases": [
        {"name": "test_insert_quoted_triple", "line": 332, "data": [],
         "steps": [{"kind": "INSERT", "triples": [[Q_AKB, iri("source"), iri("doc1")]], "result": "Update Successful"}],
         "triples": 1, "quoted_nonempty": True},
        {"name": "test_insert_normal_triple", "line": 348, "data": [],
         "steps": [{"kind": "INSERT", "triples": [[iri("alice"), iri("knows"), iri("bob")]], "result": "Update Successful"}],
         "triples": 1},
        {"name": "test_delete_basic", "line": 357,
         "data": [[EX + "alice", EX + "knows", EX + "bob"], [EX + "alice", EX + "name", "Alice"]],
         "steps": [{"kind": "DELETE", "triples": [[iri("alice"), iri("knows"), iri("bob")]], "result": "Update Successful"}],
         "triples": 1},
        {"name": "test_delete_quoted_triple", "line": 372,
         "data": [[[EX + "alice", EX + "knows", EX + "bob"], EX + "source", EX + "doc1"]],
         "steps": [{"kind": "DELETE", "triples": [[Q_AKB, iri("source"), iri("doc1")]], "result": "Update Successful"}],
         "triples": 0},
        {"name": "test_delete_where", "line": 385,
         "data": [[EX + "alice", EX + "knows", EX + "bob"], [EX + "alice", EX + "knows", EX + "carol"], [EX + "alice", EX + "name", "Alice"]],
         "steps": [{"kind": "DELETE_WHERE", "template": [["?s", iri("knows"), "?o"]], "where": [["?s", iri("knows"), "?o"]]}],
         "triples": 1},
        {"name": "test_handle_update_insert", "line": 465, "data": [],
         "steps": [{"kind": "INSERT", "triples": [[iri("a"), iri("b"), iri("c")]], "result": "Update Successful"}],
         "triples": 1},
        {"name": "test_handle_update_delete", "line": 473, "data": [],
         "steps": [{"kind": "INSERT", "triples": [[iri("a"), iri("b"), iri("c")]]},
                   {"kind": "DELETE", "triples": [[iri("a"), iri("b"), iri("c")]], "result": "Update Successful"}],
         "triples": 0},
        {"name": "test_handle_update_insert_quoted_triple", "line": 484, "data": [],
         "steps": [{"kind": "INSERT", "triples": [["<< " + iri("a") + " " + iri("b") + " " + iri("c") + " >>", iri("src"), iri("d")]],
                    "result": "Update Successful"}],
         "triples": 1, "quoted_nonempty": True},
    ]})
