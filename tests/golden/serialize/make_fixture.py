"""Writes serialize.json in this directory: a hand transcription of the INPUTS and ASSERTIONS of the reference's own serializer tests
(the "source" field cites them, by path inside the Kolibrie checkout). No reference output is captured: the fixture pins the
restatement of the serializers (tests/serialize_reference.py), which then pins the device (tests/test_gpu_serialize.py).
Run: python tests/golden/serialize/make_fixture.py"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
EX = "http://example.org/"


def dump(name, doc):
    with open(os.path.join(HERE, name), "w") as f:
        json.dump(doc, f, indent=1)


dump("serialize.json", {
    "source": "kolibrie/tests/rdf_star_test.rs:406-462 (test_generate_ntriples_basic, _star, test_generate_turtle_basic, _star); the serializers are "
              "kolibrie/src/sparql_database.rs:301-382",
    "note": "data = the triples parse_ntriples_and_add stores for the test's input (IRIs without brackets, literals without quotes; a nested "
            "[s, p, o] list is a quoted triple << s p o >>); contains / count / ends_with are the test's assertions on the output",
    "cases": [
        {"name": "test_generate_ntriples_basic", "line": 408, "format": "ntriples", "data": [[EX + "alice", EX + "knows", EX + "bob"]],
         "contains": ["<" + EX + "alice>", "<" + EX + "knows>", EX + "bob"], "ends_with": ".\n"},
        {"name": "test_generate_ntriples_star", "line": 422, "format": "ntriples",
         "data": [[[EX + "alice", EX + "knows", EX + "bob"], EX + "source", EX + "doc1"]],
         "contains": ["<<", ">>", EX + "alice", "<" + EX + "source>"]},
        {"name": "test_generate_turtle_basic", "line": 436, "format": "turtle",
         "data": [[EX + "alice", EX + "knows", EX + "bob"], [EX + "alice", EX + "name", "Alice"]],
         "count": {"<" + EX + "alice>": 1}, "contains": [";", "."]},
        {"name": "test_generate_turtle_star", "line": 452, "format": "turtle",
         "data": [[[EX + "alice", EX + "knows", EX + "bob"], EX + "source", EX + "doc1"]], "contains": ["<<", ">>"]},
    ]})
