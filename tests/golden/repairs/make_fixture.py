"""Writes repairs.json in this directory: a hand transcription of the INPUTS of the reference's two query_with_repairs examples (the
"source" field cites them, by path inside the Kolibrie checkout): the facts, the constraint and the query. No reference output is
captured: the fixture feeds the restatements of tests/repairs_reference.py, which then pin the device (tests/test_gpu_repairs.py).
Run: python tests/golden/repairs/make_fixture.py"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))

PROF_AND_STUDENT = [["?X", "isA", "professor"], ["?X", "isA", "student"]]


def case(name, lines, facts, constraints, query):
    """facts: add_abox_triple calls in order; constraints: the add_constraint premises (their conclusion is the dummy (0, 0, 0) and is
    not read); query: the query_with_repairs pattern"""
    return {"name": name, "lines": lines, "facts": facts, "constraints": constraints, "query": query}


doc = {
    "source": "kolibrie/examples/sparql_syntax/knowledge_graph/contradictions.rs:15-53,121-133 and "
              "kolibrie/examples/sparql_syntax/knowledge_graph/knowledge_graph.rs:228-272; Reasoner::query_with_repairs is "
              "datalog/src/reasoning/repairs.rs:10-43, compute_repairs datalog/src/reasoning.rs:110-150",
    "note": "strings starting with ? are variables, every other string a constant encoded by the reasoner's dictionary in order of first "
            "appearance (facts s p o each, then the constraints, then the query). contradictions.rs runs "
            "infer_new_facts_semi_naive_with_repairs before its query; that step is not transcribed (it stays on the host)",
    "cases": [
        case("contradictions", "15-53,121-133",
             [["john", "isA", "professor"], ["john", "isA", "student"], ["john", "teaches", "math101"], ["john", "enrolledIn", "physics101"]],
             [PROF_AND_STUDENT], ["john", "isA", "?Role"]),
        case("knowledge_graph_inconsistency", "228-272",
             [["john", "isA", "professor"], ["john", "isA", "student"]], [PROF_AND_STUDENT], ["?X", "isA", "?Y"]),
    ],
}

if __name__ == "__main__":
    with open(os.path.join(HERE, "repairs.json"), "w") as f:
        json.dump(doc, f, indent=1)
