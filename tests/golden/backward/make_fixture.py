"""Writes bc.json in this directory: a hand transcription of the INPUTS and ASSERTIONS of the reference's backward-chaining tests (the
"source" field cites them, by path inside the Kolibrie checkout). No reference output is captured: the fixture pins the restatement of
backward_chaining (tests/bc_reference.py), which then pins the device (tests/test_gpu_backward.py).
Run: python tests/golden/backward/make_fixture.py"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))

PARENT = [[["?X", "parent", "?Y"]], [["?X", "ancestor", "?Y"]]]
TRANS = [[["?X", "ancestor", "?Y"], ["?Y", "ancestor", "?Z"]], [["?X", "ancestor", "?Z"]]]


def case(name, line, facts, encode, rules, query, has=(), empty=None):
    """facts: add_abox_triple calls in order; encode: the later enc() calls in order (the dictionary's encode order is facts first, s p o
    each, then these); rules: [premises, conclusions]; has: bc_has(results, var, value) assertions; empty: is_empty() asserted"""
    return {"name": name, "line": line, "facts": facts, "encode": encode, "rules": rules, "query": query,
            "has": [list(h) for h in has], "empty": empty}


doc = {
    "source": "datalog/tests/reasoning_tests.rs:405-654 (the bc_* tests; bc_has is :22-24); Reasoner::backward_chaining is "
              "datalog/src/reasoning/backward_chaining.rs:165-259",
    "note": "strings starting with ? are variables (the test's Term::Variable names), every other string a constant encoded by the reasoner's "
            "dictionary; has = [variable, constant] pairs some result binds; empty = results.is_empty() asserted true / false",
    "cases": [
        case("bc_direct_fact", 409, [["A", "likes", "B"]], ["likes", "A", "B"], [], ["?X", "likes", "?Y"], has=[("X", "A"), ("Y", "B")]),
        case("bc_1hop_rule", 425, [["A", "parent", "B"]], ["parent", "ancestor", "A", "B"], [PARENT], ["A", "ancestor", "?Y"], has=[("Y", "B")]),
        case("bc_2hop_transitive", 446, [["A", "parent", "B"], ["B", "parent", "C"]], ["parent", "ancestor", "A", "B", "C"], [PARENT, TRANS],
             ["A", "ancestor", "?Y"], has=[("Y", "B"), ("Y", "C")]),
        case("bc_3hop_transitive", 477, [["A", "parent", "B"], ["B", "parent", "C"], ["C", "parent", "D"]],
             ["parent", "ancestor", "A", "B", "C", "D"], [PARENT, TRANS], ["A", "ancestor", "?Y"], has=[("Y", "B"), ("Y", "C"), ("Y", "D")]),
        case("bc_specific_target", 511, [["A", "parent", "B"], ["B", "parent", "C"]], ["parent", "ancestor", "A", "C"], [PARENT, TRANS],
             ["A", "ancestor", "C"], empty=False),
        case("bc_no_result", 540, [["A", "parent", "B"]], ["parent", "ancestor", "A", "D"], [PARENT], ["A", "ancestor", "D"], empty=True),
        case("bc_multi_rule_chain", 561, [["A", "worksFor", "Corp"]], ["worksFor", "employed", "affiliated", "A", "Corp"],
             [[[["?X", "worksFor", "?Y"]], [["?X", "employed", "?Y"]]], [[["?X", "employed", "?Y"]], [["?X", "affiliated", "?Y"]]]],
             ["A", "affiliated", "?Y"], has=[("Y", "Corp")]),
        case("bc_sibling_join", 587, [["A", "parent", "P"], ["B", "parent", "P"]], ["parent", "sibling", "B", "A"],
             [[[["?X", "parent", "?Z"], ["?Y", "parent", "?Z"]], [["?X", "sibling", "?Y"]]]], ["A", "sibling", "?Y"], has=[("Y", "B")]),
        case("bc_full_scan", 613, [["A", "parent", "B"], ["C", "parent", "D"]], ["parent", "A", "B", "C", "D"], [], ["?S", "parent", "?O"],
             has=[("S", "A"), ("O", "B"), ("S", "C"), ("O", "D")]),
        case("bc_no_spurious_negative", 639, [["A", "parent", "B"]], ["unknown"], [], ["?X", "unknown", "?Y"], empty=True),
    ],
}

if __name__ == "__main__":
    with open(os.path.join(HERE, "bc.json"), "w") as f:
        json.dump(doc, f, indent=1)
