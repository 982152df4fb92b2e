"""Writes querybuilder.json in this directory: a hand transcription of the INPUTS and ASSERTIONS of the reference's QueryBuilder tests
(kolibrie/tests/integration_test.rs:19-76 and :131-299; the "source" field cites them, by path inside the Kolibrie checkout), and
hand-worked cases for the semantics of query_builder.rs:355-643. No reference output is captured: the fixture pins the transcription
(tests/qb_reference.py), which then pins the engine and the device (tests/test_querybuilder_cpu.py, tests/test_gpu_querybuilder.py).
Run: python tests/golden/querybuilder/make_fixture.py"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
EX = "http://example.org/"


def dump(name, doc):
    with open(os.path.join(HERE, name), "w") as f:
        json.dump(doc, f, indent=1)


# the store of integration_test.rs:19-76 (setup_test_db): the dictionary in encode order and the triples as ids
terms = ["http://example.org/person1", "http://example.org/person2", "http://example.org/company1", "ex:name", "ex:age", "ex:email", "ex:worksFor",
         "ex:founded", "ex:industry", "John Smith", "Jane Doe", "ACME Corp", "30", "25", "john@example.com", "jane@example.com", "2000", "Technology"]
triples = [(0, 3, 9), (0, 4, 12), (0, 5, 14), (0, 6, 2), (1, 3, 10), (1, 4, 13), (1, 5, 15), (1, 6, 2), (2, 3, 11), (2, 7, 16), (2, 8, 17)]

# QueryBuilder (kolibrie/src/query_builder.rs:355-643). A query is {"filters": [subject, predicate, object] with each null or
# [kind, text], "join": conditions, "right": null | "R" (the case's right store) | "self" | "empty", "offset", "limit", "order_by":
# null | "asc" | "desc" (a key on the decoded object), "distinct"}; "expect" maps a result method to its answer ("error": the reference
# panics). Ids of the hand-worked store: Q is a quoted-triple id (bit 31), U an id past the dictionary.
Q, U = 1 << 31, 50
qb_strings = ["aaa", "aa", "a", "", "héllo", "日本語", "http://x/s1", "http://x/p", "lit"]
qb_store = [[6, 7, 0], [6, 7, 4], [Q, 7, 8], [6, U, 1], [3, 7, 5], [2, 7, Q]]
qb_right = [[6, 7, 8], [2, 1, 0]]
P_X = ["Exact", "http://x/p"]


def qb(filters=(None, None, None), **kw):
    return {"filters": list(filters), "join": [], "right": None, "offset": None, "limit": None, "order_by": None, "distinct": False, **kw}


store_rows = sorted(map(tuple, qb_store))
qb_hand = [
    ("contains_overlapping", qb((None, None, ["Contains", "aa"])), {"triples": [[6, 7, 0], [6, U, 1]]}),
    ("contains_empty_pattern", qb((["Contains", ""], None, None)), {"triples": [[2, 7, Q], [3, 7, 5], [6, 7, 0], [6, 7, 4], [6, U, 1]]}),
    ("exact_empty_string", qb((["Exact", ""], None, None)), {"triples": [[3, 7, 5]]}),
    ("starts_empty_pattern_skips_unknown", qb((None, ["StartsWith", ""], None)), {"count": 5}),
    ("ends_multibyte", qb((None, None, ["EndsWith", "llo"])), {"triples": [[6, 7, 4]]}),
    ("contains_multibyte", qb((None, None, ["Contains", "é"])), {"triples": [[6, 7, 4]]}),
    ("starts_multibyte", qb((None, None, ["StartsWith", "日本"])), {"triples": [[3, 7, 5]]}),
    ("ends_whole_string", qb((None, None, ["EndsWith", "日本語"])), {"triples": [[3, 7, 5]]}),
    ("pattern_longer_than_string", qb((["StartsWith", "http://x/s1/longer"], None, None)), {"count": 0}),
    ("exact_not_in_dictionary", qb((None, None, ["Exact", "zzz"])), {"count": 0}),
    ("exact_object", qb((None, None, ["Exact", "aaa"])), {"triples": [[6, 7, 0]]}),
    ("quoted_subject_fails_any_filter", qb((["EndsWith", ""], P_X, None)), {"count": 4}),
    ("join_on_subject", qb((None, P_X, None), join=["OnSubject"], right="R"), {"triples": [[2, 7, 0], [6, 7, 8]]}),
    ("join_on_predicate", qb((None, P_X, None), join=["OnPredicate"], right="R"), {"triples": [[2, 7, 8], [3, 7, 8], [6, 7, 8], [Q, 7, 8]]}),
    ("join_on_object", qb((None, P_X, None), join=["OnObject"], right="R"), {"triples": [[6, 1, 0], [Q, 7, 8]]}),
    ("join_all_three", qb((None, P_X, None), join=["OnSubject", "OnPredicate", "OnObject"], right="R"),
     {"triples": [[2, 7, 0], [2, 7, 8], [3, 7, 8], [6, 1, 0], [6, 7, 8], [Q, 7, 8]]}),
    ("join_condition_repeated", qb((None, P_X, None), join=["OnSubject", "OnSubject"], right="R"), {"triples": [[2, 7, 0], [6, 7, 8]]}),
    ("join_empty_right", qb((None, P_X, None), join=["OnSubject"], right="empty"), {"count": 0}),
    ("join_empty_left", qb((None, None, ["Exact", "zzz"]), join=["OnSubject"], right="R"), {"count": 0}),
    ("self_join_on_object", qb(join=["OnObject"], right="self"), {"triples": [list(t) for t in store_rows]}),
    ("join_without_condition", qb((None, P_X, None), right="R"), {"count": 5}),
    ("condition_without_join", qb((None, P_X, None), join=["OnSubject"]), {"count": 5}),
    ("order_by_ignored", qb(order_by="desc"), {"triples": [list(t) for t in store_rows]}),
    ("offset_at_n", qb(offset=6), {"count": 0}),
    ("offset_past_n", qb(offset=7), {"error": "offset"}),
    ("limit_zero", qb(limit=0), {"count": 0}),
    ("offset_limit_saturates", qb(offset=2, limit=(1 << 64) - 1), {"triples": [list(t) for t in store_rows[2:]]}),
    ("offset_then_limit", qb(offset=1, limit=2), {"triples": [list(t) for t in store_rows[1:3]]}),
    ("subjects_drop_undecodable", qb(), {"subjects": ["a", "", "http://x/s1", "http://x/s1", "http://x/s1"]}),
    ("subjects_distinct", qb(distinct=True), {"subjects": ["", "a", "http://x/s1"], "count": 6}),
    ("predicates", qb(), {"predicates": ["http://x/p"] * 5}),
    ("objects", qb(), {"objects": ["日本語", "aaa", "héllo", "aa", "lit"]}),
    ("objects_distinct", qb(distinct=True), {"objects": ["aa", "aaa", "héllo", "lit", "日本語"]}),
    ("decoded_none_is_empty", qb((["Exact", "a"], None, None)), {"decoded": [["a", "http://x/p", ""]]}),
    ("decoded_quoted_subject", qb((None, None, ["Exact", "lit"])), {"decoded": [["", "http://x/p", "lit"]]}),
]

P1, P2, C1 = EX + "person1", EX + "person2", EX + "company1"
qb_integration = [
    ("with_subject", qb((["Exact", P1], None, None)), {"count": 4}),
    ("with_predicate", qb((None, ["Exact", "ex:name"], None)), {"count": 3}),
    ("with_object", qb((None, None, ["Exact", "Jane Doe"])), {"count": 1}),
    ("with_subject_like", qb((["Contains", "person"], None, None)), {"count": 8}),
    ("with_predicate_like", qb((None, ["Contains", "name"], None)), {"count": 3}),
    ("with_object_like", qb((None, None, ["Contains", "example.com"])), {"count": 2}),
    ("with_subject_starting", qb((["StartsWith", EX + "person"], None, None)), {"count": 8}),
    ("with_predicate_ending", qb((None, ["EndsWith", "For"], None)), {"count": 2}),
    ("compound", qb((["Contains", "person"], ["Exact", "ex:name"], None)), {"count": 2}),
    ("name_subjects", qb((None, ["Exact", "ex:name"], None)), {"count": 3, "subjects_len": 3, "subjects_contain": P1}),
    ("person1_predicates", qb((["Exact", P1], None, None)), {"predicates_len": 4, "predicates_contain": "ex:name"}),
    ("age_objects", qb((None, ["Exact", "ex:age"], None)), {"objects_len": 2, "objects_contain": "30"}),
    ("person2_decoded", qb((["Exact", P2], None, None)), {"decoded_len": 4, "decoded_contain": [P2, "ex:name", "Jane Doe"]}),
    ("limit", qb(limit=2), {"count": 2}),
    ("offset_limit", qb(offset=2, limit=2), {"count": 2, "first_is_all_at": 2}),
    ("tech_companies", qb((None, ["Exact", "ex:industry"], ["Exact", "Technology"])), {"subjects": [C1]}),
    ("tech_employees", qb((None, ["Exact", "ex:worksFor"], ["Exact", C1])), {"subjects_len": 2, "subjects_contain": P1}),
]

dump("querybuilder.json", {
    "source": "kolibrie/tests/integration_test.rs:19-76 (fixture), :131-299 (asserted QueryBuilder answers); kolibrie/src/query_builder.rs:355-643 "
              "(the semantics of the hand-worked cases)",
    "integration": {"terms": terms, "triples": triples, "queries": [{"name": n, "query": q, "expect": e} for n, q, e in qb_integration],
                    "second_email": {"add": [P1, "ex:email", "john.smith@example.com"], "query": qb((["Exact", P1], ["Exact", "ex:email"], None)),
                                     "expect": {"count": 2}}},
    "hand": {"strings": qb_strings, "store": qb_store, "right": qb_right, "Q": Q, "U": U,
             "cases": [{"name": n, "query": q, "expect": e} for n, q, e in qb_hand]}})
