"""Hand transcriptions of the INPUTS and ASSERTIONS of the reference's tests of the Relation-to-Stream operator, in the manner of
tests/golden/make_fixtures.py: r2s.rs's three unit tests and the one RSP test of DSTREAM. `emit` is what the test asserts for that
evaluation (None: the test asserts nothing about it). Unit-test rows are given as their values in `vars` order; a firing of the RSP
test lists the window's content, and its rows are the answers of `pattern` over it (tests/r2s_reference.window_rows)."""

SOURCE = ("kolibrie/src/rsp/r2s.rs:69-127 (test_rstream, test_dstream, test_istream), "
          "kolibrie/tests/rsp_engine_test.rs:103-187 (rsp_ql_dstream_semantics)")

T = "http://test/"

CASES = [
    {"name": "test_rstream", "line": 70, "stream": "RSTREAM", "vars": ["x"],
     "firings": [{"rows": [["this"], ["is"], ["a"], ["test"]], "emit": [["this"], ["is"], ["a"], ["test"]]}]},
    {"name": "test_dstream", "line": 83, "stream": "DSTREAM", "vars": ["1", "2"],
     "firings": [{"rows": [["1", "2"], ["1.2", "2.2"]], "emit": None},
                 {"rows": [["1", "2"], ["1.3", "2.3"]], "emit": [["1.2", "2.2"]]}]},
    {"name": "test_istream", "line": 106, "stream": "ISTREAM", "vars": ["1", "2"],
     "firings": [{"rows": [["1", "2"], ["1.2", "2.2"]], "emit": None},
                 {"rows": [["1", "2"], ["1.3", "2.3"]], "emit": [["1.3", "2.3"]]}]},
    # RANGE 3 STEP 1: five firings; only the fifth emits (one consumer call, binding ?s to subjectA)
    {"name": "rsp_ql_dstream_semantics", "line": 116, "stream": "DSTREAM", "pattern": ["?s", "a", T + "DType"], "select": ["s"],
     "firings": [{"window": [[T + "subject" + x, "a", T + "DType"] for x in w], "emit": [[T + "subjectA"]] if w == "BCDE" else []}
                 for w in ("A", "AB", "ABC", "ABCD", "BCDE")]},
]
