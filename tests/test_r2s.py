"""CPU: the restatement of the Relation-to-Stream operator (tests/r2s_reference.py) against the assertions of the reference's own tests:
r2s.rs's unit tests and rsp_ql_dstream_semantics (tests/r2s_cases.py), and the ISTREAM / RSTREAM cases of
tests/golden/rsp_windows.json. The device (tests/test_gpu_r2s.py) is held to this restatement by exact list equality."""
import json
import os
import re

import pytest

from tests import r2s_cases
from tests.r2s_reference import DSTREAM, ISTREAM, RSTREAM, Relation2Stream, window_rows

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    return json.load(open(os.path.join(GOLDEN, name)))


def firing_rows(case, f):
    if "rows" in f:
        return [tuple(r) for r in f["rows"]]
    return window_rows(f["window"], case["pattern"], case["select"])


def test_r2s_cases_cite_lines_that_exist():
    from tests.test_golden_provenance import reference_sources

    ref = reference_sources()
    cited = re.findall(r"(kolibrie/[\w/\.\-]+\.rs):(\d+)-(\d+)", r2s_cases.SOURCE)
    assert len(cited) == 2
    for path, a, b in cited:
        assert path in ref and 1 <= int(a) <= int(b) <= ref[path], (path, a, b)
    for case in r2s_cases.CASES:
        path = "kolibrie/tests/rsp_engine_test.rs" if "window" in case["firings"][0] else "kolibrie/src/rsp/r2s.rs"
        assert [int(a) <= case["line"] <= int(b) for p_, a, b in cited if p_ == path] == [True], case["name"]


@pytest.mark.parametrize("case", r2s_cases.CASES, ids=lambda c: c["name"])
def test_r2s_fixture(case):
    op = Relation2Stream(case["stream"])
    for k, f in enumerate(case["firings"]):
        got = op.eval(firing_rows(case, f))
        if f["emit"] is not None:
            assert got == [tuple(r) for r in f["emit"]], (case["name"], k)


@pytest.mark.parametrize("case", [c for c in load("rsp_windows.json")["cases"] if c["stream"] in ("ISTREAM", "RSTREAM")], ids=lambda c: c["name"])
def test_rsp_windows_fixture(case):
    op = Relation2Stream(case["stream"])
    for k, f in enumerate(case["firings"]):
        assert op.eval(firing_rows(case, f)) == [tuple(r) for r in f["emit"]], (case["name"], k)


def test_order_and_bag_contract():
    ist = Relation2Stream(ISTREAM)
    assert ist.eval([(1,), (2,), (1,)]) == [(1,), (2,), (1,)]  # first firing: everything is new, duplicates kept
    assert ist.last == [(1,), (2,)]
    assert ist.eval([(3,), (2,), (3,), (4,)]) == [(3,), (3,), (4,)]  # response order, every occurrence of a new row
    dst = Relation2Stream(DSTREAM)
    assert dst.eval([(5,), (1,), (5,), (3,)]) == []
    assert dst.eval([(3,)]) == [(5,), (1,)]  # first-occurrence order of the response that set the state, each row once
    assert dst.eval([]) == [(3,)] and dst.last == []
    rst = Relation2Stream(RSTREAM)
    assert rst.eval([(1,), (1,)]) == [(1,), (1,)] and rst.last == []
