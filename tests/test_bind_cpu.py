"""CPU: ExecutionEngine._bind_host (the host restatement of Bind that kb_bind is tested against) held to a row-by-row transcription of
engine.rs:144-277 over binding rows, and to the two BIND cases of rdf_star_test.rs:281-329."""
import json
import os

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import engine as E

NONE = c.KB_ID_NONE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def reference_bind(rows, function_name, arguments, output_variable, d: E.Dictionary, qts: E.QuotedTripleStore):
    """engine.rs:144-277, statement by statement, over rows of {name: id}"""
    out = output_variable[1:] if output_variable.startswith("?") else output_variable
    strip = lambda a: a[1:] if a.startswith("?") else a
    if function_name == "CONCAT":
        decoded = []
        for row in rows:
            vals = []
            for arg in arguments:
                if arg.startswith("?"):
                    i = row.get(strip(arg))
                    vals.append((d.decode(i) or "") if i is not None else "")
                else:
                    vals.append(arg.strip('"'))
            decoded.append(vals)
        for row, vals in zip(rows, decoded):
            row[out] = d.encode("".join(vals))
    elif function_name in ("SUBJECT", "PREDICATE", "OBJECT"):
        for row in rows:
            if arguments:
                i = row.get(strip(arguments[0]))
                if i is not None and E.is_quoted_triple_id(i):
                    comp = qts.decode(i)
                    if comp is not None:
                        row[out] = comp[("SUBJECT", "PREDICATE", "OBJECT").index(function_name)]
    elif function_name == "TRIPLE":
        if len(arguments) == 3:
            for row in rows:
                args = [row.get(strip(a)) if a.startswith("?") else d.encode(strip(a)) for a in arguments]
                if all(a is not None for a in args):
                    row[out] = qts.encode(*args)
    elif function_name == "isTRIPLE":
        for row in rows:
            if arguments:
                i = row.get(strip(arguments[0]))
                if i is not None:
                    row[out] = d.encode("true" if E.is_quoted_triple_id(i) else "false")
    return rows


def cols_to_rows(cols, n):
    return [{k: int(v[i]) for k, v in cols.items() if v[i] != NONE} for i in range(n)]


def run_both(function_name, arguments, output_variable, cols, n, build):
    """the same starting dictionary / quoted store twice (`build` makes them); returns both results and both stores"""
    d1, q1 = build()
    d2, q2 = build()
    rows = reference_bind(cols_to_rows(cols, n), function_name, arguments, output_variable, d1, q1)
    out = E._strip(output_variable)
    col = E.ExecutionEngine._bind_host(function_name, arguments, cols, n, cols.get(out), d2, q2)
    want = np.array([r.get(out, NONE) for r in rows], dtype=np.uint32)
    np.testing.assert_array_equal(col, want)
    assert d1.id_to_string == d2.id_to_string, "new dictionary strings or their order differ"
    assert q1.id_to_components == q2.id_to_components and q1.next_qt_id == q2.next_qt_id
    return col, d2, q2


def store():
    d, q = E.Dictionary(), E.QuotedTripleStore()
    for t in ("a", "b", "c", "é€😀", "x\"y"):
        d.encode(t)
    q1 = q.encode(0, 1, 2)
    q.encode(q1, 1, 3)                    # nested
    q.id_to_components[0x8000_0005] = (2, 2, 2)  # a hole at 0x80000002..4 (ids the store never handed out)
    q.components_to_id[(2, 2, 2)] = 0x8000_0005
    q.next_qt_id = 0x8000_0006
    return d, q


Q0, Q1, QH = 0x8000_0000, 0x8000_0001, 0x8000_0003  # QH: a hole


def u(*v):
    return np.array(v, dtype=np.uint32)


@pytest.mark.parametrize("fn", ["SUBJECT", "PREDICATE", "OBJECT"])
def test_components(fn):
    t = u(Q0, Q1, QH, 0x8000_0005, 0x9000_0000, 2, NONE, Q1)
    run_both(fn, ["?t"], "?x", {"t": t}, len(t), store)


def test_components_overwrite_keeps_old_where_nothing_is_inserted():
    t = u(Q0, 3, NONE, QH)
    col, _, _ = run_both("OBJECT", ["?t"], "?x", {"t": t, "x": u(7, 8, NONE, 9)}, 4, store)
    assert col.tolist() == [2, 8, NONE, 9]


def test_is_triple_lazy_order():
    # "false" is needed first, then "true": encoded in that order; neither string exists yet
    col, d, _ = run_both("isTRIPLE", ["?t"], "?b", {"t": u(NONE, 1, Q0, 2)}, 4, store)
    assert d.id_to_string[-2:] == ["false", "true"]
    col, d, _ = run_both("isTRIPLE", ["?t"], "?b", {"t": u(Q1, NONE, 0)}, 3, store)
    assert d.id_to_string[-2:] == ["true", "false"]
    # only quoted ids: "false" is never encoded
    _, d, _ = run_both("isTRIPLE", ["?t"], "?b", {"t": u(Q1, Q0)}, 2, store)
    assert "false" not in d.string_to_id
    # both already held: nothing new
    def held():
        d, q = store()
        d.encode("true"); d.encode("false")
        return d, q
    _, d, _ = run_both("isTRIPLE", ["?t"], "?b", {"t": u(Q1, 0)}, 2, held)
    assert len(d.id_to_string) == 7


def test_triple_new_existing_nested_duplicates():
    s = u(0, 0, Q0, 4, 0, NONE, 4)
    p = u(1, 1, 1, 4, 1, 1, 4)
    o = u(2, 2, 3, 4, 3, 2, 4)
    col, _, q = run_both("TRIPLE", ["?s", "?p", "?o"], "?t", {"s": s, "p": p, "o": o}, 7, store)
    assert col[0] == Q0 and col[2] == Q1 and col[5] == NONE  # existing entries keep their ids; a missing argument leaves it unbound
    assert col[3] == col[6] == 0x8000_0006 and col[4] == 0x8000_0007  # first-row order of the new ones


def test_triple_constants_encoded_only_with_rows():
    cols = {"s": u(0, 1)}
    _, d, _ = run_both("TRIPLE", ["?s", "<http://new/p>", "\"lit\""], "?t", cols, 2, store)
    assert d.id_to_string[-2:] == ["<http://new/p>", "\"lit\""]
    _, d, q = run_both("TRIPLE", ["?s", "<http://new/p>", "\"lit\""], "?t", {"s": u()}, 0, store)
    assert "<http://new/p>" not in d.string_to_id and q.next_qt_id == 0x8000_0006
    # wrong arity: nothing happens
    _, d, q = run_both("TRIPLE", ["?s", "<http://new/p>"], "?t", cols, 2, store)
    assert "<http://new/p>" not in d.string_to_id


def test_concat_decode_not_decode_term_and_trim_matches():
    cols = {"a": u(0, Q0, 3, NONE, 999), "b": u(4, 1, NONE, 2, 0)}
    col, d, _ = run_both("CONCAT", ["?a", "\"a\"@en", "?b", "\"-\"", "?missing"], "?c", cols, 5, store)
    assert d.decode(int(col[0])) == 'aa"@enx"y-'  # trim_matches('"') strips every leading / trailing quote, no more
    assert d.decode(int(col[1])) == 'a"@enb-'      # a quoted id contributes "" (decode, not decode_term)
    assert d.decode(int(col[3])) == 'a"@enc-'      # a missing variable contributes ""
    assert d.decode(int(col[4])) == 'a"@ena-'      # an id the dictionary lacks contributes ""


def test_concat_duplicates_existing_and_multibyte():
    cols = {"a": u(3, 0, 3, 1, 3)}
    col, d, _ = run_both("CONCAT", ["?a", "?a"], "?c", cols, 5, store)
    assert col[0] == col[2] == col[4] and d.decode(int(col[0])) == "é€😀é€😀"
    col, d, _ = run_both("CONCAT", ["?a"], "?c", cols, 5, store)  # the strings exist: no new id
    assert len(d.id_to_string) == 5
    col, d, _ = run_both("CONCAT", [], "?c", cols, 5, store)
    assert d.decode(int(col[0])) == ""


def test_unknown_function_and_empty_input():
    run_both("NOPE", ["?a"], "?c", {"a": u(1, 2)}, 2, store)
    for fn in ("SUBJECT", "isTRIPLE", "TRIPLE", "CONCAT"):
        _, d, q = run_both(fn, ["?a", "?a", "?a"] if fn == "TRIPLE" else ["?a"], "?c", {"a": u()}, 0, store)
        assert len(d.id_to_string) == 5 and len(q) == 3


def test_unbound_propagates_through_a_chain_of_binds():
    d, q = store()
    d1, q1 = store()
    cols = {"t": u(Q1, 0, QH, NONE)}
    rows = cols_to_rows(cols, 4)
    rows = reference_bind(rows, "SUBJECT", ["?t"], "?s", d1, q1)
    rows = reference_bind(rows, "PREDICATE", ["?s"], "?p", d1, q1)
    rows = reference_bind(rows, "TRIPLE", ["?s", "?p", "?t"], "?u", d1, q1)
    rows = reference_bind(rows, "isTRIPLE", ["?u"], "?b", d1, q1)
    for fn, args, out in (("SUBJECT", ["?t"], "s"), ("PREDICATE", ["?s"], "p"), ("TRIPLE", ["?s", "?p", "?t"], "u"), ("isTRIPLE", ["?u"], "b")):
        cols[out] = E.ExecutionEngine._bind_host(fn, args, cols, 4, None, d, q)
    assert cols_to_rows(cols, 4) == rows
    assert d.id_to_string == d1.id_to_string and q.id_to_components == q1.id_to_components


def test_random_against_transcription():
    rng = np.random.default_rng(7)
    pool = u(0, 1, 2, 3, 4, 999, Q0, Q1, QH, 0x8000_0005, NONE)
    for trial in range(60):
        n = int(rng.integers(0, 40))
        cols = {k: pool[rng.integers(0, len(pool), n)] for k in ("a", "b", "c")}
        fn = ["SUBJECT", "PREDICATE", "OBJECT", "isTRIPLE", "TRIPLE", "CONCAT"][trial % 6]
        args = {"TRIPLE": ["?a", "?b", "?c"], "CONCAT": ["?a", "\"::\"", "?b"]}.get(fn, ["?a"])
        out = "?c" if trial % 4 == 0 else "?z"
        run_both(fn, args, out, cols, n, store)


def test_rdf_star_bind_cases():
    """rdf_star_test.rs:281-302 (BIND(SUBJECT(?t))) and :306-329 (BIND(TRIPLE(?s, ?p, ?o)))"""
    case = next(x for x in json.load(open(os.path.join(ROOT, "tests", "golden", "rdf_star.json")))["cases"] if x["line"] == 281)
    db = E.SparqlDatabase.__new__(E.SparqlDatabase)
    db.dictionary, db.quoted_triple_store = E.Dictionary(), E.QuotedTripleStore()
    tid = db.encode_term(tuple(case["data"][0][0]))
    db.encode_term(case["data"][0][1]); db.encode_term(case["data"][0][2])
    col = E.ExecutionEngine._bind_host("SUBJECT", ["?t"], {"t": u(tid)}, 1, None, db.dictionary, db.quoted_triple_store)
    assert db.dictionary.decode(int(col[0])) == case["subject_of_t"]
    ex = "http://example.org/"
    d, q = E.Dictionary(), E.QuotedTripleStore()
    s, p, o = (d.encode(ex + x) for x in ("alice", "knows", "bob"))
    col = E.ExecutionEngine._bind_host("TRIPLE", ["?s", "?p", "?o"], {"s": u(s), "p": u(p), "o": u(o)}, 1, None, d, q)
    db.dictionary, db.quoted_triple_store = d, q
    assert db.decode_term(int(col[0])) == f"<< {ex}alice {ex}knows {ex}bob >>"


def test_bind_abi_structs():
    import ctypes as C
    assert C.sizeof(c.KbBindSpec) == 48 and C.sizeof(c.KbBindInfo) == 32
