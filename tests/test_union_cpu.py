"""CPU: the union / par_join transcription (tests/union_reference.py) pinned to hand-worked cases, and the engine's host restatement
(SparqlDatabase.union / par_join on a context without kb_store_union / kb_store_par_join) held to the transcription."""
import pytest

from kolibrie_b200 import engine as E
from tests import union_reference as R
from tests.oracle_ctx import OracleCtx

Q = R.QUOTED_TRIPLE_ID_BIT


def db(strings, triples, quoted=()):
    return R.Db(triples, R.Dictionary(strings), quoted)


# name: (a strings, a triples, b strings, b triples, expected dictionary strings, expected triples)
UNION_CASES = {
    "disjoint": (["a", "p", "b"], [(0, 1, 2)], ["x", "q", "y"], [(0, 1, 2)],
                 ["a", "p", "b", "x", "q", "y"], [(0, 1, 2), (3, 4, 5)]),
    "overlapping": (["a", "p", "b"], [(0, 1, 2)], ["p", "c", "a"], [(1, 0, 2)],
                    ["a", "p", "b", "c"], [(0, 1, 2), (3, 1, 0)]),
    "identical": (["a", "p", "b"], [(0, 1, 2)], ["a", "p", "b"], [(0, 1, 2), (2, 1, 0)],
                  ["a", "p", "b"], [(0, 1, 2), (2, 1, 0)]),
    # "s" is id 0 in a and id 1 in b; "t" is id 1 in a and id 0 in b
    "swapped ids": (["s", "t", "p"], [(0, 2, 1)], ["t", "s", "p"], [(0, 2, 1)],
                    ["s", "t", "p"], [(0, 2, 1), (1, 2, 0)]),
    "empty a": (["a"], [], ["x", "p", "y"], [(2, 1, 0)], ["a", "y", "p", "x"], [(1, 2, 3)]),
    "empty a dictionary": ([], [], ["x", "p", "y"], [(0, 1, 2)], ["x", "p", "y"], [(0, 1, 2)]),
    "empty b": (["a", "p", "b"], [(0, 1, 2)], ["zz"], [], ["a", "p", "b"], [(0, 1, 2)]),
    # b's set in (s, p, o) order of b's ids: (0,1,2), (0,3,4) — "P" is first seen in predicate position, "O" in object position
    "first seen in p and o": (["a"], [], ["s", "P", "O", "Q", "R"], [(0, 3, 4), (0, 1, 2)],
                              ["a", "s", "P", "O", "Q", "R"], [(1, 2, 3), (1, 4, 5)]),
    # an id of b that never occurs in b's triples gets no id in the union
    "unused b string": (["a"], [(0, 0, 0)], ["u", "v"], [(1, 1, 1)], ["a", "v"], [(0, 0, 0), (1, 1, 1)]),
    # a's quoted ids are copied as they are
    "quoted in a": (["a", "p"], [(Q, 1, 0), (0, 1, Q | 1)], ["p", "b"], [(1, 0, 1)],
                    ["a", "p", "b"], [(Q, 1, 0), (0, 1, Q | 1), (2, 1, 2)]),
}


@pytest.mark.parametrize("case", sorted(UNION_CASES))
def test_union_hand_worked(case):
    sa, ta, sb, tb, want_strings, want = UNION_CASES[case]
    a, b = db(sa, ta), db(sb, tb)
    a_before = (set(a.triples), a.dictionary.strings())
    got = R.union(a, b)
    assert got.dictionary.strings() == want_strings
    assert got.dictionary.next_id == len(want_strings)
    assert got.triples == set(want)
    assert (a.triples, a.dictionary.strings()) == a_before  # a's dictionary is cloned, not changed
    assert got.quoted is a.quoted


@pytest.mark.parametrize("bad", [(0, 1, Q), (Q | 5, 1, 0), (0, 7, 1)], ids=["quoted object", "quoted subject", "id past the dictionary"])
def test_union_panics_on_ids_without_a_string(bad):
    a = db(["a"], [(0, 0, 0)])
    b = db(["x", "p"], [(0, 1, 0), bad])
    with pytest.raises(R.Panic):
        R.union(a, b)


def test_encode_asserts_below_bit_31():
    d = R.Dictionary(["a"])
    d.next_id = Q
    assert d.encode("a") == 0
    with pytest.raises(R.Panic):
        d.encode("b")


# name: (a triples, b triples, expected); a's dictionary holds "p" = 0 and "q" = 1, the predicate is "p"
PAR_CASES = {
    "key on subject": ([(10, 0, 11)], [(11, 0, 12)], [(10, 0, 12)]),
    "key on object": ([(10, 0, 11)], [(13, 0, 11)], [(10, 0, 11)]),
    "key on both": ([(10, 0, 11)], [(11, 0, 12), (13, 0, 11)], [(10, 0, 11), (10, 0, 12)]),
    "s == o in b": ([(10, 0, 11)], [(11, 0, 11)], [(10, 0, 11)]),
    "s == o in a": ([(11, 0, 11)], [(11, 0, 12)], [(11, 0, 12)]),
    "other predicate": ([(10, 1, 11), (10, 0, 11)], [(11, 1, 12), (11, 0, 13)], [(10, 0, 13)]),
    "no match": ([(10, 0, 11)], [(12, 0, 13)], []),
    "fan-out": ([(1, 0, 5), (2, 0, 5)], [(5, 0, 6), (5, 0, 7), (8, 0, 5)], [(1, 0, 5), (1, 0, 6), (1, 0, 7), (2, 0, 5), (2, 0, 6), (2, 0, 7)]),
}


@pytest.mark.parametrize("case", sorted(PAR_CASES))
def test_par_join_hand_worked(case):
    ta, tb, want = PAR_CASES[case]
    a, b = db(["p", "q"], ta), db(["zz"], tb)
    got = R.par_join(a, b, "p")
    assert got.triples == set(want)
    assert got.dictionary is a.dictionary and a.dictionary.strings() == ["p", "q"]


def test_par_join_with_a_new_predicate_adds_one_string():
    a, b = db(["p"], [(0, 0, 0)]), db(["p"], [(0, 0, 0)])
    got = R.par_join(a, b, "new")
    assert got.triples == set()
    assert a.dictionary.strings() == ["p", "new"] and got.dictionary is a.dictionary


# ---- the engine's host restatement (a context without the entry points) against the transcription
def engine_db(strings, triples, quoted=None):
    d = E.SparqlDatabase(ctx=OracleCtx())
    for s in strings:
        d.dictionary.encode(s)
    for t in triples:
        d.add_triple(tuple(t))
    if quoted:
        for comp in quoted:
            d.quoted_triple_store.encode(*comp)
    return d


@pytest.mark.parametrize("case", sorted(UNION_CASES))
def test_engine_union_host_path(case):
    sa, ta, sb, tb, _, _ = UNION_CASES[case]
    want = R.union(db(sa, ta), db(sb, tb))
    a, b = engine_db(sa, ta, quoted=[(0, 0, 0)]), engine_db(sb, tb)
    a.set_prefixes([("ex", "http://example.org/")])
    got = a.union(b)
    assert got.triples == want.triples
    assert got.dictionary.id_to_string == want.dictionary.strings()
    assert got.dictionary.string_to_id == want.dictionary.string_to_id
    assert a.dictionary.id_to_string == sa  # a's dictionary is cloned
    assert got.quoted_triple_store is a.quoted_triple_store and got.prefixes == a.prefixes
    assert got.ctx is not a.ctx


def test_engine_union_refuses_what_the_reference_panics_on():
    a, b = engine_db(["a"], [(0, 0, 0)]), engine_db(["x"], [(0, 0, Q)])
    with pytest.raises(ValueError):
        a.union(b)
    assert a.triples == {(0, 0, 0)} and a.dictionary.id_to_string == ["a"]


@pytest.mark.parametrize("case", sorted(PAR_CASES))
def test_engine_par_join_host_path(case):
    ta, tb, _ = PAR_CASES[case]
    want = R.par_join(db(["p", "q"], ta), db(["zz"], tb), "p")
    a, b = engine_db(["p", "q"], ta), engine_db(["zz"], tb)
    got = a.par_join(b, "p")
    assert got.triples == want.triples
    assert got.dictionary is a.dictionary and got.quoted_triple_store is a.quoted_triple_store
    a.dictionary.encode("later")
    assert got.dictionary.lookup("later") is not None  # the dictionary is shared, as the Arc is


def test_engine_par_join_new_predicate_and_self():
    a = engine_db(["p"], [(0, 0, 0)])
    got = a.par_join(a, "new")
    assert got.triples == set() and a.dictionary.id_to_string == ["p", "new"]
    got = a.par_join(a, "p")
    assert got.triples == R.par_join(db(["p"], [(0, 0, 0)]), db(["p"], [(0, 0, 0)]), "p").triples == {(0, 0, 0)}
