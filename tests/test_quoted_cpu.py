"""CPU: the host restatement of resolve_quoted_triple_scan (ExecutionEngine._scan_quoted over the oracle) against a literal, brute-force
transcription of engine.rs:1111-1188, and SparqlDatabase.decode_term against a restatement of Dictionary::decode_term
(dictionary.rs:60-72, "unknown" per engine.rs:42-43), on seeded random RDF-star stores. These pin the reference the GPU tests of
kb_scan_quoted and of the quoted decode compare the device with."""
import numpy as np
import pytest

from kolibrie_b200 import engine as E
from tests import quoted_cases as Q
from tests.oracle_ctx import OracleCtx


def oracle_db():
    return E.SparqlDatabase(ctx=OracleCtx())


@pytest.mark.parametrize("seed", range(12))
def test_host_quoted_scan_matches_the_entry_by_entry_transcription(seed):
    rng = np.random.default_rng(seed)
    db = oracle_db()
    Q.random_store(db, rng, n_quoted=int(rng.integers(1, 60)), n_triples=int(rng.integers(1, 160)))
    db._sync()
    for _ in range(25):
        pat = Q.random_pattern(db, rng)
        db._uploaded_version = db._version  # encoding the pattern's constants does not change the triples
        got = E.ExecutionEngine.execute_with_ids(E.TableScan(pat), db)
        assert Q.bag(got) == Q.bag(Q.brute_quoted_scan(db, pat)), pat


def test_both_positions_quoted_take_one_entry():
    """<< ?x p ?y >> q << ?y p ?x >>: ONE entry fills both positions (engine.rs:1135-1163), so only an entry with x == y qualifies"""
    db = oracle_db()
    db.add_statement(("a", "p", "b"), "q", ("a", "p", "b"))
    db.add_statement(("a", "p", "a"), "q", ("a", "p", "a"))
    db.add_statement(("b", "p", "a"), "q", ("a", "p", "b"))
    d = db.dictionary
    x, y = E.Variable("?x"), E.Variable("?y")
    pat = (E.QuotedTriple(x, E.Constant(d.lookup("p")), y), E.Constant(d.lookup("q")), E.QuotedTriple(y, E.Constant(d.lookup("p")), x))
    db._sync()
    got = E.ExecutionEngine.execute_with_ids(E.TableScan(pat), db)
    assert got == [{"x": d.lookup("a"), "y": d.lookup("a")}]
    assert Q.bag(got) == Q.bag(Q.brute_quoted_scan(db, pat))


def test_empty_quoted_store_gives_no_rows():
    db = oracle_db()
    db.add_triple_parts("a", "p", "b")
    db._sync()
    pat = (E.QuotedTriple(E.Variable("?x"), E.Variable("?y"), E.Variable("?z")), E.Variable("?p"), E.Variable("?o"))
    assert E.ExecutionEngine.execute_with_ids(E.TableScan(pat), db) == [] == Q.brute_quoted_scan(db, pat)


@pytest.mark.parametrize("seed", range(6))
def test_decode_term_matches_the_restatement(seed):
    rng = np.random.default_rng(100 + seed)
    db = oracle_db()
    qids = Q.random_store(db, rng, n_quoted=80, max_depth=5)
    qts = db.quoted_triple_store
    # dangling components: an entry whose component is an id neither table holds decodes to "unknown" as a whole
    dang = qts.encode(qids[0], db.dictionary.encode("t1"), 12345)
    dang2 = qts.encode(0x8000_7777, qids[1], qids[2])
    ids = list(qids) + [dang, dang2, qts.encode(dang, qids[3], qids[4]), 0x8000_0000 + 5000, 0, 3, 999999]
    for i in ids:
        want = Q.decode_term_ref(db, i)
        assert (db.decode_term(i) or "unknown") == want
        if i & Q.QBIT and want != "unknown":
            assert want.startswith("<< ") and want.endswith(" >>")
