"""Set-semantic writes on the device (kb_store_insert, kb_store_remove, kb_store_remove_template) against the restatement in
tests/update_reference.py: per-triple flags, the stored set, the index kept alive, the segment count, and every refusal."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200 import engine
from tests import oracle_api as O
from tests.update_reference import RefDb, batch_insert, batch_remove, run_fixture_case

pytestmark = pytest.mark.gpu


def stored(ctx):
    s, p, o = ctx.store_download()
    rows = list(zip(s.tolist(), p.tolist(), o.tolist()))
    assert len(rows) == len(set(rows)), "the store holds a triple twice"
    return set(rows)


def cols(batch):
    a = np.array(batch, dtype=np.uint32).reshape(-1, 3)
    return a[:, 0], a[:, 1], a[:, 2]


@pytest.mark.parametrize("indexed", [False, True])
def test_seeded_mixed_batches_match_the_restatement(ctx, indexed):
    rng = np.random.default_rng(7 + indexed)
    # ids at both ends of the u32 domain next to small ones: 0 and 0xFFFFFFFE are ordinary ids
    pool_s = np.array([0, 1, 2, 3, 5, 8, 13, 0xFFFFFFFE, 0xFFFFFFFD, 1000], np.uint32)
    pool_p = np.array([0, 7, 9, 0xFFFFFFFE], np.uint32)

    def rand_batch(n):
        return [(int(rng.choice(pool_s)), int(rng.choice(pool_p)), int(rng.choice(pool_s))) for _ in range(n)]

    base = sorted(set(rand_batch(60)))
    ctx.store_load(*cols(base))
    want = set(base)
    if indexed:
        ctx.build_index()
    for step in range(40):
        batch = rand_batch(int(rng.integers(1, 30)))
        if rng.random() < 0.5:
            got = ctx.store_insert(*cols(batch), tag=int(rng.integers(0, 3)))
            exp = batch_insert(want, batch)
        else:
            got = ctx.store_remove(*cols(batch))
            exp = batch_remove(want, batch)
        assert got.tolist() == exp, f"step {step}"
        assert stored(ctx) == want, f"step {step}"
        assert ctx.store_size()[0] == len(want)
        if indexed:  # the index answers (?s P ?o) by itself: its chunks must hold exactly the stored triples of P
            for pred in pool_p.tolist():
                rel = ctx.scan([c.pattern(c.V(0), c.K(pred), c.V(1))])[0]
                rows = rel.to_numpy([0, 1])
                rel.free()
                assert sorted(map(tuple, rows.tolist())) == sorted((s, o) for s, p, o in want if p == pred), f"step {step}, predicate {pred}"


def test_remove_takes_every_stored_copy_and_evict_after_removes(ctx):
    # a bag built by appends: the same triple in two tagged segments
    ctx.store_load(*cols([(1, 1, 1), (2, 2, 2)]))
    ctx.store_append(*cols([(3, 3, 3), (1, 1, 1), (4, 4, 4)]), 5)
    ctx.store_append(*cols([(1, 1, 1), (6, 6, 6)]), 6)
    assert ctx.store_remove(*cols([(1, 1, 1), (1, 1, 1)])).tolist() == [True, False]
    assert stored(ctx) == {(2, 2, 2), (3, 3, 3), (4, 4, 4), (6, 6, 6)} and ctx.store_size()[0] == 4
    assert ctx.store_remove(*cols([(3, 3, 3)])).tolist() == [True]
    ctx.store_evict(5)  # what is left of tag 5 goes
    assert stored(ctx) == {(2, 2, 2), (6, 6, 6)}


def test_delete_then_insert_of_the_same_triple(ctx):
    ctx.store_load(*cols([(1, 2, 3)]))
    assert ctx.store_remove(*cols([(1, 2, 3)])).tolist() == [True]
    assert ctx.store_insert(*cols([(1, 2, 3), (1, 2, 3)])).tolist() == [True, False]
    assert stored(ctx) == {(1, 2, 3)}


def test_refusals_leave_the_store_unchanged(ctx):
    ctx.store_load(*cols([(1, 2, 3), (4, 5, 6)]))
    before = (ctx.store_size(), stored(ctx))
    for pos in range(3):
        bad = [[7, 8, 9], [1, 2, 3]]
        bad[1][pos] = c.KB_ID_NONE
        for call in (ctx.store_insert, ctx.store_remove):
            with pytest.raises(c.KolibrieError) as e:
                call(*cols(bad))
            assert e.value.status == c.KB_E_INVALID and ("subject", "predicate", "object")[pos] in str(e.value)
            assert (ctx.store_size(), stored(ctx)) == before
    n = C.c_uint64()
    assert c.lib().kb_store_insert(ctx.h, None, None, None, 1, 0, None, C.byref(n)) == c.KB_E_INVALID
    assert c.lib().kb_store_remove(ctx.h, None, None, None, 1, None, C.byref(n)) == c.KB_E_INVALID
    assert (ctx.store_size(), stored(ctx)) == before


def test_one_triple_inserts_stay_few_segments_and_upload_only_the_batch(ctx):
    ctx.store_load(*cols([(0, 0, 0)]))
    ctx.get_stats(reset=True)
    want = {(0, 0, 0)}
    for i in range(1000):
        h0 = ctx.get_stats()["h2d_bytes"]
        assert ctx.store_insert(*cols([(i + 1, 3, i)]), tag=9).tolist() == [True]
        assert ctx.get_stats()["h2d_bytes"] - h0 <= 12 + 64
        want.add((i + 1, 3, i))
    n, n_seg = ctx.store_size()
    assert n == 1001 and n_seg <= 12, n_seg
    assert stored(ctx) == want


def test_index_stays_alive_across_writes(ctx):
    d = datagen.employee_dataset(5000)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    rng = np.random.default_rng(3)
    rows = set(zip(d.s.tolist(), d.p.tolist(), d.o.tolist()))
    gone = [tuple(int(x) for x in t) for t in np.array(sorted(rows))[rng.choice(len(rows), 200, replace=False)]]
    ctx.store_remove(*cols(gone))
    rows -= set(gone)
    back = gone[:50]
    ctx.store_insert(*cols(back), tag=1)
    rows |= set(back)
    assert stored(ctx) == rows
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    n0 = ctx.get_stats()["index_joins"]
    got = ctx.star_join(js, pats, filt)
    assert ctx.get_stats()["index_joins"] > n0, "the star join left the index path"
    a = np.array(sorted(rows), dtype=np.uint32)
    want = O.Db(a[:, 0], a[:, 1], a[:, 2], d.num_or0, d.is_num).bgp(pats, filt)
    assert np.array_equal(datagen.canonical_rows(got.to_numpy(sorted(got.slots))), datagen.canonical_rows(want.to_numpy(sorted(want.slots))))


def test_remove_template_fills_from_the_relation(ctx):
    strings = ["a", "knows", "b", "c", "name", "Alice", "<<x>>", '"q"', "\u00a0x", "x\u3000"]
    ctx.dict_strings_load(strings)
    ctx.store_load(*cols([(0, 1, 2), (0, 1, 3), (0, 4, 5), (6, 1, 2)]))
    rel = ctx.rel_from_host([0, 1], [np.array([0, 0], np.uint32), np.array([2, 3], np.uint32)])
    tmpl = [c.pattern(c.V(0), c.K(1), c.V(1)), c.pattern(c.V(1), c.K(1), c.V(0))]
    assert ctx.store_remove_template(rel, tmpl) == 2
    assert stored(ctx) == {(0, 4, 5), (6, 1, 2)}
    before = stored(ctx)
    refusals = [
        (rel, [c.pattern(c.V(0), c.K(1), c.V(7))]),                                          # not a slot of rel
        (ctx.rel_from_host([0], [np.array([0, c.KB_ID_NONE], np.uint32)]), [c.pattern(c.V(0), c.K(4), c.K(5))]),  # unbound
        (ctx.rel_from_host([0], [np.array([6], np.uint32)]), [c.pattern(c.V(0), c.K(1), c.K(2))]),    # "<<x>>" re-encodes otherwise
        (ctx.rel_from_host([0], [np.array([7], np.uint32)]), [c.pattern(c.K(0), c.K(4), c.V(0))]),    # a quoted literal too
        (ctx.rel_from_host([0], [np.array([0x80000000], np.uint32)]), [c.pattern(c.V(0), c.K(1), c.K(2))]),
        (ctx.rel_from_host([0], [np.array([99], np.uint32)]), [c.pattern(c.V(0), c.K(1), c.K(2))]),   # no string for the id
        (ctx.rel_from_host([0], [np.array([8], np.uint32)]), [c.pattern(c.V(0), c.K(1), c.K(2))]),    # str::trim strips U+00A0
        (ctx.rel_from_host([0], [np.array([9], np.uint32)]), [c.pattern(c.V(0), c.K(1), c.K(2))]),    # and U+3000
    ]
    for r, t in refusals:
        with pytest.raises(c.KolibrieError) as e:
            ctx.store_remove_template(r, t)
        assert e.value.status == c.KB_E_UNSUPPORTED
        assert stored(ctx) == before


def test_engine_handle_update_matches_the_restatement(ctx):
    db = engine.SparqlDatabase(ctx)
    ref = RefDb()
    A, B, Cc, D = "<http://example.org/a>", "<http://example.org/b>", "<http://example.org/c>", "<http://example.org/d>"
    q = f"<< {A} {B} {Cc} >>"
    steps = [
        ("INSERT", [(A, B, Cc)]),
        ("INSERT", [(q, "<http://example.org/src>", D), (A, B, Cc), (A, B, '"12.5"')]),
        ("DELETE", [(A, B, Cc), (A, B, "<http://example.org/never>")]),
        ("INSERT", [(f"<< {q} {B} \"x y\" >>", B, D)]),
        ("DELETE", [(q, "<http://example.org/src>", D)]),
        ("LOAD", [(A, B, Cc)]),
    ]
    for kind, triples in steps:
        assert db.handle_update(kind, triples) == ref.handle_update(kind, triples)
        assert db.triples == ref.triples
        assert db.dictionary.id_to_string == ref.id_to_string
        assert db.quoted_triple_store.components_to_id == ref.qt_to_id
        assert db._uploaded_version == db._version
        assert stored(ctx) == ref.triples
    assert ctx.dict_strings_info()[0] == len(ref.id_to_string)


FIXTURE = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "update", "update.json")))


def load_engine(db, data):
    """parse_ntriples_and_add of a fixture's data on the engine (the ids RefDb.load gives)"""
    def enc(x):
        return db.quoted_triple_store.encode(*[enc(y) for y in x]) if isinstance(x, list) else db.dictionary.encode(x)
    for s, p, o in data:
        db.add_triple((enc(s), enc(p), enc(o)))


@pytest.mark.parametrize("case", FIXTURE["cases"], ids=lambda x: x["name"])
def test_engine_passes_the_reference_update_tests(ctx, case):
    db = engine.SparqlDatabase(ctx)
    load_engine(db, case["data"])
    ref = RefDb()
    ref.load(case["data"])
    run_fixture_case(db, case)
    run_fixture_case(ref, case)
    assert db.triples == ref.triples and db.dictionary.id_to_string == ref.id_to_string
    assert stored(ctx) == ref.triples


EX = "http://example.org/"
DATA = [[EX + "a", EX + "knows", EX + "b"], [EX + "a", EX + "knows", EX + "c"], [EX + "b", EX + "knows", 'say "hi"'],
        [EX + "a", EX + "age", "42"], [[EX + "a", EX + "knows", EX + "b"], EX + "source", EX + "doc"]]


@pytest.mark.parametrize("template,where,insert", [
    ([["?s", "<" + EX + "knows>", "?o"]], [["?s", "<" + EX + "knows>", "?o"]], None),                  # device path
    ([["?o", "<" + EX + "knows>", "?s"], ["?s", "<" + EX + "age>", '"42"']], [["?s", "<" + EX + "knows>", "?o"]], None),
    ([["?s", "<" + EX + "knows>", "?o"]], [["?s", "<" + EX + "knows>", "?o"]], [["?s", "<" + EX + "p>", "<" + EX + "q>"]]),  # INSERT literal
    ([["?s", "<" + EX + "never>", "<" + EX + "unknown>"]], [["?s", "<" + EX + "knows>", "?o"]], None),  # unknown terms join the dictionary
    ([["?s", "<" + EX + "knows>", "?o"]], [["?s", "<" + EX + "nothing>", "?o"]], None),                 # no rows: nothing is encoded
    ([["?x", "<" + EX + "source>", "<" + EX + "doc>"]], [["?x", "<" + EX + "source>", "?d"]], None),     # quoted binding: the host loop
    ([["?s", "<" + EX + "knows>", "?o"]], [["<" + EX + "b>", "<" + EX + "knows>", "?o"], ["?s", "<" + EX + "knows>", "<" + EX + "b>"]], None),
    ([["?s", "?p", "?z"]], [["?s", "?p", "?o"]], None),                                                    # ?z unbound: the host loop
])
def test_engine_delete_where_matches_the_restatement(ctx, template, where, insert):
    db = engine.SparqlDatabase(ctx)
    load_engine(db, DATA)
    db.build_all_indexes()
    ref = RefDb()
    ref.load(DATA)
    db.execute_delete_where(template, where, insert)
    ref.execute_delete_where(template, where, insert)
    assert db.triples == ref.triples
    assert db.dictionary.id_to_string == ref.id_to_string
    assert db.quoted_triple_store.components_to_id == ref.qt_to_id
    assert stored(ctx) == ref.triples


def test_cfg3_store_mixed_updates_then_delete_of_a_predicate(ctx):
    """the 100 M-triple store of BASELINE config 3: 1,000 mixed one-triple updates, then the DELETE of one predicate's 16.7 M triples
    (the WHERE's rows as one kb_store_remove batch), checked by digest against the generated arrays; the star join stays on the index"""
    d = datagen.employee_dataset(16_666_667)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    rng = np.random.default_rng(11)
    big = int(max(d.s.max(), d.o.max())) + 1
    keep = np.ones(len(d.s), bool)
    extra = set()
    loaded_removed = rng.choice(len(d.s), 10, replace=False)
    for i in range(1000):
        if i % 100 == 99:  # a loaded triple
            j = int(loaded_removed[i // 100])
            t = (int(d.s[j]), int(d.p[j]), int(d.o[j]))
            assert ctx.store_remove(*cols([t])).tolist() == [True]
            keep[j] = False
        elif i % 2 == 0 or not extra:
            t = (big + i, int(d.p[0]), big + i)
            assert ctx.store_insert(*cols([t]), tag=3).tolist() == [True]
            extra.add(t)
        else:
            t = extra.pop()
            assert ctx.store_remove(*cols([t])).tolist() == [True]
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    P = sorted(set(np.unique(d.p).tolist()) - {pt.p.value for pt in pats})[0]
    rel = ctx.scan([c.pattern(c.V(0), c.K(P), c.V(1))])[0]
    rows = rel.to_numpy([0, 1])
    rel.free()
    assert len(rows) == int(((d.p == P) & keep).sum())
    assert int(ctx.store_remove(rows[:, 0], np.full(len(rows), P, np.uint32), rows[:, 1]).sum()) == len(rows)
    keep &= d.p != P

    def digest(s, p, o):
        h = (s.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) ^ (p.astype(np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F)) ^ o.astype(np.uint64)
        return len(s), int(np.bitwise_xor.reduce(h)), int(h.sum(dtype=np.uint64))

    e = np.array(sorted(extra), np.uint32).reshape(-1, 3)
    want = digest(np.concatenate([d.s[keep], e[:, 0]]), np.concatenate([d.p[keep], e[:, 1]]), np.concatenate([d.o[keep], e[:, 2]]))
    s, p, o = ctx.store_download()
    assert digest(s, p, o) == want
    n0 = ctx.get_stats()["index_joins"]
    got = ctx.star_join(js, pats, filt)
    assert ctx.get_stats()["index_joins"] > n0, "the star join left the index path"
    got.free()
    ctx.store_clear()
