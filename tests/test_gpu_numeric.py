"""GPU (-m gpu): the numeric side tables derived on the device (kb_dict_numeric_derive) against the host loops they replace
(Dictionary.numeric_table for num_or0 / is_num, the rust_parse_i32 loop for the legacy i32 view), bit for bit: the parse corpus of
tests/numparse_corpus.py, incremental derives across kb_dict_encode batches and a CONCAT, the refusals, what a derive voids, the mirror's
paths with and without the device derive, the per-firing upload of a window, and the full-size employee dictionary. The tests run on
contexts of their own, so no derived table reaches the session context."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200 import engine as E
from tests import numparse_corpus as NC

pytestmark = pytest.mark.gpu

BOTH = c.NUMERIC_F64 | c.NUMERIC_I32


@pytest.fixture(scope="module")
def nctx():
    ctx = c.Context(0)
    yield ctx
    ctx.close()


@pytest.fixture(scope="module")
def hctx():
    """a second context for the host-loop side of the mirror comparisons"""
    ctx = c.Context(0)
    yield ctx
    ctx.close()


class NoDerive:
    """the same context without kb_dict_numeric_derive: the mirror takes the host loops"""

    def __init__(self, ctx):
        self._ctx = ctx

    def __getattr__(self, k):
        if k == "dict_numeric_derive":
            raise AttributeError(k)
        return getattr(self._ctx, k)


def host_tables(strings):
    d = E.Dictionary()
    d.id_to_string = list(strings)
    num, isn = d.numeric_table()
    val = np.zeros(len(strings), np.int32)
    isi = np.zeros(len(strings), np.uint8)
    for i, s in enumerate(strings):
        v = E.rust_parse_i32(s)
        if v is not None:
            val[i], isi[i] = v, 1
    return num.view(np.uint64), isn, val, isi


def assert_tables(ctx, strings):
    num, isn, val, isi = ctx.dict_numeric_download(0, len(strings), f64=True, i32=True)
    hnum, hisn, hval, hisi = host_tables(strings)
    bad = np.nonzero((num.view(np.uint64) != hnum) | (isn != hisn))[0]
    assert not len(bad), [(strings[i][:60], hex(int(num.view(np.uint64)[i])), hex(int(hnum[i]))) for i in bad[:8]]
    bad = np.nonzero((val != hval) | (isi != hisi))[0]
    assert not len(bad), [(strings[i][:60], int(val[i]), int(hval[i])) for i in bad[:8]]


def test_corpus_parity_with_the_host_loops(nctx):
    strings = NC.corpus()
    nctx.dict_strings_load(strings)
    nctx.get_stats(reset=True)
    info = nctx.dict_numeric_derive(BOTH, 0)
    st = nctx.get_stats(reset=True)
    assert st["h2d_bytes"] == 0 and st["other_launches"] >= 1
    bits, isn, val, isi = NC.reference(strings)
    assert info["n_ids"] == info["n_derived"] == len(strings)
    assert info["n_numeric"] == int(isn.sum()) and info["n_i32"] == int(isi.sum()) and info["n_slow"] > 0
    num, dn, dv, di = nctx.dict_numeric_download(0, len(strings), f64=True, i32=True)
    bad = np.nonzero((num.view(np.uint64) != bits) | (dn != isn))[0]
    assert not len(bad), [(strings[i][:60], hex(int(num.view(np.uint64)[i])), hex(int(bits[i]))) for i in bad[:8]]
    assert np.array_equal(dv, val) and np.array_equal(di, isi)
    # and equal to what Dictionary.numeric_table uploads (the same loop as NC.reference)
    d = E.Dictionary()
    d.id_to_string = strings
    hnum, hisn = d.numeric_table()
    assert np.array_equal(num.view(np.uint64), hnum.view(np.uint64)) and np.array_equal(dn, hisn)


def test_incremental_derive_equals_a_full_derive(nctx):
    strings = NC.corpus(seed=7, scale=0.02)
    rng = np.random.default_rng(3)
    d = E.Dictionary()
    nctx.dict_strings_load([])
    nctx.dict_numeric_load([], [])
    nctx.dict_legacy_i32_load([], [])
    cuts = sorted(rng.choice(len(strings), 5, replace=False).tolist())
    for a, b in zip([0] + cuts, cuts + [len(strings)]):
        d.encode_bulk(nctx, strings[a:b])
        info = nctx.dict_numeric_derive(BOTH, c.NUMERIC_APPEND)
        assert info["n_ids"] == len(d.id_to_string)
    assert_tables(nctx, d.id_to_string)
    # a CONCAT creates strings on the device (numeric ones among them: "<number>5")
    ids = np.array([i for i, s in enumerate(d.id_to_string) if E.rust_parse_f64(s) is not None][:500], np.uint32)
    rel = nctx.rel_from_host([0], [ids])
    _, info = nctx.bind(rel, c.BIND_CONCAT, [c.V(0), c.K(0)], 1, 0, [b"5"])
    assert info["dict_new"] > 0
    d.id_to_string += nctx.dict_strings_download(info["dict_first"], info["dict_new"])
    inc = nctx.dict_numeric_derive(BOTH, c.NUMERIC_APPEND)
    assert inc["n_derived"] == info["dict_new"]
    got = nctx.dict_numeric_download(0, len(d.id_to_string), True, True)
    assert_tables(nctx, d.id_to_string)
    full = nctx.dict_numeric_derive(BOTH, 0)
    assert full["n_derived"] == len(d.id_to_string)
    again = nctx.dict_numeric_download(0, len(d.id_to_string), True, True)
    assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(got, again))
    # an append after a host load keeps the loaded entries
    nctx.dict_numeric_load(np.full(10, 7.0), np.ones(10, np.uint8))
    nctx.dict_numeric_derive(c.NUMERIC_F64, c.NUMERIC_APPEND)
    num, isn = nctx.dict_numeric_download(0, len(d.id_to_string))
    assert (num[:10] == 7.0).all() and isn[:10].all()
    hnum, hisn, _, _ = host_tables(d.id_to_string[10:])
    assert np.array_equal(num[10:].view(np.uint64), hnum) and np.array_equal(isn[10:], hisn)


def test_refusals_leave_the_tables_unchanged(nctx):
    strings = ["1", "x", "2.5", "-3", "nan", "abc", "7e1", "+8", "0", "y"]
    nctx.dict_strings_load(strings)
    nctx.dict_numeric_derive(BOTH, 0)
    nctx.dict_encode(["11", "12", "13", "z", "15"])
    assert nctx.dict_strings_info()[0] == 15
    before = nctx.dict_numeric_download(0, 10, True, True)

    def refused(tables, first):
        with pytest.raises(c.KolibrieError) as e:
            nctx.dict_numeric_derive(tables, first)
        assert e.value.status == c.KB_E_INVALID
        after = nctx.dict_numeric_download(0, 10, True, True)
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(before, after))
        with pytest.raises(c.KolibrieError):  # the tables still hold 10 ids
            nctx.dict_numeric_download(0, 11, True, True)

    refused(c.NUMERIC_F64, 11)   # a hole: the table holds 10
    refused(c.NUMERIC_I32, 12)
    refused(BOTH, 16)            # past the dictionary
    for bad in (0, 4, c.NUMERIC_F64 | 8, 0x80000000):
        refused(bad, 0)
    info = nctx.dict_numeric_derive(BOTH, c.NUMERIC_APPEND)
    assert info["n_derived"] == 5 and info["n_numeric"] == 4 and info["n_i32"] == 4
    with pytest.raises(c.KolibrieError):
        nctx.dict_numeric_derive(c.NUMERIC_F64, 16)
    assert nctx.dict_numeric_derive(c.NUMERIC_F64, 15)["n_derived"] == 0  # nothing to add


def employee_strings(d):
    """the employee dictionary as strings: the salary literals (the ids is_num marks) print as integers, every other id as a name"""
    out = np.array(["ex:t%d" % i for i in range(d.n_ids)], dtype=object)
    k = np.nonzero(d.is_num)[0]
    out[k] = [str(int(v)) for v in d.num_or0[k]]
    return out.tolist()


def test_versioning_like_a_load(nctx):
    d = datagen.employee_dataset(20000)
    nctx.store_load(d.s, d.p, d.o)
    nctx.dict_strings_load(employee_strings(d))
    nctx.dict_numeric_derive(c.NUMERIC_F64, 0)
    nctx.build_index()
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    plan = nctx.prepare_star_join(js, pats, filt, ring=1)
    plan.collect(plan.submit())
    nctx.dict_numeric_derive(c.NUMERIC_I32, 0)  # the i32 view voids nothing
    plan.collect(plan.submit())
    nctx.dict_numeric_derive(c.NUMERIC_F64, c.NUMERIC_APPEND)
    with pytest.raises(c.KolibrieError) as e:
        plan.submit()
    assert e.value.status == c.KB_E_INVALID and "stale" in e.value.message
    plan.free()
    # the closed-store token: voided only when a rule filter compares numbers
    PAR, ANC = 3, 4
    nctx.dict_strings_load([str(i) for i in range(16)])
    nctx.dict_numeric_derive(c.NUMERIC_F64, 0)
    nctx.store_clear()
    nctx.store_append(np.array([1, 2], np.uint32), np.array([PAR, PAR], np.uint32), np.array([2, 3], np.uint32), 1)
    V, K = c.V, c.K
    plain = [{"premise": [c.pattern(V(0), K(PAR), V(1))], "conclusion": [c.pattern(V(0), K(ANC), V(1))], "filters": []}]
    numeric = [dict(plain[0], filters=[c.KbRuleFilter(0, c.CMP_GT, 0, 0, 1.0)])]
    nctx.datalog_fixpoint(plain)
    nctx.dict_numeric_derive(c.NUMERIC_F64, 0)
    nctx.datalog_maintain(plain, [], np.array([[3, PAR, 4]], np.uint32), 2)
    nctx.store_evict(c.KB_TAG_INFERRED)
    nctx.datalog_fixpoint(numeric)
    nctx.dict_numeric_derive(c.NUMERIC_F64, 0)
    with pytest.raises(c.KolibrieError) as e:
        nctx.datalog_maintain(numeric, [], np.array([[4, PAR, 5]], np.uint32), 3)
    assert e.value.status == c.KB_E_INVALID
    nctx.store_clear()


# ------------------------------------------------------------------------------------------------ the mirror with and without it
def salary_rows(rng, k0, n):
    return [(f"ex:e{k}", "ex:salary", [str(int(rng.integers(0, 200))), f"{rng.integers(0, 200)}.5", "n/a", "1e2", "-7"][k % 5]) for k in range(k0, k0 + n)]


def test_sparql_database_and_reasoner_answers_are_unchanged(nctx, hctx):
    rng = np.random.default_rng(11)
    rows = salary_rows(rng, 0, 400)
    res = []
    for ctx in (nctx, NoDerive(hctx)):
        db = E.SparqlDatabase(ctx=ctx)
        for t in rows:
            db.add_triple_parts(*t)
        V, K = E.Variable, E.Constant
        sal = K(db.dictionary.encode("ex:salary"))
        q = E.Filter(E.TableScan((V("?e"), sal, V("?s"))), E.Condition(E.Or(E.Comparison("?s", ">", "120"), E.Comparison("?s", "<=", "3.5"))))
        a = sorted(tuple(sorted(r.items())) for r in E.ExecutionEngine.execute(q, db))
        r = E.Reasoner(ctx=ctx)
        for t in rows[:200]:
            r.add_abox_triple(*t)
        rule = E.Rule([(V("?e"), K(r.dictionary.encode("ex:salary")), V("?s"))], [(V("?e"), K(r.dictionary.encode("ex:high")), V("?s"))],
                      [E.FilterCondition("?s", ">", "100")])
        r.add_rule(rule)
        first = sorted(r.infer_new_facts_semi_naive())
        seeds = []
        for k in range(3):  # incremental seeds that bring new literals
            for t in salary_rows(np.random.default_rng(100 + k), 1000 + 50 * k, 50):
                r.add_abox_triple(*t)
            seeds.append(sorted(r.infer_new_facts_incremental()))
        res.append((a, first, seeds, list(r.dictionary.id_to_string)))
    assert res[0] == res[1]
    assert res[0][0] and res[0][1] and all(res[0][2])


def test_legacy_executor_answers_are_unchanged(nctx, hctx):
    from tests.test_legacy_path import QUERIES, employee4_triples, bag

    fx, tr = employee4_triples()
    for k in range(60):
        tr += [(f"http://example.org/gen{k}", "https://data.cityofchicago.org/resource/xzkq-xp2w/annual_salary", ["70000", "-12", "80000.5", "2147483648"][k % 4])]
    for what, patterns, filters in QUERIES:
        got = []
        for ctx in (nctx, NoDerive(hctx)):
            db = E.SparqlDatabase(ctx=ctx)
            for t in tr:
                db.add_triple_parts(*t)
            keys = sorted({t for pt in patterns for t in (pt[0], pt[2]) if t.startswith("?")})
            got.append(bag(E.LegacyExecutor(db).execute_bgp(patterns, filters), keys))
        assert got[0] == got[1], what


def window_run(ctx, firings):
    w = E.SimpleR2R(ctx=ctx)
    d = w.item.dictionary
    V, K = E.Variable, E.Constant
    sal, high = d.encode("ex:salary"), d.encode("ex:high")
    w.add_reasoning_rules([E.Rule([(V("?e"), K(sal), V("?s"))], [(V("?e"), K(high), V("?s"))], [E.FilterCondition("?s", ">", "100")])])
    q = E.Filter(E.TableScan((V("?e"), K(sal), V("?s"))), E.Condition(E.Comparison("?s", ">=", "50")))
    out, uploads, prev = [], [], []
    for rows in firings:
        for t in prev:
            w.remove(t)
        n0 = len(d.id_to_string)
        cur = [(d.encode(s), d.encode(p), d.encode(o)) for s, p, o in rows]
        for t in cur:
            w.add(t)
        added = d.id_to_string[n0:]
        ctx.get_stats(reset=True)
        w._load_tables()
        uploads.append((ctx.get_stats(reset=True)["h2d_bytes"], added))
        out.append((w.materialize(), sorted(tuple(sorted(r.items())) for r in w.execute_query(q)), w.last_mode))
        prev = cur
    return out, uploads


def test_window_sequence_answers_and_uploads(nctx, hctx):
    firings = [salary_rows(np.random.default_rng(k), 40 * k, 80) for k in range(5)]
    nctx.store_clear()
    hctx.store_clear()
    dev, up = window_run(nctx, firings)
    host, _ = window_run(NoDerive(hctx), firings)
    assert dev == host
    assert any(m[0] for m in dev) and all(m[1] for m in dev)  # (the rule filter compares numbers and every firing adds literals: each
    # derive voids the closed store, as a load does, and the window is closed again by a fixpoint on both sides)
    for i, (h2d, added) in enumerate(up[1:], 1):  # a firing uploads the strings it added (bytes + offsets), nothing per dictionary id
        assert added, i
        assert h2d == sum(len(s.encode()) for s in added) + 8 * (len(added) + 1), (i, h2d, len(added))
    nctx.store_clear()
    hctx.store_clear()


def test_filter_and_join_over_a_concat_output_run_on_the_device(nctx):
    db = E.SparqlDatabase(ctx=nctx)
    for k in range(300):
        db.add_triple_parts(f"ex:e{k}", "ex:salary", str(k % 23))
        db.add_triple_parts(f"ex:e{k}", "ex:dept", f"d{k % 5}")
    db.add_triple_parts("ex:x", "ex:code", "75")
    db.add_triple_parts("ex:y", "ex:code", "225")
    V, K = E.Variable, E.Constant
    enc = db.dictionary.encode
    scan = E.TableScan((V("?e"), K(enc("ex:salary")), V("?s")))
    bind = E.Bind(scan, "CONCAT", ["?s", "\"5\""], "?c")
    plan = E.Filter(bind, E.Condition(E.Comparison("?c", ">", "100")))
    nctx.get_stats(reset=True)
    rows = E.ExecutionEngine.execute(plan, db)
    assert nctx.get_stats()["filter_launches"] >= 1  # kb_filter over the BIND output, no KB_E_UNSUPPORTED
    # the host restatement: _bind_host over the scan's columns, then rust_parse_f64 of the output strings
    d2 = E.Dictionary()
    for t in db.dictionary.id_to_string:
        d2.encode(t)
    srel = nctx.scan([c.pattern(c.V(0), c.K(enc("ex:salary")), c.V(1))])[0]
    e_col, s_col = srel.column(srel.slots.index(0)), srel.column(srel.slots.index(1))
    out = E.ExecutionEngine._bind_host("CONCAT", ["?s", "\"5\""], {"s": s_col}, len(s_col), None, d2, E.QuotedTripleStore())
    want = sorted((d2.decode(int(e)), d2.decode(int(s)), d2.decode(int(o))) for e, s, o in zip(e_col, s_col, out)
                  if E.rust_parse_f64(d2.decode(int(o))) > 100)
    assert len(want) > 0
    assert sorted((r["e"], r["s"], r["c"]) for r in rows) == want
    # a join over the CONCAT output: ?c equals a code's object
    join = E.HashJoin(bind, E.TableScan((V("?k"), K(enc("ex:code")), V("?c"))))
    rows = E.ExecutionEngine.execute(join, db)
    assert sorted((r["e"], r["k"]) for r in rows) == sorted([(f"ex:e{k}", "ex:x") for k in range(300) if k % 23 == 7] +
                                                            [(f"ex:e{k}", "ex:y") for k in range(300) if k % 23 == 22])
    nctx.store_clear()


def test_full_size_employee_dictionary(nctx):
    d = datagen.employee_dataset(1_666_667)
    strings = employee_strings(d)
    assert len(strings) > 1_700_000
    nctx.dict_strings_load(strings)
    info = nctx.dict_numeric_derive(c.NUMERIC_F64, 0)
    assert info["n_numeric"] == int(d.is_num.sum())
    num, isn = nctx.dict_numeric_download(0, len(strings))
    host = E.Dictionary()
    host.id_to_string = strings
    hnum, hisn = host.numeric_table()
    assert np.array_equal(num.view(np.uint64), hnum.view(np.uint64)) and np.array_equal(isn, hisn)
    nctx.dict_strings_load([])
