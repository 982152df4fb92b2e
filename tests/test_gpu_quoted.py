"""GPU (-m gpu): RDF-star quoted-triple patterns on the device — the quoted-triple table (kb_quoted_load), the match pass + bind join
(kb_scan_quoted) and the decode of quoted ids (kb_rel_decode) — against the host restatement (ExecutionEngine._scan_quoted, pinned to
engine.rs:1111-1188 by tests/test_quoted_cpu.py) and SparqlDatabase.decode_term. Bags are compared exactly, with the store index on and
off. The tests run on a context of their own, so no quoted table reaches the session context."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200 import engine as E
from tests import helpers as H
from tests import quoted_cases as Q

pytestmark = pytest.mark.gpu

STAR = H.load("rdf_star.json")
QB = Q.QBIT


@pytest.fixture(scope="module")
def qctx():
    ctx = c.Context(0)
    yield ctx
    ctx.close()


@pytest.fixture(params=["scan", "index"])
def mode(request):
    return request.param


def make_db(ctx):
    return E.SparqlDatabase(ctx=ctx)


def sync(db, mode):
    db._sync()
    if mode == "index":
        db.ctx.set_use_index(True)
        db.ctx.build_index()
    else:
        db.ctx.set_use_index(False)


def rows_of(rel, slots):
    n, rs = rel.info()
    cols = [rel.column(i) for i in range(len(rs))]
    names = [slots.names[s] for s in rs]
    return [{names[j]: int(cols[j][i]) for j in range(len(names))} for i in range(n)]


def device_rows(db, pat):
    db._uploaded_version = db._version  # (encoding a query constant does not change the triples)
    return E.ExecutionEngine.execute_with_ids(E.TableScan(pat), db)


def host_rows(db, pat):
    slots = E.SlotMap()
    return rows_of(E.ExecutionEngine._scan_quoted(pat, db, slots), slots)


def check(db, pat):
    got = device_rows(db, pat)
    want = host_rows(db, pat)
    assert Q.bag(got) == Q.bag(want), pat
    return got


def pattern_term(db, t):
    if isinstance(t, list):
        return E.QuotedTriple(*(pattern_term(db, x) for x in t))
    return E.Variable(t) if t.startswith("?") else E.Constant(db.dictionary.encode(t))


def data_term(t):
    return tuple(data_term(x) for x in t) if isinstance(t, list) else t


QUOTED_CASES = [x for x in STAR["cases"] if any(isinstance(t, list) for t in x["pattern"])]


@pytest.mark.parametrize("case", QUOTED_CASES, ids=[x["name"] for x in QUOTED_CASES])
def test_rdf_star_fixture_cases(qctx, mode, case):
    db = make_db(qctx)
    for s, p, o in case["data"]:
        db.add_statement(data_term(s), data_term(p), data_term(o))
    pat = tuple(pattern_term(db, t) for t in case["pattern"])
    sync(db, mode)
    check(db, pat)
    rows = E.ExecutionEngine.execute(E.Projection(E.TableScan(pat), ["?" + v for v in case["select"]]), db)
    assert sorted(tuple(r[v] for v in case["select"]) for r in rows) == sorted(tuple(r) for r in case["rows"])


def corner_db(ctx):
    db = make_db(ctx)
    ex = "http://example.org/"
    db.add_statement((ex + "a", ex + "says", ex + "a"), ex + "by", ex + "a")
    db.add_statement((ex + "a", ex + "says", ex + "b"), ex + "by", ex + "b")
    db.add_statement((ex + "b", ex + "says", ex + "a"), ex + "by", ex + "c")
    db.add_statement(ex + "d", ex + "cites", (ex + "a", ex + "says", ex + "b"))
    db.add_statement(((ex + "a", ex + "says", ex + "b"), ex + "in", ex + "g"), ex + "by", ex + "e")
    db.add_statement((ex + "a", ex + "says", ex + "b"), ex + "echo", (ex + "a", ex + "says", ex + "b"))
    db.add_statement((ex + "a", ex + "says", ex + "a"), ex + "echo", (ex + "b", ex + "says", ex + "a"))
    return db


def test_corner_cases(qctx, mode):
    """the shapes of test_quoted_scan_semantics_beyond_the_fixtures plus both positions quoted, repeated variables within and across
    the inner and outer terms, nested terms and absent constants"""
    db = corner_db(qctx)
    ex = "http://example.org/"
    sync(db, mode)
    P = lambda t: pattern_term(db, t)  # noqa: E731
    says, by = ex + "says", ex + "by"
    cases = [
        ([["?x", says, "?y"], by, "?y"], 2),
        ([["?x", says, "?x"], by, "?w"], 1),
        (["?who", ex + "cites", ["?x", says, "?y"]], 1),
        ([[["?p", "?q", "?r"], ex + "in", "?g"], by, "?w"], 1),
        ([["?x", ex + "nothing", "?y"], by, "?w"], 0),
        ([["?x", says, "?y"], ex + "echo", ["?x", says, "?y"]], 1),  # one entry fills both positions: << a says a >> echo << b says a >> is out
        ([["?x", says, "?y"], ex + "echo", ["?y", says, "?x"]], 0),  # ... and would need x == y
        ([["?x", "?p", "?y"], "?p", "?o"], 0),                       # inner and outer predicate variable
        ([["?x", says, ex + "absent"], by, "?w"], 0),
        ([["?x", says, "?y"], "?p", "?x"], None),
    ]
    for pat, n in cases:
        got = check(db, tuple(P(t) for t in pat))
        if n is not None:
            assert len(got) == n, pat


def test_empty_table_and_no_table(qctx, mode):
    db = make_db(qctx)
    db.add_triple_parts("a", "p", "b")
    sync(db, mode)
    pat = (E.QuotedTriple(E.Variable("?x"), E.Variable("?y"), E.Variable("?z")), E.Variable("?p"), E.Variable("?o"))
    assert device_rows(db, pat) == []
    rel = qctx.scan_quoted(E.SlotMap().quoted_pattern(pat))
    assert rel.info() == (0, [0, 1, 2, 3, 4])  # one column per variable, in reading order


@pytest.mark.parametrize("seed", range(8))
def test_random_stores_and_patterns(qctx, mode, seed):
    rng = np.random.default_rng(seed)
    db = make_db(qctx)
    Q.random_store(db, rng, n_quoted=int(rng.integers(1, 80)), n_triples=int(rng.integers(1, 200)))
    sync(db, mode)
    for _ in range(20):
        pat = Q.random_pattern(db, rng)
        got = check(db, pat)
        assert Q.bag(got) == Q.bag(Q.brute_quoted_scan(db, pat))


@pytest.mark.parametrize("n_entries", [0, 1, 1000, 200_000])
def test_fuzz_holes_permuted_ids_nesting(qctx, mode, n_entries):
    rng = np.random.default_rng(n_entries + 3)
    db = make_db(qctx)
    live = Q.holey_store(db, rng, n_entries)
    d = db.dictionary
    sync(db, mode)
    src, ann = E.Constant(d.lookup("ex:src")), E.Constant(d.lookup("ex:source"))
    pats = [
        (E.QuotedTriple(E.Variable("?s"), E.Variable("?p"), E.Variable("?o")), ann, E.Variable("?w")),
        (E.QuotedTriple(E.QuotedTriple(E.Variable("?a"), E.Variable("?b"), E.Variable("?c")), E.Variable("?p"), E.Variable("?o")), ann, src),
        (E.QuotedTriple(E.Variable("?s"), E.Constant(d.lookup("w3")), E.Variable("?s")), E.Variable("?q"), E.Variable("?w")),
    ]
    for pat in pats:
        check(db, pat)
    if n_entries:  # every live id renders as decode_term renders it
        ids = live[rng.permutation(len(live))[:5000]].astype(np.uint32)
        got = qctx.rel_from_host([0], [ids]).decode_strings(0)
        assert got == [Q.decode_term_ref(db, int(i)) for i in ids]


def test_decode_renders_like_decode_term(qctx):
    rng = np.random.default_rng(11)
    db = make_db(qctx)
    qids = Q.random_store(db, rng, n_quoted=200, max_depth=6)
    qts = db.quoted_triple_store
    dang = [qts.encode(qids[0], 1, 777777), qts.encode(0x8000_5555, 2, 3), qts.encode(qids[1], 0x8000_6666, qids[2])]
    dang.append(qts.encode(dang[0], 0, 1))
    db._sync()
    ids = np.array(list(qids) + dang + [0x8000_7000, 0, 5, 999999], dtype=np.uint32)
    rng.shuffle(ids)
    rel = qctx.rel_from_host([0], [ids])
    assert rel.decode_strings(0) == [Q.decode_term_ref(db, int(i)) for i in ids]
    # execute() decodes quoted columns on the device: no host decode_term call when the table is loaded
    calls = []
    orig = db.decode_term
    db.decode_term = lambda i: calls.append(i) or orig(i)
    pat = (E.Variable("?s"), E.Variable("?p"), E.Variable("?o"))
    rows = E.ExecutionEngine.execute(E.TableScan(pat), db)
    assert not calls
    want = sorted((Q.decode_term_ref(db, s), Q.decode_term_ref(db, p), Q.decode_term_ref(db, o)) for s, p, o in db.triples)
    assert sorted((r["s"], r["p"], r["o"]) for r in rows) == want


def test_decode_depth_cap_and_clearing(qctx):
    qctx.dict_strings_load(["a", "b", "c"])
    chain = [(QB, 0, 1, 2)] + [(QB + k, QB + k - 1, 1, 2) for k in range(1, 17)]
    cyc = [(QB + 100, QB + 101, 0, 0), (QB + 101, QB + 100, 0, 0)]
    ent = np.array(chain + cyc, dtype=np.uint32)
    qctx.quoted_load(ent[:, 0], ent[:, 1], ent[:, 2], ent[:, 3])
    ok = qctx.rel_from_host([0], [np.array([QB + 15], np.uint32)]).decode_strings(0)[0]  # 16 levels: the cap
    assert ok == "<< " * 16 + "a b c >>" + " b c >>" * 15
    for bad in (QB + 16, QB + 100):  # 17 levels; a cycle
        with pytest.raises(c.KolibrieError) as e:
            qctx.rel_from_host([0], [np.array([0, bad], np.uint32)]).decode(0)
        assert e.value.status == c.KB_E_LIMIT
    qctx.quoted_load([], [], [], [])
    with pytest.raises(c.KolibrieError) as e:
        qctx.rel_from_host([0], [np.array([1, QB], np.uint32)]).decode(0)
    assert e.value.status == c.KB_E_UNSUPPORTED


def test_refusals_leave_the_table(qctx):
    qctx.dict_strings_load(["a", "b", "c"])
    qctx.quoted_load([QB + 1], [0], [1], [2])
    probe = lambda: qctx.rel_from_host([0], [np.array([QB + 1], np.uint32)]).decode_strings(0)  # noqa: E731
    assert probe() == ["<< a b c >>"]
    for args, status in (
        (([5], [0], [1], [2]), c.KB_E_INVALID),                          # no bit 31
        (([c.KB_ID_NONE], [0], [1], [2]), c.KB_E_INVALID),               # KB_ID_NONE
        (([QB + 2, QB + 2], [0, 1], [1, 1], [2, 2]), c.KB_E_INVALID),    # repeated id
        (([QB + 3], [0], [c.KB_ID_NONE], [2]), c.KB_E_INVALID),          # reserved component
        (([QB + (1 << 28)], [0], [1], [2]), c.KB_E_LIMIT),               # beyond the table's slots
    ):
        with pytest.raises(c.KolibrieError) as e:
            qctx.quoted_load(*args)
        assert e.value.status == status
        assert probe() == ["<< a b c >>"]
    qp = c.KbQuotedPattern(c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.KbTerm(c.KB_TERM_QUOTED, 0), c.V(1)), c.pattern(c.V(2), c.V(3), c.V(4)),
                           c.KbPattern())
    with pytest.raises(c.KolibrieError) as e:
        qctx.scan_quoted(qp)
    assert e.value.status == c.KB_E_UNSUPPORTED
    qp = c.KbQuotedPattern(c.pattern(c.V(0), c.K(1), c.V(1)), c.KbPattern(), c.KbPattern())
    with pytest.raises(c.KolibrieError) as e:
        qctx.scan_quoted(qp)
    assert e.value.status == c.KB_E_INVALID
    with pytest.raises(c.KolibrieError) as e:  # the other entry points keep refusing is_var > 1
        qctx.scan([c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.K(1), c.V(1))])
    assert e.value.status == c.KB_E_INVALID
    qctx.quoted_load([], [], [], [])


def test_mirror_keeps_the_work_on_the_device(qctx):
    """a query with a quoted pattern uploads nothing per query (no kb_rel_from_host) once the store and the table are synced"""
    db = corner_db(qctx)
    ex = "http://example.org/"
    sync(db, "index")
    pat = (pattern_term(db, ["?x", ex + "says", "?y"]), pattern_term(db, ex + "by"), E.Variable("?w"))
    qctx.get_stats(reset=True)
    rows = E.ExecutionEngine.execute(E.TableScan(pat), db)
    st = qctx.get_stats(reset=True)
    assert len(rows) == 3 and st["h2d_bytes"] == 0


def annotated_db(ctx, a):
    ctx.store_load(a.s, a.p, a.o)
    ctx.dict_numeric_load(a.num_or0, a.is_num)
    ctx.quoted_load(a.qt_ids, a.qt_s, a.qt_p, a.qt_o)


def bench_query(ctx, a):
    qp = c.KbQuotedPattern(c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.K(a.source), c.V(2)),
                           c.pattern(c.V(0), c.K(a.d.ids["ds:annual_salary"]), c.V(1)), c.KbPattern())
    rel = ctx.scan_quoted(qp)
    st = ctx.get_stats()
    return rel, ctx.filter(rel, [c.fop(c.F_CMP_NUM, slot=1, cmp=c.CMP_GT, value=100000.0)]), st


def test_bench_workload_full_size(qctx):
    """the workload of scripts/quoted_bench.py at full size (cfg2's 10 M-triple employee store + 1.67 M annotations) against its closed
    form; on this shape (unique, dense quoted subjects of ex:source) the indexed scan is one match launch plus one probe launch"""
    a = datagen.annotated_salary_dataset(1_666_667)
    want = datagen.row_checksums(datagen.annotated_salary_answer(a))
    annotated_db(qctx, a)
    for use_index in (True, False):
        qctx.set_use_index(use_index)
        if use_index:
            qctx.build_index()
        qctx.get_stats(reset=True)
        rel, f, st = bench_query(qctx, a)
        assert rel.info() == (a.d.n_employees, [0, 1, 2])
        assert datagen.row_checksums(f.to_numpy([0, 1, 2])) == want
        if use_index:
            assert st["scan_launches"] == 1 and st["probe_launches"] == 1 and st["kernel_launches"] == 2, st
    qctx.set_use_index(True)
    qctx.quoted_load([], [], [], [])
    qctx.store_clear()
