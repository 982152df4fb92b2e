"""GPU (-m gpu): BIND built-ins on the device (kb_bind) against the host restatement ExecutionEngine._bind_host (pinned to
engine.rs:144-277 by tests/test_bind_cpu.py): the output column, n_unbound, the new dictionary strings and the new quoted-triple entries,
ids and order included, for relations from kb_rel_from_host, kb_scan and kb_scan_quoted. Then what follows a TRIPLE (decode, quoted
scans, a second TRIPLE, a reload), refusals, ordering, the mirror's route and the full-size workload of scripts/quoted_bench.py. The
tests run on contexts of their own, so no grown table or dictionary reaches the session context."""
import copy
import os

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200 import engine as E
from tests import quoted_cases as Q

pytestmark = pytest.mark.gpu

NONE = c.KB_ID_NONE
QB = Q.QBIT
FN = {"SUBJECT": c.BIND_SUBJECT, "PREDICATE": c.BIND_PREDICATE, "OBJECT": c.BIND_OBJECT, "isTRIPLE": c.BIND_IS_TRIPLE,
      "TRIPLE": c.BIND_TRIPLE, "CONCAT": c.BIND_CONCAT}


@pytest.fixture(scope="module")
def bctx():
    ctx = c.Context(0)
    yield ctx
    ctx.close()


def new_db(ctx, n_entries=300, seed=3):
    """a dictionary with multibyte strings and a quoted-triple store with holes, permuted ids and nesting"""
    db = E.SparqlDatabase(ctx=ctx)
    for t in ("é", "€uro", "😀", "\"lit\"@en", ""):
        db.dictionary.encode(t)
    if n_entries:
        Q.holey_store(db, np.random.default_rng(seed), n_entries)
    return db


def upload(ctx, db):
    """the device mirrors the host: dictionary strings and the quoted-triple table (kb_quoted_load drops the reverse index)"""
    ctx.dict_strings_load(db.dictionary.id_to_string)
    qts = db.quoted_triple_store
    ids = np.array(sorted(qts.id_to_components), dtype=np.uint32)
    comp = np.array([qts.id_to_components[int(i)] for i in ids], dtype=np.uint32).reshape(-1, 3)
    ctx.quoted_load(ids, comp[:, 0], comp[:, 1], comp[:, 2])


def apply_tails(ctx, db, info):
    d, qts = db.dictionary, db.quoted_triple_store
    for t in ctx.dict_strings_download(info["dict_first"], info["dict_new"]):
        d.string_to_id[t] = len(d.id_to_string)
        d.id_to_string.append(t)
    if info["quoted_new"]:
        s, p, o = ctx.quoted_download(info["quoted_first"], info["quoted_new"])
        for k in range(info["quoted_new"]):
            key = (int(s[k]), int(p[k]), int(o[k]))
            qts.id_to_components[info["quoted_first"] + k] = key
            qts.components_to_id[key] = info["quoted_first"] + k
        qts.next_qt_id = info["quoted_first"] + info["quoted_new"]


def check(ctx, db, rel, names, fn, args, out, consts=()):
    """kb_bind on `rel` (columns = names by slot) against _bind_host on its downloaded columns; both stores compared afterwards"""
    n, rslots = rel.info()
    cols = {names[s]: rel.column(i) for i, s in enumerate(rslots)}
    want_d, want_q = copy.deepcopy(db.dictionary), copy.deepcopy(db.quoted_triple_store)
    host_args = []
    for a in args:  # the reference's argument strings
        if a.is_var:
            host_args.append("?" + names[a.value])
        elif fn == "TRIPLE":
            host_args.append(db.dictionary.id_to_string[a.value])
        else:
            host_args.append('"' + consts[a.value].decode("utf-8") + '"')
    want = E.ExecutionEngine._bind_host(fn, host_args, cols, n, cols.get(out), want_d, want_q)
    slot_of = {v: k for k, v in names.items()}
    res, info = ctx.bind(rel, FN[fn], args, slot_of[out], db.quoted_triple_store.next_qt_id if fn == "TRIPLE" else 0, consts)
    apply_tails(ctx, db, info)
    rn, rs = res.info()
    assert rn == n and set(rs) == set(rslots) | {slot_of[out]} and len(rs) == len(set(rs))
    got = res.column(rs.index(slot_of[out]))
    np.testing.assert_array_equal(got, want)
    for i, s in enumerate(rs):  # the other columns are the input's
        if s != slot_of[out]:
            np.testing.assert_array_equal(res.column(i), cols[names[s]])
    assert info["n_rows"] == n and info["n_unbound"] == int((want == NONE).sum())
    assert db.dictionary.id_to_string == want_d.id_to_string
    assert list(db.quoted_triple_store.id_to_components.items()) == list(want_q.id_to_components.items())
    assert db.quoted_triple_store.next_qt_id == want_q.next_qt_id
    return got, info


def pools(db):
    d, qts = db.dictionary, db.quoted_triple_store
    quoted = np.array(sorted(qts.id_to_components), dtype=np.uint32)
    holes = np.setdiff1d(np.arange(QB, QB + 40, dtype=np.uint32), quoted)[:5]
    plain = np.arange(len(d.id_to_string), dtype=np.uint32)
    return np.concatenate([quoted, holes, plain, np.array([NONE, len(d.id_to_string) + 7, QB + 0x0FFF_FFFF], dtype=np.uint32)])


SIZES = [0, 1, 255, 256, 257, (1 << 20) + 3]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("fn", ["SUBJECT", "PREDICATE", "OBJECT", "isTRIPLE", "TRIPLE", "CONCAT"])
def test_parity_from_host(bctx, fn, n):
    db = new_db(bctx)
    upload(bctx, db)
    rng = np.random.default_rng(n + len(fn))
    pool = pools(db)
    names = {0: "a", 1: "b", 2: "c", 3: "x"}
    if fn == "TRIPLE":  # small pools: duplicates in the batch, existing entries, nested quoted components, missing arguments
        qts = db.quoted_triple_store
        have = np.array(list(qts.id_to_components.values()), dtype=np.uint32)
        pick = have[rng.integers(0, len(have), n)]
        alt = np.stack([pool[rng.integers(0, 12, n)], pool[rng.integers(0, 4, n)], pool[rng.integers(0, 30, n)]], axis=1)
        use = rng.random(n) < 0.4
        rows = np.where(use[:, None], pick, alt).astype(np.uint32)
        rows[rng.random(n) < 0.05, 1] = NONE
        cols = [rows[:, 0], rows[:, 1], rows[:, 2]]
        args = [c.V(0), c.V(1), c.V(2)]
    else:
        cols = [pool[rng.integers(0, len(pool), n)] for _ in range(3)]
        args = {"CONCAT": [c.V(0), c.K(0), c.V(1), c.K(1)]}.get(fn, [c.V(0)])
    cols.append(pool[rng.integers(0, len(pool), n)])  # an output variable the input binds already: overwritten where the reference inserts
    rel = bctx.rel_from_host([0, 1, 2, 3], cols)
    consts = ("→ ".encode(), b'a"@en') if fn == "CONCAT" else ()
    check(bctx, db, rel, names, fn, args, "x", consts)
    rel2 = bctx.rel_from_host([0, 1, 2], cols[:3])  # and a new output column
    names[5] = "y"
    check(bctx, db, rel2, names, fn, args, "y", consts)


def test_parity_from_scans_and_empty_context(bctx):
    db = new_db(bctx, n_entries=2000, seed=11)
    db._sync()
    upload(bctx, db)
    names = {0: "t", 1: "p", 2: "o", 3: "s2", 4: "p2", 5: "o2", 9: "x"}
    rel = bctx.scan([c.pattern(c.V(0), c.V(1), c.V(2))])[0]
    for fn in ("SUBJECT", "OBJECT", "isTRIPLE", "CONCAT"):
        check(bctx, db, rel, names, fn, [c.V(0)] if fn != "CONCAT" else [c.V(0), c.V(2)], "x")
    qp = c.KbQuotedPattern(c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.V(1), c.V(2)), c.pattern(c.V(3), c.V(4), c.V(5)), c.KbPattern())
    qrel = bctx.scan_quoted(qp)
    for fn, args in (("PREDICATE", [c.V(3)]), ("TRIPLE", [c.V(5), c.V(4), c.V(3)]), ("TRIPLE", [c.V(3), c.V(4), c.V(5)])):
        check(bctx, db, qrel, names, fn, args, "x")
    # an empty context (no table, nothing in the dictionary beyond the store's terms): TRIPLE starts one
    db2 = new_db(bctx, n_entries=0)
    upload(bctx, db2)
    rel = bctx.rel_from_host([0, 1, 2], [np.array([0, 1, 0, 2], np.uint32), np.array([1, 1, 1, 1], np.uint32), np.array([2, 2, 2, 0], np.uint32)])
    got, info = check(bctx, db2, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "x")
    assert info["quoted_new"] == 3 and got.tolist() == [QB, QB + 1, QB, QB + 2]
    got, info = check(bctx, db2, rel, names, "SUBJECT", [c.V(0)], "x")
    assert (got == NONE).all()


def test_after_triple_decode_scan_second_call_and_reload(bctx):
    db = new_db(bctx, n_entries=500, seed=5)
    upload(bctx, db)
    rng = np.random.default_rng(1)
    n = 5000
    plain = np.arange(len(db.dictionary.id_to_string), dtype=np.uint32)
    quoted = np.array(sorted(db.quoted_triple_store.id_to_components), dtype=np.uint32)
    s = np.where(rng.random(n) < 0.3, quoted[rng.integers(0, len(quoted), n)], plain[rng.integers(0, 20, n)]).astype(np.uint32)
    p = plain[rng.integers(0, 3, n)]
    o = plain[rng.integers(0, 40, n)]
    names = {0: "s", 1: "p", 2: "o", 3: "t"}
    rel = bctx.rel_from_host([0, 1, 2], [s, p, o])
    got, info = check(bctx, db, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "t")
    assert info["quoted_new"] > 0
    res, _ = bctx.bind(rel, c.BIND_TRIPLE, [c.V(0), c.V(1), c.V(2)], 3, db.quoted_triple_store.next_qt_id)
    col = res.slots.index(3)
    # kb_rel_decode renders the new ids as << s p o >>
    assert res.decode_strings(col) == [db.decode_term(int(x)) for x in res.column(col)]
    # a second TRIPLE over the same rows adds nothing and gives the same ids
    again, info2 = check(bctx, db, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "t")
    assert info2["quoted_new"] == 0 and np.array_equal(again, got)
    # kb_scan_quoted matches the new entries, index on and off
    ann, src = db.dictionary.encode("ex:ann"), db.dictionary.encode("ex:src")
    for q in np.unique(got).tolist():
        db.triples.add((q, ann, src))
    db._version += 1
    db._sync()
    db._uploaded_quoted = len(db.quoted_triple_store)
    pat = (E.QuotedTriple(E.Variable("?a"), E.Variable("?b"), E.Variable("?c")), E.Constant(ann), E.Variable("?w"))
    for use_index in (False, True):
        bctx.set_use_index(use_index)
        if use_index:
            bctx.build_index()
        slots = E.SlotMap()
        dev = Q.bag(E.ExecutionEngine.execute_with_ids(E.TableScan(pat), db))
        assert dev == Q.bag(Q.brute_quoted_scan(db, pat)) and sum(dev.values()) == len(np.unique(got))
    bctx.set_use_index(True)
    # kb_quoted_load, then TRIPLE: the same ids as the restatement (the reverse index is rebuilt from the loaded table)
    upload(bctx, db)
    check(bctx, db, rel, names, "TRIPLE", [c.V(2), c.V(1), c.V(0)], "t")
    bctx.store_clear()


def state(ctx, db):
    n_ids, n_bytes = ctx.dict_strings_info()
    qts = db.quoted_triple_store
    lo = min(qts.id_to_components) if len(qts) else QB
    return n_ids, n_bytes, [x.tolist() for x in ctx.quoted_download(lo, qts.next_qt_id - lo + 8)]


def test_refusals_leave_everything_unchanged(bctx):
    db = new_db(bctx, n_entries=100)
    upload(bctx, db)
    rel = bctx.rel_from_host([0, 1, 2], [np.array([0, 1], np.uint32), np.array([1, 2], np.uint32), np.array([3, 4], np.uint32)])
    names = {0: "a", 1: "b", 2: "c", 3: "t"}
    check(bctx, db, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "t")  # builds the reverse index
    before = state(bctx, db)
    nxt = db.quoted_triple_store.next_qt_id
    cases = [
        (7, [c.V(0)], nxt, (), c.KB_E_INVALID),                             # unknown function
        (c.BIND_SUBJECT, [c.V(0), c.V(1)], 0, (), c.KB_E_INVALID),          # wrong number of arguments
        (c.BIND_TRIPLE, [c.V(0), c.V(1)], nxt, (), c.KB_E_INVALID),
        (c.BIND_SUBJECT, [c.K(0)], 0, (), c.KB_E_INVALID),                  # SUBJECT of a constant
        (c.BIND_OBJECT, [c.V(9)], 0, (), c.KB_E_INVALID),                   # not a column of the input
        (c.BIND_CONCAT, [c.K(1)], 0, (b"x",), c.KB_E_INVALID),              # constant index past n_const
        (c.BIND_TRIPLE, [c.V(2), c.V(1), c.V(0)], QB, (), c.KB_E_INVALID),  # next_qt_id not above the table's ids
        (c.BIND_TRIPLE, [c.V(2), c.V(1), c.V(0)], 5, (), c.KB_E_INVALID),   # next_qt_id without bit 31
        (c.BIND_TRIPLE, [c.V(2), c.V(1), c.V(0)], QB + (1 << 28) - 1, (), c.KB_E_LIMIT),  # 2 new entries past KB_QUOTED_MAX_SLOTS
    ]
    for fn, args, nq, consts, status in cases:
        with pytest.raises(c.KolibrieError) as e:
            bctx.bind(rel, fn, args, 3, nq, consts)
        assert e.value.status == status, (fn, e.value)
        assert state(bctx, db) == before
    # the reverse index still answers: the next TRIPLE gives the restatement's ids
    check(bctx, db, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "t")
    check(bctx, db, rel, names, "TRIPLE", [c.V(2), c.V(1), c.V(0)], "t")


def test_ordered_mode_gives_identical_ids():
    old = os.environ.get("KOLIBRIE_ORDERED")
    os.environ["KOLIBRIE_ORDERED"] = "1"
    try:
        outs = []
        for _ in range(2):
            ctx = c.Context(0)
            db = new_db(ctx, n_entries=200)
            upload(ctx, db)
            rng = np.random.default_rng(9)
            cols = [rng.integers(0, 30, 300_000).astype(np.uint32) for _ in range(3)]
            rel = ctx.rel_from_host([0, 1, 2], cols)
            a, _ = ctx.bind(rel, c.BIND_TRIPLE, [c.V(0), c.V(1), c.V(2)], 3, db.quoted_triple_store.next_qt_id)
            b, _ = ctx.bind(rel, c.BIND_CONCAT, [c.V(0), c.K(0), c.V(2)], 4, 0, (b"-",))
            outs.append((a.column(a.slots.index(3)), b.column(b.slots.index(4))))
            ctx.close()
        assert all(np.array_equal(x, y) for x, y in zip(*outs))
    finally:
        if old is None:
            os.environ.pop("KOLIBRIE_ORDERED", None)
        else:
            os.environ["KOLIBRIE_ORDERED"] = old


class HostOnly:
    """the same context without kb_bind: ExecutionEngine takes the host restatement"""

    def __init__(self, ctx):
        self._ctx = ctx

    def __getattr__(self, k):
        if k == "bind":
            raise AttributeError(k)
        return getattr(self._ctx, k)


def emp_db(ctx):
    db = E.SparqlDatabase(ctx=ctx)
    for i in range(300):
        e = f"ex:e{i}"
        db.add_triple_parts(e, "ex:salary", str(1000 * (i % 17)))
        db.add_triple_parts(e, "ex:dept", f"ex:d{i % 5}")
        db.add_statement((e, "ex:salary", str(1000 * (i % 17))), "ex:source", f"ex:doc{i % 3}")
    return db


def test_mirror_route_stays_on_the_device(bctx):
    sal, dept, src = "ex:salary", "ex:dept", "ex:source"
    for fn, args in (("SUBJECT", ["?t"]), ("OBJECT", ["?t"]), ("TRIPLE", ["?e", "?d", "?s"]), ("isTRIPLE", ["?t"]), ("CONCAT", ["?e", "\"/\"", "?d"]),
                     ("TRIPLE", ["?e", "ex:new", "?s"])):
        res = []
        for host in (False, True):
            db = emp_db(bctx)
            V, K = E.Variable, E.Constant
            cid = lambda t: K(db.dictionary.encode(t))
            star = E.StarJoin("?e", [(V("?e"), cid(sal), V("?s")), (V("?e"), cid(dept), V("?d"))])
            qscan = E.TableScan((E.QuotedTriple(V("?e"), cid(sal), V("?s")), cid(src), V("?doc")))
            if fn in ("SUBJECT", "OBJECT", "isTRIPLE"):
                inner = E.Filter(E.TableScan((V("?t"), cid(src), V("?doc"))), E.Condition(E.Comparison("?doc", "=", "ex:doc1")))
            elif fn == "TRIPLE" and args[1] == "?d":
                inner = E.Filter(star, E.Condition(E.Comparison("?s", ">", "5000")))
            else:
                inner = E.Filter(qscan, E.Condition(E.Comparison("?s", ">", "5000")))
                if fn == "CONCAT":
                    inner = E.Filter(E.HashJoin(qscan, E.TableScan((V("?e"), cid(dept), V("?d")))), E.Condition(E.Comparison("?s", ">", "5000")))
            plan = E.Projection(E.Bind(inner, fn, args, "?x"), ["e", "x"] if "?e" in args else ["t", "x"])
            db._sync()
            if host:
                db.ctx = HostOnly(bctx)
            bctx.get_stats(reset=True)
            rows = E.ExecutionEngine.execute(plan, db)
            st = bctx.get_stats(reset=True)
            if not host and fn in ("SUBJECT", "OBJECT") and args == ["?t"]:
                assert st["h2d_bytes"] == 0, st  # no relation went through the host
            res.append((sorted(tuple(sorted(r.items())) for r in rows), db.dictionary.id_to_string, dict(db.quoted_triple_store.id_to_components)))
        assert res[0] == res[1], fn
        assert len(res[0][0]) > 0
    # unbound keys are absent: SUBJECT of a plain id
    db = emp_db(bctx)
    plan = E.Bind(E.TableScan((E.Variable("?e"), E.Constant(db.dictionary.encode(dept)), E.Variable("?d"))), "SUBJECT", ["?e"], "?x")
    rows = E.ExecutionEngine.execute_with_ids(plan, db)
    assert rows and all("x" not in r for r in rows)
    # a FILTER over a BIND output with unbound rows is left to the CPU
    with pytest.raises(c.KolibrieError) as e:
        E.ExecutionEngine.execute_with_ids(E.Filter(plan, E.Condition(E.Comparison("?x", "=", "ex:d1"))), db)
    assert e.value.status == c.KB_E_UNSUPPORTED
    bctx.store_clear()
    bctx.quoted_load([], [], [], [])


def test_full_size_workload(bctx):
    """scripts/quoted_bench.py's workload (cfg2's 10 M-triple employee store + 1.67 M annotations): SUBJECT / OBJECT over the annotation
    scan, TRIPLE over the salary scan (every triple quoted already: no new id) and over its swap (every triple new), each against its
    closed form"""
    a = datagen.annotated_salary_dataset(1_666_667)
    E_ = a.d.n_employees
    bctx.store_load(a.s, a.p, a.o)
    bctx.dict_strings_load(["t%d" % i for i in range(a.n_ids)])
    bctx.quoted_load(a.qt_ids, a.qt_s, a.qt_p, a.qt_o)
    ann = bctx.scan([c.pattern(c.V(0), c.K(a.source), c.V(1))])[0]
    assert ann.n_rows == E_
    for fn, comp in ((c.BIND_SUBJECT, a.qt_s), (c.BIND_OBJECT, a.qt_o)):
        r, info = bctx.bind(ann, fn, [c.V(0)], 2)
        assert info["n_unbound"] == 0 and info["quoted_new"] == 0 and info["dict_new"] == 0
        want = np.stack([a.qt_ids, a.src_of_employee, comp], axis=1)
        assert datagen.row_checksums(r.to_numpy([0, 1, 2])) == datagen.row_checksums(want)
    P = a.d.ids["ds:annual_salary"]
    salr = bctx.scan([c.pattern(c.V(0), c.K(P), c.V(1))])[0]
    nxt = int(QB + E_)
    r, info = bctx.bind(salr, c.BIND_TRIPLE, [c.V(0), c.K(P), c.V(1)], 2, nxt)
    assert info["quoted_new"] == 0 and info["n_unbound"] == 0
    want = np.stack([a.qt_s, a.qt_o, a.qt_ids], axis=1)
    assert datagen.row_checksums(r.to_numpy([0, 1, 2])) == datagen.row_checksums(want)
    r, info = bctx.bind(salr, c.BIND_TRIPLE, [c.V(1), c.K(P), c.V(0)], 2, nxt)
    assert info["quoted_new"] == E_ and info["quoted_first"] == nxt and info["n_unbound"] == 0
    t = r.column(r.slots.index(2))
    assert np.array_equal(np.sort(t), np.arange(nxt, nxt + E_, dtype=np.uint32))
    qs, qp, qo = bctx.quoted_download(nxt, E_)
    rows = r.to_numpy([0, 1])
    k = (t - np.uint32(nxt)).astype(np.int64)
    assert np.array_equal(qs[k], rows[:, 1]) and np.array_equal(qo[k], rows[:, 0]) and (qp == P).all()
    want = np.stack([a.qt_s, a.qt_o, a.qt_o, a.qt_s], axis=1)
    assert datagen.row_checksums(np.stack([rows[:, 0], rows[:, 1], qs[k], qo[k]], axis=1)) == datagen.row_checksums(want)
    bctx.quoted_load([], [], [], [])
    bctx.store_clear()
