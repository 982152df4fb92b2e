"""GPU (-m gpu): kb_values and the joins above a VALUES block against the restatement (tests/values_reference.py), compared as bags:
the ids, the dictionary's growth and the numeric side table over the new ids, every join operator over seeded ragged relations, the
refusals, and the engine mirror on plans the planner mirror builds for queries with VALUES."""
import ctypes as C
import random

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import engine as E
from kolibrie_b200 import planner as PL
from tests import values_reference as V

pytestmark = pytest.mark.gpu
NONE = c.KB_ID_NONE


def fresh_ctx(strings):
    ctx = c.Context(0)
    ctx.dict_strings_load(strings)
    ctx.dict_numeric_derive(c.NUMERIC_F64, 0)
    return ctx


def host_dict(strings):
    d = E.Dictionary()
    for t in strings:
        d.encode(t)
    return d


def device_rows(rel, names):
    n, slots = rel.info()
    cols = [rel.column(i) for i in range(len(slots))]
    return [{names[s]: int(cols[j][i]) for j, s in enumerate(slots) if cols[j][i] != NONE} for i in range(n)]


def random_block(rng, n_rows, header, vocab, p_undef=0.2, p_short=0.1):
    rows = []
    for _ in range(n_rows):
        row = [None if rng.random() < p_undef else rng.choice(vocab) for _ in header]
        if rng.random() < p_short:
            row = row[: rng.randrange(len(header) + 1)]
        rows.append(row)
    return rows


def check_values(strings, header, rows):
    ctx = fresh_ctx(strings)
    try:
        d = host_dict(strings)
        want = V.values(header, rows, d.encode)
        slot_of = {}
        slots = [slot_of.setdefault(V.strip(v), len(slot_of)) for v in header]
        names = {s: n for n, s in slot_of.items()}
        rel, info = ctx.values(slots, rows)
        assert rel.info()[1] == list(dict.fromkeys(slots))
        assert device_rows(rel, names) == want  # kb_values keeps the row order
        assert info["dict_first"] == len(strings) and info["dict_new"] == len(d.id_to_string) - len(strings)
        assert info["rows_dropped"] == len(rows) - len(want)
        assert ctx.dict_strings_download(len(strings), info["dict_new"]) == d.id_to_string[len(strings):]
        num, isn = ctx.dict_numeric_download(0, len(d.id_to_string))
        for i, t in enumerate(d.id_to_string):
            v = E.rust_parse_f64(t)
            assert bool(isn[i]) == (v is not None), t
            if v is not None:
                assert num[i] == v or (np.isnan(v) and np.isnan(num[i])), t
    finally:
        ctx.close()


def test_hand_worked_block():
    check_values(["<pre>", "7"], ["?a", "?b", "?a"], [["x", "<pre>", None], [None, None, None], ["1.5", "x", "y"], ["7"], [], [None, "z"]])


@pytest.mark.parametrize("seed", range(6))
def test_seeded_blocks(seed):
    rng = random.Random(seed)
    vocab = ["s%d" % k for k in range(40)] + ["%d" % k for k in range(10)] + ["-0.0", "1e3", "NaN", "inf", "<http://x/%d>" % seed, ""]
    header = [rng.choice(["?a", "?b", "?c", "?d"]) for _ in range(rng.randrange(1, 6))]
    check_values(vocab[::3], header, random_block(rng, rng.randrange(0, 400), header, vocab))


def test_a_numeric_table_that_does_not_cover_the_dictionary_is_left_alone():
    ctx = c.Context(0)
    try:
        ctx.dict_strings_load(["a", "1"])  # no f64 table derived
        _, info = ctx.values([0], [["2"], ["b"]])
        assert info["dict_new"] == 2
        with pytest.raises(c.KolibrieError):
            ctx.dict_numeric_download(0, 1)  # still no table: kb_values did not parse the whole dictionary
    finally:
        ctx.close()


def test_empty_header_and_no_rows():
    check_values(["a"], [], [[], []])
    check_values(["a"], ["?x"], [])


def test_refusals_leave_out_and_the_dictionary_untouched():
    ctx = fresh_ctx(["a", "b"])
    try:
        sentinel = C.c_void_p(0x1234)
        L = c.lib()
        slots = (C.c_uint32 * 17)(*range(17))
        undef = np.zeros(17, np.uint8)
        off = np.arange(18, dtype=np.uint64)
        data = np.frombuffer(b"q" * 17, np.uint8).copy()
        rc = L.kb_values(ctx.h, slots, 17, 1, c._ptr(undef), c._ptr(off), c._ptr(data), C.byref(sentinel), None)
        assert rc == c.KB_E_LIMIT and sentinel.value == 0x1234
        undef2 = np.array([1], np.uint8)
        off2 = np.array([0, 1], np.uint64)
        rc = L.kb_values(ctx.h, slots, 1, 1, c._ptr(undef2), c._ptr(off2), c._ptr(data), C.byref(sentinel), None)
        assert rc == c.KB_E_INVALID and sentinel.value == 0x1234  # a non-empty UNDEF cell
        assert ctx.dict_strings_info()[0] == 2
        # a key cell without a value
        left = ctx.rel_from_host([0, 1], [np.array([1, NONE], np.uint32), np.array([5, 6], np.uint32)])
        right = ctx.rel_from_host([0], [np.array([1], np.uint32)])
        keys = (C.c_uint32 * 1)(0)
        rc = L.kb_hash_join_keyed(ctx.h, left.h, right.h, keys, 1, c.MERGE_LEFT_FIRST, C.byref(sentinel))
        assert rc == c.KB_E_UNSUPPORTED and sentinel.value == 0x1234
        rc = L.kb_hash_join_keyed(ctx.h, left.h, right.h, keys, 1, 7, C.byref(sentinel))
        assert rc == c.KB_E_INVALID and sentinel.value == 0x1234
        wide = [ctx.rel_from_host(list(range(6)), [np.array([k], np.uint32) for k in range(6)]) for _ in range(2)]
        keys5 = (C.c_uint32 * 5)(*range(5))
        ctx.get_stats(reset=True)
        rc = L.kb_hash_join_keyed(ctx.h, wide[0].h, wide[1].h, keys5, 5, c.MERGE_LEFT_FIRST, C.byref(sentinel))
        assert rc == c.KB_E_LIMIT and sentinel.value == 0x1234 and ctx.get_stats()["kernel_launches"] == 0
    finally:
        ctx.close()


def ragged_rows(rng, n, names, unbound, mode):
    """mode: 'none' no cell unbound, 'one' exactly one row unbound in each `unbound` name, 'all' every row, 'some' a random share"""
    rows = []
    for i in range(n):
        row = {}
        for k in names:
            if k in unbound and (mode == "all" or (mode == "one" and i == n - 1) or (mode == "some" and rng.random() < 0.3)):
                continue
            row[k] = rng.randrange(4)
        rows.append(row)
    return rows


def rel_of(ctx, slots, rows):
    names = list(slots)
    return ctx.rel_from_host([slots[k] for k in names], [np.array([r.get(k, NONE) for r in rows], np.uint32) for k in names])


def run_join(ctx, kind, lnames, lrows, rnames, rrows):
    sm = E.SlotMap()
    ls = {k: sm.of(k) for k in lnames}
    rs = {k: sm.of(k) for k in rnames}
    sm.ragged.update(ls.values())
    sm.ragged.update(rs.values())
    rel = E.ExecutionEngine._join(ctx, sm, rel_of(ctx, ls, lrows), rel_of(ctx, rs, rrows), kind)
    return device_rows(rel, sm.names)


MODES = ["none", "one", "some", "all"]


@pytest.mark.parametrize("kind", sorted(V.JOINS))
@pytest.mark.parametrize("mode", MODES)
def test_every_join_operator_over_ragged_rows(ctx, kind, mode):
    rng = random.Random(100 * sorted(V.JOINS).index(kind) + MODES.index(mode))
    for trial in range(8):
        lnames, rnames = ["x", "y", "a"], ["y", "x", "b"][: 2 + trial % 2]
        unbound = {"y"} if trial % 2 else {"x", "y"}
        sizes = [(0, 5), (5, 0), (0, 0)] if trial == 0 else [(rng.randrange(1, 60), rng.randrange(1, 60))]
        for nl, nr in sizes:
            lrows = ragged_rows(rng, nl, lnames, unbound, mode)
            rrows = ragged_rows(rng, nr, rnames, unbound if trial % 3 else set(), mode)
            try:
                want = V.JOINS[kind](lrows, rrows)
            except V.Panic:
                with pytest.raises(c.KolibrieError) as e:
                    run_join(ctx, kind, lnames, lrows, rnames, rrows)
                assert e.value.status == c.KB_E_UNSUPPORTED
                continue
            assert V.bag(run_join(ctx, kind, lnames, lrows, rnames, rrows)) == V.bag(want), (kind, mode, trial, nl, nr)


@pytest.mark.parametrize("kind", sorted(V.JOINS))
def test_cartesian_case(ctx, kind):
    lrows = [{"y": 5}, {"x": 1}, {"x": 2, "y": 6}]
    rrows = [{"x": 2}, {"z": 3}]
    assert V.bag(run_join(ctx, kind, ["x", "y"], lrows, ["x", "z"], rrows)) == V.bag(V.JOINS[kind](lrows, rrows))


def test_bind_join_route_unchanged_without_unbound_cells():
    """a ParallelJoin with a scan on the right, over a left side without KB_ID_NONE, is one kb_bind_join: the same result and the same
    kb_stats counters as calling kb_bind_join directly"""
    ctx = c.Context(0)
    try:
        db = E.SparqlDatabase(ctx)
        for i in range(200):
            db.add_triple_parts("e%d" % i, "p", "v%d" % (i % 13))
            db.add_triple_parts("e%d" % i, "q", "w%d" % (i % 7))
        db.build_all_indexes()
        p, q = db.dictionary.lookup("p"), db.dictionary.lookup("q")
        s_, o, w = E.Variable("s"), E.Variable("o"), E.Variable("w")
        plan = E.ParallelJoin(E.IndexScan((s_, E.Constant(p), o)), E.IndexScan((s_, E.Constant(q), w)))
        db._sync()
        sm = E.SlotMap()
        ctx.get_stats(reset=True)
        left = E.ExecutionEngine._run(plan.left, db, sm)
        direct = ctx.bind_join(left, sm.pattern(plan.right.pattern))
        s1 = ctx.get_stats(reset=True)
        via = E.ExecutionEngine._run(plan, db, E.SlotMap())
        s2 = ctx.get_stats(reset=True)
        assert direct.n_rows == via.n_rows == 200
        assert np.array_equal(np.sort(direct.to_numpy(), axis=0), np.sort(via.to_numpy(), axis=0))
        for k in ("kernel_launches", "scan_launches", "build_launches", "probe_launches", "other_launches", "index_joins", "d2h_bytes", "h2d_bytes"):
            assert s1[k] == s2[k], k
    finally:
        ctx.close()


def test_launch_counts_unchanged_without_unbound_cells(ctx):
    """the engine's join route adds nothing to kb_hash_join over relations without KB_ID_NONE"""
    sm = E.SlotMap()
    x, y, z = sm.of("x"), sm.of("y"), sm.of("z")
    a = ctx.rel_from_host([x, y], [np.arange(100, dtype=np.uint32) % 7, np.arange(100, dtype=np.uint32)])
    b = ctx.rel_from_host([x, z], [np.arange(50, dtype=np.uint32) % 7, np.arange(50, dtype=np.uint32)])
    ctx.get_stats(reset=True)
    direct = ctx.hash_join(a, b).n_rows
    s1 = ctx.get_stats(reset=True)
    via = E.ExecutionEngine._join(ctx, sm, a, b, "HashJoin").n_rows
    s2 = ctx.get_stats(reset=True)
    assert direct == via
    for k in ("kernel_launches", "build_launches", "probe_launches", "other_launches", "d2h_bytes"):
        assert s1[k] == s2[k], k


def ref_exec(plan, d, triples):
    if isinstance(plan, E.Values):
        return V.values(plan.variables, plan.values, d.encode)
    if isinstance(plan, (E.TableScan, E.IndexScan)):
        return V.scan(tuple("?" + t.name if isinstance(t, E.Variable) else t.id for t in plan.pattern), triples)
    if isinstance(plan, E.ParallelJoin) and isinstance(plan.right, (E.TableScan, E.IndexScan)):
        pat = tuple("?" + t.name if isinstance(t, E.Variable) else t.id for t in plan.right.pattern)
        return V.bind_join(ref_exec(plan.left, d, triples), pat, triples)
    if isinstance(plan, (E.HashJoin, E.OptimizedHashJoin, E.NestedLoopJoin, E.ParallelJoin)):
        return V.JOINS[type(plan).__name__](ref_exec(plan.left, d, triples), ref_exec(plan.right, d, triples))
    raise TypeError(plan)


@pytest.mark.parametrize("seed", range(4))
def test_engine_end_to_end_on_planner_plans(seed):
    rng = random.Random(seed)
    ctx = c.Context(0)
    try:
        db = E.SparqlDatabase(ctx)
        for i in range(60):
            db.add_triple_parts("e%d" % rng.randrange(20), rng.choice(["p", "q"]), "v%d" % rng.randrange(15))
        db.build_all_indexes()
        p, q = db.dictionary.lookup("p"), db.dictionary.lookup("q")
        pats = [(E.Variable("s"), E.Constant(p), E.Variable("o")), (E.Variable("s"), E.Constant(q), E.Variable("w"))][: 1 + seed % 2]
        header = [["?s"], ["?s", "?o"], ["?o", "?s", "?x"], ["?w", "?s"]][seed]
        vocab = ["e%d" % k for k in range(25)] + ["v%d" % k for k in range(18)]
        rows = random_block(rng, 30 + 400 * (seed == 3), header, vocab, p_undef=0.15 * (seed > 0))
        stats = PL.DatabaseStats(db.triples)
        logical = PL.build_logical_plan(pats, values=PL.LValues(header, rows))
        plan = PL.lower_to_engine(PL.Streamertail(stats).find_best_plan(logical))
        d = host_dict(db.dictionary.id_to_string)
        try:
            want = ref_exec(plan, d, sorted(db.triples))
        except V.Panic:
            with pytest.raises(c.KolibrieError) as e:
                E.ExecutionEngine.execute_with_ids(plan, db)
            assert e.value.status == c.KB_E_UNSUPPORTED
            return
        got = E.ExecutionEngine.execute_with_ids(plan, db)
        assert V.bag(got) == V.bag(want), plan
        assert db.dictionary.id_to_string == d.id_to_string
    finally:
        ctx.close()


def test_million_row_block_at_cfg2_size():
    """10^6 subject IRIs (about 5 % new, 2 % UNDEF) against a dictionary of cfg2's 10 M-triple store"""
    from kolibrie_b200 import datagen

    dd = datagen.employee_dataset(1_666_667)
    strings = ["<http://example.org/t%d>" % i for i in range(dd.n_ids)]
    ctx = fresh_ctx(strings)
    try:
        rng = np.random.default_rng(3)
        subj = rng.choice(np.unique(dd.s), 1_000_000)
        rows = [[None] if rng.random() < 0.02 else (["<http://example.org/new%d>" % k] if k % 20 == 0 else [strings[int(sj)]])
                for k, sj in enumerate(subj.tolist())]
        rel, info = ctx.values([0], rows)
        d = host_dict(strings)
        want = [d.encode(r[0]) for r in rows if r[0] is not None]
        assert np.array_equal(rel.column(0), np.array(want, np.uint32))
        assert info["dict_new"] == len(d.id_to_string) - len(strings) and info["rows_dropped"] == len(rows) - len(want)
        assert ctx.dict_strings_download(len(strings), info["dict_new"]) == d.id_to_string[len(strings):]
    finally:
        ctx.close()
