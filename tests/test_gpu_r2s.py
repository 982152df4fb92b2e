"""GPU (-m gpu): kb_r2s_eval, the Relation-to-Stream operators on device relations, against the restatement of r2s.rs in
tests/r2s_reference.py. Every case compares the emitted rows by exact list equality, order included: ISTREAM in response order with
duplicates kept, DSTREAM in the order the rows first appeared in the response that set the state."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200.engine import Dictionary, Relation2StreamOperator
from tests import r2s_cases
from tests.r2s_reference import DSTREAM, ISTREAM, RSTREAM, Relation2Stream
from tests.test_r2s import load

pytestmark = pytest.mark.gpu


def rows_of(rel, slots):
    return list(map(tuple, rel.to_numpy(slots).tolist()))


def rel_of(ctx, slots, rows, order=None):
    """a relation holding `rows` (tuples in `slots` order), its columns stored in `order`"""
    a = np.asarray(rows, dtype=np.uint32).reshape(-1, len(slots))
    order = list(range(len(slots))) if order is None else list(order)
    return ctx.rel_from_host([slots[j] for j in order], [np.ascontiguousarray(a[:, j]) for j in order])


def check(op, ref, rel, slots, what):
    want = ref.eval(rows_of(rel, slots))
    got = op.eval(rel)
    assert got.slots == list(slots), what
    assert rows_of(got, slots) == want, what
    assert op.info() == (len(ref.last), ref.stream_operator), what
    return got


# ------------------------------------------------------------------ the reference's tests
@pytest.mark.parametrize("case", [c_ for c_ in r2s_cases.CASES if "vars" in c_], ids=lambda c_: c_["name"])
def test_r2s_unit_tests(ctx, case):
    d = Dictionary()
    slots = list(range(len(case["vars"])))
    ref = Relation2Stream(case["stream"])
    op = ctx.r2s(ref.stream_operator, slots)
    for k, f in enumerate(case["firings"]):
        rows = [tuple(d.encode(v) for v in r) for r in f["rows"]]
        got = check(op, ref, rel_of(ctx, slots, rows), slots, (case["name"], k))
        if f["emit"] is not None:
            assert [[d.decode(i) for i in r] for r in rows_of(got, slots)] == f["emit"], (case["name"], k)
    op.free()


def window_cases():
    out = [c_ for c_ in r2s_cases.CASES if "window" in c_["firings"][0]]
    return out + [c_ for c_ in load("rsp_windows.json")["cases"] if c_["stream"] in ("ISTREAM", "RSTREAM")]


@pytest.mark.parametrize("case", window_cases(), ids=lambda c_: c_["name"])
def test_window_firings_through_device_segments(ctx, case):
    """each firing: the segments whose triples left the window are evicted, the firing's new triples are appended as one segment, the
    pattern is scanned and the operator runs on the scan's rows"""
    d = Dictionary()
    ctx.store_clear()
    pat = case["pattern"]
    slot = {v: k for k, v in enumerate(case["select"])}
    term = lambda x: c.V(slot[x[1:]]) if x.startswith("?") else c.K(d.encode(x))
    ref = Relation2Stream(case["stream"])
    op = ctx.r2s(ref.stream_operator, list(range(len(slot))))
    live, seg_rows = {}, {}
    for k, f in enumerate(case["firings"]):
        win = [tuple(d.encode(x) for x in t) for t in f["window"]]
        for t in [t for t in live if t not in set(win)]:
            tag = live.pop(t)
            seg_rows[tag] -= 1
            if seg_rows[tag] == 0:
                ctx.store_evict(tag)
        new = [t for t in dict.fromkeys(win) if t not in live]
        if new:
            a = np.array(new, dtype=np.uint32)
            ctx.store_append(a[:, 0], a[:, 1], a[:, 2], tag=100 + k)
            live.update({t: 100 + k for t in new})
            seg_rows[100 + k] = len(new)
        assert ctx.store_size()[0] == len(set(win))
        scanned = ctx.scan([c.pattern(term(pat[0]), term(pat[1]), term(pat[2]))])[0]
        resp = ctx.project(scanned, list(range(len(slot))))
        got = check(op, ref, resp, list(range(len(slot))), (case["name"], k))
        assert [[d.decode(i) for i in r] for r in rows_of(got, list(range(len(slot))))] == f["emit"], (case["name"], k)
    op.free()
    ctx.store_clear()


# ------------------------------------------------------------------ seeded random firing sequences
def firing_plan(rng, n_cols):
    """(name, rows) per firing: empty first / middle / last, heavy duplication, 0 / ~50 / 100 % overlap with the previous firing, rows
    that differ only by a swap of two columns' values or only in one column's high bits"""
    fresh = lambda n: rng.integers(0, 1 << 32, (n, n_cols), dtype=np.uint64).astype(np.uint32)
    dup = lambda n, dom: rng.integers(0, dom, (n, n_cols), dtype=np.uint32)
    plan, prev = [], np.zeros((0, n_cols), np.uint32)

    def add(name, rows):
        nonlocal prev
        plan.append((name, rows))
        prev = rows

    add("empty first", prev)
    add("heavy duplication", dup(5000, 6))
    add("0% overlap", fresh(3000))
    half = prev[rng.integers(0, len(prev), 1500)]
    add("~50% overlap", rng.permutation(np.concatenate([half, fresh(1500)])))
    add("100% overlap", rng.permutation(np.concatenate([prev, prev[: len(prev) // 3]])))
    add("empty middle", np.zeros((0, n_cols), np.uint32))
    base = fresh(2000)
    add("base", base)
    if n_cols >= 2:
        sw = base.copy()
        sw[:, [0, n_cols - 1]] = sw[:, [n_cols - 1, 0]]
        add("columns swapped", rng.permutation(np.concatenate([base[:1000], sw])))
    hb = prev.copy()
    hb[:, n_cols // 2] ^= np.uint32(0x80000000)
    hb[::7, 0] = np.uint32(0xFFFFFFFF)
    add("high bits", np.concatenate([hb, prev[:500]]))
    add("large bag", dup(300_000, 40 if n_cols <= 2 else 4))
    add("large, ~50% overlap", rng.permutation(np.concatenate([prev[:150_000], fresh(150_000)])))
    add("empty last", np.zeros((0, n_cols), np.uint32))
    return plan


@pytest.mark.parametrize("n_cols", [1, 2, 3, 8, 16])
@pytest.mark.parametrize("stream", [ISTREAM, DSTREAM], ids=["ISTREAM", "DSTREAM"])
def test_random_firings(ctx, stream, n_cols):
    rng = np.random.default_rng(97 * n_cols + stream)
    slots = [int(x) for x in rng.permutation(40)[:n_cols]]
    ref = Relation2Stream(stream)
    op = ctx.r2s(stream, slots)
    for name, rows in firing_plan(rng, n_cols):
        order = rng.permutation(n_cols)  # the response's column order changes between firings
        rel = rel_of(ctx, slots, rows, order)
        check(op, ref, rel, slots, name)
        rel.free()
    op.free()


def test_rstream_returns_the_response(ctx):
    ist = ctx.r2s(ISTREAM, [3, 7])
    ist.eval(rel_of(ctx, [3, 7], [(1, 2), (1, 2), (5, 6)]))
    op = ctx.r2s(RSTREAM, [3, 7])
    rel = rel_of(ctx, [3, 7], [(9, 8), (1, 2), (9, 8)], order=[1, 0])
    got = op.eval(rel)
    assert got.slots == rel.slots == [7, 3]
    assert np.array_equal(got.to_numpy(), rel.to_numpy())
    assert op.info() == (0, RSTREAM) and ist.info() == (2, ISTREAM)
    assert op.eval(rel_of(ctx, [3, 7], [])).n_rows == 0 and op.info() == (0, RSTREAM)
    op.free()
    ist.free()


@pytest.mark.parametrize("stream", [ISTREAM, DSTREAM], ids=["ISTREAM", "DSTREAM"])
def test_other_slot_set_is_refused_and_changes_nothing(ctx, stream):
    ref = Relation2Stream(stream)
    op = ctx.r2s(stream, [1, 2])
    check(op, ref, rel_of(ctx, [1, 2], [(1, 1), (2, 2), (3, 3)]), [1, 2], "first")
    for bad in ([1, 3], [1], [1, 2, 3], [2, 5]):
        with pytest.raises(c.KolibrieError) as e:
            op.eval(rel_of(ctx, bad, [tuple(range(len(bad)))] * 2))
        assert e.value.status == c.KB_E_INVALID, bad
        assert op.info() == (3, stream)
    check(op, ref, rel_of(ctx, [1, 2], [(3, 3), (4, 4)], order=[1, 0]), [1, 2], "after the refusals")
    with pytest.raises(c.KolibrieError) as e:
        ctx.r2s(stream, [4, 4])
    assert e.value.status == c.KB_E_INVALID
    with pytest.raises(c.KolibrieError):
        ctx.r2s(stream, [])
    with pytest.raises(c.KolibrieError):
        ctx.r2s(3, [1])
    op.free()


def test_engine_operator_over_a_window(ctx):
    """engine.Relation2StreamOperator (rsp/r2s.rs) over SimpleR2R.execute_query_rel: the rows of rsp_ql_dstream_semantics"""
    from kolibrie_b200.engine import Constant, SimpleR2R, TableScan, Variable

    case = [c_ for c_ in r2s_cases.CASES if c_["name"] == "rsp_ql_dstream_semantics"][0]
    r2r = SimpleR2R(ctx)
    ctx.store_clear()
    d = r2r.item.dictionary
    a, dtype = d.encode("a"), d.encode(case["pattern"][2])
    q = TableScan((Variable("s"), Constant(a), Constant(dtype)))
    r2s = Relation2StreamOperator(ctx, "DSTREAM")
    prev = []
    emitted = []
    for f in case["firings"]:
        win = [tuple(d.encode(x) for x in t) for t in f["window"]]
        for t in prev:
            if t not in win:
                r2r.remove(t)
        for t in win:
            if t not in prev:
                r2r.add(t)
        prev = win
        rel = r2r.execute_query_rel(q)
        out = r2s.eval(rel, 0)
        emitted.append([[d.decode(int(x)) for x in row] for row in out.to_numpy().tolist()])
    assert emitted == [f["emit"] for f in case["firings"]]
    assert r2r.slot_names == ["s"] and r2s.last_rows() == 4
    r2s.free()
    ctx.store_clear()


# ------------------------------------------------------------------ the cfg5 window (10 slides, query cfg2, index path)
def run_cfg5(per_slide, n_slides, check_rows):
    ctx = c.Context(0)
    try:
        width, per_e = 10, per_slide // 6
        d = datagen.employee_dataset(per_e * n_slides)
        ctx.dict_numeric_load(d.num_or0, d.is_num)
        js, pats, filt = datagen.employee_queries(d)["cfg2"]
        slots = [0, 1, 2, 3]  # e, t, s, n
        ist, dst = ctx.r2s(ISTREAM, slots), ctx.r2s(DSTREAM, slots)
        ref_i, ref_d = Relation2Stream(ISTREAM), Relation2Stream(DSTREAM)
        rich = lambda t: d.subj_prefix[t * per_e + np.nonzero(d.salary_of_employee[t * per_e:(t + 1) * per_e] > 100000)[0]]
        live = []
        for t in range(n_slides):
            lo, hi = t * per_slide, (t + 1) * per_slide
            if len(live) == width:
                ctx.store_evict(live.pop(0))
            ctx.store_append(d.s[lo:hi], d.p[lo:hi], d.o[lo:hi], tag=100 + t)
            live.append(100 + t)
            if t == 0:
                ctx.build_index()
            n0 = ctx.get_stats()["index_joins"]
            r = ctx.star_join(js, pats, filt)
            assert ctx.get_stats()["index_joins"] > n0, "cfg2 left the index path"
            ei, ed = ist.eval(r), dst.eval(r)
            # closed form: ISTREAM = the new slide's employees with salary > 100000, DSTREAM = the evicted slide's
            assert np.array_equal(np.sort(ei.column(0)), np.sort(rich(t))), t
            if t >= width:
                assert np.array_equal(np.sort(ed.column(0)), np.sort(rich(t - width))), t
            else:
                assert ed.n_rows == 0, t
            assert ist.info()[0] == dst.info()[0] == r.n_rows
            if check_rows:
                rows = rows_of(r, slots)
                assert rows_of(ei, slots) == ref_i.eval(rows), t
                assert rows_of(ed, slots) == ref_d.eval(rows), t
            for x in (r, ei, ed):
                x.free()
        ist.free()
        dst.free()
    finally:
        ctx.close()


def test_cfg5_window_tenth_scale():
    run_cfg5(100_002, 12, check_rows=True)


def test_cfg5_window_full_scale():
    run_cfg5(1_000_002, 12, check_rows=False)
