"""GPU (-m gpu): kb_order_by (ORDER BY + LIMIT on the device) against the restatement of apply_order_by in tests/order_reference.py,
row for row: numeric and string keys, 1-4 keys, every LIMIT around the cut, both routes, the refusals, the engine mirror, and the
100 M-triple headline result."""
import ctypes as C

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200.engine import ExecutionEngine, InMemoryBuffer, OrderCondition, SortDirection, SparqlDatabase
from tests import order_reference as R

pytestmark = pytest.mark.gpu
NONE = c.KB_ID_NONE


@pytest.fixture(scope="module")
def cx():
    x = c.Context(0)
    yield x
    x.close()


def load_dict(cx, strings, quoted=None):
    cx.dict_strings_load(strings)
    cx.dict_numeric_derive(c.NUMERIC_F64, 0)
    q = quoted or {}
    ids = np.array(list(q.keys()), np.uint32)
    comp = np.array(list(q.values()), np.uint32).reshape(-1, 3)
    cx.quoted_load(ids, comp[:, 0], comp[:, 1], comp[:, 2])


def check(cx, strings, quoted, slots, cols, keys, limit, route=None):
    """kb_order_by of the relation (slots, cols) against the restatement; keys = [(slot, desc)]"""
    rel = cx.rel_from_host(slots, cols)
    out, info = cx.order_by(rel, keys, limit)
    n = len(cols[0]) if cols else 0
    rows = [{s: R.render(int(col[i]), strings, quoted) for s, col in zip(slots, cols)} for i in range(n)]
    want = R.order_rows(rows, keys, limit)
    got = out.to_numpy(slots)
    assert out.slots == list(slots)
    expect = np.stack([np.asarray(col)[want] for col in cols], axis=1) if cols else got
    assert got.shape == expect.shape and np.array_equal(got, expect), (keys, limit, info)
    assert info["n_rows_in"] == n and info["n_rows_out"] == len(want)
    if route is not None:
        assert info["route"] == route, info
    assert np.array_equal(rel.to_numpy(slots), np.stack(cols, axis=1)), "the input relation changed"
    return info


NUMBERS = ["0", "-0", "0.0", "-0.0", "1", "-1", "10", "9", "2.5", "2.50", "1e3", "999", "1E-3", "-1e308", "1e308", "inf", "-inf", "+inf",
           "Infinity", "-Infinity", "123456789012345678901234567890", "0.1", "0.30000000000000004", "5.", ".5", "7"]


@pytest.mark.parametrize("desc", [False, True])
def test_numeric_key_every_limit(cx, desc):
    strings = NUMBERS + [""]
    load_dict(cx, strings)
    rng = np.random.default_rng(1 + desc)
    n = 300
    ids = rng.integers(0, len(strings), n).astype(np.uint32)
    ids[::17] = NONE
    other = rng.integers(0, 1 << 30, n).astype(np.uint32)
    info = check(cx, strings, {}, [3, 5], [ids, other], [(3, desc)], 0, c.ORDER_SORT)
    assert info["key_kind"] == [c.ORDER_NUMERIC] and info["string_rounds"] == [0]
    for limit in (1, 7, 18, 19, n - 1, n, n + 1):  # 7 and 18/19 cut through runs of ties
        check(cx, strings, {}, [3, 5], [ids, other], [(3, desc)], limit, c.ORDER_TOPK if limit * 16 <= n else c.ORDER_SORT)


def test_all_nan_column_and_nan_refused_with_numbers(cx):
    strings = ["NaN", "nan", "-nan", "", "1", "2"]
    load_dict(cx, strings)
    ids = np.array([0, 3, 1, 2, NONE, 0, 3], np.uint32)
    info = check(cx, strings, {}, [0], [ids], [(0, True)], 0)
    assert info["key_kind"] == [c.ORDER_NUMERIC]
    with pytest.raises(c.KolibrieError) as e:
        cx.order_by(cx.rel_from_host([0], [np.array([0, 4, 5], np.uint32)]), [(0, False)])
    assert e.value.status == c.KB_E_UNSUPPORTED


def string_dictionary(rng):
    prefix = "http://example.org/a/very/long/shared/prefix/that/runs/past/sixty/four/bytes/"
    assert len(prefix) > 64
    out = ["", "a", "ab", "ab\0", "ab\x01", "z", "é", "éa", "中文", "🙂", "Z", "b"]
    out += [prefix + s for s in ["", "x", "xy", "x\0", "é", "zz", "x" * 30, "x" * 29 + "y"]]
    base = "abcdefghijklmnop"
    for k in (6, 7, 13, 14):  # first difference at bytes 6, 7, 13 and 14
        out += [base[:k] + "a" + "q" * 5, base[:k] + "b", base[:k]]
    alphabet = list("abcxyz/:#") + ["é", "ß"]
    out += ["".join(rng.choice(alphabet, int(rng.integers(1, 40)))) for _ in range(300)]
    return out


@pytest.mark.parametrize("desc", [False, True])
def test_string_key(cx, desc):
    rng = np.random.default_rng(7)
    strings = string_dictionary(rng)
    nd = len(strings)
    # quoted ids: << 1 2 1 >>, a nested one, one with a component past the dictionary ("unknown") and one the table lacks
    quoted = {0x80000000: (1, 2, 1), 0x80000001: (0x80000000, 5, 0), 0x80000002: (1, nd + 50, 1)}
    load_dict(cx, strings, quoted)
    n = 2000
    ids = rng.integers(0, nd, n).astype(np.uint32)
    ids[::23] = NONE
    ids[5::31] = rng.integers(nd, nd + 1000, len(ids[5::31]))  # "unknown": past the dictionary, all one value
    ids[7::41] = rng.choice([0x80000000, 0x80000001, 0x80000002, 0x80000007], len(ids[7::41]))
    payload = np.arange(n, dtype=np.uint32)
    info = check(cx, strings, quoted, [1, 2], [ids, payload], [(1, desc)], 0, c.ORDER_SORT)
    assert info["key_kind"] == [c.ORDER_STRING] and info["string_rounds"][0] >= 11  # the 80-byte strings take 12 rounds
    for limit in (1, 10, 125, n - 1, n, n + 1):
        check(cx, strings, quoted, [1, 2], [ids, payload], [(1, desc)], limit)


@pytest.mark.parametrize("seed", range(6))
def test_several_keys(cx, seed):
    rng = np.random.default_rng(100 + seed)
    strings = ["a", "b", "ab", "", "ba", "1", "2", "10", "-3", "2.0", "x" * 20, "x" * 21]
    load_dict(cx, strings)
    n = 1500
    num = rng.choice([5, 6, 7, 8, 9, 3], n).astype(np.uint32)  # numbers and ""
    txt = rng.choice([0, 1, 2, 3, 4, 10, 11], n).astype(np.uint32)  # strings and ""
    num2 = rng.choice([5, 6, 9, NONE], n).astype(np.uint32)
    txt2 = rng.choice([0, 1, NONE], n).astype(np.uint32)
    slots = [10, 11, 12, 13]
    cols = [num, txt, num2, txt2]
    n_keys = 1 + seed % 4
    keys = [(int(s), bool(rng.integers(0, 2))) for s in rng.permutation(slots)[:n_keys]]
    for limit in (0, 1, 50, 93, n):
        check(cx, strings, {}, slots, cols, keys, limit)


def test_routes_agree(cx):
    rng = np.random.default_rng(3)
    strings = [str(v) for v in range(40)] + ["w%d" % v for v in range(40)]
    load_dict(cx, strings)
    n = 20000
    a = rng.integers(0, 40, n).astype(np.uint32)
    b = rng.integers(40, 80, n).astype(np.uint32)
    rel = cx.rel_from_host([0, 1], [a, b])
    for keys in ([(0, True)], [(0, False), (1, True)], [(1, False)]):
        full, fi = cx.order_by(rel, keys, 0)
        for limit in (1, 10, 500, 1250):  # 1250 * 16 == n: the largest limit top-k takes
            top, ti = cx.order_by(rel, keys, limit)
            assert fi["route"] == c.ORDER_SORT and ti["route"] == c.ORDER_TOPK, (fi, ti)
            assert np.array_equal(top.to_numpy([0, 1]), full.to_numpy([0, 1])[:limit])
        check(cx, strings, {}, [0, 1], [a, b], keys, 10, c.ORDER_TOPK)


def test_empty_no_keys_duplicates_and_absent_slot(cx):
    strings = ["b", "a", "3", "1"]
    load_dict(cx, strings)
    empty = cx.rel_from_host([0, 1], [np.zeros(0, np.uint32), np.zeros(0, np.uint32)])
    out, info = cx.order_by(empty, [(0, False)], 5)
    assert out.n_rows == 0 and out.slots == [0, 1] and info["route"] == c.ORDER_VIEW
    ids = np.array([0, 1, 0, 1, 1, 0], np.uint32)
    tag = np.array([7, 7, 7, 7, 8, 7], np.uint32)  # duplicate rows
    for limit in (0, 4):
        info = check(cx, strings, {}, [0, 1], [ids, tag], [], limit, c.ORDER_VIEW)
        assert info["key_kind"] == []
        check(cx, strings, {}, [0, 1], [ids, tag], [(9, True)], limit, c.ORDER_VIEW)  # slot 9 is "" in every row
        info = check(cx, strings, {}, [0, 1], [ids, tag], [(9, False), (0, True), (1, False)], limit)
        # tags 7 and 8 are past the dictionary: both "unknown", one value
        assert info["key_kind"] == [c.ORDER_CONST, c.ORDER_STRING, c.ORDER_CONST] and info["n_distinct"] == [0, 2, 2]
    check(cx, strings, {}, [0, 1], [ids, np.full(6, 2, np.uint32)], [(1, False)], 0, c.ORDER_VIEW)  # one value: nothing to sort


def test_unbound_cells_from_natural_join_and_bind(cx):
    strings = ["x", "y", "5", "6", "z"]
    load_dict(cx, strings)
    left = cx.rel_from_host([0, 1], [np.array([0, 1, 4, 0], np.uint32), np.array([2, NONE, 3, NONE], np.uint32)])
    right = cx.rel_from_host([0, 2], [np.array([0, 1, 4], np.uint32), np.array([NONE, 2, 3], np.uint32)])
    joined = cx.natural_join(left, right)
    slots = joined.slots
    cols = [joined.column(i) for i in range(len(slots))]
    assert any((col == NONE).any() for col in cols)
    for desc in (False, True):
        check(cx, strings, {}, slots, cols, [(1, desc), (2, not desc)], 0)
    bound, _ = cx.bind(left, c.BIND_SUBJECT, [c.V(0)], 3)  # no quoted ids: every output cell is KB_ID_NONE
    out, info = cx.order_by(bound, [(3, False), (1, True)])
    assert info["key_kind"] == [c.ORDER_CONST, c.ORDER_NUMERIC]
    assert out.column(1).tolist() == [3, 2, NONE, NONE]


def raw_order_by(cx, rel, keys, n_keys=None, limit=0):
    arr = (c.KbOrderKey * max(len(keys), 1))(*[c.KbOrderKey(s, d) for s, d in keys])
    out = C.c_void_p(0x1234)
    rc = c.lib().kb_order_by(cx.h, rel.h, arr, len(keys) if n_keys is None else n_keys, limit, C.byref(out), None)
    return rc, out.value


def test_refusals_leave_out_untouched(cx):
    strings = ["10", "9", "1a", "NaN", "1", "a", "b"]
    load_dict(cx, strings)
    mixed = cx.rel_from_host([0], [np.array([0, 1, 2], np.uint32)])
    assert raw_order_by(cx, mixed, [(0, 0)]) == (c.KB_E_UNSUPPORTED, 0x1234)
    assert "mixes" in c.lib().kb_last_error(cx.h).decode()
    assert raw_order_by(cx, cx.rel_from_host([0], [np.array([3, 4], np.uint32)]), [(0, 1)]) == (c.KB_E_UNSUPPORTED, 0x1234)
    assert raw_order_by(cx, mixed, [(0, 0)] * 17) == (c.KB_E_INVALID, 0x1234)
    rc = c.lib().kb_order_by(cx.h, mixed.h, None, 1, 0, C.byref(C.c_void_p()), None)
    assert rc == c.KB_E_INVALID
    # quoted ids without a quoted-triple table
    cx.quoted_load(np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    q = cx.rel_from_host([0], [np.array([5, 0x80000000], np.uint32)])
    assert raw_order_by(cx, q, [(0, 0)]) == (c.KB_E_UNSUPPORTED, 0x1234)
    # a numeric side table that covers fewer ids than the dictionary
    cx.dict_strings_load(strings + ["c", "d"])
    s = cx.rel_from_host([0], [np.array([5, 6], np.uint32)])
    assert raw_order_by(cx, s, [(0, 0)]) == (c.KB_E_UNSUPPORTED, 0x1234)
    cx.dict_numeric_derive(c.NUMERIC_F64, c.NUMERIC_APPEND)
    assert cx.order_by(s, [(0, 1)])[0].column(0).tolist() == [6, 5]
    # a string key without device dictionary strings; a numeric one still runs on the numeric table
    cx.dict_strings_load([])
    assert raw_order_by(cx, s, [(0, 0)]) == (c.KB_E_UNSUPPORTED, 0x1234)
    num = cx.rel_from_host([0], [np.array([0, 4, 1], np.uint32)])
    assert cx.order_by(num, [(0, 0)])[0].column(0).tolist() == [4, 1, 0]


def test_engine_execute_orders_like_the_reference(cx):
    db = SparqlDatabase(cx)
    content = []
    for i in range(1, 61):
        iri = "http://example.org/employee%d" % i
        title = ["Manager", "Developer", "Salesperson"][i % 3]
        sal = str(30000 + (977 * i) % 5000)
        code = ["10", "9", "1a", "b"][i % 4] if i < 50 else str(i)
        db.add_triple_parts(iri, "foaf:title", title)
        db.add_triple_parts(iri, "ds:annual_salary", sal)
        db.add_triple_parts(iri, "ex:code", code)
        content.append({k: db.dictionary.lookup(v) for k, v in (("e", iri), ("t", title), ("s", sal), ("k", code))})
    op = InMemoryBuffer(content)  # rows in a fixed order, so that ties have one stable answer
    rows = ExecutionEngine.execute(op, db)
    assert R.is_mixed([r["k"] for r in rows])
    cases = [([OrderCondition("?s", SortDirection.DESC)], 10), ([OrderCondition("t"), OrderCondition("s", SortDirection.DESC)], 0),
             ([OrderCondition("e")], 7), ([OrderCondition("t", SortDirection.DESC)], 25), ([], 5), ([OrderCondition("missing")], 3),
             ([OrderCondition("k")], 0), ([OrderCondition("t"), OrderCondition("k", SortDirection.DESC)], 12)]  # the last two: host fallback
    for conds, limit in cases:
        got = ExecutionEngine.execute(op, db, order_by=conds, limit=limit)
        want = R.order_rows(rows, [(o.variable.lstrip("?"), o.direction == SortDirection.DESC) for o in conds], limit)
        assert got == [rows[i] for i in want], conds


E_FULL = 16_666_667  # 100 000 002 triples: the headline star join


def test_headline_result_at_full_size():
    d = datagen.employee_dataset(E_FULL)
    x = c.Context(0)
    try:
        x.dict_numeric_load(d.num_or0, d.is_num)
        x.store_load(d.s, d.p, d.o)
        js, pats, filt = datagen.employee_queries(d)["cfg2"]  # slots e, t, s, n
        rel = x.star_join(js, pats, filt)
        n = rel.n_rows
        assert n == 6_945_872
        cols = rel.to_numpy([0, 1, 2, 3])
        # ORDER BY DESC(?s) LIMIT 10: every salary id is numeric, so the order is that of its value
        out, info = x.order_by(rel, [(2, True)], 10)
        assert info["route"] == c.ORDER_TOPK and info["key_kind"] == [c.ORDER_NUMERIC]
        want = np.argsort(-d.num_or0[cols[:, 2]], kind="stable")[:10]
        assert np.array_equal(out.to_numpy([0, 1, 2, 3]), cols[want])
        # a full sort by a string key: ?e rendered as an IRI whose digits do not follow the id order
        strings = [(repr(float(d.num_or0[i])) if d.is_num[i] else "http://example.org/e/%010d" % ((i * 2654435761) % (1 << 32)))
                   for i in range(d.n_ids)]
        x.dict_strings_load(strings)
        full, info = x.order_by(rel, [(0, False)], 0)
        assert info["route"] == c.ORDER_SORT and info["key_kind"] == [c.ORDER_STRING] and info["string_rounds"] == [5]
        keys = np.array(strings, dtype=object)[cols[:, 0]].astype("S")
        assert np.array_equal(full.to_numpy([0, 1, 2, 3]), cols[np.argsort(keys, kind="stable")])
    finally:
        x.close()
