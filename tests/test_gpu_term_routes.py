"""GPU (-m gpu): what every entry point over the device dictionary and the quoted-triple table costs, pinned for each shape it takes.

Like test_gpu_group_routes.py: every case runs twice on a context of its own and checks, for each call, the result against the
existing references and the *fingerprint* against a literal: the change of every integer counter of kb_stats across the call (launches
per family, kernel launches, rows, bytes copied). d2h_bytes counts whole control-arena reads, so it also pins the number of host
synchronisations. The state a case starts from is rebuilt before each of its two calls. Counters that did not move are left out of the
literals.

The shapes:
  kb_dict_encode          first batch into an empty dictionary, repeats inside a batch, a batch the dictionary holds, a batch that
                          forces the persistent index to be rebuilt, the first encode after kb_dict_strings_load (lazy index build)
  kb_rel_decode           plain ids, ids past the dictionary, nested quoted ids, an empty relation
  kb_order_by             one string key holding KB_ID_NONE, quoted ids and ids past the dictionary
  kb_serialize_*          N-Triples and Turtle of a small store with quoted terms and missing ids
  kb_quoted_load          replacing a table, n = 0; kb_quoted_download over a range that runs past the table
  kb_scan_quoted          index on, index off, no table
  kb_bind                 SUBJECT / PREDICATE / OBJECT with and without an old column; isTRIPLE needing "true", "false", both,
                          neither; TRIPLE all hits, all new, repeats in the batch, first after kb_quoted_load; CONCAT
  kb_values               a block that adds strings
and the status code of each invalid call at each entry point.
"""
import ctypes as C

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import engine as E
from tests import order_reference as OR
from tests import quoted_cases as Q
from tests import serialize_reference as SR
from tests import values_reference as VR
from tests.test_gpu_bind import check as bind_check
from tests.test_gpu_bind import new_db, pools, upload
from tests.test_gpu_dict_encode import batch, seq_encode
from tests.test_gpu_quoted import corner_db, host_rows, pattern_term, rows_of, sync
from tests.test_gpu_serialize import seeded_store

pytestmark = pytest.mark.gpu

NONE = c.KB_ID_NONE
QB = Q.QBIT
FIELDS = ("scan_launches", "build_launches", "probe_launches", "filter_launches", "group_launches", "other_launches", "kernel_launches",
          "rows_scanned", "rows_built", "rows_probed", "h2d_bytes", "d2h_bytes", "fused_scan_builds", "index_joins")

# name -> fingerprints of the first and the second call (recorded on an H100)
ROUTES = {
    "encode_first_batch": [{"other_launches": 2, "kernel_launches": 12, "h2d_bytes": 1107096, "d2h_bytes": 175248}] * 2,
    "encode_repeats": [{"other_launches": 2, "kernel_launches": 13, "h2d_bytes": 87, "d2h_bytes": 98372}] * 2,
    "encode_all_held": [{"other_launches": 2, "kernel_launches": 11, "h2d_bytes": 45078, "d2h_bytes": 70268}] * 2,
    "encode_index_rebuild": [{"other_launches": 2, "kernel_launches": 13, "h2d_bytes": 2269639, "d2h_bytes": 365816}] * 2,
    "encode_after_strings_load": [{"other_launches": 2, "kernel_launches": 13, "h2d_bytes": 273881, "d2h_bytes": 124000}] * 2,
    "encode_null_offsets": [{}] * 2,
    "encode_null_ids": [{}] * 2,
    "encode_offsets_not_at_0": [{}] * 2,
    "encode_null_bytes": [{}] * 2,
    "encode_too_many_terms": [{}] * 2,
    "encode_too_many_bytes": [{}] * 2,
    "decode_plain": [{"other_launches": 2, "kernel_launches": 5, "d2h_bytes": 295400}] * 2,
    "decode_unknown": [{"other_launches": 2, "kernel_launches": 5, "d2h_bytes": 32825}] * 2,
    "decode_quoted_nested": [{"other_launches": 2, "kernel_launches": 5, "d2h_bytes": 33275}] * 2,
    "decode_quoted_without_table": [{"other_launches": 1, "kernel_launches": 4, "d2h_bytes": 32768}] * 2,
    "decode_too_deep": [{"other_launches": 1, "kernel_launches": 4, "d2h_bytes": 32768}] * 2,
    "decode_empty": [{"other_launches": 2, "kernel_launches": 5, "d2h_bytes": 32772}] * 2,
    "order_by_string_key": [{"other_launches": 12, "kernel_launches": 22, "d2h_bytes": 163848}] * 2,
    "serialize_nt": [{"other_launches": 10, "kernel_launches": 20, "d2h_bytes": 176261}] * 2,
    "serialize_ttl": [{"other_launches": 15, "kernel_launches": 35, "d2h_bytes": 239960}] * 2,
    "quoted_load_replace": [{"h2d_bytes": 96}] * 2,
    "quoted_load_empty": [{}] * 2,
    "quoted_load_not_quoted_id": [{}] * 2,
    "quoted_load_id_none": [{}] * 2,
    "quoted_load_repeated_id": [{}] * 2,
    "quoted_load_reserved_component": [{}] * 2,
    "quoted_load_past_slots": [{}] * 2,
    "quoted_download_past_table": [{"d2h_bytes": 24}] * 2,
    "quoted_download_all_past": [{}] * 2,
    "quoted_download_null": [{}] * 2,
    "quoted_download_not_quoted": [{}] * 2,
    "quoted_download_past_id_space": [{}] * 2,
    "scan_quoted_index": [{"scan_launches": 1, "probe_launches": 1, "kernel_launches": 2, "rows_scanned": 4, "rows_probed": 3, "d2h_bytes": 65536, "index_joins": 1}] * 2,
    "scan_quoted_scan": [{"scan_launches": 2, "build_launches": 2, "probe_launches": 2, "kernel_launches": 10, "rows_scanned": 11, "rows_built": 3, "rows_probed": 4, "d2h_bytes": 131072}] * 2,
    "scan_quoted_no_table": [{}] * 2,
    "scan_quoted_predicate": [{}] * 2,
    "scan_quoted_nothing_quoted": [{}] * 2,
    "bind_subject_old": [{"other_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "bind_subject_new": [{"other_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "bind_predicate_old": [{"other_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "bind_predicate_new": [{"other_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "bind_object_old": [{"other_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "bind_object_new": [{"other_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "bind_istriple_true": [{"other_launches": 4, "kernel_launches": 15, "h2d_bytes": 28, "d2h_bytes": 163840}] * 2,
    "bind_istriple_false": [{"other_launches": 4, "kernel_launches": 15, "h2d_bytes": 29, "d2h_bytes": 163840}] * 2,
    "bind_istriple_both": [{"other_launches": 4, "kernel_launches": 15, "h2d_bytes": 33, "d2h_bytes": 163840}] * 2,
    "bind_istriple_neither": [{"other_launches": 2, "kernel_launches": 2, "d2h_bytes": 65536}] * 2,
    "bind_triple_hits": [{"other_launches": 2, "kernel_launches": 7, "d2h_bytes": 98304}] * 2,
    "bind_triple_new": [{"other_launches": 2, "kernel_launches": 11, "d2h_bytes": 131072}] * 2,
    "bind_triple_repeats": [{"other_launches": 2, "kernel_launches": 11, "d2h_bytes": 131072}] * 2,
    "bind_triple_after_load": [{"other_launches": 2, "kernel_launches": 11, "d2h_bytes": 131072}] * 2,
    "bind_triple_empty_table": [{"other_launches": 2, "kernel_launches": 10, "d2h_bytes": 98304}] * 2,
    "bind_concat": [{"other_launches": 4, "kernel_launches": 18, "h2d_bytes": 9, "d2h_bytes": 163840}] * 2,
    "bind_unknown_function": [{}] * 2,
    "bind_arity": [{}] * 2,
    "bind_triple_arity": [{}] * 2,
    "bind_subject_of_constant": [{}] * 2,
    "bind_not_a_column": [{}] * 2,
    "bind_concat_constant_past": [{}] * 2,
    "bind_triple_constant_none": [{}] * 2,
    "bind_triple_next_not_above": [{}] * 2,
    "bind_triple_next_not_quoted": [{}] * 2,
    "bind_triple_past_slots": [{"other_launches": 1, "kernel_launches": 5, "d2h_bytes": 32768}] * 2,
    "values_new_strings": [{"other_launches": 6, "kernel_launches": 19, "h2d_bytes": 228, "d2h_bytes": 163840}] * 2,
}


@pytest.fixture
def make_ctx():
    made = []

    def make():
        cx = c.Context(0)
        made.append(cx)
        return cx

    yield make
    for cx in made:
        cx.close()


def fingerprint(cx, call):
    a = cx.get_stats()
    try:
        out = call()
    except c.KolibrieError as e:
        out = e
    b = cx.get_stats()
    return out, {f: b[f] - a[f] for f in FIELDS if b[f] != a[f]}


def twice(name, run):
    """run() sets the case's state up, measures the call (fingerprint) and checks its result; it returns the fingerprint"""
    fps = [run() for _ in range(2)]
    assert fps == ROUTES.get(name), f"{name}: {fps!r}"


def status(out):
    return out.status if isinstance(out, c.KolibrieError) else c.KB_OK


# ---------------------------------------------------------------- kb_dict_encode

def strings_of(seed, n, vocab, tag):
    return batch(np.random.default_rng(seed), n, vocab, tag)


HELD = list(dict.fromkeys(strings_of(1, 3000, 2000, "h")))  # distinct: string i has id i
# name -> (dictionary before the call, terms encoded outside the fingerprint first, terms of the call)
ENCODE_CASES = {
    "encode_first_batch": (None, None, strings_of(2, 20000, 6000, "a")),
    "encode_repeats": (["x"], None, ["a", "b", "a", "a", "", "c", "b", "", "x"]),
    "encode_all_held": ([], HELD, HELD[::-1]),
    "encode_index_rebuild": ([], ["a", "b", "c"], strings_of(3, 40000, 30000, "r")),
    "encode_after_strings_load": (HELD, None, strings_of(4, 5000, 3000, "h")),
}


@pytest.mark.parametrize("name", list(ENCODE_CASES))
def test_dict_encode_route(make_ctx, name):
    before, warm, terms = ENCODE_CASES[name]
    cx = make_ctx()

    def run():
        d = E.Dictionary()
        for t in before or []:
            d.encode(t)
        cx.dict_strings_load(before or [])
        if warm:
            seq_encode(d, warm)
            cx.dict_encode(warm)
        n0 = len(d.id_to_string)
        (got, first), fp = fingerprint(cx, lambda: cx.dict_encode(terms))
        assert np.array_equal(got, seq_encode(d, terms)), name
        assert [terms[int(p)] for p in first] == d.id_to_string[n0:]
        assert cx.dict_strings_info()[0] == len(d.id_to_string)
        return fp

    twice(name, run)


def raw_encode(cx, off, data, n, ids):
    p = lambda a: None if a is None else c._ptr(a)  # noqa: E731
    n_new = C.c_uint32(0)
    rc = c.lib().kb_dict_encode(cx.h, p(off), p(data), n, p(ids), C.byref(n_new), None)
    if rc != c.KB_OK:
        raise c.KolibrieError(rc, "")


ONE = np.zeros(4, np.uint8)
ENCODE_REFUSALS = {
    "encode_null_offsets": (None, ONE, 2, np.zeros(2, np.uint32), c.KB_E_INVALID),
    "encode_null_ids": (np.array([0, 1, 2], np.uint64), ONE, 2, None, c.KB_E_INVALID),
    "encode_offsets_not_at_0": (np.array([1, 1, 2], np.uint64), ONE, 2, np.zeros(2, np.uint32), c.KB_E_INVALID),
    "encode_null_bytes": (np.array([0, 1, 2], np.uint64), None, 2, np.zeros(2, np.uint32), c.KB_E_INVALID),
    "encode_too_many_terms": (np.array([0, 1, 2], np.uint64), ONE, 0xFFFFFFF0, np.zeros(2, np.uint32), c.KB_E_LIMIT),
    "encode_too_many_bytes": (np.array([0, 1 << 33], np.uint64), ONE, 1, np.zeros(1, np.uint32), c.KB_E_LIMIT),
}


@pytest.mark.parametrize("name", list(ENCODE_REFUSALS))
def test_dict_encode_refusal(make_ctx, name):
    off, data, n, ids, want = ENCODE_REFUSALS[name]
    cx = make_ctx()

    def run():
        cx.dict_strings_load(["a", "b"])
        out, fp = fingerprint(cx, lambda: raw_encode(cx, off, data, n, ids))
        assert status(out) == want and cx.dict_strings_info() == (2, 2)
        return fp

    twice(name, run)


# ---------------------------------------------------------------- kb_rel_decode

WORDS = ["a", "b", "c", "", "é中🙂", "x" * 300, "http://example.org/p"]
CHAIN = {QB: (0, 1, 2)}
CHAIN.update({QB + k: (QB + k - 1, 1, 2) for k in range(1, 17)})  # QB + 15: 16 levels (the cap); QB + 16: 17
NESTED = {QB: (0, 1, 2), QB + 1: (QB, 6, 4), QB + 2: (QB + 1, 1, QB), QB + 3: (0, 1, 99), QB + 5: (QB + 4, 1, 2)}
rng_ = np.random.default_rng(5)
# name -> (quoted table or None, ids, expected status)
DECODE_CASES = {
    "decode_plain": (None, rng_.integers(0, len(WORDS), 5000).astype(np.uint32), c.KB_OK),
    "decode_unknown": (None, np.array([0, 7, 1 << 20, 0x7FFFFFFF, 3, 8], np.uint32), c.KB_OK),
    "decode_quoted_nested": (NESTED, np.array([QB, 1, QB + 1, QB + 2, QB + 3, QB + 4, QB + 5, QB + 9, 5, 40], np.uint32), c.KB_OK),
    "decode_quoted_without_table": (None, np.array([1, QB, 2], np.uint32), c.KB_E_UNSUPPORTED),
    "decode_too_deep": (CHAIN, np.array([QB + 15, 0, QB + 16], np.uint32), c.KB_E_LIMIT),
    "decode_empty": (None, np.zeros(0, np.uint32), c.KB_OK),
}


def load_quoted(cx, quoted):
    ids = np.array(list(quoted), np.uint32)
    comp = np.array(list(quoted.values()), np.uint32).reshape(-1, 3)
    cx.quoted_load(ids, comp[:, 0], comp[:, 1], comp[:, 2])


@pytest.mark.parametrize("name", list(DECODE_CASES))
def test_rel_decode_route(make_ctx, name):
    quoted, ids, want = DECODE_CASES[name]
    cx = make_ctx()

    def run():
        cx.dict_strings_load(WORDS)
        load_quoted(cx, quoted or {})
        rel = cx.rel_from_host([3], [ids])
        out, fp = fingerprint(cx, lambda: rel.decode_strings(0))
        assert status(out) == want, out
        if want == c.KB_OK:
            assert out == [OR.render(int(i), WORDS, quoted or {}) for i in ids]
        return fp

    twice(name, run)


# ---------------------------------------------------------------- kb_order_by

def test_order_by_string_key_route(make_ctx):
    strings = ["b", "a", "", "ab", "é", "B"]
    quoted = {QB: (1, 0, 3), QB + 1: (QB, 0, 0), QB + 2: (0, 0, 77)}
    cx = make_ctx()
    key = np.array([1, NONE, QB, 0, 9, QB + 1, 3, 2, NONE, QB + 2, 4, 5, 0, 1000] * 7, np.uint32)
    tag = np.arange(len(key), dtype=np.uint32)

    def run():
        cx.dict_strings_load(strings)
        cx.dict_numeric_derive(c.NUMERIC_F64, 0)
        load_quoted(cx, quoted)
        rel = cx.rel_from_host([0, 1], [key, tag])
        (out, info), fp = fingerprint(cx, lambda: cx.order_by(rel, [(0, True)], 0))
        rows = [{0: OR.render(int(k), strings, quoted), 1: str(int(t))} for k, t in zip(key, tag)]
        want = OR.order_rows(rows, [(0, True)], 0)
        assert np.array_equal(out.to_numpy([0, 1]), np.stack([key[want], tag[want]], axis=1))
        assert info["key_kind"] == [c.ORDER_STRING]
        return fp

    twice("order_by_string_key", run)


# ---------------------------------------------------------------- kb_serialize_begin / next

@pytest.mark.parametrize("fmt", [c.SER_NTRIPLES, c.SER_TURTLE], ids=["nt", "ttl"])
def test_serialize_route(make_ctx, fmt):
    words, quoted, trip = seeded_store(4, 300)
    prefixes = [("x", "http://x/")]
    cx = make_ctx()

    def run():
        t = np.array(trip, dtype=np.uint32)
        cx.store_load(t[:, 0], t[:, 1], t[:, 2])
        cx.dict_strings_load(words)
        load_quoted(cx, quoted)
        s, p, o = cx.store_download()
        held = list(zip(s.tolist(), p.tolist(), o.tolist()))
        got, fp = fingerprint(cx, lambda: b"".join(cx.serialize(fmt, prefixes, 1 << 20)).decode("utf-8"))
        want = SR.generate_ntriples(held, words, quoted) if fmt == c.SER_NTRIPLES else SR.generate_turtle(held, words, quoted, prefixes)
        assert got == want
        return fp

    twice("serialize_" + ("nt" if fmt == c.SER_NTRIPLES else "ttl"), run)


# ---------------------------------------------------------------- kb_quoted_load / kb_quoted_download

TABLE_A = {QB + 1: (0, 1, 2), QB + 4: (QB + 1, 1, 0)}
TABLE_B = {QB + 2: (2, 1, 0), QB: (0, 0, 0), QB + 7: (QB, 1, QB + 2)}
# name -> (table before, arguments of kb_quoted_load, expected status, table after)
QLOAD_CASES = {
    "quoted_load_replace": (TABLE_A, TABLE_B, c.KB_OK, TABLE_B),
    "quoted_load_empty": (TABLE_A, {}, c.KB_OK, {}),
    "quoted_load_not_quoted_id": (TABLE_A, ([5], [0], [1], [2]), c.KB_E_INVALID, TABLE_A),
    "quoted_load_id_none": (TABLE_A, ([NONE], [0], [1], [2]), c.KB_E_INVALID, TABLE_A),
    "quoted_load_repeated_id": (TABLE_A, ([QB + 2, QB + 2], [0, 1], [1, 1], [2, 2]), c.KB_E_INVALID, TABLE_A),
    "quoted_load_reserved_component": (TABLE_A, ([QB + 3], [0], [NONE], [2]), c.KB_E_INVALID, TABLE_A),
    "quoted_load_past_slots": (TABLE_A, ([QB + (1 << 28)], [0], [1], [2]), c.KB_E_LIMIT, TABLE_A),
}


def table_args(t):
    if isinstance(t, tuple):
        return t
    ids = list(t)
    return ids, [t[i][0] for i in ids], [t[i][1] for i in ids], [t[i][2] for i in ids]


def downloaded(cx, lo, n):
    s, p, o = cx.quoted_download(lo, n)
    return {lo + k: (int(s[k]), int(p[k]), int(o[k])) for k in range(n) if s[k] != NONE}


@pytest.mark.parametrize("name", list(QLOAD_CASES))
def test_quoted_load_route(make_ctx, name):
    before, args, want, after = QLOAD_CASES[name]
    cx = make_ctx()

    def run():
        load_quoted(cx, before)
        out, fp = fingerprint(cx, lambda: cx.quoted_load(*table_args(args)))
        assert status(out) == want
        assert downloaded(cx, QB, 16) == after
        return fp

    twice(name, run)


def raw_download(cx, first, n, null=False):
    bufs = [np.empty(max(n, 1), np.uint32) for _ in range(3)]
    ptrs = [None if null else c._ptr(b) for b in bufs]
    rc = c.lib().kb_quoted_download(cx.h, first, n, *ptrs)
    if rc != c.KB_OK:
        raise c.KolibrieError(rc, "")
    return [b[:n].tolist() for b in bufs]


# name -> (first id, n, NULL outputs, expected status)
QDOWN_CASES = {
    "quoted_download_past_table": (QB + 3, 6, False, c.KB_OK),
    "quoted_download_all_past": (QB + 100, 3, False, c.KB_OK),
    "quoted_download_null": (QB, 2, True, c.KB_E_INVALID),
    "quoted_download_not_quoted": (3, 2, False, c.KB_E_INVALID),
    "quoted_download_past_id_space": (0xFFFFFFFE, 2, False, c.KB_E_INVALID),
}


@pytest.mark.parametrize("name", list(QDOWN_CASES))
def test_quoted_download_route(make_ctx, name):
    first, n, null, want = QDOWN_CASES[name]
    cx = make_ctx()

    def run():
        load_quoted(cx, TABLE_A)
        out, fp = fingerprint(cx, lambda: raw_download(cx, first, n, null))
        assert status(out) == want
        if want == c.KB_OK:
            assert out == [[TABLE_A.get(first + k, (NONE,) * 3)[j] for k in range(n)] for j in range(3)]
        return fp

    twice(name, run)


# ---------------------------------------------------------------- kb_scan_quoted

@pytest.mark.parametrize("mode", ["index", "scan", "no_table"])
def test_scan_quoted_route(make_ctx, mode):
    cx = make_ctx()

    def run():
        db = corner_db(cx)
        sync(db, "scan" if mode == "no_table" else mode)
        if mode == "no_table":
            cx.quoted_load([], [], [], [])
        ex = "http://example.org/"
        pat = (pattern_term(db, ["?x", ex + "says", "?y"]), pattern_term(db, ex + "by"), E.Variable("?w"))
        slots = E.SlotMap()
        qp = slots.quoted_pattern(pat)
        rel, fp = fingerprint(cx, lambda: cx.scan_quoted(qp))
        got = rows_of(rel, slots)
        if mode == "no_table":
            assert got == []
        else:
            assert Q.bag(got) == Q.bag(host_rows(db, pat)) and len(got) == 3
        return fp

    twice("scan_quoted_" + mode, run)


def test_scan_quoted_refusals(make_ctx):
    cx = make_ctx()
    cases = {
        "scan_quoted_predicate": (c.KbQuotedPattern(c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.KbTerm(c.KB_TERM_QUOTED, 0), c.V(1)),
                                                    c.pattern(c.V(2), c.V(3), c.V(4)), c.KbPattern()), c.KB_E_UNSUPPORTED),
        "scan_quoted_nothing_quoted": (c.KbQuotedPattern(c.pattern(c.V(0), c.K(1), c.V(1)), c.KbPattern(), c.KbPattern()), c.KB_E_INVALID),
    }
    for name, (qp, want) in cases.items():
        def run():
            cx.dict_strings_load(["a", "b", "c"])
            load_quoted(cx, TABLE_A)
            out, fp = fingerprint(cx, lambda: cx.scan_quoted(qp))
            assert status(out) == want
            return fp

        twice(name, run)


# ---------------------------------------------------------------- kb_bind

class Measured:
    """the context, with kb_bind's fingerprint kept: what tests.test_gpu_bind.check calls"""

    def __init__(self, cx):
        self.cx, self.fp = cx, None

    def __getattr__(self, k):
        return getattr(self.cx, k)

    def bind(self, *a, **k):
        out, self.fp = fingerprint(self.cx, lambda: self.cx.bind(*a, **k))
        if isinstance(out, c.KolibrieError):
            raise out
        return out


NAMES = {0: "a", 1: "b", 2: "c", 3: "x", 5: "y"}


def bind_columns(db, kind, seed, n=3000):
    """columns a, b, c, x of `n` rows of one kind (seeded)"""
    rng = np.random.default_rng(seed)
    pool = pools(db)
    qts = db.quoted_triple_store
    quoted = np.array(sorted(qts.id_to_components), dtype=np.uint32)
    plain = np.arange(len(db.dictionary.id_to_string), dtype=np.uint32)
    have = np.array(list(qts.id_to_components.values()), dtype=np.uint32)
    pick = lambda a: a[rng.integers(0, len(a), n)]  # noqa: E731
    if kind == "is_true":
        return [pick(quoted), pick(plain), pick(plain), pick(pool)]
    if kind == "is_false":
        return [pick(plain), pick(plain), pick(plain), pick(pool)]
    if kind == "is_neither":
        return [np.full(n, NONE, np.uint32), pick(plain), pick(plain), pick(pool)]
    if kind == "triple_hits":
        rows = pick(have)
        return [rows[:, 0], rows[:, 1], rows[:, 2], pick(pool)]
    if kind == "triple_new":  # (o, p, s) of entries: none of them is an entry (the components are 0..49 and quoted ids)
        s = np.arange(n, dtype=np.uint32) + np.uint32(len(db.dictionary.id_to_string) + 1000)
        return [s, pick(plain[:5]), pick(plain), pick(pool)]
    if kind == "triple_repeats":
        return [pick(plain[:4]), pick(plain[:3]), pick(plain[:5]), pick(pool)]
    return [pick(pool) for _ in range(4)]


# name -> (function, argument terms, output variable, kind of the columns (bind_columns), entries of the table, the warm TRIPLE before the call)
BIND_CASES = {
    "bind_subject_old": ("SUBJECT", [c.V(0)], "x", "mixed", 300, False),
    "bind_subject_new": ("SUBJECT", [c.V(0)], "y", "mixed", 300, False),
    "bind_predicate_old": ("PREDICATE", [c.V(0)], "x", "mixed", 300, False),
    "bind_predicate_new": ("PREDICATE", [c.V(0)], "y", "mixed", 300, False),
    "bind_object_old": ("OBJECT", [c.V(0)], "x", "mixed", 300, False),
    "bind_object_new": ("OBJECT", [c.V(0)], "y", "mixed", 300, False),
    "bind_istriple_true": ("isTRIPLE", [c.V(0)], "y", "is_true", 300, False),
    "bind_istriple_false": ("isTRIPLE", [c.V(0)], "y", "is_false", 300, False),
    "bind_istriple_both": ("isTRIPLE", [c.V(0)], "x", "mixed", 300, False),
    "bind_istriple_neither": ("isTRIPLE", [c.V(0)], "x", "is_neither", 300, False),
    "bind_triple_hits": ("TRIPLE", [c.V(0), c.V(1), c.V(2)], "y", "triple_hits", 300, True),
    "bind_triple_new": ("TRIPLE", [c.V(0), c.V(1), c.V(2)], "x", "triple_new", 300, True),
    "bind_triple_repeats": ("TRIPLE", [c.V(0), c.V(1), c.V(2)], "y", "triple_repeats", 300, True),
    "bind_triple_after_load": ("TRIPLE", [c.V(2), c.V(1), c.V(0)], "y", "mixed", 300, False),
    "bind_triple_empty_table": ("TRIPLE", [c.V(0), c.V(1), c.V(2)], "y", "triple_repeats", 0, False),
    "bind_concat": ("CONCAT", [c.V(0), c.K(0), c.V(1), c.K(1)], "x", "mixed", 300, False),
}


def fresh_bind_db(cx, n_entries, warm):
    db = new_db(cx, n_entries=n_entries)
    upload(cx, db)
    if warm:  # a TRIPLE of one row the table holds: the reverse index is built, nothing is added
        s, p, o = next(iter(db.quoted_triple_store.id_to_components.values()))
        rel = cx.rel_from_host([0, 1, 2], [np.array([s], np.uint32), np.array([p], np.uint32), np.array([o], np.uint32)])
        _, info = cx.bind(rel, c.BIND_TRIPLE, [c.V(0), c.V(1), c.V(2)], 3, db.quoted_triple_store.next_qt_id)
        assert info["quoted_new"] == 0
    return db


@pytest.mark.parametrize("name", list(BIND_CASES))
def test_bind_route(make_ctx, name):
    fn, args, out, kind, n_entries, warm = BIND_CASES[name]
    cx = make_ctx()
    m = Measured(cx)

    def run():
        db = fresh_bind_db(cx, n_entries, warm)
        cols = bind_columns(db, kind, len(name))
        consts = ("→ ".encode(), b'a"@en') if fn == "CONCAT" else ()
        rel = cx.rel_from_host([0, 1, 2, 3] if out == "x" else [0, 1, 2], cols if out == "x" else cols[:3])
        bind_check(m, db, rel, NAMES, fn, args, out, consts)
        return m.fp

    twice(name, run)


# name -> (function, arguments, next_qt_id (None: the table's next id), constants, expected status)
BIND_REFUSALS = {
    "bind_unknown_function": (7, [c.V(0)], None, (), c.KB_E_INVALID),
    "bind_arity": (c.BIND_SUBJECT, [c.V(0), c.V(1)], 0, (), c.KB_E_INVALID),
    "bind_triple_arity": (c.BIND_TRIPLE, [c.V(0), c.V(1)], None, (), c.KB_E_INVALID),
    "bind_subject_of_constant": (c.BIND_SUBJECT, [c.K(0)], 0, (), c.KB_E_INVALID),
    "bind_not_a_column": (c.BIND_OBJECT, [c.V(9)], 0, (), c.KB_E_INVALID),
    "bind_concat_constant_past": (c.BIND_CONCAT, [c.K(1)], 0, (b"x",), c.KB_E_INVALID),
    "bind_triple_constant_none": (c.BIND_TRIPLE, [c.V(0), c.K(NONE), c.V(2)], None, (), c.KB_E_INVALID),
    "bind_triple_next_not_above": (c.BIND_TRIPLE, [c.V(2), c.V(1), c.V(0)], QB, (), c.KB_E_INVALID),
    "bind_triple_next_not_quoted": (c.BIND_TRIPLE, [c.V(2), c.V(1), c.V(0)], 5, (), c.KB_E_INVALID),
    "bind_triple_past_slots": (c.BIND_TRIPLE, [c.V(2), c.V(1), c.V(0)], QB + (1 << 28) - 1, (), c.KB_E_LIMIT),
}


@pytest.mark.parametrize("name", list(BIND_REFUSALS))
def test_bind_refusal(make_ctx, name):
    fn, args, nq, consts, want = BIND_REFUSALS[name]
    cx = make_ctx()

    def run():
        db = fresh_bind_db(cx, 100, True)
        rel = cx.rel_from_host([0, 1, 2], [np.array([0, 1], np.uint32), np.array([1, 2], np.uint32), np.array([3, 4], np.uint32)])
        before = (cx.dict_strings_info(), downloaded(cx, QB, 300))
        nxt = db.quoted_triple_store.next_qt_id if nq is None else nq
        out, fp = fingerprint(cx, lambda: cx.bind(rel, fn, args, 3, nxt, consts))
        assert status(out) == want
        assert (cx.dict_strings_info(), downloaded(cx, QB, 300)) == before
        return fp

    twice(name, run)


# ---------------------------------------------------------------- kb_values

def test_values_route(make_ctx):
    strings = ["<pre>", "7", "a"]
    header = ["?a", "?b", "?c"]
    rows = [["x", "<pre>", None], [None, None, None], ["1.5", "x", "y"], ["7"], [], [None, "z", "a"], ["w", "w", "1e3"]]
    cx = make_ctx()

    def run():
        cx.dict_strings_load(strings)
        cx.dict_numeric_derive(c.NUMERIC_F64, 0)
        d = E.Dictionary()
        for t in strings:
            d.encode(t)
        want = VR.values(header, rows, d.encode)
        (rel, info), fp = fingerprint(cx, lambda: cx.values([0, 1, 2], rows))
        n, slots = rel.info()
        cols = [rel.column(i) for i in range(len(slots))]
        got = [{"abc"[s]: int(cols[j][i]) for j, s in enumerate(slots) if cols[j][i] != NONE} for i in range(n)]
        assert got == want and info["dict_new"] == len(d.id_to_string) - len(strings)
        assert cx.dict_strings_download(len(strings), info["dict_new"]) == d.id_to_string[len(strings):]
        return fp

    twice("values_new_strings", run)
