"""GPU: QueryBuilder triple queries on the device (kb_qb_triples / kb_qb_terms, and the engine's QueryBuilder over them) against the
transcription of query_builder.rs (tests/qb_reference.py), row for row and string for string: the fixture, seeded multi-segment stores
with repeats, the store after appends / evictions / deletes / set-semantic inserts and removes with the index on and off, every mode in
every position, strings of 64 KB and more, quoted ids and ids past the dictionary, the id-domain remaps, joins with a second context and
with the context itself, OFFSET / LIMIT at both ends, the refusals, and cfg2's 10 M-triple and the 100 M-triple store by count and
SHA-256. Every call leaves the store, its index route and its digest as they were."""
import hashlib
import os
import random

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200 import engine as E
from tests import helpers as H
from tests import id_domain_cases as D
from tests import qb_reference as R

pytestmark = pytest.mark.gpu

FX = H.load(os.path.join("querybuilder", "querybuilder.json"))
INT, HAND = FX["integration"], FX["hand"]
Q = 1 << 31
MODES = {"Exact": c.QB_EXACT, "Contains": c.QB_CONTAINS, "StartsWith": c.QB_STARTS, "EndsWith": c.QB_ENDS}
JOINS = {"OnSubject": c.QB_ON_SUBJECT, "OnPredicate": c.QB_ON_PREDICATE, "OnObject": c.QB_ON_OBJECT}


@pytest.fixture(scope="module")
def ctx():
    x = c.Context(0)
    yield x
    x.close()


@pytest.fixture(scope="module")
def ctx2():
    x = c.Context(0)
    yield x
    x.close()


def held(ctx):
    s, p, o = ctx.store_download()
    return list(zip(s.tolist(), p.tolist(), o.tolist()))


def digest(ctx):
    s, p, o = ctx.store_download()
    return hashlib.sha256(np.stack([s, p, o], 1).tobytes()).hexdigest()


def device_spec(q, strings):
    """a fixture query's filters as qb_triples' (an Exact string resolved through the dictionary, KB_ID_NONE when it lacks it)"""
    out = []
    for f in q["filters"]:
        if f is None:
            out.append(None)
        elif f[0] == "Exact":
            out.append((c.QB_EXACT, strings.index(f[1]) if f[1] in strings else c.KB_ID_NONE))
        else:
            out.append((MODES[f[0]], f[1]))
    return out


def run_device(ctx, q, strings, right=None):
    """(rows, subjects / predicates / objects as get_* gives them, decoded triples) of a query on the device"""
    join = 0
    for j in q["join"]:
        join |= JOINS[j]
    rel, info = ctx.qb_triples(device_spec(q, strings), join, right, q["offset"] or 0, q["limit"])
    try:
        rows = [tuple(int(x) for x in r) for r in rel.to_numpy()]
        mode = c.QB_TERMS_DISTINCT if q["distinct"] else c.QB_TERMS_DROP
        terms = [ctx.qb_terms(rel, k, mode) for k in range(3)]
        decoded = list(zip(*[ctx.qb_terms(rel, k, c.QB_TERMS_EMPTY) for k in range(3)]))
    finally:
        rel.free()
    _, count = ctx.qb_triples(device_spec(q, strings), join, right, q["offset"] or 0, q["limit"], count_only=True)
    assert count["n_rows"] == len(rows) == info["n_rows"]
    return rows, terms, decoded


def check_query(ctx, q, triples, strings, right_ctx=None, right_rows=None):
    ref = R.ref_query(triples, strings, q, right_rows)
    rows, terms, decoded = run_device(ctx, q, strings, right_ctx)
    assert rows == ref.get_triples()
    assert terms == [ref.terms(k) for k in range(3)]
    assert [tuple(t) for t in decoded] == ref.get_decoded_triples()


def load(ctx, strings, rows, quoted=None):
    t = np.array(rows, dtype=np.uint32).reshape(-1, 3)
    ctx.store_load(t[:, 0], t[:, 1], t[:, 2])
    ctx.dict_strings_load(strings)
    q = quoted or {}
    comp = np.array(list(q.values()), dtype=np.uint32).reshape(-1, 3)
    ctx.quoted_load(np.array(list(q), dtype=np.uint32), comp[:, 0], comp[:, 1], comp[:, 2])


# ---- the fixture
@pytest.mark.parametrize("case", HAND["cases"], ids=lambda c_: c_["name"])
def test_hand_worked_cases(ctx, ctx2, case):
    q = case["query"]
    load(ctx, HAND["strings"], HAND["store"])
    right_rows = {None: None, "R": HAND["right"], "self": HAND["store"], "empty": []}[q["right"]]
    right = {None: None, "R": ctx2, "self": ctx, "empty": ctx2}[q["right"]]
    if q["right"] in ("R", "empty"):
        load(ctx2, [], right_rows)
    if "error" in case["expect"]:
        with pytest.raises(c.KolibrieError) as e:
            ctx.qb_triples(device_spec(q, HAND["strings"]), 0, None, q["offset"], q["limit"])
        assert e.value.status == c.KB_E_INVALID
        return
    check_query(ctx, q, HAND["store"], HAND["strings"], right, right_rows)
    R.assert_expect(lambda: _Dev(ctx, q, HAND["strings"], right), case["expect"])


class _Dev:
    """the result methods of one fixture query answered by qb_triples / qb_terms"""

    def __init__(self, ctx, q, strings, right):
        self.rows, self.terms, self.decoded = run_device(ctx, q, strings, right)

    def get_triples(self):
        return set(self.rows)

    def count(self):
        return len(self.rows)

    def get_decoded_triples(self):
        return self.decoded

    def get_subjects(self):
        return self.terms[0]

    def get_predicates(self):
        return self.terms[1]

    def get_objects(self):
        return self.terms[2]


def _engine_db(strings, rows, ctx):
    db = E.SparqlDatabase(ctx=ctx)
    for s in strings:
        db.dictionary.encode(s)
    for t in rows:
        db.add_triple(tuple(t))
    return db


@pytest.mark.parametrize("case", INT["queries"], ids=lambda c_: c_["name"])
def test_engine_mirror_on_the_integration_fixture(ctx, case):
    db = _engine_db(INT["terms"], INT["triples"], ctx)
    all_rows = [list(t) for t in sorted(db.query().get_triples())]
    R.assert_expect(lambda: R.engine_query(db, case["query"]), case["expect"], all_rows)
    b = R.engine_query(db, case["query"])
    b.count()
    assert b.last_path == "device"
    se = INT["second_email"]
    db.add_statement(*se["add"])
    R.assert_expect(lambda: R.engine_query(db, se["query"]), se["expect"])


@pytest.mark.parametrize("case", HAND["cases"], ids=lambda c_: c_["name"])
def test_engine_mirror_on_the_hand_worked_cases(ctx, ctx2, case):
    q = case["query"]
    db = _engine_db(HAND["strings"], HAND["store"], ctx)
    right_db = {None: None, "R": _engine_db([], HAND["right"], ctx2), "self": db, "empty": _engine_db([], [], ctx2)}[q["right"]]
    R.assert_expect(lambda: R.engine_query(db, q, right_db), case["expect"])
    b = R.engine_query(db, q, right_db)
    if "error" not in case["expect"]:
        b.get_subjects()
        assert b.last_path == "device"


def test_engine_takes_the_host_path_for_closures_and_shared_contexts(ctx):
    db = _engine_db(HAND["strings"], HAND["store"], ctx)
    b = db.query().filter(lambda t: t[1] == 7)
    assert sorted(b.get_triples()) == [t for t in sorted(map(tuple, HAND["store"])) if t[1] == 7]
    assert b.last_path == "host"
    other = _engine_db(HAND["strings"], HAND["right"], ctx)  # the same context cannot hold both stores
    b = db.query().join(other).join_on_subject()
    ref = R.Ref(HAND["store"], HAND["strings"], HAND["right"])
    ref.join_conditions = ["OnSubject"]
    assert sorted(b.get_triples()) == ref.get_triples()
    assert b.last_path == "host"
    ctx.dict_strings_load([])  # no device strings: a text filter is refused and the host path answers
    db2 = E.SparqlDatabase(ctx=ctx)
    db2.dictionary = db.dictionary
    db2.triples = set(db.triples)
    db2._uploaded_version = db2._version  # (the store is current; the device dictionary is not)
    ctx.store_load(*np.array(sorted(db.triples), dtype=np.uint32).T)
    b = db2.query().with_object_like("aa")
    assert sorted(b.get_triples()) == [(6, 7, 0), (6, 50, 1)]
    assert b.last_path == "host"


# ---- seeded stores
def seeded(seed, n, n_words=300, long_words=2):
    rng = random.Random(seed)
    alphabet = ["a", "b", "ab", "ba", "é", "日", "x/", "http://", "aa"]
    words = list(dict.fromkeys("".join(rng.choice(alphabet) for _ in range(rng.randrange(0, 12))) for _ in range(n_words)))
    for k in range(long_words):  # strings of 64 KB and more: the warp-cooperative CONTAINS
        w = "".join(rng.choice("ab") for _ in range(65536 + 977 * k)) + "needle%d" % k + "ab" * 50
        words.append(w)
    nw = len(words)
    ids = list(range(nw)) + [nw, nw + 5, Q, Q + 1, Q + 7]  # ids past the dictionary, quoted ids
    trip = [(rng.choice(ids), rng.choice(ids[: 12] + [Q]), rng.choice(ids)) for _ in range(n)]
    return words, trip + [trip[rng.randrange(n)] for _ in range(n // 5)]


def random_query(rng, words):
    def pattern():
        w = rng.choice(words)
        w = w if len(w) < 70000 else w[-200:]
        if not w or rng.random() < 0.1:
            return ""
        a = rng.randrange(len(w))
        return w[a: a + rng.randrange(1, 6)] if rng.random() < 0.8 else w + "x"  # a piece, or longer than the string
    filters = []
    for _ in range(3):
        r = rng.random()
        if r < 0.45:
            filters.append(None)
        elif r < 0.6:
            filters.append(["Exact", rng.choice(words + ["missing"])])
        else:
            filters.append([rng.choice(["Contains", "StartsWith", "EndsWith"]), pattern()])
    return {"filters": filters, "join": [], "right": None, "offset": None, "limit": None, "order_by": None, "distinct": rng.random() < 0.5}


@pytest.mark.parametrize("seed", range(3))
def test_seeded_multi_segment_stores(ctx, seed):
    words, trip = seeded(seed, 3000)
    load(ctx, words, trip[:2000], {Q: (0, 1, 2)} if seed else None)
    more = np.array(trip[1500:] + trip[:300], dtype=np.uint32)
    ctx.store_append(more[:, 0], more[:, 1], more[:, 2], tag=7)
    rows = held(ctx)
    rng = random.Random(100 + seed)
    for _ in range(25):
        check_query(ctx, random_query(rng, words), rows, words)


def test_every_mode_in_every_position_at_string_boundaries(ctx):
    words, trip = seeded(21, 1500)
    load(ctx, words, trip)
    rows = held(ctx)
    rng = random.Random(5)
    for pos in range(3):
        for mode in ("Contains", "StartsWith", "EndsWith", "Exact"):
            for _ in range(4):
                w = rng.choice(words[:-2])
                for pat in {w, w[:1], w[-1:], w[1:], w[:-1], w + "a", "a" + w, ""}:
                    f = [None, None, None]
                    f[pos] = [mode, pat]
                    q = {"filters": f, "join": [], "right": None, "offset": None, "limit": None, "order_by": None, "distinct": False}
                    assert run_device(ctx, q, words)[0] == R.ref_query(rows, words, q).get_triples(), (pos, mode, pat)


def test_long_strings_are_matched_by_the_warp(ctx):
    words, trip = seeded(3, 500, long_words=4)
    long_ids = [i for i, w in enumerate(words) if len(w) >= 65536]
    trip = trip + [(i, 1, i) for i in long_ids]
    load(ctx, words, trip)
    rows = held(ctx)
    for k in range(4):
        for mode, pat in (("Contains", "needle%d" % k), ("Contains", "needle%dab" % k), ("EndsWith", "needle%d" % k + "ab" * 50),
                          ("Contains", "needle%dx" % k), ("StartsWith", words[long_ids[k]][:3000]), ("Contains", words[long_ids[k]][-4096:])):
            q = {"filters": [[mode, pat], None, None], "join": [], "right": None, "offset": None, "limit": None, "order_by": None, "distinct": False}
            check_query(ctx, q, rows, words)


@pytest.mark.parametrize("indexed", [False, True], ids=["no_index", "index"])
def test_after_store_mutations(ctx, indexed):
    words, trip = seeded(11, 4000)
    load(ctx, words, trip[:1000])
    if indexed:
        ctx.build_index()
    ctx.set_use_index(indexed)
    for tag, part in ((1, trip[1000:2500]), (2, trip[2000:4000]), (3, trip[:500])):
        a = np.array(part, dtype=np.uint32)
        ctx.store_append(a[:, 0], a[:, 1], a[:, 2], tag)
    ctx.store_evict(2)
    d = np.array(trip[:200] + trip[1200:1300], dtype=np.uint32)
    ctx.store_delete(d[:, 0], d[:, 1], d[:, 2])
    ins = np.array(trip[2200:2600] + [(0, 1, 2), (3, 4, 5)], dtype=np.uint32)
    ctx.store_insert(ins[:, 0], ins[:, 1], ins[:, 2])
    rem = np.array(trip[1000:1100], dtype=np.uint32)
    ctx.store_remove(rem[:, 0], rem[:, 1], rem[:, 2])
    rows = held(ctx)
    rng = random.Random(7)
    for _ in range(15):
        check_query(ctx, random_query(rng, words), rows, words)
    ctx.set_use_index(True)


@pytest.mark.parametrize("family", D.FAMILIES)
def test_id_domain_remaps(ctx, family):
    """ids at the u32 edges: a remapped id past the dictionary or with bit 31 does not decode and fails every text filter"""
    words, trip = seeded(31, 800, n_words=60, long_words=0)
    plain = [t for t in trip if all(x < Q for x in t)]
    f = D.Remap(family, np.unique(np.array(plain, dtype=np.uint64)), (), seed=3)
    rows = [tuple(r) for r in f(np.array(plain, dtype=np.uint32)).tolist()]
    load(ctx, words, rows)
    rng = random.Random(9)
    for _ in range(12):
        check_query(ctx, random_query(rng, words), held(ctx), words)


# ---- joins
@pytest.mark.parametrize("seed", range(2))
def test_joins_with_a_second_context_and_with_itself(ctx, ctx2, seed):
    words, trip = seeded(40 + seed, 600, n_words=40, long_words=0)
    rtrip = seeded(50 + seed, 500, n_words=40, long_words=0)[1]
    load(ctx, words, trip[:400])
    a = np.array(trip[300:], dtype=np.uint32)
    ctx.store_append(a[:, 0], a[:, 1], a[:, 2], 5)
    load(ctx2, [], rtrip[:300])
    b = np.array(rtrip[250:], dtype=np.uint32)
    ctx2.store_append(b[:, 0], b[:, 1], b[:, 2], 6)
    rows, rrows = held(ctx), held(ctx2)
    rng = random.Random(seed)
    for joins in (["OnSubject"], ["OnPredicate"], ["OnObject"], ["OnSubject", "OnObject"], ["OnSubject", "OnPredicate", "OnObject"]):
        for right, rr in ((ctx2, rrows), (ctx, rows)):
            q = random_query(rng, words)
            q["join"] = joins
            if rng.random() < 0.5:
                q["filters"] = [None, None, None]
            check_query(ctx, q, rows, words, right, rr)


def test_offset_and_limit_around_both_ends(ctx):
    words, trip = seeded(60, 300, n_words=30, long_words=0)
    load(ctx, words, trip)
    rows = held(ctx)
    n = len(set(rows))
    for off in (None, 0, 1, n - 1, n):
        for lim in (None, 0, 1, n - 1, n, n + 1, (1 << 64) - 1):
            q = {"filters": [None, None, None], "join": [], "right": None, "offset": off, "limit": lim, "order_by": None, "distinct": False}
            check_query(ctx, q, rows, words)
    with pytest.raises(c.KolibrieError) as e:
        ctx.qb_triples(offset=n + 1)
    assert e.value.status == c.KB_E_INVALID


# ---- refusals and what no call changes
def test_refusals(ctx, ctx2):
    words, trip = seeded(70, 200, n_words=30, long_words=0)
    load(ctx, words, trip)

    def status(**kw):
        with pytest.raises(c.KolibrieError) as e:
            ctx.qb_triples(**kw)
        return e.value.status

    assert status(filters=[(c.QB_CONTAINS, "a" * (c.QB_PATTERN_MAX + 1)), None, None]) == c.KB_E_LIMIT
    assert ctx.qb_triples(filters=[(c.QB_CONTAINS, "a" * c.QB_PATTERN_MAX), None, None], count_only=True)[1]["n_rows"] == 0
    assert status(filters=[(9, "a"), None, None]) == c.KB_E_INVALID
    assert status(join=8, right=ctx2) == c.KB_E_INVALID
    spec = c.KbQbSpec()
    spec.pos[0].mode, spec.pos[0].len = c.QB_CONTAINS, 3  # a NULL pattern
    sl = (c.C.c_uint32 * 3)(0, 1, 2)
    assert c.lib().kb_qb_triples(ctx.h, c.C.byref(spec), None, sl, None, None) == c.KB_E_INVALID
    assert c.lib().kb_qb_triples(ctx.h, None, None, sl, None, None) == c.KB_E_INVALID
    rel, _ = ctx.qb_triples()
    assert c.lib().kb_qb_terms(ctx.h, rel.h, 3, 0, c.C.byref(c.C.c_void_p())) == c.KB_E_INVALID
    assert c.lib().kb_qb_terms(ctx.h, rel.h, 0, 3, c.C.byref(c.C.c_void_p())) == c.KB_E_INVALID
    ctx.dict_strings_load([])
    assert status(filters=[None, (c.QB_ENDS, "a"), None]) == c.KB_E_UNSUPPORTED
    assert c.lib().kb_qb_terms(ctx.h, rel.h, 0, 0, c.C.byref(c.C.c_void_p())) == c.KB_E_UNSUPPORTED
    rel.free()
    assert ctx.qb_triples(filters=[(c.QB_EXACT, trip[0][0]), None, None], count_only=True)[1]["n_rows"] > 0  # EXACT needs no strings
    # a join whose output reaches 2^32 - 16 rows: 70 000 x 70 000 pairs on one predicate, refused before anything is allocated
    n = 70000
    big = np.stack([np.arange(n), np.full(n, 3), np.arange(n) + n], 1).astype(np.uint32)
    ctx2.store_load(big[:, 0], big[:, 1], big[:, 2])
    ctx.store_load(big[:, 0], big[:, 1], big[:, 2])
    with pytest.raises(c.KolibrieError) as e:
        ctx.qb_triples(join=c.QB_ON_PREDICATE, right=ctx2, count_only=True)
    assert e.value.status == c.KB_E_LIMIT
    assert ctx.qb_triples(join=c.QB_ON_SUBJECT, right=ctx2, count_only=True)[1]["n_rows"] == n
    ctx.set_sharding(0, 2)
    try:
        assert status() == c.KB_E_UNSUPPORTED
    finally:
        ctx.set_sharding(0, 1)


def test_store_version_index_route_and_digest_unchanged(ctx, ctx2):
    d = datagen.employee_dataset(20000)
    strings = datagen.employee_strings(d)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_strings_load(strings)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    ctx2.store_load(d.s[:500], d.p[:500], d.o[:500])
    before = digest(ctx)
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    n0 = ctx.get_stats()["index_joins"]
    want = ctx.star_join(js, pats, filt).to_numpy()
    n1 = ctx.get_stats()["index_joins"]
    assert n1 > n0
    for kw in ({"filters": [None, (c.QB_ENDS, "annual_salary"), None]}, {"filters": [(c.QB_STARTS, "http://example.org/employee1"), None, None]},
               {"filters": [None, None, (c.QB_CONTAINS, "Developer")], "offset": 3, "limit": 10}, {"join": 7, "right": ctx2}, {"join": 1, "right": ctx}):
        rel, _ = ctx.qb_triples(**kw)
        ctx.qb_terms(rel, 0, c.QB_TERMS_DISTINCT)
        rel.free()
    assert digest(ctx) == before
    got = ctx.star_join(js, pats, filt).to_numpy()
    assert ctx.get_stats()["index_joins"] > n1, "the star join left the index route: the index was dropped"
    assert np.array_equal(datagen.canonical_rows(got), datagen.canonical_rows(want))
    # the store version: a prepared plan of the star join is still valid after the queries (a mutation would void it)
    plan = ctx.prepare_star_join(js, pats, filt)
    ctx.qb_triples(filters=[None, (c.QB_ENDS, "annual_salary"), None], count_only=True)
    assert plan.collect(plan.submit()) == len(want)
    plan.free()


# ---- the large stores, by count and SHA-256 against a numpy restatement
def _np_match(strings, mode, pat):
    if mode == c.QB_CONTAINS:
        return np.fromiter((pat in s for s in strings), bool, len(strings))
    if mode == c.QB_STARTS:
        return np.fromiter((s.startswith(pat) for s in strings), bool, len(strings))
    return np.fromiter((s.endswith(pat) for s in strings), bool, len(strings))


def _np_rows(d, strings, pos, mode, pat):
    """the distinct rows of the store whose position `pos` matches, in (s, p, o) order"""
    col = (d.s, d.p, d.o)[pos]
    ok = _np_match(strings, mode, pat)[col]
    t = np.stack([d.s[ok], d.p[ok], d.o[ok]], 1).astype(np.uint64)
    rows = np.unique(t.view([("s", np.uint64), ("p", np.uint64), ("o", np.uint64)]).ravel())
    return np.stack([rows["s"], rows["p"], rows["o"]], 1).astype(np.uint32)


def _device_rows(ctx, filters):
    rel, info = ctx.qb_triples(filters=filters)
    try:
        return rel.to_numpy(), info
    finally:
        rel.free()


@pytest.mark.parametrize("n_employees", [1_666_667, 16_666_667], ids=["cfg2_10m", "bench_100m"])
def test_large_stores_by_count_and_digest(ctx, n_employees):
    d = datagen.employee_dataset(n_employees)
    strings = datagen.employee_strings(d)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_strings_load(strings)
    for pos, mode, pat in ((1, c.QB_ENDS, "annual_salary"), (2, c.QB_CONTAINS, "Developer"), (0, c.QB_STARTS, "http://example.org/employee1")):
        f = [None, None, None]
        f[pos] = (mode, pat)
        got, info = _device_rows(ctx, f)
        want = _np_rows(d, strings, pos, mode, pat)
        assert info["n_raw"] == len(d.s) and len(got) == len(want)
        assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == hashlib.sha256(want.tobytes()).hexdigest()
    assert ctx.qb_triples(count_only=True)[1]["n_rows"] == len(d.s)  # every triple of the generator is distinct
    rel, _ = ctx.qb_triples(filters=[None, (c.QB_EXACT, d.ids["foaf:title"]), None])
    try:
        assert ctx.qb_terms(rel, 2, c.QB_TERMS_DISTINCT) == sorted({strings[i] for i in d.o[d.p == d.ids["foaf:title"]].tolist()})
    finally:
        rel.free()
