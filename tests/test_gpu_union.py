"""GPU: SparqlDatabase::union and par_join on the device (kb_store_union / kb_store_par_join, and the engine's SparqlDatabase.union /
par_join over them) against the transcription of sparql_database.rs:1874-2005 (tests/union_reference.py), triple for triple and string
for string: the hand-worked cases, seeded multi-segment stores with repeats, stores after appends / evictions / deletes / set-semantic
inserts and removes with and without the index, the id-domain remaps, a == b, every refusal with dst unchanged, a and b untouched,
queries on the result, the engine mirror, and the cfg2 union and the cfg4 self-join by count and SHA-256."""
import hashlib
import random

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200 import engine as E
from tests import id_domain_cases as D
from tests import union_reference as R
from tests.test_union_cpu import PAR_CASES, UNION_CASES

pytestmark = pytest.mark.gpu

Q = 1 << 31


@pytest.fixture(scope="module")
def ctxs():
    xs = [c.Context(0) for _ in range(3)]
    yield xs
    for x in xs:
        x.close()


def held(ctx):
    s, p, o = ctx.store_download()
    return list(zip(s.tolist(), p.tolist(), o.tolist()))


def digest(ctx):
    s, p, o = ctx.store_download()
    return hashlib.sha256(np.stack([s, p, o], 1).tobytes()).hexdigest()


def strings_of(ctx):
    n, _ = ctx.dict_strings_info()
    return ctx.dict_strings_download(0, n)


def quoted_of(ctx, n=16):
    return [tuple(x.tolist()) for x in ctx.quoted_download(Q, n)]


def load(ctx, strings, rows, quoted=None, parts=1):
    """rows in `parts` segments (the later ones appended), the dictionary strings and the quoted table"""
    t = np.array(rows, dtype=np.uint32).reshape(-1, 3)
    cuts = np.linspace(0, len(t), parts + 1).astype(int)
    ctx.store_load(t[: cuts[1], 0], t[: cuts[1], 1], t[: cuts[1], 2])
    for k in range(1, parts):
        seg = t[cuts[k]: cuts[k + 1]]
        ctx.store_append(seg[:, 0], seg[:, 1], seg[:, 2], 100 + k)
    ctx.dict_strings_load(strings)
    q = quoted or {}
    comp = np.array(list(q.values()), dtype=np.uint32).reshape(-1, 3)
    ctx.quoted_load(np.array(list(q), dtype=np.uint32), comp[:, 0], comp[:, 1], comp[:, 2])


def check_union(dst, a, b, a_strings, a_rows, b_strings, b_rows):
    want = R.union(R.Db(a_rows, R.Dictionary(a_strings)), R.Db(b_rows, R.Dictionary(b_strings)))
    qa = quoted_of(a)
    info = dst.store_union(a, b)
    assert held(dst) == sorted(want.triples)  # one segment, in ascending (s, p, o) order
    assert strings_of(dst) == want.dictionary.strings()
    assert info["dict_first"] == len(a_strings) and info["dict_first"] + info["dict_new"] == want.dictionary.next_id
    assert info["n_a"] == len(set(a_rows)) and info["n_b"] == len(set(b_rows)) and info["n_rows"] == len(want.triples)
    assert quoted_of(dst) == qa
    return info


def ref_par_join(a_rows, b_rows, pid):
    d = R.Dictionary()
    d.string_to_id["P"] = pid  # the predicate as a's dictionary resolves it
    return R.par_join(R.Db(a_rows, d), R.Db(b_rows), "P").triples


def check_par_join(dst, a, b, a_rows, b_rows, pid):
    want = ref_par_join(a_rows, b_rows, pid)
    info = dst.store_par_join(a, b, pid)
    assert held(dst) == sorted(want)
    assert strings_of(dst) == strings_of(a) and quoted_of(dst) == quoted_of(a)
    assert info["n_rows"] == len(want)
    assert info["n_a"] == len({t for t in a_rows if t[1] == pid}) and info["n_b"] == len({t for t in b_rows if t[1] == pid})
    return info


# ---- the hand-worked cases
@pytest.mark.parametrize("case", sorted(UNION_CASES))
def test_union_hand_worked_cases(ctxs, case):
    dst, a, b = ctxs
    sa, ta, sb, tb, want_strings, want = UNION_CASES[case]
    load(a, sa, ta, quoted={Q: (0, 0, 0), Q | 1: (Q, 0, 0)} if case == "quoted in a" else None)
    load(b, sb, tb)
    check_union(dst, a, b, sa, ta, sb, tb)
    assert held(dst) == sorted(want) and strings_of(dst) == want_strings


@pytest.mark.parametrize("case", sorted(PAR_CASES))
def test_par_join_hand_worked_cases(ctxs, case):
    dst, a, b = ctxs
    ta, tb, want = PAR_CASES[case]
    load(a, ["p", "q"], ta, quoted={Q: (0, 1, 0)})
    load(b, ["zz"], tb)
    check_par_join(dst, a, b, ta, tb, 0)
    assert held(dst) == sorted(want)


def test_par_join_with_a_predicate_no_triple_carries(ctxs):
    dst, a, b = ctxs
    load(a, ["p", "new"], [(0, 0, 0)])
    load(b, ["p"], [(0, 0, 0)])
    info = check_par_join(dst, a, b, [(0, 0, 0)], [(0, 0, 0)], 1)
    assert info["n_rows"] == 0 and held(dst) == [] and strings_of(dst) == ["p", "new"]


# ---- seeded stores
def seeded(seed, n, n_words, plain=True):
    rng = random.Random(seed)
    words = list(dict.fromkeys("w%d_%s" % (rng.randrange(4 * n_words), "ab" * rng.randrange(4)) for _ in range(n_words)))
    nw = len(words)
    ids = list(range(nw)) + ([] if plain else [nw + 3, Q, Q + 2])
    trip = [(rng.choice(ids), rng.choice(ids[:8]), rng.choice(ids)) for _ in range(n)]
    return words, trip + [trip[rng.randrange(n)] for _ in range(n // 4)]


@pytest.mark.parametrize("seed", range(4))
def test_seeded_multi_segment_stores(ctxs, seed):
    dst, a, b = ctxs
    wa, ta = seeded(seed, 3000, 400)
    wb, tb = seeded(100 + seed, 2500, 350)
    wb = wb[: len(wb) // 2] + wa[: 150] + wb[len(wb) // 2:]  # shared strings at other ids
    wb = list(dict.fromkeys(wb))
    tb = [tuple(min(x, len(wb) - 1) for x in t) for t in tb]
    load(a, wa, ta, quoted={Q: (1, 2, 3)}, parts=3)
    load(b, wb, tb + tb[:300], parts=4)  # repeats inside and across segments
    check_union(dst, a, b, wa, ta, wb, tb)
    pid = ta[0][1]
    check_par_join(dst, a, b, ta, tb, pid)


@pytest.mark.parametrize("indexed", [False, True], ids=["no_index", "index"])
def test_after_store_mutations(ctxs, indexed):
    dst, a, b = ctxs
    words, trip = seeded(11, 4000, 300)
    for x in (a, b):
        load(x, words, trip[:1000])
        if indexed:
            x.build_index()
        for tag, part in ((1, trip[1000:2500]), (2, trip[2000:4000]), (3, trip[:500])):
            t = np.array(part, dtype=np.uint32)
            x.store_append(t[:, 0], t[:, 1], t[:, 2], tag)
    a.store_evict(2)
    d = np.array(trip[:200] + trip[1200:1300], dtype=np.uint32)
    a.store_delete(d[:, 0], d[:, 1], d[:, 2])
    ins = np.array(trip[2200:2600] + [(0, 1, 2), (3, 4, 5)], dtype=np.uint32)
    b.store_insert(ins[:, 0], ins[:, 1], ins[:, 2])
    rem = np.array(trip[1000:1100], dtype=np.uint32)
    b.store_remove(rem[:, 0], rem[:, 1], rem[:, 2])
    b.store_evict(1)
    ra, rb = held(a), held(b)
    check_union(dst, a, b, words, ra, words, rb)
    check_par_join(dst, a, b, ra, rb, trip[5][1])


@pytest.mark.parametrize("family", D.FAMILIES)
def test_id_domain_remaps(ctxs, family):
    """a's ids anywhere in the u32 domain are copied as they are by the union; par_join compares both stores' remapped ids raw"""
    dst, a, b = ctxs
    words, trip = seeded(31, 800, 60)
    wb, tb = seeded(32, 600, 50)
    f = D.Remap(family, np.unique(np.array(trip + tb, dtype=np.uint64)), (), seed=3)
    ra = [tuple(r) for r in f(np.array(trip, dtype=np.uint32)).tolist()]
    rb = [tuple(r) for r in f(np.array(tb, dtype=np.uint32)).tolist()]
    load(a, words, ra)
    load(b, wb, tb)
    check_union(dst, a, b, words, ra, wb, tb)
    load(b, wb, rb)
    check_par_join(dst, a, b, ra, rb, ra[0][1])


def test_a_equals_b(ctxs):
    dst, a, _ = ctxs
    words, trip = seeded(5, 2000, 200)
    load(a, words, trip, quoted={Q: (0, 0, 0)}, parts=2)
    info = check_union(dst, a, a, words, trip, words, trip)
    assert info["dict_new"] == 0 and held(dst) == sorted(set(trip))
    check_par_join(dst, a, a, trip, trip, trip[0][1])


# ---- refusals: dst exactly as it was
def test_refusals_leave_dst_unchanged(ctxs):
    dst, a, b = ctxs
    d = datagen.employee_dataset(3000)
    dst.store_load(d.s, d.p, d.o)
    dst.dict_strings_load(datagen.employee_strings(d))
    dst.dict_numeric_load(d.num_or0, d.is_num)
    dst.build_index()
    dst.quoted_load(np.array([Q], np.uint32), np.array([1], np.uint32), np.array([2], np.uint32), np.array([3], np.uint32))
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    n_want = dst.star_join(js, pats, filt).n_rows
    plan = dst.prepare_star_join(js, pats, filt)  # voided by any change of dst's store version
    before = (digest(dst), dst.dict_strings_info(), quoted_of(dst))
    words, trip = seeded(3, 300, 40)
    load(a, words, trip)

    def refused(status, call):
        with pytest.raises(c.KolibrieError) as e:
            call()
        assert e.value.status == status, str(e.value)
        assert (digest(dst), dst.dict_strings_info(), quoted_of(dst)) == before

    for bad in ((0, 1, Q), (Q + 3, 1, 0), (0, len(words) + 2, 1)):  # quoted ids and an id past b's dictionary
        load(b, words, trip + [bad])
        refused(c.KB_E_INVALID, lambda: dst.store_union(a, b))
    load(b, words, trip)
    refused(c.KB_E_INVALID, lambda: dst.store_union(dst, b))
    refused(c.KB_E_INVALID, lambda: dst.store_union(a, dst))
    refused(c.KB_E_INVALID, lambda: dst.store_par_join(a, dst, 0))
    refused(c.KB_E_INVALID, lambda: dst.store_par_join(a, b, c.KB_ID_NONE))
    assert c.lib().kb_store_union(dst.h, None, b.h, None) == c.KB_E_INVALID
    assert c.lib().kb_store_par_join(dst.h, a.h, None, 0, None) == c.KB_E_INVALID
    b.dict_strings_load([])
    refused(c.KB_E_UNSUPPORTED, lambda: dst.store_union(a, b))
    a.dict_strings_load([])
    refused(c.KB_E_UNSUPPORTED, lambda: dst.store_union(a, b))
    refused(c.KB_E_UNSUPPORTED, lambda: dst.store_par_join(a, b, 0))
    load(a, words, trip)
    load(b, words, trip)
    b.set_sharding(0, 2)
    try:
        refused(c.KB_E_UNSUPPORTED, lambda: dst.store_union(a, b))
        refused(c.KB_E_UNSUPPORTED, lambda: dst.store_par_join(a, b, 0))
    finally:
        b.set_sharding(0, 1)
    # a join of 70 000 x 70 000 rows on one key, refused before anything is allocated
    n = 70000
    big = np.concatenate([np.stack([np.arange(n), np.zeros(n), np.full(n, 7)], 1), np.stack([np.full(n, 7), np.zeros(n), np.arange(n) + n], 1)]).astype(np.uint32)
    a.store_load(big[:, 0], big[:, 1], big[:, 2])
    refused(c.KB_E_LIMIT, lambda: dst.store_par_join(a, a, 0))
    assert plan.collect(plan.submit()) == n_want  # dst's store version did not move
    plan.free()


def test_a_and_b_untouched(ctxs):
    dst, a, b = ctxs
    d = datagen.employee_dataset(20000)
    strings = datagen.employee_strings(d)
    a.store_load(d.s, d.p, d.o)
    a.dict_strings_load(strings)
    a.dict_numeric_load(d.num_or0, d.is_num)
    a.build_index()
    d2 = datagen.employee_dataset(5000, seed=45)
    load(b, datagen.employee_strings(d2), list(zip(d2.s.tolist(), d2.p.tolist(), d2.o.tolist())))
    before = (digest(a), digest(b), strings_of(b), a.dict_strings_info())
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    want = a.star_join(js, pats, filt).to_numpy()
    plan = a.prepare_star_join(js, pats, filt)
    n1 = a.get_stats()["index_joins"]
    dst.store_union(a, b)
    dst.store_union(b, a)
    dst.store_par_join(a, b, d.ids["foaf:title"])
    dst.store_par_join(a, a, d.ids["foaf:title"])
    assert (digest(a), digest(b), strings_of(b), a.dict_strings_info()) == before
    got = a.star_join(js, pats, filt).to_numpy()
    assert a.get_stats()["index_joins"] > n1, "a's star join left the index route: a's index was dropped"
    assert np.array_equal(datagen.canonical_rows(got), datagen.canonical_rows(want))
    assert plan.collect(plan.submit()) == len(want)  # a's store version did not move
    plan.free()


def test_queries_on_the_result(ctxs):
    """dst after kb_store_build_index and kb_dict_numeric_derive answers a FILTER star and decodes its rows as the same store built on
    the host does"""
    dst, a, b = ctxs
    da, db_ = datagen.employee_dataset(4000), datagen.employee_dataset(4000, seed=45)
    sa, sb = datagen.employee_strings(da), datagen.employee_strings(db_)
    ra = list(zip(da.s.tolist(), da.p.tolist(), da.o.tolist()))
    rb = list(zip(db_.s.tolist(), db_.p.tolist(), db_.o.tolist()))
    load(a, sa, ra)
    load(b, sb, rb)
    want = R.union(R.Db(ra, R.Dictionary(sa)), R.Db(rb, R.Dictionary(sb)))
    dst.store_union(a, b)
    dst.build_index()
    dst.dict_numeric_derive(c.NUMERIC_F64, 0)
    host = c.Context(0)
    try:
        load(host, want.dictionary.strings(), sorted(want.triples))
        host.dict_numeric_derive(c.NUMERIC_F64, 0)
        js, pats, filt = datagen.employee_queries(da)["cfg2"]
        got, ref = dst.star_join(js, pats, filt), host.star_join(js, pats, filt)
        order = sorted(got.slots)
        assert np.array_equal(datagen.canonical_rows(got.to_numpy(order)), datagen.canonical_rows(ref.to_numpy(order)))
        assert got.n_rows > 0
        key = lambda rel: sorted(zip(*[rel.decode_strings(k) for k in range(len(rel.slots))]))
        assert key(got) == key(ref)
    finally:
        host.close()


# ---- the engine mirror
def test_engine_mirror(ctxs):
    words, trip = seeded(21, 1500, 200)
    wb, tb = seeded(22, 1200, 150)
    x, y = E.SparqlDatabase(device=0), E.SparqlDatabase(device=0)
    for w in words:
        x.dictionary.encode(w)
    for w in wb:
        y.dictionary.encode(w)
    for t in trip:
        x.add_triple(t)
    for t in tb:
        y.add_triple(t)
    x.quoted_triple_store.encode(0, 1, 2)
    x.dictionary.encode("encoded after the last upload")
    want = R.union(R.Db(trip, R.Dictionary(x.dictionary.id_to_string)), R.Db(tb, R.Dictionary(wb)))
    u = x.union(y)
    assert u.triples == want.triples and u.dictionary.id_to_string == want.dictionary.strings()
    assert u.ctx is not x.ctx and u.quoted_triple_store is x.quoted_triple_store
    assert held(u.ctx) == sorted(want.triples) and strings_of(u.ctx) == want.dictionary.strings()
    assert x.last_union_info["n_rows"] == len(want.triples)
    pj = x.par_join(y, words[trip[0][1]])
    assert pj.triples == ref_par_join(trip, tb, trip[0][1]) and pj.dictionary is x.dictionary
    x.dictionary.encode("later")
    assert pj.dictionary.lookup("later") is not None
    pj2 = x.par_join(y, "a predicate x lacks")
    assert pj2.triples == set() and x.dictionary.id_to_string[-1] == "a predicate x lacks"
    assert x.union(x).triples == x.triples  # a == b on the device
    # an `other` that shares x's context takes the host restatement
    z = E.SparqlDatabase(ctx=x.ctx)
    z.dictionary = y.dictionary
    z.triples = set(y.triples)
    want2 = R.union(R.Db(x.triples, R.Dictionary(x.dictionary.id_to_string)), R.Db(tb, R.Dictionary(wb)))
    assert x.union(z).triples == want2.triples
    bad = E.SparqlDatabase(device=0)
    bad.dictionary.encode("s")
    bad.add_triple((0, 0, Q))
    with pytest.raises(ValueError):
        x.union(bad)
    for db in (x, y, u, pj, pj2, bad):
        db.ctx.close()


# ---- full size, against a numpy restatement
def _rows_sha(t):
    return hashlib.sha256(np.ascontiguousarray(t, dtype=np.uint32).tobytes()).hexdigest()


def _np_set_rows(t):
    """the distinct rows of an (n, 3) uint32 array in (s, p, o) order (packed into one u64 key when the ids' bits fit)"""
    t = np.asarray(t, dtype=np.uint64).reshape(-1, 3)
    if not len(t):
        return t.astype(np.uint32)
    bits = [max(int(t[:, k].max()).bit_length(), 1) for k in range(3)]
    if sum(bits) <= 64:
        key = (t[:, 0] << np.uint64(bits[1] + bits[2])) | (t[:, 1] << np.uint64(bits[2])) | t[:, 2]
        u = np.sort(key)
        u = u[np.concatenate(([True], u[1:] != u[:-1]))]
        m1, m2 = np.uint64((1 << bits[1]) - 1), np.uint64((1 << bits[2]) - 1)
        return np.stack([u >> np.uint64(bits[1] + bits[2]), (u >> np.uint64(bits[2])) & m1, u & m2], 1).astype(np.uint32)
    t = t[np.lexsort((t[:, 2], t[:, 1], t[:, 0]))]
    keep = np.ones(len(t), bool)
    keep[1:] = (t[1:] != t[:-1]).any(axis=1)
    return t[keep].astype(np.uint32)


def _np_set(s, p, o):
    return _np_set_rows(np.stack([s, p, o], 1))


def np_union(da, sa, db_, sb):
    """the union of two employee stores by numpy: b's set, its terms in first-seen order, new ids in that order, the set union"""
    bset = _np_set(db_.s, db_.p, db_.o)
    seq = bset.reshape(-1)
    order = np.argsort(seq, kind="stable")
    ss = seq[order]
    terms = seq[np.sort(order[np.concatenate(([True], ss[1:] != ss[:-1]))])]  # distinct ids by first position
    a_id = {s: i for i, s in enumerate(sa)}
    new_id = np.empty(len(terms), np.uint32)
    nxt = len(sa)
    added = []
    for k, t in enumerate(terms.tolist()):
        i = a_id.get(sb[t])
        if i is None:
            i = nxt
            nxt += 1
            added.append(sb[t])
        new_id[k] = i
    remap = np.zeros(len(sb), np.uint32)
    remap[terms] = new_id
    rb = remap[bset]
    aset = _np_set(da.s, da.p, da.o)
    return _np_set(np.concatenate([aset[:, 0], rb[:, 0]]), np.concatenate([aset[:, 1], rb[:, 1]]), np.concatenate([aset[:, 2], rb[:, 2]])), sa + added


def test_cfg2_union_by_count_and_digest(ctxs):
    dst, a, b = ctxs
    da, db_ = datagen.employee_dataset(1_666_667, seed=42), datagen.employee_dataset(1_666_667, seed=45)
    sa, sb = datagen.employee_strings(da), datagen.employee_strings(db_)
    a.store_load(da.s, da.p, da.o)
    a.dict_strings_load(sa)
    b.store_load(db_.s, db_.p, db_.o)
    b.dict_strings_load(sb)
    info = dst.store_union(a, b)
    want, strings = np_union(da, sa, db_, sb)
    got = np.stack(dst.store_download(), 1)
    assert info["n_rows"] == len(want) == len(got)
    assert _rows_sha(got) == _rows_sha(want)
    assert info["dict_first"] == len(sa) and info["dict_first"] + info["dict_new"] == len(strings)
    assert dst.dict_strings_download(len(sa), info["dict_new"]) == strings[len(sa):]


def test_cfg4_par_join_with_itself(ctxs):
    dst, a, _ = ctxs
    t = datagen.taxonomy_dataset()
    sc = t.ids["rdfs:subClassOf"]
    a.store_load(t.s, t.p, t.o)
    a.dict_strings_load(["rdfs:subClassOf", "rdf:type"])
    info = dst.store_par_join(a, a, sc)
    e = t.p == sc
    child, parent = t.s[e].astype(np.int64), t.o[e].astype(np.int64)
    par = np.full(int(max(child.max(), parent.max())) + 1, -1, np.int64)
    par[child] = parent
    g = par[parent]
    joined = np.stack([child[g >= 0], np.full(int((g >= 0).sum()), sc), g[g >= 0]], 1)
    semi = np.isin(parent, parent)
    kept = np.stack([child[semi], np.full(int(semi.sum()), sc), parent[semi]], 1)
    both = np.concatenate([joined, kept]).astype(np.uint32)
    want = _np_set(both[:, 0], both[:, 1], both[:, 2])
    got = np.stack(dst.store_download(), 1)
    assert info["n_rows"] == len(want) == len(got) and info["n_a"] == int(e.sum())
    assert _rows_sha(got) == _rows_sha(want)
