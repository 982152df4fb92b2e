"""GPU (-m gpu): the device's open-addressing hash tables on keys built to collide (tests/hash_mirror.py), against the references the
suite already trusts. Random data almost never reaches these branches:

  tag tables (kb_tagtab.cuh)  two different keys with the same 32-bit tag and home slot, told apart only by the caller's comparison:
                              the dictionary's batch table and persistent index (kb_dict_encode, against engine.Dictionary), the
                              quoted-triple batch table and reverse index (kb_bind TRIPLE, against ExecutionEngine._bind_host)
  GROUP BY                    two-column keys with the same in-warp match hash (group_kernel), more than 64 keys at CTA home 63
                              (group1_kernel and the index probe's fused GROUP BY: the CTA table wraps and spills), and keys at the
                              last slot of the 4096-slot global table and of its 16x retry (against tests/agg_reference.py)
  distinct set                255 and 256 objects at slot 511 of the subject codes' 512-slot set (kb_store_build_index)
  96-bit key set              INSERT / DELETE batches whose triples all share the last slot (kb_store_insert / kb_store_remove)
  64-bit fact set             inferred facts that all share the last slot of the Datalog known-fact set (against the oracle)

Keys that share a home slot at the end of a table form a probe chain that wraps to slot 0. Every case runs on a context of its own."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import engine as En
from tests import agg_reference as R
from tests import hash_mirror as M
from tests import helpers as H
from tests import oracle_api as O
from tests.test_gpu_aggregate import E as SE, K as SK, ORDERS, V as SV, load_star
from tests.test_gpu_bind import QB, check as bind_check, new_db, upload
from tests.test_gpu_probe_codes import Store, star, subj

pytestmark = pytest.mark.gpu

KINDS = [R.COUNT, R.SUM, R.MIN, R.MAX, R.AVG]


@pytest.fixture
def cx():
    x = c.Context(0)
    yield x
    x.close()


# ---- the dictionary: kb_dict_encode against engine.Dictionary

def twins(wide=False):
    """tag twins of the dictionary hash; wide: those that also share their home in a 2048-slot table"""
    out = [p for p in M.tag_twin_strings() if not wide or M.fnv1a64_folded(p[0]) & 2047 == M.fnv1a64_folded(p[1]) & 2047]
    assert len(out) >= (2 if wide else 6)
    return out


def fillers(tag, n):
    return [f"http://example.org/fill/{tag}/{k}" for k in range(n)]


def encode_and_check(cx, d: En.Dictionary, terms, what):
    """one batch: ids equal the sequential encode, `first` names the first occurrence of every new string in id order"""
    before = len(d.id_to_string)
    want = np.array([d.encode(t) for t in terms], dtype=np.uint32)
    got, first = cx.dict_encode(terms)
    assert np.array_equal(got, want), f"{what}: ids differ from the sequential encode at {np.flatnonzero(got != want)[:10]}"
    assert [terms[int(p)] for p in first] == d.id_to_string[before:], f"{what}: first-seen positions"
    for p in first:  # ... and it is the FIRST occurrence
        assert terms.index(terms[int(p)]) == int(p), what
    assert cx.dict_strings_info()[0] == len(d.id_to_string), what


def decode_all(cx, d: En.Dictionary):
    rel = cx.rel_from_host([0], [np.arange(len(d.id_to_string), dtype=np.uint32)])
    assert rel.decode_strings(0) == d.id_to_string
    rel.free()


def scatter(rng, terms, n):
    """n terms drawn from `terms`, every one of them at least twice, shuffled"""
    out = list(terms) * 2 + [terms[int(i)] for i in rng.integers(0, len(terms), max(0, n - 2 * len(terms)))]
    return [out[int(i)] for i in rng.permutation(len(out))]


def test_dict_twins_new_in_one_batch(cx):
    """both strings of every tag-twin pair are new in the same batch, each at scattered positions (batch table of 1024 slots)"""
    rng = np.random.default_rng(1)
    pool = [s for p in twins() for s in p] + fillers("a", 30)
    terms = scatter(rng, pool, 400)
    assert M.tag_batch_slots(len(terms)) == 1024
    cx.dict_strings_load([])
    d = En.Dictionary()
    encode_and_check(cx, d, terms, "twins in one batch")
    encode_and_check(cx, d, scatter(rng, pool, 300), "the same strings again (all in the persistent index)")
    decode_all(cx, d)


@pytest.mark.parametrize("route", ["encode", "load"])
def test_dict_twin_in_the_index_other_in_a_later_batch(cx, route):
    """one string of every pair is in the dictionary (encoded earlier, or loaded and indexed lazily); its twin arrives later: the
    persistent index's probe meets the same tag and home, the comparison says no, the string goes to the batch table"""
    rng = np.random.default_rng(2)
    tw = twins()
    first_half = [a for a, _ in tw] + fillers("b", 40)
    d = En.Dictionary()
    if route == "encode":
        cx.dict_strings_load([])
        encode_and_check(cx, d, scatter(rng, first_half, 120), "first members")
    else:
        for t in first_half:
            d.encode(t)
        cx.dict_strings_load(d.id_to_string)
    later = scatter(rng, [b for _, b in tw] + [a for a, _ in tw] + fillers("c", 20), 120)
    assert M.tag_index_slots(len(d.id_to_string), len(later), current=1024 if route == "encode" else 0) == 1024
    encode_and_check(cx, d, later, f"second members ({route})")
    encode_and_check(cx, d, scatter(rng, [s for p in tw for s in p], 100), "both members, both known")
    decode_all(cx, d)


def test_dict_chain_wraps_the_table(cx):
    """12 strings whose home is the last slot of every 1024-slot table: the batch table's chain and then the persistent index's
    chain run from slot 1023 through slot 0"""
    rng = np.random.default_rng(3)
    chain = list(M.home_strings(12, 1024, 1023))
    tw = twins()
    cx.dict_strings_load([])
    d = En.Dictionary()
    encode_and_check(cx, d, scatter(rng, chain[:8] + [tw[0][0]], 60), "8 of the chain, new")
    encode_and_check(cx, d, scatter(rng, chain + [tw[0][1]] + fillers("d", 10), 200), "the chain again, 4 more of it new")
    encode_and_check(cx, d, scatter(rng, chain[::-1], 40), "the chain, all known")
    decode_all(cx, d)


def test_dict_rebuild_with_twins_in_the_index(cx):
    """300 ids in a 1024-slot persistent index with tag twins in it; a batch of 200 more passes its threshold and rebuilds it at 2048
    slots, where the twins still share their home, while the twin of an indexed string arrives"""
    rng = np.random.default_rng(4)
    (a1, b1), (a2, b2) = twins(wide=True)[:2]
    cx.dict_strings_load([])
    d = En.Dictionary()
    batch1 = [a1, b1, a2] + fillers("e", 297)
    encode_and_check(cx, d, [batch1[int(i)] for i in rng.permutation(300)], "300 ids, twins among them")
    assert len(d.id_to_string) == 300 and M.tag_index_slots(300, 0) == 1024
    assert M.tag_index_slots(300, 200, current=1024) == 2048  # the next batch rebuilds the index
    batch2 = [b2, a1, b1, a2] + fillers("f", 196)
    batch2 = [batch2[int(i)] for i in rng.permutation(200)]
    encode_and_check(cx, d, batch2, "rebuild, then the twin of an indexed string")
    encode_and_check(cx, d, scatter(rng, [a1, b1, a2, b2], 40), "all twins known after the rebuild")
    decode_all(cx, d)


# ---- quoted triples: kb_bind TRIPLE against ExecutionEngine._bind_host

def quoted_db(cx, entries):
    """a dictionary of 5 strings and a quoted-triple table holding `entries` under ids QB + 2k (every other id a hole)"""
    db = new_db(cx, n_entries=0)
    qts = db.quoted_triple_store
    for k, t in enumerate(entries):
        qts.id_to_components[QB + 2 * k] = t
        qts.components_to_id[t] = QB + 2 * k
    qts.next_qt_id = QB + 2 * len(entries) + 1
    upload(cx, db)
    return db


def triple_rows(rng, triples, n):
    t = np.array(triples, dtype=np.uint32).reshape(-1, 3)
    pick = np.concatenate([np.arange(len(t)), np.arange(len(t)), rng.integers(0, len(t), max(0, n - 2 * len(t)))])
    return t[pick[rng.permutation(len(pick))]]


def test_quoted_twin_of_a_table_entry(cx):
    """the table holds one triple of every tag-twin pair; TRIPLE over rows of both: the reverse index meets the twin's tag at the
    twin's home and must answer 'not held' for the new one and the table's id for the old one"""
    tt = M.tag_twin_triples()
    db = quoted_db(cx, [a for a, _ in tt] + [(9000 + k, 3, 9100 + k) for k in range(20)])
    rng = np.random.default_rng(5)
    rows = triple_rows(rng, [b for _, b in tt] + [a for a, _ in tt], 200)
    assert M.tag_index_slots(2 * (len(tt) + 20), len(rows)) == 1024 == M.tag_batch_slots(len(rows))  # (the table's slots, holes included)
    names = {0: "s", 1: "p", 2: "o", 3: "t"}
    rel = cx.rel_from_host([0, 1, 2], [rows[:, 0], rows[:, 1], rows[:, 2]])
    got, info = bind_check(cx, db, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "t")
    assert info["quoted_new"] == len(tt)
    got2, info2 = bind_check(cx, db, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "t")  # now both twins are in the table
    assert info2["quoted_new"] == 0 and np.array_equal(got, got2)
    rel.free()


def test_quoted_twins_new_in_one_batch(cx):
    """both triples of every pair are new in the same batch: the batch table keeps them apart"""
    tt = M.tag_twin_triples()
    db = quoted_db(cx, [(9000 + k, 3, 9100 + k) for k in range(20)])
    rng = np.random.default_rng(6)
    rows = triple_rows(rng, [t for p in tt for t in p], 300)
    names = {0: "s", 1: "p", 2: "o", 3: "t"}
    rel = cx.rel_from_host([0, 1, 2], [rows[:, 0], rows[:, 1], rows[:, 2]])
    got, info = bind_check(cx, db, rel, names, "TRIPLE", [c.V(0), c.V(1), c.V(2)], "t")
    assert info["quoted_new"] == 2 * len(tt) and len(np.unique(got)) == 2 * len(tt)
    rel.free()


# ---- GROUP BY against tests/agg_reference.py

def value_table(n_ids):
    """small integers, so that every SUM is exact; ids of the value column index it"""
    num = (np.arange(n_ids, dtype=np.float64) % 97) - 40.0
    return num, np.ones(n_ids, dtype=np.uint8)


N_VALS = 4096
NUM, ISN = value_table(N_VALS)


def value_col(rng, n):
    return rng.integers(0, N_VALS, n).astype(np.uint32)


def check_groups(cx, rel, rows, group_cols, aggs_list, what):
    msgs = []
    for aggs in aggs_list:
        g = cx.group_aggregate(rel, group_cols, aggs)
        try:
            R.assert_groups_match(g, rows, NUM, group_cols, aggs, f"{what} aggs={aggs}")
        except AssertionError as e:
            msgs.append(str(e))
    assert not msgs, "\n".join(msgs)


def twin_pairs(rng, n_pairs):
    out = []
    for _ in range(n_pairs):
        k0, k1, k0b = (int(x) for x in rng.integers(0, 1 << 31, 3))
        k1b = M.group_kernel_twin(k0, k1, k0b)
        out.append(((k0, k1), (k0b, k1b)))
    return out


@pytest.mark.parametrize("layout", ["same warp", "same CTA"])
def test_group_kernel_match_hash_twins(cx, layout):
    """8 pairs of two-column keys with equal group_kernel match hashes (so equal CTA homes): in the same warp the match groups must
    split on the key comparison; in different warps of one CTA the CTA table must keep them apart"""
    rng = np.random.default_rng(7)
    pairs = twin_pairs(rng, 8)
    keys = np.array([k for p in pairs for k in p], dtype=np.uint32)  # 16 groups: 2q, 2q+1 are twins
    h = M.group_kernel_hash([keys[:, 0], keys[:, 1]])
    assert (h[0::2] == h[1::2]).all() and len({tuple(k) for k in keys.tolist()}) == 16
    n = 4096
    i = np.arange(n)
    if layout == "same warp":  # every warp holds one pair, alternating lane by lane
        g = 2 * ((i // 32) % 8) + (i % 2)
    else:  # every warp one key; the eight warps of a 256-row CTA stride hold four pairs
        g = ((i // 32) % 8) + 8 * ((i // 256) % 2)
    rows = np.concatenate([keys[g], value_col(rng, n)[:, None], value_col(rng, n)[:, None]], axis=1).astype(np.uint32)
    cx.dict_numeric_load(NUM, ISN)
    rel = cx.rel_from_host([0, 1, 2, 3], [rows[:, j] for j in range(4)])
    check_groups(cx, rel, rows, [0, 1], [[(R.COUNT, 0)], [(k, 2) for k in KINDS] + [(R.SUM, 3)]], f"group_kernel twins, {layout}")
    rel.free()


def cta63_keys(n):
    """n one-column keys at CTA home 63 that also sit at the last slot of the 4096-slot global table"""
    k = M.group_slot_keys(128 * n, low_bits=12, low=0xFFF)
    k = k[M.group1_cta_home(k) == 63][:n]
    assert len(k) == n
    return k


def test_group1_cta_table_wraps_and_spills(cx):
    """100 keys at CTA home 63, 8 rows each, in one CTA (800 rows): the CTA table's chain wraps from 63 to 0, fills, and the last 36
    keys go to the global table, where all of them sit at slot 4095"""
    rng = np.random.default_rng(8)
    keys = cta63_keys(100)
    kc = np.repeat(keys, 8)[rng.permutation(800)]
    rows = np.stack([kc, value_col(rng, 800)], axis=1).astype(np.uint32)
    cx.dict_numeric_load(NUM, ISN)
    rel = cx.rel_from_host([0, 1], [rows[:, 0], rows[:, 1]])
    check_groups(cx, rel, rows, [0], [[]] + [[(k, 1)] for k in KINDS], "group1_kernel, 100 keys at CTA home 63")
    rel.free()


def test_fused_probe_cta_table_wraps_and_spills(cx):
    """the index probe's fused GROUP BY (the star (?e P_key ?k) . (?e P_val ?v) grouped by ?k) with 300 keys at CTA home 63"""
    rng = np.random.default_rng(9)
    keys = cta63_keys(300)
    n = 1200
    rows = np.stack([np.repeat(keys, 4)[rng.permutation(n)], value_col(rng, n)], axis=1).astype(np.uint32)
    load_star(cx, rows, NUM, ISN)
    msgs = []
    for what, pats in ORDERS.items():
        for aggs in [[]] + [[(k, SV)] for k in KINDS]:
            n0 = cx.get_stats()["kernel_launches"]
            g, n_joined = cx.star_join_aggregate(SE, pats, None, [SK], aggs)
            assert cx.get_stats()["kernel_launches"] - n0 <= 2, f"fused path not taken ({what}, {aggs})"
            assert n_joined == n
            try:
                R.assert_groups_match(g, rows, NUM, [0], [(k, 1) for k, _ in aggs], f"fused probe, {what}, aggs={aggs}")
            except AssertionError as e:
                msgs.append(str(e))
    assert not msgs, "\n".join(msgs)


@pytest.mark.parametrize("n_keys", [1, 2])
def test_global_table_last_slot_and_retry(cx, n_keys):
    """5000 groups whose global home is the last slot of the 4096-slot table and of the 65536-slot retry: the first table fills
    through its wrapped chain and overflows, the retry chains 5000 groups from slot 65535 through slot 0. With two columns every
    group has the same first column, so only the second tells them apart."""
    rng = np.random.default_rng(10 + n_keys)
    ng = 5000
    if n_keys == 1:
        keys = M.group_slot_keys(ng)[:, None]
    else:
        keys = np.stack([np.full(ng, 77, np.uint32), M.group_slot_second_cols(77, ng)], axis=1)
    assert (M.group_slot_home([keys[:, j] for j in range(n_keys)], M.group_table_slots(0)) == 4095).all()
    assert (M.group_slot_home([keys[:, j] for j in range(n_keys)], M.group_table_slots(1)) == 65535).all()
    n = 2 * ng
    rows = np.concatenate([keys[np.tile(np.arange(ng), 2)[rng.permutation(n)]], value_col(rng, n)[:, None]], axis=1).astype(np.uint32)
    cx.dict_numeric_load(NUM, ISN)
    slots = list(range(n_keys + 1))
    rel = cx.rel_from_host(slots, [rows[:, j] for j in slots])
    aggs = [(R.COUNT, 0)] if n_keys == 1 else [(R.COUNT, 0), (R.SUM, n_keys), (R.MIN, n_keys), (R.MAX, n_keys)]
    g0 = cx.get_stats()["group_launches"]
    check_groups(cx, rel, rows, list(range(n_keys)), [aggs], f"{n_keys}-column keys at the last global slot")
    assert cx.get_stats()["group_launches"] - g0 == 2, "the 4096-slot table must overflow into the 16x retry"
    rel.free()


# ---- the one-byte subject codes: distinct_kernel's 512-slot set

@pytest.mark.parametrize("k", [255, 256])
def test_subject_code_objects_at_one_slot(monkeypatch, k):
    """k title objects that all home to slot 511 of the distinct set: 255 are coded (the chain wraps and holds them all), 256 are not"""
    objs = M.keys_with_mix32_low(256, 9, 511)[:k]
    assert (M.distinct_home(objs, M.CODE_SET_SLOTS) == 511).all()
    st = Store(monkeypatch)
    st.append(1, star(subj(0, 6000), objs, seed=61))
    s, p, o = st.triples()
    present = np.unique(o[p == 1])
    assert len(present) == k
    _, h2d = st.build()
    assert h2d == (4 * k if k <= M.CODE_MAX else 0), (k, h2d)
    st.check(filters=(None, int(objs[0]), int(objs[-1])))
    st.ctx.close()


# ---- set-semantic store writes: the 96-bit batch set

def store_set(cx):
    s, p, o = cx.store_download()
    return set(zip(s.tolist(), p.tolist(), o.tolist()))


def test_store_insert_remove_at_one_home(cx):
    """every triple of the batches shares one set_hash home, the last slot of every batch set: the batch set's chain wraps, and the
    pass over the store finds its triples along it"""
    S, P = 123457, 41
    objs = M.objects_for_set_hash(S, P, 300).tolist()
    rng = np.random.default_rng(12)
    base = {(S, P, x) for x in objs[:150]} | {(int(a), 42, int(b)) for a, b in rng.integers(0, 1 << 20, (200, 2))}
    b = np.array(sorted(base), dtype=np.uint32)
    cx.store_load(b[:, 0], b[:, 1], b[:, 2])
    model = set(base)

    def apply(kind, trip):
        t = np.array(trip, dtype=np.uint32)
        got = (cx.store_insert if kind == "insert" else cx.store_remove)(t[:, 0], t[:, 1], t[:, 2])
        want = []
        for x in trip:
            if kind == "insert":
                want.append(x not in model)
                model.add(x)
            else:
                want.append(x in model)
                model.discard(x)
        assert got.tolist() == want, f"{kind}: per-triple results differ at {np.flatnonzero(got != np.array(want))[:10]}"
        assert store_set(cx) == model, f"{kind}: the store differs from the set"

    ins = [(S, P, x) for x in objs[100:250]]
    ins += [ins[int(i)] for i in rng.integers(0, len(ins), 60)]  # repeats within the batch
    apply("insert", [ins[int(i)] for i in rng.permutation(len(ins))])
    rem = [(S, P, x) for x in objs[50:200] + objs[250:300]]  # held, and never held (same home)
    rem += [rem[int(i)] for i in rng.integers(0, len(rem), 60)]
    apply("remove", [rem[int(i)] for i in rng.permutation(len(rem))])
    apply("insert", [(S, P, x) for x in objs[::-1]])


# ---- Datalog: the 64-bit known-fact set

def test_datalog_facts_at_one_home(cx):
    """a rule whose 300 inferred facts (S, Q, o) share one set64 home, the last slot of the known-fact set (whatever its size up to
    65536 slots), 40 of them in the store already; a second rule infers from the first's facts"""
    S, P1, Q, P3 = 5150, 7, 8, 9
    objs = M.objects_for_set64(S, 300)
    assert (M.set64_home(1024, np.full(300, S, np.uint32), objs) == 1023).all()
    s = np.concatenate([np.full(300, S), np.full(40, S), np.arange(100, 160)]).astype(np.uint32)
    p = np.concatenate([np.full(300, P1), np.full(40, Q), np.full(60, P1)]).astype(np.uint32)
    o = np.concatenate([objs, objs[::7][:40], np.arange(200, 260)]).astype(np.uint32)
    rules = [{"premise": [c.pattern(c.V(0), c.K(P1), c.V(1))], "conclusion": [c.pattern(c.V(0), c.K(Q), c.V(1))], "filters": []},
             {"premise": [c.pattern(c.V(0), c.K(Q), c.V(1))], "conclusion": [c.pattern(c.V(0), c.K(P3), c.V(1))], "filters": []}]
    cx.store_load(s, p, o)
    rel, st = cx.datalog_fixpoint(rules, c.SEMI_NAIVE)
    want = O.Db(s, p, o).fixpoint(rules, c.SEMI_NAIVE)
    assert want["status"] == 0
    H.assert_same_bag(rel.to_numpy([0, 1, 2]), want["facts"], "closure")
    assert len(want["facts"]) == (360 - 40) + 360
    rel2, st2 = cx.datalog_fixpoint(rules, c.SEMI_NAIVE)
    assert rel2.n_rows == 0
