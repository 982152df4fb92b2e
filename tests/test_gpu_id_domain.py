"""GPU (-m gpu): the join, scan, index and Datalog routes on term ids at the edges of the u32 domain, and on both sides of every
id-range threshold that selects a route.

Every case runs through the C ABI on a context of its own and is checked two ways: against the oracle (the same bag, row for row on
the u32 ids), and against the remap (tests/id_domain_cases.py): op(f(x)) == f(op(x)), with op(x) the device's own answer on the
identity. Where a threshold selects the route, the kb_stats delta of the call proves which route ran:

  kb_hash_join, join_grouped (range <= max(16 n, 2^20))   probe_launches 2 (the grouped probe) vs 1 (the chained table's)
  star join R3, fused scan build (range <= max(4 n, 2^16))  fused_scan_builds 1 vs 0 (index off)
  store slice tables (range <= max(4 n + 65536, 2^16))   the one-kernel index join: index_joins 1 with a one-word read-back
                                                           (d2h_bytes 4) vs no index join
  star join R2, tables built from slices (range <= max(8 n, 2^16))   index_joins 1 vs 0
  index-lookup directories (range <= max(8 n, 2^20))     scan_launches 0 (answered from the directory) vs a scan
  kb_bgp_execute reduce bitmaps ([lo, lo + 2^28))          no counter: the plan must show a reduction round, and an id at
                                                           lo + 2^28 passes the reduction and must survive in the bag

A store holding KB_ID_NONE (reserved: the direct tables use it as their empty slot) is refused by every store entry point.
"""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import helpers as H
from tests import id_domain_cases as D
from tests import oracle_api as O
from tests import rsp_join_reference as J

pytestmark = pytest.mark.gpu

NONE = c.KB_ID_NONE
FIELDS = ("scan_launches", "build_launches", "probe_launches", "kernel_launches", "fused_scan_builds", "index_joins", "d2h_bytes")
DEFAULT_ENV = {"KOLIBRIE_USE_INDEX": "1", "KOLIBRIE_INDEX_KERNEL": "1", "KOLIBRIE_PROBE_TABLE": "1", "KOLIBRIE_CSR_JOIN": "1",
               "KOLIBRIE_INDEX_MAINTAIN": "1"}
ROWS = D.star_store()
MAPS = D.remaps(ROWS)
# remaps that keep every predicate slice's id range and density: the star join takes the identity's route under them
SAME_ROUTE = ("identity", "top_plain", "quoted")
HIS = {"top": 0xFFFFFFFE, "straddle": 0x80000000 + (1 << 15)}


@pytest.fixture
def make_ctx(monkeypatch):
    """a fresh context, created after the route switches are set (they are read when a context is created); KOLIBRIE_ORDERED is
    left as the caller's environment has it"""
    made = []

    def make(**env):
        for k, v in {**DEFAULT_ENV, **env}.items():
            monkeypatch.setenv(k, v)
        cx = c.Context(0)
        made.append(cx)
        return cx

    yield make
    for cx in made:
        cx.close()


def u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def delta(cx, call):
    a = cx.get_stats()
    out = call()
    b = cx.get_stats()
    return out, {f: b[f] - a[f] for f in FIELDS}


def rows(rel, slots):
    return rel.to_numpy(slots) if rel.n_rows else np.empty((0, len(slots)), np.uint32)


def load(cx, tr, index, numeric=True):
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    if numeric:
        num, isn = D.numeric_table()
        cx.dict_numeric_load(num, isn)
    if index:
        cx.build_index()


def db_of(tr, numeric=True):
    if numeric:
        num, isn = D.numeric_table()
        return O.Db(tr[:, 0], tr[:, 1], tr[:, 2], num, isn)
    return O.Db(tr[:, 0], tr[:, 1], tr[:, 2])


def ordered():
    import os

    return os.environ.get("KOLIBRIE_ORDERED", "0") == "1"


# ---------------------------------------------------------------- the reserved id in the store
def put(cx, entry, tr, tmp_path, tag=5):
    """one store entry point on the triples `tr`; returns the status"""
    import torch

    s, p, o = (u32(tr[:, j]) for j in range(3))
    L = c.lib()
    if entry in ("load", "append"):
        fn = L.kb_store_load if entry == "load" else L.kb_store_append
        args = (cx.h, s.ctypes.data, p.ctypes.data, o.ctypes.data, len(tr)) + ((tag,) if entry == "append" else ())
        return fn(*args)
    if entry in ("load_device", "append_device"):
        cols = [torch.from_numpy(x).cuda() for x in (s, p, o)]
        fn = L.kb_store_load_device if entry == "load_device" else L.kb_store_append_device
        args = (cx.h, cols[0].data_ptr(), cols[1].data_ptr(), cols[2].data_ptr(), len(tr)) + ((tag,) if entry == "append_device" else ())
        rc = fn(*args)
        torch.cuda.synchronize()
        return rc
    if entry == "star_join_host":
        try:
            cx.star_join_host(s, p, o, 0, [c.pattern(c.V(0), c.K(D.P_NAME), c.V(1))])
            return c.KB_OK
        except c.KolibrieError as e:
            return e.status
    assert entry == "append_file"
    path = str(tmp_path / "seg.kbs")
    c.segment_write(path, s, p, o, tag=tag)
    return L.kb_store_append_file(cx.h, path.encode(), tag, 1)


ENTRIES = ("load", "load_device", "append", "append_device", "append_file", "star_join_host")
POSITIONS = ("subject", "predicate", "object")


@pytest.mark.parametrize("position", POSITIONS)
@pytest.mark.parametrize("entry", ENTRIES)
def test_store_refuses_the_reserved_id(make_ctx, tmp_path, entry, position):
    """a triple holding KB_ID_NONE anywhere is refused with KB_E_INVALID naming the position. A refused load has emptied the store
    (and so voided the closed token); a refused append changes nothing"""
    cx = make_ctx()
    base = ROWS[:400]
    rules = D.store_rules()
    load(cx, base, index=True)
    cx.datalog_fixpoint(rules)
    before = np.stack(cx.store_download(), axis=1)
    bad = u32(ROWS[400:460].copy())
    bad[17, POSITIONS.index(position)] = NONE
    rc = put(cx, entry, bad, tmp_path)
    assert rc == c.KB_E_INVALID, entry
    msg = c.lib().kb_last_error(cx.h).decode()
    assert position in msg and "reserved" in msg, msg
    after = np.stack(cx.store_download(), axis=1)
    if entry.startswith("load") or entry == "star_join_host":  # (the one-shot host call replaces the store, as a load does)
        assert cx.store_size()[0] == 0 and len(after) == 0
        with pytest.raises(c.KolibrieError) as e:
            cx.datalog_maintain(rules)
        assert e.value.status == c.KB_E_INVALID and "not closed" in e.value.message
    else:
        assert np.array_equal(after, before), "a refused append changed the store"
        cx.datalog_maintain(rules)  # still the closed store
    # the same triples without the reserved id are accepted
    assert put(cx, entry, u32(ROWS[400:460]), tmp_path) == c.KB_OK


# ---------------------------------------------------------------- remaps: scan, star join, BGP, GROUP BY, fixpoint
def both_ways(got_f, want_f, got_id, f, what):
    """the device's answer on f(x) against the oracle on f(x), and against f(the device's answer on x)"""
    H.assert_same_bag(got_f, want_f, f"{what}: oracle")
    H.assert_same_bag(got_f, f(got_id), f"{what}: remap")


def scan_patterns():
    some = ROWS[7]
    return [c.pattern(c.V(0), c.K(D.P_KNOWS), c.V(1)), c.pattern(c.K(int(some[0])), c.V(1), c.V(2)),
            c.pattern(c.K(int(some[0])), c.K(int(some[1])), c.V(2)), c.pattern(c.V(0), c.K(D.P_DEPT), c.K(int(ROWS[ROWS[:, 1] == D.P_DEPT][0, 2]))),
            c.pattern(c.V(0), c.V(1), c.K(int(some[2]))), c.pattern(c.V(0), c.K(D.P_KNOWS), c.V(0)), c.pattern(c.V(0), c.K(D.P_TAG), c.K(1))]


@pytest.mark.parametrize("index", [True, False])
@pytest.mark.parametrize("family", D.FAMILIES)
def test_scan_under_remap(make_ctx, family, index):
    """kb_scan with constants at the moved ids in each position, a repeated variable, index lookups with a bound subject or object.
    In ordered mode the output is in store order, which a remap does not change: the image sequence must be exact"""
    f = MAPS[family]
    cx0, cx = make_ctx(), make_ctx()
    load(cx0, ROWS, index)
    load(cx, f(ROWS), index)
    db = db_of(f(ROWS))
    for i, pat in enumerate(scan_patterns()):
        a = cx0.scan([pat])[0]
        b = cx.scan([f.pattern(pat)])[0]
        w = db.scan(f.pattern(pat))
        slots = sorted(w.slots)
        assert sorted(b.slots) == slots
        both_ways(rows(b, slots), rows(w, slots), rows(a, slots), f, f"{family} scan {i}")
        if ordered() and not index:  # (the scan path: output in store order)
            assert np.array_equal(rows(b, slots), f(rows(a, slots))), f"{family} scan {i}: ordered sequence"


@pytest.mark.parametrize("index", [True, False])
@pytest.mark.parametrize("family", D.FAMILIES)
def test_star_join_under_remap(make_ctx, family, index):
    """kb_star_join and kb_star_join_aggregate (COUNT by ?3) on the moved store, index on (table mode / slice mode) and off (fused
    scan build, chained). Under the SAME_ROUTE remaps the route is pinned to the identity's, and in ordered mode the exact image
    sequence too"""
    f = MAPS[family]
    cx0, cx = make_ctx(), make_ctx()
    load(cx0, ROWS, index)
    load(cx, f(ROWS), index)
    db = db_of(f(ROWS))
    for name, (js, pats, filt) in D.star_queries().items():
        fp = [f.pattern(p) for p in pats]
        a, da = delta(cx0, lambda: cx0.star_join(js, pats, filt))
        b, db_ = delta(cx, lambda: cx.star_join(js, fp, f.filt(filt)))
        w = db.bgp(fp, f.filt(filt))
        slots = sorted(w.slots)
        both_ways(rows(b, slots), rows(w, slots), rows(a, slots), f, f"{family} {name}")
        if family in SAME_ROUTE:
            route = ("index_joins", "fused_scan_builds", "scan_launches")
            assert {k: db_[k] for k in route} == {k: da[k] for k in route}, f"{family} {name}: {db_} vs {da}"
            if ordered():  # output in store order (table mode, slice mode and the scan path alike), which the remap keeps
                assert np.array_equal(rows(b, slots), f(rows(a, slots))), f"{family} {name}: ordered sequence"
        ga, na = cx0.star_join_aggregate(js, pats, filt, [3], [(c.AGG_COUNT, 0)])
        gb, nb = cx.star_join_aggregate(js, fp, f.filt(filt), [3], [(c.AGG_COUNT, 0)])
        assert na == nb == w.n_rows
        want = np.unique(rows(w, [3])[:, 0], return_counts=True)
        got = np.stack([gb["keys"][0], gb["counts"]], axis=1)
        H.assert_same_bag(got, np.stack([want[0], want[1]], axis=1).astype(np.uint64), f"{family} {name} aggregate")
        H.assert_same_bag(got, np.stack([f(ga["keys"][0]).astype(np.uint64), ga["counts"]], axis=1), f"{family} {name} aggregate remap")


def annotation_store(seed=8):
    """RDF-star annotations: subjects are quoted ids, << s p o >> ex:source ?s ; ex:certainty ?c (numeric)"""
    g = np.random.default_rng(seed)
    n = 3000
    q = u32(0x80000000 + np.sort(g.choice(1 << 20, n, replace=False)))
    q[0], q[-1] = 0x80000000, 0x80000000 + (D.QUOTED_LIMIT - 1)
    src = np.stack([q, np.full(n, 140), 4000 + g.integers(0, 60, n)], axis=1)
    cer = np.stack([q, np.full(n, 141), g.integers(D.NUM_LO, D.NUM_HI, n)], axis=1)
    return u32(np.concatenate([src, cer])[g.permutation(2 * n)])


@pytest.mark.parametrize("index", [True, False])
def test_star_join_on_quoted_subjects(make_ctx, index):
    """?q ex:source ?s . ?q ex:certainty ?c FILTER(?c > 0): the join key is a quoted-triple id in every row"""
    cx = make_ctx()
    tr = annotation_store()
    load(cx, tr, index)
    pats = [c.pattern(c.V(0), c.K(140), c.V(1)), c.pattern(c.V(0), c.K(141), c.V(2))]
    filt = [c.fop(c.F_CMP_NUM, slot=2, cmp=c.CMP_GT, value=0.0)]
    w = db_of(tr).bgp(pats, filt)
    assert 0 < w.n_rows < len(tr) // 2
    got = cx.star_join(0, pats, filt)
    H.assert_same_bag(rows(got, [0, 1, 2]), rows(w, [0, 1, 2]), "annotations")
    g, n = cx.star_join_aggregate(0, pats, filt, [1], [(c.AGG_COUNT, 0)])
    assert n == w.n_rows and int(g["counts"].sum()) == n


@pytest.mark.parametrize("family", D.FAMILIES)
def test_bgp_under_remap(make_ctx, family):
    """kb_bgp_execute's component route on a chain BGP over the moved store"""
    f = MAPS[family]
    cx0, cx = make_ctx(), make_ctx()
    load(cx0, ROWS, False)
    load(cx, f(ROWS), False)
    pats = [f.pattern(p) for p in D.bgp_chain()]
    a = cx0.bgp_execute(D.bgp_chain())
    b = cx.bgp_execute(pats)
    assert cx.bgp_last_plan()["route"] == c.BGP_COMPONENTS
    w = db_of(f(ROWS)).bgp(pats)
    slots = sorted(w.slots)
    assert w.n_rows > 0
    both_ways(rows(b, slots), rows(w, slots), rows(a, slots), f, f"{family} chain")


@pytest.mark.parametrize("lo", [16, 0x7FF00000, 0xFFFFFFFE - (1 << 28) - 200], ids=["low", "straddle", "top"])
def test_bgp_reduce_bitmap_edge(make_ctx, lo):
    """a variable taking lo, lo + 2^28 - 1 and lo + 2^28: the last id is past the 32 MB bitmap and must pass the reduction"""
    cx = make_ctx()
    tr, pats = D.bitmap_store(lo)
    load(cx, tr, False, numeric=False)
    got = cx.bgp_execute(pats)
    plan = cx.bgp_last_plan()
    assert plan["route"] == c.BGP_COMPONENTS and sum(plan["reduce_rounds"]) > 0, plan
    w = db_of(tr, numeric=False).bgp(pats)
    slots = sorted(w.slots)
    H.assert_same_bag(rows(got, slots), rows(w, slots), f"bitmap edge {lo:#x}")
    assert lo + D.RED_MAX_BITS in set(rows(got, [1])[:, 0].tolist())


def test_group_aggregate_edge_keys(make_ctx):
    """group keys 0, 0x7FFFFFFF, 0x80000000 and 0xFFFFFFFE among 300 groups (more than one CTA's 64: the global table too)"""
    cx = make_ctx()
    g = np.random.default_rng(12)
    n = 40000
    keys = np.concatenate([[0, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE], 0x7FFF0000 + np.arange(296)]).astype(np.uint32)
    kc = u32(keys[g.integers(0, len(keys), n)])
    kc[:4] = keys[:4]
    vc = u32(g.integers(D.NUM_LO, D.NUM_HI, n))
    num, isn = D.numeric_table()
    cx.dict_numeric_load(num, isn)
    rel = cx.rel_from_host([0, 1], [kc, vc])
    got = cx.group_aggregate(rel, [0], [(c.AGG_COUNT, 1), (c.AGG_SUM, 1), (c.AGG_MIN, 1), (c.AGG_MAX, 1)])
    db = O.Db(np.zeros(1, np.uint32), np.zeros(1, np.uint32), np.zeros(1, np.uint32), num, isn)
    want = db.group(O.rel_from_host([0, 1], [kc, vc]), [0], [(c.AGG_COUNT, 1), (c.AGG_SUM, 1), (c.AGG_MIN, 1), (c.AGG_MAX, 1)])
    assert len(got["keys"][0]) == len(keys)
    og, ow = np.argsort(got["keys"][0]), np.argsort(want["keys"][0])
    assert np.array_equal(got["keys"][0][og], want["keys"][0][ow])
    assert np.array_equal(got["counts"][og], want["counts"][ow])
    for j in range(4):
        assert np.array_equal(got["values"][j][og], want["values"][j][ow]), j


STRATEGIES = {"semi_naive": c.SEMI_NAIVE, "naive": c.NAIVE, "parallel": c.SEMI_NAIVE_PARALLEL}


def datalog_edge_store():
    """star_store with link chains through 0x7FFFFFFF, 0x80000000 and 0xFFFFFFFE, the fact (0xFFFFFFFE link 0xFFFFFFFE) — whose
    64-bit known-fact key differs from the tombstone only in bit 32 — and tags at 0xFFFFFFFE, the constant of the third rule"""
    top, mid_lo, mid_hi = 0xFFFFFFFE, 0x7FFFFFFF, 0x80000000
    subj = np.unique(ROWS[:, 0])
    extra = np.array([[subj[0], D.P_LINK, mid_lo], [mid_lo, D.P_LINK, mid_hi], [mid_hi, D.P_LINK, top], [top, D.P_LINK, top],
                      [subj[0], D.P_TAG, top], [mid_lo, D.P_TAG, top], [top, D.P_TAG, top]], dtype=np.uint64)
    return u32(np.concatenate([ROWS.astype(np.uint64), extra]))


def edge_rules():
    rules = D.store_rules()
    r = rules[2]
    r["premise"][0] = c.pattern(c.V(0), c.K(D.P_TAG), c.K(0xFFFFFFFE))
    r["conclusion"][0] = c.pattern(c.V(1), c.K(D.P_TAG), c.K(0xFFFFFFFE))
    return rules


def fix_check(rel, st, want, what):
    H.assert_same_bag(rows(rel, [0, 1, 2]), want["facts"], f"{what}: facts")
    assert st.rounds == len(want["round_new"]), what
    assert list(st.round_new[: st.rounds]) == want["round_new"], what
    assert st.derivations == want["derivations"], what


@pytest.mark.parametrize("strategy", list(STRATEGIES))
@pytest.mark.parametrize("family", D.FAMILIES)
def test_fixpoint_under_remap(make_ctx, family, strategy):
    f = MAPS[family]
    cx = make_ctx()
    load(cx, f(ROWS), False, numeric=False)
    rules = [f.rule(r) for r in D.store_rules()]
    rel, st = cx.datalog_fixpoint(rules, STRATEGIES[strategy])
    fix_check(rel, st, db_of(f(ROWS), numeric=False).fixpoint(rules, STRATEGIES[strategy]), f"{family} {strategy}")


@pytest.mark.parametrize("strategy", list(STRATEGIES))
def test_fixpoint_seed_and_maintain_at_the_top_ids(make_ctx, strategy):
    """kb_datalog_fixpoint, kb_datalog_maintain (the closed token is recorded for the sequential strategies only) and
    kb_datalog_fixpoint_seed over facts at 2^31 +- 1 and 0xFFFFFFFE; the store after each call = base + the oracle's closure"""
    tr = datalog_edge_store()
    rules = edge_rules()
    k = STRATEGIES[strategy]
    cx = make_ctx()
    later, base = tr[:40], tr[40:]  # (the edge facts are the last rows: they stay in the base)
    cx.store_load(base[:, 0], base[:, 1], base[:, 2])
    cx.store_append(later[:, 0], later[:, 1], later[:, 2], 9)
    rel, st = cx.datalog_fixpoint(rules, k)
    fix_check(rel, st, db_of(tr, numeric=False).fixpoint(rules, k), f"edge fixpoint {strategy}")
    assert (0xFFFFFFFE, D.P_REACH, 0xFFFFFFFE) in set(map(tuple, rows(rel, [0, 1, 2]).tolist()))

    def check_store(facts, what):
        want = db_of(facts, numeric=False).fixpoint(rules, k)["facts"]
        s, p, o = cx.store_download()
        H.assert_same_bag(np.stack([s, p, o], axis=1), np.concatenate([facts, want]), what)

    def closure(facts):
        return set(map(tuple, db_of(facts, numeric=False).fixpoint(rules, k)["facts"].tolist()))

    facts, inferred = tr, closure(tr)
    if k != c.SEMI_NAIVE_PARALLEL:
        add = u32([[0x80000000, D.P_LINK, 0xFFFFFFFD], [0xFFFFFFFD, D.P_LINK, 0xFFFFFFFE]])
        gone, new, mst = cx.datalog_maintain(rules, [9], add, 10, k)
        facts = np.concatenate([base, add])
        check_store(facts, f"maintain {strategy}")
        after = closure(facts)
        # the inferred facts that left and arrived are exactly the oracle closures' difference
        assert set(map(tuple, rows(gone, [0, 1, 2]).tolist())) == inferred - after, strategy
        assert set(map(tuple, rows(new, [0, 1, 2]).tolist())) == after - inferred, strategy
        assert mst.inferred_removed == len(inferred - after) and mst.inferred_added == len(after - inferred)
        inferred = after
    seed_rows = u32([[0xFFFFFFFE, D.P_LINK, 0x7FFFFFFF]])
    seed = cx.rel_from_host([0, 1, 2], [seed_rows[:, j] for j in range(3)])
    out, n_new, sst = cx.datalog_fixpoint_seed(rules, seed, k)
    assert n_new == 1
    facts = np.concatenate([facts, seed_rows])
    check_store(facts, f"seed {strategy}")
    # the accepted seed fact, then exactly the facts the oracle's closure gains from it
    after = closure(facts)
    got = rows(out, [0, 1, 2])
    assert tuple(got[0]) == tuple(seed_rows[0]) and set(map(tuple, got[1:].tolist())) == after - inferred, strategy
    assert sst.inferred == len(after - inferred) == len(got) - 1


# ---------------------------------------------------------------- thresholds
@pytest.mark.parametrize("past", [False, True], ids=["at", "past"])
@pytest.mark.parametrize("hi", list(HIS))
def test_hash_join_grouped_threshold(make_ctx, hi, past):
    cx = make_ctx()
    (ls, lc), (rs, rc), route = D.grouped_pair(HIS[hi], past)
    want = O.hash_join(O.rel_from_host(ls, lc), O.rel_from_host(rs, rc))
    left, right = cx.rel_from_host(ls, lc), cx.rel_from_host(rs, rc)
    got, d = delta(cx, lambda: cx.hash_join(left, right))
    H.assert_same_bag(rows(got, [0, 1, 2]), rows(want, [0, 1, 2]), f"{hi} {route}")
    assert d["probe_launches"] == (2 if route == "grouped" else 1), d


@pytest.mark.parametrize("heavy", [0xFFFFFFFE, 0x80000000])
def test_hash_join_heavy_key_at_the_edge(make_ctx, heavy):
    """a third of the probe rows and 40 build rows on one key at an edge id: the output passes PROBEG_HEAVY, so the grouped join makes
    its heavy-tile launch (one kernel launch more than the control with one build row on that key), and the route equals that of the
    same join with every key shifted down to small ids"""
    cx, cx0, cxc = make_ctx(), make_ctx(), make_ctx()
    (ls, lc), (rs, rc) = D.heavy_pair(heavy)
    want = O.hash_join(O.rel_from_host(ls, lc), O.rel_from_host(rs, rc))
    assert want.n_rows > D.PROBEG_HEAVY
    got, d = delta(cx, lambda: cx.hash_join(cx.rel_from_host(ls, lc), cx.rel_from_host(rs, rc)))
    H.assert_same_bag(rows(got, [0, 1, 2]), rows(want, [0, 1, 2]), f"heavy {heavy:#x}")
    (cls, clc), (crs, crc) = D.heavy_pair(heavy, n_heavy=1)
    assert O.hash_join(O.rel_from_host(cls, clc), O.rel_from_host(crs, crc)).n_rows < D.PROBEG_HEAVY
    _, dc = delta(cxc, lambda: cxc.hash_join(cxc.rel_from_host(cls, clc), cxc.rel_from_host(crs, crc)))
    assert d["kernel_launches"] == dc["kernel_launches"] + 1 and d["build_launches"] == dc["build_launches"], (d, dc)
    shift = int(min(lc[0].min(), rc[0].min())) - 1000
    lo_l, lo_r = [u32(lc[0] - shift), lc[1]], [u32(rc[0] - shift), rc[1]]
    got0, d0 = delta(cx0, lambda: cx0.hash_join(cx0.rel_from_host(ls, lo_l), cx0.rel_from_host(rs, lo_r)))
    assert d == d0, (d, d0)
    a = rows(got0, [0, 1, 2])
    a[:, 0] += np.uint32(shift)
    H.assert_same_bag(rows(got, [0, 1, 2]), a, "heavy remap")


@pytest.mark.parametrize("past", [False, True], ids=["at", "past"])
@pytest.mark.parametrize("hi", list(HIS))
@pytest.mark.parametrize("kind", ["r3", "slice", "r2"])
def test_star_join_threshold(make_ctx, kind, hi, past):
    tr, on = D.star_threshold(kind, HIS[hi], past)
    cx = make_ctx(KOLIBRIE_USE_INDEX="0" if kind == "r3" else "1")
    load(cx, tr, index=kind != "r3", numeric=False)
    pats = D.star_pats()
    want = db_of(tr, numeric=False).bgp(pats)
    got, d = delta(cx, lambda: cx.star_join(0, pats, []))
    H.assert_same_bag(rows(got, [0, 1, 2, 3]), rows(want, [0, 1, 2, 3]), f"{kind} {hi} {'at' if on else 'past'}")
    if kind == "r3":
        assert d["fused_scan_builds"] == (1 if on else 0), d
    elif kind == "slice":
        assert (d["index_joins"] == 1 and d["d2h_bytes"] == 4) == on, d
    else:
        assert d["index_joins"] == (1 if on else 0), d


@pytest.mark.parametrize("past", [False, True], ids=["at", "past"])
@pytest.mark.parametrize("hi", list(HIS))
def test_index_lookup_directory_threshold(make_ctx, hi, past):
    """(c P ?o) on a multi-valued subject column, c at both ends of the range: a key-grouped directory answers it, or a scan"""
    tr, lo, top = D.directory_store(HIS[hi], past)
    cx = make_ctx()
    load(cx, tr, True, numeric=False)
    db = db_of(tr, numeric=False)
    for k in (lo, top):
        pat = c.pattern(c.K(k), c.K(120), c.V(1))
        got, d = delta(cx, lambda: cx.scan([pat])[0])
        w = db.scan(pat)
        assert w.n_rows > 0
        H.assert_same_bag(rows(got, [1]), rows(w, [1]), f"{k:#x}")
        assert (d["scan_launches"] == 0) == (not past), d


def test_window_slides_to_the_top_of_the_domain(make_ctx):
    """slides with the index maintained. A window of dense low ids is replaced by one just below 0xFFFFFF00: the subject tables are
    built anew there with headroom past 2^32 (tmin + cap > 2^32), and the next slide's keys land in that headroom; then quoted
    subjects join the same predicates, and the top slide leaves. After each slide the index path answers like the oracle"""
    cx = make_ctx()
    g = np.random.default_rng(30)
    pats = D.star_pats()
    top = 0xFFFFFF00 - 4000  # two slides of 2 000 ids each end below 0xFFFFFF00

    def slide(lo, n=500):
        return D.star_over_subjects(u32(lo + np.sort(g.choice(4 * n, n, replace=False))), seed=int(g.integers(1 << 30)))

    keep = u32([[5, 99, 6]])  # a predicate of its own that stays: the index is never empty, so it is maintained throughout
    held = {0: keep, 1: slide(1000)}
    for tag in (0, 1):
        cx.store_append(held[tag][:, 0], held[tag][:, 1], held[tag][:, 2], tag)
    cx.build_index()
    # tag, first subject, tag evicted before it arrives, whether the one-kernel index join (persistent tables) must answer
    for tag, lo, evict, r1 in [(2, top, 1, True), (3, top + 2000, None, True), (4, 0x80000000, None, False), (5, 0x80000000 + 2000, 2, False)]:
        if evict is not None:
            cx.store_evict(evict)
            del held[evict]
        tr = slide(lo)
        cx.store_append(tr[:, 0], tr[:, 1], tr[:, 2], tag)
        held[tag] = tr
        all_rows = np.concatenate(list(held.values()))
        db = db_of(all_rows, numeric=False)
        want = db.bgp(pats)
        got, d = delta(cx, lambda: cx.star_join(0, pats, []))
        H.assert_same_bag(rows(got, [0, 1, 2, 3]), rows(want, [0, 1, 2, 3]), f"slide {tag}")
        if r1:
            assert d["index_joins"] == 1 and d["d2h_bytes"] == 4, (tag, d)
        subj = all_rows[all_rows[:, 1] == 101, 0]
        for k in (int(tr[:, 0].min()), int(tr[:, 0].max()), int(subj.min()), int(subj.max())):
            pat = c.pattern(c.K(k), c.K(101), c.V(1))
            H.assert_same_bag(rows(cx.scan([pat])[0], [1]), rows(db.scan(pat), [1]), f"slide {tag} lookup {k:#x}")


def test_slide_into_table_headroom_past_2_32(make_ctx):
    """a slide of ten predicates (the batched index path) whose subjects land in the headroom of the subject tables: near the top of
    the domain tmin + cap passes 2^32, and the keys must still be found to fit — the append costs what it costs at low ids (no table
    rebuild), and the one-kernel index join answers like the oracle"""
    preds = tuple(range(101, 111))
    costs = {}
    for lo in (1000, 0xFFFF0000):
        g = np.random.default_rng(31)
        first = D.star_over_subjects(u32(lo + np.sort(g.choice(1500, 500, replace=False))), preds, seed=1)
        second = D.star_over_subjects(u32(lo + 1500 + np.sort(g.choice(1500, 500, replace=False))), preds, seed=2)
        cx = make_ctx()
        cx.store_append(first[:, 0], first[:, 1], first[:, 2], 1)
        cx.build_index()
        _, costs[lo] = delta(cx, lambda: cx.store_append(second[:, 0], second[:, 1], second[:, 2], 2))
        pats = D.star_pats()
        want = db_of(np.concatenate([first, second]), numeric=False).bgp(pats)
        got, d = delta(cx, lambda: cx.star_join(0, pats, []))
        H.assert_same_bag(rows(got, [0, 1, 2, 3]), rows(want, [0, 1, 2, 3]), f"{lo:#x}")
        assert d["index_joins"] == 1 and d["d2h_bytes"] == 4, (lo, d)
    assert costs[1000] == costs[0xFFFF0000], costs


def test_joins_keep_the_top_id_apart_from_unbound(make_ctx):
    """0xFFFFFFFE is a bound value and KB_ID_NONE an unbound cell: kb_natural_join never confuses them; kb_bind_join joins on the edge
    ids (its contract defines no unbound cell on the left, so none is given)"""
    cx = make_ctx()
    g = np.random.default_rng(61)
    vals = np.array([0xFFFFFFFE, 0x80000000, 0x7FFFFFFF, 0, 5], dtype=np.uint32)

    def side(n, slots, unbound):
        a = vals[g.integers(0, len(vals), (n, len(slots)))]
        for j, s in enumerate(slots):
            if s in unbound:
                a[g.random(n) < 0.3, j] = NONE
        return a

    ls, rs = [10, 11, 20], [30, 11, 10]
    la, ra = side(300, ls, {10}), side(200, rs, {11})
    left = cx.rel_from_host(ls, [u32(la[:, j]) for j in range(3)])
    right = cx.rel_from_host(rs, [u32(ra[:, j]) for j in range(3)])
    ref = J.natural_join([{s: v for s, v in zip(ls, r) if v != NONE} for r in la.tolist()],
                         [{s: v for s, v in zip(rs, r) if v != NONE} for r in ra.tolist()])
    out_slots = [10, 11, 20, 30]
    want = np.array([[r.get(s, NONE) for s in out_slots] for r in ref], dtype=np.uint32).reshape(-1, 4)
    assert len(want) > 0
    H.assert_same_bag(rows(cx.natural_join(left, right), out_slots), want, "natural join")
    # bind join: subjects at the edge ids in the store and in the left relation
    tr = u32([[v, 100, 7000 + i] for i, v in enumerate(vals.tolist())] + [[v, 101, 8000 + i] for i, v in enumerate(vals.tolist())])
    load(cx, tr, True, numeric=False)
    lc = [u32(vals[g.integers(0, len(vals), 1000)]), u32(g.integers(0, 9, 1000))]
    pat = c.pattern(c.V(0), c.K(100), c.V(1))
    want = O.hash_join(O.rel_from_host([0, 5], lc), db_of(tr, numeric=False).scan(pat))
    got = cx.bind_join(cx.rel_from_host([0, 5], lc), pat)
    H.assert_same_bag(rows(got, [0, 1, 5]), rows(want, [0, 1, 5]), "bind join")


def keyed_reference(la, ls, ra, rs, keys, left_first):
    """kb_hash_join_keyed: rows paired on the key slots, every other shared slot coalesced (the first side's bound cell, else the
    other's); output columns by slot"""
    out_slots = sorted(set(ls) | set(rs))
    out = []
    for l in la.tolist():
        lv = dict(zip(ls, l))
        for r in ra.tolist():
            rv = dict(zip(rs, r))
            if any(lv[k] != rv[k] for k in keys):
                continue
            first, second = (lv, rv) if left_first else (rv, lv)
            out.append([first[s] if first.get(s, NONE) != NONE else second.get(s, NONE) for s in out_slots])
    return out_slots, np.array(out, dtype=np.uint32).reshape(-1, len(out_slots))


@pytest.mark.parametrize("merge", [0, 1], ids=["left_first", "right_first"])
def test_hash_join_keyed_top_id_and_unbound(make_ctx, merge):
    """kb_hash_join_keyed with 0xFFFFFFFE and 0x80000000 as key values and, in a shared non-key slot, next to unbound cells (which
    coalesce); an unbound key cell is refused with KB_E_UNSUPPORTED, as DESIGN §8 states"""
    cx = make_ctx()
    g = np.random.default_rng(71)
    vals = np.array([0xFFFFFFFE, 0x80000000, 0x7FFFFFFF, 0, 5], dtype=np.uint32)
    ls, rs = [10, 11, 20], [10, 11, 30]
    la = vals[g.integers(0, len(vals), (200, 3))]
    ra = vals[g.integers(0, len(vals), (150, 3))]
    la[g.random(200) < 0.3, 1] = NONE  # slot 11: shared, not a key
    ra[g.random(150) < 0.3, 1] = NONE
    left = cx.rel_from_host(ls, [u32(la[:, j]) for j in range(3)])
    right = cx.rel_from_host(rs, [u32(ra[:, j]) for j in range(3)])
    out_slots, want = keyed_reference(la, ls, ra, rs, [10], merge == 0)
    assert len(want) > 0 and np.any(want[:, 0] == 0xFFFFFFFE)
    got = cx.hash_join_keyed(left, right, [10], merge)
    assert sorted(got.slots) == out_slots
    H.assert_same_bag(rows(got, out_slots), want, "keyed")
    la[3, 0] = NONE
    bad = cx.rel_from_host(ls, [u32(la[:, j]) for j in range(3)])
    with pytest.raises(c.KolibrieError) as e:
        cx.hash_join_keyed(bad, right, [10], merge)
    assert e.value.status == c.KB_E_UNSUPPORTED


@pytest.mark.parametrize("index", [True, False])
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_store_in_the_top_shard_blocks(make_ctx, world, index):
    """kb_set_sharding: one rank's shard whose subjects are in the last shard blocks below 2^32, so compact_key folds keys near the
    top of the domain; star joins (index on: persistent tables; off: the fused scan build) equal the oracle"""
    rank = world - 1
    cand = np.arange(0xFFFFFFFE - 60000, 0xFFFFFFFF, dtype=np.uint64)
    mine = np.array([x for x in cand.tolist() if c.lib().kb_shard_of(x, world) == rank], dtype=np.uint64)
    assert len(mine) >= 3000 and int(mine.max()) >= 0xFFFFFFFE - 4096
    subj = u32(np.sort(np.random.default_rng(81).choice(mine, 3000, replace=False)))
    tr = D.star_over_subjects(subj)
    cx = make_ctx(KOLIBRIE_USE_INDEX="1" if index else "0")
    cx.set_sharding(rank, world)
    load(cx, tr, index, numeric=False)
    pats = D.star_pats()
    want = db_of(tr, numeric=False).bgp(pats)
    got, d = delta(cx, lambda: cx.star_join(0, pats, []))
    H.assert_same_bag(rows(got, [0, 1, 2, 3]), rows(want, [0, 1, 2, 3]), f"world {world}")
    if index:
        assert d["index_joins"] == 1, d
    else:
        assert d["fused_scan_builds"] == 1, d
