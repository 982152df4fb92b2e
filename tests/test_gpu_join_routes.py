"""GPU (-m gpu): which route the join operators take for each input shape, pinned by what it costs.

Every case runs its call twice on a context of its own and checks, for each call, the result against a reference and the
*fingerprint* against a literal: the change of every integer counter of kb_stats across the call (launches per family, kernel
launches, rows scanned / built / probed, bytes copied, fused scan builds, index joins). d2h_bytes counts whole control-arena reads, so
it also pins the number of host synchronisations. Counters that did not move are left out of the literals. Every case runs in
unordered and in ordered mode (KOLIBRIE_ORDERED=1: output in input order, the look-back prefix of every compacting kernel).

The routes:
  kb_hash_join      cartesian (no common variable); grouped (CSR directory: one dense key column), with heavy tiles spread over the
                    grid by a second launch; chained (multimap: several key columns, a sparse key range, or KOLIBRIE_CSR_JOIN=0), whose
                    first pass either fits its output or doubles as the exact count for a second pass; a post-filter rides on the
                    chained join (through a star join that reaches its chained route)
  kb_bind_join      one probe against a persistent table of the store index; else a scan of the pattern and a natural join
  kb_filter         the direct probe with zero tables
  kb_scan_quoted    the match pass, then a bind join (index on and off)
  kb_natural_join   kb_hash_join when no shared column holds an unbound cell; else check, mask, partition, sub-joins and coalesce
"""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import helpers as H
from tests import oracle_api as O
from tests import rsp_join_reference as J

pytestmark = pytest.mark.gpu

FIELDS = ("scan_launches", "build_launches", "probe_launches", "filter_launches", "group_launches", "other_launches", "kernel_launches",
          "rows_scanned", "rows_built", "rows_probed", "h2d_bytes", "d2h_bytes", "fused_scan_builds", "index_joins")
# switches that select routes: pinned to their defaults, so that the literals hold whatever the caller's environment says
DEFAULT_ENV = {"KOLIBRIE_ORDERED": "0", "KOLIBRIE_USE_INDEX": "1", "KOLIBRIE_INDEX_KERNEL": "1", "KOLIBRIE_PROBE_TABLE": "1",
               "KOLIBRIE_CSR_JOIN": "1", "KOLIBRIE_INDEX_MAINTAIN": "1"}
NONE = c.KB_ID_NONE

# name -> fingerprints of the first and the second call (recorded on an H100)
ROUTES = {
    "cartesian": [{"probe_launches": 1, "kernel_launches": 1}] * 2,
    "cartesian_ordered": [{"probe_launches": 1, "kernel_launches": 1}] * 2,
    "grouped": [{"build_launches": 2, "probe_launches": 2, "kernel_launches": 8, "rows_built": 4000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "grouped_ordered": [{"build_launches": 2, "probe_launches": 2, "kernel_launches": 8, "rows_built": 4000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "grouped_heavy": [{"build_launches": 2, "probe_launches": 2, "kernel_launches": 9, "rows_built": 120, "rows_probed": 9000, "d2h_bytes": 65536}] * 2,
    "grouped_heavy_ordered": [{"build_launches": 2, "probe_launches": 2, "kernel_launches": 9, "rows_built": 120, "rows_probed": 9000, "d2h_bytes": 65536}] * 2,
    "chained_fits": [{"build_launches": 1, "probe_launches": 1, "kernel_launches": 2, "rows_built": 5000, "rows_probed": 20000, "d2h_bytes": 32768}] * 2,
    "chained_fits_ordered": [{"build_launches": 1, "probe_launches": 1, "kernel_launches": 2, "rows_built": 5000, "rows_probed": 20000, "d2h_bytes": 32768}] * 2,
    "chained_resize": [{"build_launches": 1, "probe_launches": 2, "kernel_launches": 3, "rows_built": 5000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "chained_resize_ordered": [{"build_launches": 1, "probe_launches": 2, "kernel_launches": 3, "rows_built": 5000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "chained_csr_off": [{"build_launches": 1, "probe_launches": 1, "kernel_launches": 2, "rows_built": 4000, "rows_probed": 20000, "d2h_bytes": 32768}] * 2,
    "chained_csr_off_ordered": [{"build_launches": 1, "probe_launches": 1, "kernel_launches": 2, "rows_built": 4000, "rows_probed": 20000, "d2h_bytes": 32768}] * 2,
    "sparse_keys": [{"build_launches": 2, "probe_launches": 1, "kernel_launches": 3, "rows_built": 3000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "sparse_keys_ordered": [{"build_launches": 2, "probe_launches": 1, "kernel_launches": 3, "rows_built": 3000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "multi_column_keys": [{"build_launches": 1, "probe_launches": 2, "kernel_launches": 3, "rows_built": 6000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "multi_column_keys_ordered": [{"build_launches": 1, "probe_launches": 2, "kernel_launches": 3, "rows_built": 6000, "rows_probed": 20000, "d2h_bytes": 65536}] * 2,
    "star_post_filter": [{"scan_launches": 2, "build_launches": 4, "probe_launches": 3, "other_launches": 2, "kernel_launches": 10, "rows_scanned": 7778, "rows_built": 3825, "rows_probed": 3840, "d2h_bytes": 163840, "fused_scan_builds": 1},
                         {"scan_launches": 1, "build_launches": 1, "probe_launches": 1, "other_launches": 2, "kernel_launches": 5, "rows_scanned": 3889, "rows_built": 1270, "rows_probed": 1285, "d2h_bytes": 65536}],
    "star_post_filter_ordered": [{"scan_launches": 2, "build_launches": 5, "probe_launches": 3, "other_launches": 2, "kernel_launches": 10, "rows_scanned": 7778, "rows_built": 3825, "rows_probed": 3840, "d2h_bytes": 163840, "fused_scan_builds": 1},
                                 {"scan_launches": 1, "build_launches": 1, "probe_launches": 1, "other_launches": 2, "kernel_launches": 5, "rows_scanned": 3889, "rows_built": 1270, "rows_probed": 1285, "d2h_bytes": 65536}],
    "bind_index": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 30000, "d2h_bytes": 32768, "index_joins": 1}] * 2,
    "bind_index_ordered": [{"probe_launches": 1, "kernel_launches": 1, "rows_probed": 30000, "d2h_bytes": 32768, "index_joins": 1}] * 2,
    "bind_scan": [{"scan_launches": 1, "build_launches": 2, "probe_launches": 2, "kernel_launches": 9, "rows_scanned": 7000, "rows_built": 3000, "rows_probed": 30000, "d2h_bytes": 98304}] * 2,
    "bind_scan_ordered": [{"scan_launches": 1, "build_launches": 2, "probe_launches": 2, "kernel_launches": 9, "rows_scanned": 7000, "rows_built": 3000, "rows_probed": 30000, "d2h_bytes": 98304}] * 2,
    "filter": [{"filter_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "filter_ordered": [{"filter_launches": 1, "kernel_launches": 1, "d2h_bytes": 32768}] * 2,
    "quoted_index": [{"scan_launches": 1, "probe_launches": 1, "kernel_launches": 2, "rows_scanned": 5000, "rows_probed": 3488, "d2h_bytes": 65536, "index_joins": 1}] * 2,
    "quoted_index_ordered": [{"scan_launches": 1, "probe_launches": 1, "kernel_launches": 2, "rows_scanned": 5000, "rows_probed": 3488, "d2h_bytes": 65536, "index_joins": 1}] * 2,
    "quoted_scan": [{"scan_launches": 2, "build_launches": 2, "probe_launches": 2, "kernel_launches": 10, "rows_scanned": 9064, "rows_built": 3488, "rows_probed": 4064, "d2h_bytes": 131072}] * 2,
    "quoted_scan_ordered": [{"scan_launches": 2, "build_launches": 2, "probe_launches": 2, "kernel_launches": 10, "rows_scanned": 9064, "rows_built": 3488, "rows_probed": 4064, "d2h_bytes": 131072}] * 2,
    "natjoin_fast": [{"build_launches": 1, "probe_launches": 1, "other_launches": 1, "kernel_launches": 3, "rows_built": 400, "rows_probed": 600, "d2h_bytes": 65536}] * 2,
    "natjoin_fast_ordered": [{"build_launches": 1, "probe_launches": 1, "other_launches": 1, "kernel_launches": 3, "rows_built": 400, "rows_probed": 600, "d2h_bytes": 65536}] * 2,
    "natjoin_unbound": [{"build_launches": 5, "probe_launches": 6, "other_launches": 4, "kernel_launches": 26, "rows_built": 593, "rows_probed": 1095, "d2h_bytes": 229376}] * 2,
    "natjoin_unbound_ordered": [{"build_launches": 5, "probe_launches": 6, "other_launches": 4, "kernel_launches": 26, "rows_built": 593, "rows_probed": 1095, "d2h_bytes": 229376}] * 2,
}


def rng(seed):
    return np.random.default_rng(seed)


def u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def two_sides(seed, n_l, n_r, ls, rs, key_of):
    """left and right columns by slot; key_of(rng, n) gives the shared key columns"""
    g = rng(seed)
    lk, rk = key_of(g, n_l), key_of(g, n_r)
    left = {**lk, **{s: g.integers(0, 1000, n_l) for s in ls if s not in lk}}
    right = {**rk, **{s: g.integers(0, 1000, n_r) for s in rs if s not in rk}}
    return (ls, [u32(left[s]) for s in ls]), (rs, [u32(right[s]) for s in rs])


def one_key(lo, hi):
    return lambda g, n: {0: g.integers(lo, hi, n)}


def skewed_key(g, n):
    """a third of the rows share key 7: a probe tile of them expands past PROBEG_HEAVY rows"""
    k = g.integers(0, 3000, n)
    k[: n // 3] = 7
    return {0: g.permutation(k)}


SPARSE_POOL = np.sort(rng(5).choice(2_000_000_000, 5000, replace=False))


def sparse_key(g, n):
    return {0: SPARSE_POOL[g.integers(0, len(SPARSE_POOL), n)]}


def keys_of(*ranges):
    return lambda g, n: {q: g.integers(0, r, n) for q, r in enumerate(ranges)}


# name -> (switches, (left, right) = ((slots, columns), (slots, columns)))
HASH_CASES = {
    "cartesian": ({}, lambda: two_sides(1, 300, 200, [1, 2], [3, 4], lambda g, n: {})),
    "grouped": ({}, lambda: two_sides(2, 20000, 4000, [0, 1], [0, 2], one_key(0, 5000))),
    "grouped_heavy": ({}, lambda: two_sides(3, 9000, 120, [0, 1], [0, 2], skewed_key)),
    "chained_fits": ({}, lambda: two_sides(4, 20000, 5000, [0, 1, 2], [1, 0, 3], keys_of(2000, 5))),
    "chained_resize": ({}, lambda: two_sides(6, 20000, 5000, [0, 1, 2], [0, 1, 3], keys_of(50, 2))),
    "chained_csr_off": ({"KOLIBRIE_CSR_JOIN": "0"}, lambda: two_sides(2, 20000, 4000, [0, 1], [0, 2], one_key(0, 5000))),
    "sparse_keys": ({}, lambda: two_sides(7, 20000, 3000, [0, 1], [0, 2], sparse_key)),
    "multi_column_keys": ({}, lambda: two_sides(8, 20000, 6000, [0, 1, 2, 5], [2, 3, 1, 0], keys_of(40, 3, 30))),
}
MODES = {"": {}, "_ordered": {"KOLIBRIE_ORDERED": "1"}}


@pytest.fixture
def make_ctx(monkeypatch):
    """a fresh context, created after the route switches are set (they are read when a context is created)"""
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


def fingerprint(cx, call):
    a = cx.get_stats()
    out = call()
    b = cx.get_stats()
    return out, {f: b[f] - a[f] for f in FIELDS if b[f] != a[f]}


def twice(cx, name, call, check):
    fps = []
    for rep in range(2):
        out, fp = fingerprint(cx, call)
        check(out, f"{name} call {rep + 1}")
        fps.append(fp)
    assert fps == ROUTES.get(name), f"{name}: {fps!r}"


def same_bag(want_rows, want_slots):
    def check(got, what):
        assert sorted(got.slots) == sorted(want_slots), what
        H.assert_same_bag(got.to_numpy(sorted(want_slots)), want_rows, what)
    return check


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("case", list(HASH_CASES))
def test_hash_join_route(make_ctx, case, mode):
    env, sides = HASH_CASES[case]
    cx = make_ctx(**env, **MODES[mode])
    (ls, lc), (rs, rc) = sides()
    want = O.hash_join(O.rel_from_host(ls, lc), O.rel_from_host(rs, rc))
    want_slots = sorted(want.slots)
    left, right = cx.rel_from_host(ls, lc), cx.rel_from_host(rs, rc)

    def check(got, what):
        assert got.slots == ls + [s for s in rs if s not in ls], what  # left columns, then the right side's new ones
        same_bag(want.to_numpy(want_slots), want_slots)(got, what)

    twice(cx, case + mode, lambda: cx.hash_join(left, right), check)


def multivalued():
    """1:N predicates 100..102 over 600 subjects"""
    g = rng(3)
    n = 4000
    return np.unique(np.stack([g.integers(0, 600, n), g.integers(100, 103, n), g.integers(1000, 1040, n)], axis=1).astype(np.uint32), axis=0)


@pytest.mark.parametrize("mode", list(MODES))
def test_star_join_post_filter_route(make_ctx, mode):
    """a conjunct over two patterns' variables is evaluated by the last chained join of the star join's chained route"""
    cx = make_ctx(**MODES[mode])
    tr = multivalued()
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    db = O.Db(tr[:, 0], tr[:, 1], tr[:, 2])
    pats = [c.pattern(c.V(0), c.K(100), c.V(1)), c.pattern(c.V(0), c.K(101), c.V(2))]
    filt = [c.fop(c.F_EQ_ID, slot=1, id=1003), c.fop(c.F_EQ_ID, slot=2, id=1017), c.fop(c.F_OR)]
    want = db.bgp(pats, filt)
    twice(cx, "star_post_filter" + mode, lambda: cx.star_join(0, pats, filt), same_bag(want.to_numpy(sorted(want.slots)), want.slots))


def functional_store():
    """P100 maps 3 000 dense subjects to one object each (its subject column has a persistent table); P101 is 1:N"""
    g = rng(21)
    subj = np.arange(100, 3100)
    p100 = np.stack([subj, np.full(3000, 100), 5000 + g.integers(0, 400, 3000)], axis=1)
    p101 = np.stack([g.integers(100, 3100, 4000), np.full(4000, 101), 6000 + g.integers(0, 50, 4000)], axis=1)
    return u32(np.concatenate([p100, p101]))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("route", ["index", "scan"])
def test_bind_join_route(make_ctx, route, mode):
    cx = make_ctx(**MODES[mode])
    tr = functional_store()
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    if route == "index":
        cx.build_index()
    db = O.Db(tr[:, 0], tr[:, 1], tr[:, 2])
    g = rng(22)
    lc = [u32(g.integers(0, 4000, 30000)), u32(g.integers(0, 100, 30000))]  # subjects (a quarter unknown to P100), a payload
    pat = c.pattern(c.V(0), c.K(100), c.V(1))
    want = O.hash_join(O.rel_from_host([0, 5], lc), db.scan(pat))
    left = cx.rel_from_host([0, 5], lc)
    twice(cx, f"bind_{route}{mode}", lambda: cx.bind_join(left, pat), same_bag(want.to_numpy(sorted(want.slots)), want.slots))


@pytest.mark.parametrize("mode", list(MODES))
def test_filter_route(make_ctx, mode):
    cx = make_ctx(**MODES[mode])
    g = rng(31)
    cols = [u32(g.integers(0, 10, 50000)), u32(g.integers(0, 1000, 50000))]
    rel = cx.rel_from_host([1, 2], cols)
    prog = [c.fop(c.F_NE_ID, slot=1, id=3), c.fop(c.F_EQ_ID, slot=2, id=7), c.fop(c.F_OR)]
    keep = (cols[0] != 3) | (cols[1] == 7)
    want = np.stack([cols[0][keep], cols[1][keep]], axis=1)
    twice(cx, "filter" + mode, lambda: cx.filter(rel, prog), same_bag(want, [1, 2]))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("index", [True, False])
def test_scan_quoted_route(make_ctx, index, mode):
    """<< ?1 P200 ?2 >> P300 ?3: the match pass gives (entry, ?1, ?2), the bind join adds ?3"""
    cx = make_ctx(**MODES[mode])
    g = rng(41)
    n = 5000
    ids = u32(0x80000000 + np.arange(n))
    qp_ = u32(np.where(g.random(n) < 0.7, 200, 201))
    qs, qo = u32(g.integers(0, 500, n)), u32(g.integers(0, 500, n))
    cx.quoted_load(ids, qs, qp_, qo)
    annotated = g.random(n) < 0.8  # entries that are the subject of a P300 triple
    s3 = ids[annotated]
    o3 = u32(9000 + g.integers(0, 30, len(s3)))
    cx.store_load(s3, u32(np.full(len(s3), 300)), o3)
    if index:
        cx.build_index()
    else:
        cx.set_use_index(False)
    inner = c.pattern(c.V(1), c.K(200), c.V(2))
    qpat = c.KbQuotedPattern(c.pattern(c.KbTerm(c.KB_TERM_QUOTED, 0), c.K(300), c.V(3)), inner, c.pattern(c.V(0), c.V(0), c.V(0)))
    hit = annotated & (qp_ == 200)
    want = np.stack([qs[hit], qo[hit], o3[hit[annotated]]], axis=1)
    twice(cx, f"quoted_{'index' if index else 'scan'}{mode}", lambda: cx.scan_quoted(qpat), same_bag(want, [1, 2, 3]))


def nat_side(g, n, slots, unbound):
    a = g.integers(0, 40, (n, len(slots))).astype(np.uint32)
    for j, s in enumerate(slots):
        if s in unbound:
            a[g.random(n) < 0.3, j] = NONE
    return a


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("unbound", [False, True])
def test_natural_join_route(make_ctx, unbound, mode):
    cx = make_ctx(**MODES[mode])
    g = rng(51 + unbound)
    ls, rs = [10, 11, 20], [30, 11, 10]
    la = nat_side(g, 600, ls, {10} if unbound else set())
    ra = nat_side(g, 400, rs, {11} if unbound else set())
    left = cx.rel_from_host(ls, [u32(la[:, j]) for j in range(3)])
    right = cx.rel_from_host(rs, [u32(ra[:, j]) for j in range(3)])
    ref = J.natural_join([{s: v for s, v in zip(ls, r) if v != NONE} for r in la.tolist()],
                         [{s: v for s, v in zip(rs, r) if v != NONE} for r in ra.tolist()])
    out_slots = [10, 11, 20, 30]
    want = np.array([[r.get(s, NONE) for s in out_slots] for r in ref], dtype=np.uint32).reshape(-1, 4)

    def check(got, what):
        assert got.slots == ls + [30], what
        H.assert_same_bag(got.to_numpy(out_slots), want, what)

    twice(cx, f"natjoin_{'unbound' if unbound else 'fast'}{mode}", lambda: cx.natural_join(left, right), check)
