"""GPU (-m gpu): which route kb_scan takes for each pattern shape, pinned by what it costs.

Every case runs its call twice on a context of its own and checks, for each call, the result against a numpy brute force over the
triples and the *fingerprint* against a literal: the change of every integer counter of kb_stats across the call (launches per family,
kernel launches, rows scanned, bytes copied, index joins). d2h_bytes counts whole control-arena reads and the index's key lookups, so it
also pins the number of host synchronisations. Counters that did not move are left out of the literals. Every case runs in unordered
and in ordered mode (KOLIBRIE_ORDERED=1: output in store order, the look-back prefix with ping-pong totals across launches).

The routes:
  fused scan        1..8 patterns in one pass over the store (9 is refused): constants in any position, a variable repeated within a
                    pattern (quirk Q4), a pushed-down FILTER; a store of more than 16 segments takes a launch per 16
  index lookup      with a valid index, a pattern with a constant predicate is answered from the predicate's slice: (?s P ?o) is the
                    slice (one unpair per chunk), (c P ?o) one slot of a unique subject table (a key of another shard: no lookup at
                    all), (?s P c) the key's run in a directory (a view when the run starts 16-byte aligned, else a copy), an absent
                    predicate nothing; two constants and ?x P ?x fall back to the scan, a pushdown is applied to the looked-up rows,
                    and a call mixing both shapes scans only what the index cannot answer. KOLIBRIE_USE_INDEX=0 scans everything.
"""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import helpers as H

pytestmark = pytest.mark.gpu

FIELDS = ("scan_launches", "build_launches", "probe_launches", "filter_launches", "group_launches", "other_launches", "kernel_launches",
          "rows_scanned", "rows_built", "rows_probed", "h2d_bytes", "d2h_bytes", "fused_scan_builds", "index_joins")
# switches that select routes: pinned to their defaults, so that the literals hold whatever the caller's environment says
DEFAULT_ENV = {"KOLIBRIE_ORDERED": "0", "KOLIBRIE_USE_INDEX": "1", "KOLIBRIE_INDEX_MAINTAIN": "1"}
MODES = {"": {}, "_ordered": {"KOLIBRIE_ORDERED": "1"}}

# name -> fingerprints of the first and the second call (recorded on an H100)
ROUTES = {
    "k1": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "k1_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "constants": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "constants_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "k8": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "k8_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "repeated": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "repeated_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "pushdown": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "pushdown_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "k9": [{}] * 2,
    "k9_ordered": [{}] * 2,
    "idx_all": [{"scan_launches": 1, "kernel_launches": 1, "index_joins": 1}] * 2,
    "idx_all_ordered": [{"scan_launches": 1, "kernel_launches": 1, "index_joins": 1}] * 2,
    "idx_all_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_all_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_unique_hit": [{"d2h_bytes": 4, "index_joins": 1}] * 2,
    "idx_unique_hit_ordered": [{"d2h_bytes": 4, "index_joins": 1}] * 2,
    "idx_unique_hit_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_unique_hit_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_unique_miss": [{"d2h_bytes": 4, "index_joins": 1}] * 2,
    "idx_unique_miss_ordered": [{"d2h_bytes": 4, "index_joins": 1}] * 2,
    "idx_unique_miss_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_unique_miss_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_dir_view": [{"d2h_bytes": 8, "index_joins": 1}] * 2,
    "idx_dir_view_ordered": [{"d2h_bytes": 8, "index_joins": 1}] * 2,
    "idx_dir_view_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_dir_view_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_dir_copy": [{"d2h_bytes": 8, "index_joins": 1}] * 2,
    "idx_dir_copy_ordered": [{"d2h_bytes": 8, "index_joins": 1}] * 2,
    "idx_dir_copy_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_dir_copy_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_absent_predicate": [{}] * 2,
    "idx_absent_predicate_ordered": [{}] * 2,
    "idx_absent_predicate_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_absent_predicate_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_two_constants": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_two_constants_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_two_constants_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_two_constants_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_same_variable": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_same_variable_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_same_variable_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_same_variable_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_pushdown": [{"scan_launches": 1, "filter_launches": 1, "kernel_launches": 2, "d2h_bytes": 32768, "index_joins": 1}] * 2,
    "idx_pushdown_ordered": [{"scan_launches": 1, "filter_launches": 1, "kernel_launches": 2, "d2h_bytes": 32768, "index_joins": 1}] * 2,
    "idx_pushdown_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_pushdown_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_mixed": [{"scan_launches": 2, "kernel_launches": 2, "rows_scanned": 7600, "d2h_bytes": 32772, "index_joins": 2}] * 2,
    "idx_mixed_ordered": [{"scan_launches": 2, "kernel_launches": 2, "rows_scanned": 7600, "d2h_bytes": 32772, "index_joins": 2}] * 2,
    "idx_mixed_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_mixed_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "idx_chunks": [{"scan_launches": 2, "kernel_launches": 3, "index_joins": 2}] * 2,
    "idx_chunks_ordered": [{"scan_launches": 2, "kernel_launches": 3, "index_joins": 2}] * 2,
    "idx_chunks_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 8600, "d2h_bytes": 32768}] * 2,
    "idx_chunks_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 8600, "d2h_bytes": 32768}] * 2,
    "idx_shard_hit": [{"d2h_bytes": 4, "index_joins": 1}] * 2,
    "idx_shard_hit_ordered": [{"d2h_bytes": 4, "index_joins": 1}] * 2,
    "idx_shard_hit_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 3000, "d2h_bytes": 32768}] * 2,
    "idx_shard_hit_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 3000, "d2h_bytes": 32768}] * 2,
    "idx_shard_other_shard": [{}] * 2,
    "idx_shard_other_shard_ordered": [{}] * 2,
    "idx_shard_other_shard_off": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 3000, "d2h_bytes": 32768}] * 2,
    "idx_shard_other_shard_off_ordered": [{"scan_launches": 1, "kernel_launches": 1, "rows_scanned": 3000, "d2h_bytes": 32768}] * 2,
    "many_segments": [{"scan_launches": 2, "kernel_launches": 2, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
    "many_segments_ordered": [{"scan_launches": 2, "kernel_launches": 2, "rows_scanned": 7600, "d2h_bytes": 32768}] * 2,
}


def u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def base_store():
    """P100: 3 000 even subjects, one object each (a unique subject table; the objects 7000..7399 get a directory).
    P101: 1:N over 600 subjects. Then 600 triples over ids 0..7, where subject, predicate and object often coincide."""
    g = np.random.default_rng(11)
    p100 = np.stack([2 * np.arange(3000), np.full(3000, 100), 7000 + g.integers(0, 400, 3000)], axis=1)
    p101 = np.stack([g.integers(0, 600, 4000), np.full(4000, 101), g.integers(1000, 1040, 4000)], axis=1)
    small = g.integers(0, 8, (600, 3))
    return u32(np.concatenate([p100, p101, small]))


def sharded_store(rank, world):
    """P100 over 3 000 subjects of shard `rank` of `world`, one object each"""
    subj = [x for x in range(20000) if c.lib().kb_shard_of(x, world) == rank][:3000]
    g = np.random.default_rng(12)
    return u32(np.stack([subj, np.full(3000, 100), 7000 + g.integers(0, 400, 3000)], axis=1))


def other_shard_key(rank, world):
    return next(k for k in range(1, 20000, 97) if c.lib().kb_shard_of(k, world) != rank)


def directory_keys(tr):
    """objects of P100 whose run in the object directory (a counting sort by object) starts 16-byte aligned, and one whose does not"""
    o = np.sort(tr[tr[:, 1] == 100, 2])
    keys, first = np.unique(o, return_index=True)
    aligned = keys[(first % 4 == 0) & (first > 0)]
    unaligned = keys[first % 4 != 0]
    return int(aligned[0]), int(unaligned[0])


def brute(tr, pat, keep=None):
    """slots and rows of one pattern over the triples: constants select, a repeated variable is an equality (quirk Q4), columns come
    out in the order of each variable's first appearance (s, p, o); keep: the pushed-down FILTER over {slot: column}"""
    m = np.ones(len(tr), dtype=bool)
    first = {}
    for i, t in enumerate((pat.s, pat.p, pat.o)):
        if not t.is_var:
            m &= tr[:, i] == t.value
        elif t.value in first:
            m &= tr[:, i] == tr[:, first[t.value]]
        else:
            first[t.value] = i
    cols = {v: tr[m, i] for v, i in first.items()}
    n = int(m.sum())
    if keep is not None:
        k = keep(cols)
        cols = {v: col[k] for v, col in cols.items()}
        n = int(k.sum())
    slots = list(first)
    return slots, n, np.stack([cols[s] for s in slots], axis=1) if slots else None


def P(s, p, o):
    return c.pattern(s, p, o)


V, K = c.V, c.K
# a pushed-down FILTER(?1 != 1003 || ?0 = 17) and its numpy form
PUSH_OPS = [c.fop(c.F_NE_ID, slot=1, id=1003), c.fop(c.F_EQ_ID, slot=0, id=17), c.fop(c.F_OR)]


def push_keep(cols):
    return (cols[1] != 1003) | (cols[0] == 17)


# name -> (patterns, pushdown per pattern (None: no FILTER) with its numpy form) over base_store; scanned without an index
SCAN_CASES = {
    "k1": lambda tr: ([P(V(0), K(101), V(1))], None),
    "constants": lambda tr: ([P(K(24), V(1), V(2)), P(V(0), K(101), V(2)), P(V(0), V(1), K(1005))], None),
    "k8": lambda tr: ([P(V(0), K(100), V(1)), P(V(0), K(101), V(2)), P(V(3), V(4), K(7003)), P(K(40), V(1), V(5)),
                       P(V(0), V(1), V(2)), P(V(0), K(3), V(1)), P(K(5), V(1), K(1)), P(V(0), K(102), V(1))], None),
    "repeated": lambda tr: ([P(V(0), V(0), V(1)), P(V(0), V(1), V(0)), P(V(1), V(0), V(0)), P(V(0), V(0), V(0))], None),
    "pushdown": lambda tr: ([P(V(0), K(101), V(1)), P(V(0), K(100), V(1))], [(PUSH_OPS, push_keep), None]),
}
# the same over base_store with the index built (cases named idx_*); KOLIBRIE_USE_INDEX=0 runs them through the scan
INDEX_CASES = {
    "all": lambda tr: ([P(V(0), K(100), V(1))], None),
    "unique_hit": lambda tr: ([P(K(24), K(100), V(1))], None),
    "unique_miss": lambda tr: ([P(K(25), K(100), V(1))], None),
    "dir_view": lambda tr: ([P(V(0), K(100), K(directory_keys(tr)[0]))], None),
    "dir_copy": lambda tr: ([P(V(0), K(100), K(directory_keys(tr)[1]))], None),
    "absent_predicate": lambda tr: ([P(V(0), K(555), V(1))], None),
    "two_constants": lambda tr: ([P(K(24), K(100), K(int(tr[12, 2])))], None),
    "same_variable": lambda tr: ([P(V(0), K(3), V(0))], None),
    "pushdown": lambda tr: ([P(V(0), K(101), V(1))], [(PUSH_OPS, push_keep)]),
    "mixed": lambda tr: ([P(V(0), K(100), V(1)), P(V(0), V(2), K(1005)), P(K(24), K(100), V(3)), P(V(0), K(3), V(0))], None),
}


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


def run_scan(cx, name, tr, pats, pushdown):
    """kb_scan twice; each call's relations against the brute force, the two fingerprints against ROUTES[name]"""
    ops = [pd[0] if pd else None for pd in pushdown] if pushdown else None
    keeps = [pd[1] if pd else None for pd in pushdown] if pushdown else [None] * len(pats)
    wants = [brute(tr, p, k) for p, k in zip(pats, keeps)]
    fps = []
    for rep in range(2):
        got, fp = fingerprint(cx, lambda: cx.scan(pats, ops))
        for k, (rel, (slots, n, rows)) in enumerate(zip(got, wants)):
            what = f"{name} call {rep + 1} pattern {k}"
            assert rel.slots == slots, what
            assert rel.n_rows == n, what
            if slots:
                H.assert_same_bag(rel.to_numpy(slots), rows, what)
        fps.append(fp)
    assert fps == ROUTES.get(name), f"{name}: {fps!r}"


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("case", list(SCAN_CASES))
def test_scan_route(make_ctx, case, mode):
    cx = make_ctx(**MODES[mode])
    tr = base_store()
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    run_scan(cx, case + mode, tr, *SCAN_CASES[case](tr))


@pytest.mark.parametrize("mode", list(MODES))
def test_scan_nine_patterns_refused(make_ctx, mode):
    cx = make_ctx(**MODES[mode])
    tr = base_store()
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    fps = []
    for _ in range(2):
        def call():
            with pytest.raises(c.KolibrieError) as e:
                cx.scan([P(V(0), K(101), V(1))] * 9)
            return e.value.status
        status, fp = fingerprint(cx, call)
        assert status == c.KB_E_LIMIT
        fps.append(fp)
    assert fps == ROUTES.get("k9" + mode), f"k9{mode}: {fps!r}"


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("use_index", ["1", "0"], ids=["index", "no_index"])
@pytest.mark.parametrize("case", list(INDEX_CASES))
def test_index_route(make_ctx, case, use_index, mode):
    cx = make_ctx(KOLIBRIE_USE_INDEX=use_index, **MODES[mode])
    tr = base_store()
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    cx.build_index()
    name = f"idx_{case}" + ("" if use_index == "1" else "_off") + mode
    run_scan(cx, name, tr, *INDEX_CASES[case](tr))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("use_index", ["1", "0"], ids=["index", "no_index"])
def test_index_route_chunks(make_ctx, use_index, mode):
    """(?s P ?o) over a slice of two chunks: the store is indexed, then a segment with more P100 rows arrives (index maintained)"""
    cx = make_ctx(KOLIBRIE_USE_INDEX=use_index, **MODES[mode])
    tr = base_store()
    cx.store_append(tr[:, 0], tr[:, 1], tr[:, 2], 0)
    cx.build_index()
    more = u32(np.stack([2 * np.arange(1000) + 1, np.full(1000, 100), 7000 + np.arange(1000) % 400], axis=1))
    cx.store_append(more[:, 0], more[:, 1], more[:, 2], 1)
    name = "idx_chunks" + ("" if use_index == "1" else "_off") + mode
    run_scan(cx, name, np.concatenate([tr, more]), [P(V(0), K(100), V(1)), P(V(0), K(101), V(1))], None)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("use_index", ["1", "0"], ids=["index", "no_index"])
@pytest.mark.parametrize("key", ["hit", "other_shard"])
def test_index_route_sharded(make_ctx, key, use_index, mode):
    """(c P ?o) on the unique subject table of rank 0's shard of a 2-way subject-sharded store: a key of this shard is one table slot;
    a key of the other shard is not in this store and needs no lookup"""
    cx = make_ctx(KOLIBRIE_USE_INDEX=use_index, **MODES[mode])
    cx.set_sharding(0, 2)
    tr = sharded_store(0, 2)
    cx.store_load(tr[:, 0], tr[:, 1], tr[:, 2])
    cx.build_index()
    k = int(tr[77, 0]) if key == "hit" else other_shard_key(0, 2)
    name = f"idx_shard_{key}" + ("" if use_index == "1" else "_off") + mode
    run_scan(cx, name, tr, [P(K(k), K(100), V(1))], None)


@pytest.mark.parametrize("mode", list(MODES))
def test_scan_many_segments(make_ctx, mode):
    """24 segments, every fourth empty: 18 non-empty ones take two launches (16 + 2); ordered mode carries the totals across them"""
    cx = make_ctx(**MODES[mode])
    tr = base_store()
    parts = np.array_split(tr, 18)
    held = []
    for t in range(24):
        part = tr[:0] if t % 4 == 3 else parts.pop()
        cx.store_append(part[:, 0], part[:, 1], part[:, 2], t)
        held.append(part)
    assert not parts
    run_scan(cx, "many_segments" + mode, np.concatenate(held), [P(V(0), K(101), V(1)), P(V(0), V(1), K(1005))], None)
