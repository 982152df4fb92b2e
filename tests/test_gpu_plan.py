"""GPU (-m gpu): prepared star joins (kb_star_join_prepare / kb_plan_submit / kb_plan_collect) and the cross-rank GROUP BY merge
(kb_groups_pack / kb_groups_merge) against the oracle and against the synchronous operators they shadow."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import agg_reference as AR
from tests import helpers as H
from tests import oracle_api as O

pytestmark = pytest.mark.gpu

_EMP = {}


@pytest.fixture
def emp(ctx):
    if "d" not in _EMP:
        _EMP["d"] = datagen.employee_dataset(20000)
    d = _EMP["d"]
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    return d, O.Db(d.s, d.p, d.o, d.num_or0, d.is_num)


def table(x):
    keys = np.stack(x["keys"], axis=1)
    order = np.lexsort(tuple(keys[:, k] for k in range(keys.shape[1] - 1, -1, -1)))
    return keys[order], x["counts"][order], [v[order] for v in x["values"]]


@pytest.mark.parametrize("q", ["cfg1", "cfg2", "cfg3", "star3"])
def test_prepared_rows_equal_oracle_and_sync_path(ctx, emp, q):
    d, db = emp
    js, pats, filt = datagen.employee_queries(d)[q]
    want = db.bgp(pats, filt)
    want_rows = want.to_numpy(sorted(want.slots))
    plan = ctx.prepare_star_join(js, pats, filt, ring=3)
    assert plan.ring == 3 and not plan.grouped and sorted(plan.slots) == sorted(want.slots)
    launches0 = ctx.get_stats()["kernel_launches"]
    # 7 queries through a ring of 3: the host stays two launches ahead of the collect
    tickets, seen = [], 0
    for i in range(7):
        tickets.append(plan.submit())
        if len(tickets) == plan.ring:
            r = plan.collect_rows(tickets.pop(0))
            H.assert_same_bag(r.to_numpy(sorted(r.slots)), want_rows, f"{q} ticket {i}")
            r.free()
            seen += 1
    while tickets:
        assert plan.collect(tickets.pop(0)) == len(want_rows)
        seen += 1
    assert seen == 7
    assert ctx.get_stats()["kernel_launches"] - launches0 == 7, "one kernel per prepared query"
    # the synchronous operator gives the same bag
    got = ctx.star_join(js, pats, filt)
    H.assert_same_bag(got.to_numpy(sorted(got.slots)), want_rows, q)
    plan.free()


def test_prepared_group_by_equals_oracle(ctx, emp):
    d, db = emp
    js, pats, _ = datagen.employee_queries(d)["cfg3"]
    _, pats2, filt2 = datagen.employee_queries(d)["cfg2"]
    for pp, ff, gslot, aggs in [(pats, None, 1, [(c.AGG_COUNT, 0)]), (pats, None, 1, [(c.AGG_AVG, 2)]), (pats2, filt2, 1, [(c.AGG_SUM, 2)]),
                                (pats2, filt2, 1, [(c.AGG_MIN, 2)]), (pats, None, 1, [(c.AGG_MAX, 2)]), (pats, None, 1, [])]:
        plan = ctx.prepare_star_join(js, pp, ff, group_slots=[gslot], aggs=aggs, ring=2)
        assert plan.grouped
        orel = db.bgp(pp, ff)
        w = db.group(orel, [gslot], aggs)
        osl = sorted(orel.slots)
        orows = orel.to_numpy(osl)
        for rep in range(3):
            t = plan.submit()
            g, n_rows = plan.collect_groups(t)
            assert n_rows == orel.n_rows
            gk, gc, _ = table(g)
            wk, wc, _ = table(w)
            assert np.array_equal(gk, wk) and np.array_equal(gc, wc)
            AR.assert_groups_match_slots(g, orows, osl, d.num_or0, [gslot], aggs, f"{aggs} rep {rep}")
        plan.free()
    # a GROUP BY with thousands of groups does not fit the plan's fixed table: reported at collect, not silently truncated
    plan = ctx.prepare_star_join(js, pats, None, group_slots=[2], aggs=[(c.AGG_COUNT, 0)], ring=1)
    t = plan.submit()
    with pytest.raises(c.KolibrieError) as e:
        plan.collect_groups(t)
    assert e.value.status == c.KB_E_LIMIT
    plan.free()


def test_plan_errors(ctx, emp):
    d, db = emp
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    plan = ctx.prepare_star_join(js, pats, filt, ring=2)
    t1, t2 = plan.submit(), plan.submit()
    with pytest.raises(c.KolibrieError) as e:  # ring of 2, both slots in flight
        plan.submit()
    assert e.value.status == c.KB_E_LIMIT
    n = plan.collect(t1)
    assert n == plan.collect(t2)
    with pytest.raises(c.KolibrieError) as e:  # collected twice
        plan.collect(t1)
    assert e.value.status == c.KB_E_NOT_FOUND
    # any store mutation makes the plan stale (its slices and tables describe the old store)
    ctx.store_append(d.s[:6], d.p[:6], d.o[:6], tag=5)
    with pytest.raises(c.KolibrieError) as e:
        plan.submit()
    assert e.value.status == c.KB_E_INVALID and "stale" in e.value.message
    plan.free()
    # without an index, or for a shape the one-kernel path does not take, prepare says so
    with pytest.raises(c.KolibrieError) as e:
        ctx.prepare_star_join(js, pats, filt)
    assert e.value.status == c.KB_E_UNSUPPORTED
    ctx.build_index()
    bound = [c.pattern(c.V(0), c.K(d.ids["foaf:title"]), c.K(d.ids["Manager"])), pats[1]]
    with pytest.raises(c.KolibrieError) as e:
        ctx.prepare_star_join(js, bound, None)
    assert e.value.status == c.KB_E_UNSUPPORTED


@pytest.mark.parametrize("n_parts", [2, 3, 8])
def test_groups_merge_of_shard_partials_equals_global_group_by(ctx, n_parts):
    """what N ranks do: every shard (kb_shard_of(subject)) aggregates locally, the packed partials are merged on the device; the
    result must be the GROUP BY of the unsharded store (oracle), for every aggregate kind, few and many groups"""
    d = datagen.employee_dataset(30000)
    db = O.Db(d.s, d.p, d.o, d.num_or0, d.is_num)
    js, pats, _ = datagen.employee_queries(d)["cfg3"]
    orel = db.bgp(pats)
    owner = datagen.shard_of_np(d.s, n_parts)
    cases = [([1], [(c.AGG_COUNT, 0)]), ([1], [(c.AGG_AVG, 2)]), ([1], [(c.AGG_SUM, 2)]), ([1], [(c.AGG_MIN, 2)]), ([1], [(c.AGG_MAX, 2)]),
             ([2], [(c.AGG_COUNT, 0)]), ([1, 2], [(c.AGG_COUNT, 0), (c.AGG_AVG, 2), (c.AGG_MAX, 2)])]
    parts = {i: [] for i in range(len(cases))}
    rows = 0
    for r in range(n_parts):
        keep = owner == r
        ctx.store_load(d.s[keep], d.p[keep], d.o[keep])
        ctx.dict_numeric_load(d.num_or0, d.is_num)
        ctx.build_index()
        for i, (gs, aggs) in enumerate(cases):
            packed, n_rows = ctx.star_join_aggregate_packed(js, pats, None, gs, aggs)
            parts[i].append(packed)
            if i == 0:
                rows += n_rows
    assert rows == orel.n_rows
    osl = sorted(orel.slots)
    orows = orel.to_numpy(osl)
    for i, (gs, aggs) in enumerate(cases):
        g = ctx.groups_merge(parts[i])
        w = db.group(orel, gs, aggs)
        gk, gc, _ = table(g)
        wk, wc, _ = table(w)
        assert np.array_equal(gk, wk) and np.array_equal(gc, wc), (gs, aggs)
        AR.assert_groups_match_slots(g, orows, osl, d.num_or0, gs, aggs, f"{gs} {aggs}")
    # merging a single partial is the identity; garbage is rejected
    g1 = ctx.groups_merge([parts[0][0]])
    assert int(g1["counts"].sum()) > 0
    with pytest.raises(c.KolibrieError):
        ctx.groups_merge([np.zeros(64, dtype=np.uint8)])
    with pytest.raises(c.KolibrieError):  # partials of different GROUP BYs
        ctx.groups_merge([parts[0][0], parts[1][0]])


@pytest.mark.parametrize("n_parts,n_cols,n", [(2, 2, 100_003), (8, 2, 1_000_000), (5, 3, 70_001), (64, 1, 300_000), (3, 9, 20_000), (8, 2, 0), (8, 2, 17)])
def test_shuffle_kernel_single_gpu(ctx, n_parts, n_cols, n):
    """the fused partition+transfer kernel with every 'peer' buffer on this GPU: both reservation modes (precomputed ranges =
    kb_shuffle_scatter, receiver-owned cursors = kb_shuffle_push) must deliver to destination d exactly the rows whose key maps to d"""
    import torch

    rng = np.random.default_rng(n_parts * 1000 + n_cols)
    cols = [rng.integers(0, 1 << 22, n).astype(np.uint32) for _ in range(n_cols)]
    slots = list(range(10, 10 + n_cols))
    key_col = n_cols - 1
    rel = ctx.rel_from_host(slots, cols) if n else ctx.rel_from_host(slots, [np.empty(0, np.uint32)] * n_cols)
    dest = datagen.shard_of_np(cols[key_col], n_parts) if n else np.empty(0, np.int64)
    counts = np.bincount(dest, minlength=n_parts)
    assert ctx.partition_counts(rel, slots[key_col], n_parts) == [int(x) for x in counts]
    cap = int(counts.max(initial=0)) + 64
    dev = torch.device("cuda", ctx.device)
    full = np.stack(cols, axis=1) if n else np.empty((0, n_cols), np.uint32)
    for mode in ("planned", "push"):
        bufs = torch.full((n_parts, n_cols, cap), -1, dtype=torch.int32, device=dev)
        cursors = torch.zeros(n_parts, 64, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        peer_cols = [bufs[d_, c_].data_ptr() for d_ in range(n_parts) for c_ in range(n_cols)]
        if mode == "planned":
            ctx.shuffle_scatter(rel, slots[key_col], n_parts, peer_cols, [0] * n_parts, cap)
            got_counts = counts
        else:
            ctx.shuffle_push(rel, slots[key_col], n_parts, peer_cols, [cursors[d_].data_ptr() for d_ in range(n_parts)], cap)
            got_counts = cursors[:, 0].cpu().numpy()
            assert np.array_equal(got_counts, counts)
        host = bufs.cpu().numpy().astype(np.uint32)
        for d_ in range(n_parts):
            m = int(got_counts[d_])
            got = host[d_, :, :m].T
            H.assert_same_bag(got, full[dest == d_], f"{mode} destination {d_}")
            assert (host[d_, :, m:] == 0xFFFFFFFF).all(), "nothing written past the reserved range"
    # a receive buffer that is too small is reported, not overrun
    if n > 1000:
        small = torch.zeros((n_parts, n_cols, 8), dtype=torch.int32, device=dev)
        cursors = torch.zeros(n_parts, 64, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        with pytest.raises(c.KolibrieError) as e:
            ctx.shuffle_push(rel, slots[key_col], n_parts, [small[d_, c_].data_ptr() for d_ in range(n_parts) for c_ in range(n_cols)],
                             [cursors[d_].data_ptr() for d_ in range(n_parts)], 8)
        assert e.value.status == c.KB_E_LIMIT
    # the wrapped (zero-copy) relation over caller-owned columns behaves like an owned one
    if n:
        t = [torch.from_numpy(x.astype(np.int32)).to(dev) for x in cols]
        pad = [torch.cat([x, torch.zeros(64, dtype=torch.int32, device=dev)]) for x in t]
        torch.cuda.synchronize()
        w = ctx.rel_wrap_device(slots, [x.data_ptr() for x in pad], n)
        H.assert_same_bag(w.to_numpy(slots), full, "wrapped relation")
        w.free()
    rel.free()


def test_peer_merged_group_plan_world_of_one(ctx):
    """kb_plan_attach_peers with a world of one rank (its own scratch is its only peer): submit runs join+group -> barrier -> merge
    kernel -> compaction, and collect returns the same groups as the oracle. The two-and-more-rank protocol needs one process per GPU
    (two spinning kernels of one process may share a hardware queue): scripts/dist_group_check.py under torchrun, and bench.py's cfg3
    leg, assert it against the oracle / the closed form at N >= 2."""
    import torch

    d = datagen.employee_dataset(30000)
    db = O.Db(d.s, d.p, d.o, d.num_or0, d.is_num)
    js, pats, _ = datagen.employee_queries(d)["cfg3"]
    orel = db.bgp(pats)
    osl = sorted(orel.slots)
    orows = orel.to_numpy(osl)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    dev = torch.device("cuda", ctx.device)
    for aggs in ([(c.AGG_COUNT, 0)], [(c.AGG_AVG, 2)], [(c.AGG_MIN, 2)], [(c.AGG_MAX, 2)], [(c.AGG_SUM, 2)], []):
        plan = ctx.prepare_star_join(js, pats, None, group_slots=[1], aggs=aggs, ring=2)
        nbytes = plan.peer_scratch_bytes()
        assert nbytes > 0
        scratch = torch.zeros((nbytes + 3) // 4, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        plan.attach_peers(0, 1, [scratch.data_ptr()], keep=scratch)
        w = db.group(orel, [1], aggs)
        wk, wc, _ = table(w)
        tickets = []
        for rep in range(5):  # more queries than ring slots: the slots and the barrier epochs are reused
            tickets.append(plan.submit())
            if len(tickets) == 2:
                g, n_rows = plan.collect_groups(tickets.pop(0))
                assert n_rows == orel.n_rows
                gk, gc, _ = table(g)
                assert np.array_equal(gk, wk) and np.array_equal(gc, wc), (aggs, rep)
                AR.assert_groups_match_slots(g, orows, osl, d.num_or0, [1], aggs, f"{aggs} rep {rep}")
        plan.collect_groups(tickets.pop(0))
        plan.free()
    # a row plan has nothing to merge; a ring of one cannot be attached
    p1 = ctx.prepare_star_join(js, pats, None, ring=2)
    with pytest.raises(c.KolibrieError):
        p1.attach_peers(0, 1, [scratch.data_ptr()])
    p1.free()
    p2 = ctx.prepare_star_join(js, pats, None, group_slots=[1], aggs=[(c.AGG_COUNT, 0)], ring=1)
    with pytest.raises(c.KolibrieError):
        p2.attach_peers(0, 1, [scratch.data_ptr()])
    p2.free()


def test_bind_join_vs_oracle(ctx):
    """kb_bind_join (engine.rs:840-885): a relation joined with one store pattern — through the index's persistent tables when they
    exist (subject-bound and object-bound lookups), through scan + hash join otherwise; always the oracle's natural join"""
    d = datagen.employee_dataset(20000)
    db = O.Db(d.s, d.p, d.o, d.num_or0, d.is_num)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    rng = np.random.default_rng(5)
    subj = d.s[0::6]
    e_col = np.concatenate([rng.choice(subj, 30000), np.array([0xFFFFFF0, 3], dtype=np.uint32)]).astype(np.uint32)  # duplicates + keys that match nothing
    tag = rng.integers(0, 1000, len(e_col)).astype(np.uint32)
    E, T, X, N = 0, 1, 7, 3
    title_p, name_p, sal_p = (c.pattern(c.V(E), c.K(d.ids[k]), c.V(v)) for k, v in (("foaf:title", T), ("foaf:name", N), ("ds:annual_salary", 2)))
    cases = [("subject-bound, unique dense column", title_p, E), ("object-bound (name object = employee id, unique)", c.pattern(c.V(9), c.K(d.ids["foaf:name"]), c.V(E)), E),
             ("bound through the object of a multi-valued column", c.pattern(c.V(9), c.K(d.ids["foaf:title"]), c.V(E)), E)]
    for indexed in (False, True):
        if indexed:
            ctx.build_index()
        for what, pat, key in cases:
            col = e_col if "multi" not in what else np.array([d.ids["Manager"], d.ids["Developer"], 5], dtype=np.uint32)
            tg = tag[: len(col)]
            left = ctx.rel_from_host([key, X], [col, tg])
            n0 = ctx.get_stats()["index_joins"]
            got = ctx.bind_join(left, pat)
            want = O.hash_join(O.rel_from_host([key, X], [col, tg]), db.bgp([pat]))
            H.assert_same_bag(got.to_numpy(sorted(got.slots)), want.to_numpy(sorted(want.slots)), f"{what} indexed={indexed}")
            took_index = ctx.get_stats()["index_joins"] > n0
            if "multi" not in what:  # (a multi-valued column has no table: the pattern's slice still comes from the index, then a hash join)
                assert took_index == indexed, (what, indexed)
    # both variables bound, or none: natural join / cartesian semantics through the general path
    left = ctx.rel_from_host([E, T], [subj[:50], d.o[1::6][:50]])
    got = ctx.bind_join(left, title_p)
    assert got.n_rows == 50
