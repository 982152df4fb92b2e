"""GPU (-m gpu): every device entry point of GROUP BY against the exact reference of tests/agg_reference.py, on inputs whose every
value is under the test's control (tests/agg_cases.py: exact V1, rounding V2, special-value V3 groups), at the shapes where the
aggregation kernels change behaviour — the 64-entry CTA tables, the 4096-slot first global table and its 16x rerun, warp and
4 x 256-row load boundaries, one grid-stride pass at 132 SMs.

  E1 kb_group_aggregate, 1 key, <= 1 aggregate        group1_kernel<COUNT/SUM/AVG/MIN/MAX>
  E2 kb_group_aggregate, 2-4 keys or 2-8 aggregates   group_kernel
  E3 kb_star_join_aggregate, indexed, fused           the AGG branch of probe_index_kernel
  E4 kb_star_join_aggregate, no index / 2 aggregates  join, then E1 / E2
  E5 prepared grouped plan                             probe_index_kernel + group_compact_kernel
  E6 kb_groups_pack -> kb_groups_merge                 group_merge_kernel
  E7 prepared plan with attach_peers, world of one     group_merge_peers_kernel
"""
import ctypes as C

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import agg_cases as AC
from tests import agg_reference as R

pytestmark = pytest.mark.gpu

KINDS = [R.COUNT, R.SUM, R.MIN, R.MAX, R.AVG]
PASS_E1 = 132 * 8 * 1024  # rows of one grid-stride pass of group1_kernel at 132 SMs (8 CTAs x 256 threads x 4 rows)
PASS_E2 = 132 * 8 * 256   # group_kernel
N_SPECIAL = len(AC.SPECIAL_GROUPS)


class Failures:
    """every disagreement of one test, reported together: a kernel that is wrong for several aggregates shows all of them"""

    def __init__(self):
        self.msgs = []

    def check(self, *args):
        try:
            R.assert_groups_match(*args)
        except AssertionError as e:
            self.msgs.append(str(e))

    def done(self):
        assert not self.msgs, "\n".join(self.msgs)


def make_rows(seed, n_rows, n_groups, vset, n_key_cols=1, key_none=False):
    """rows u32 [n, n_key_cols + 2] = (key columns..., value id, second value id), num_or0, is_num. V3: the special groups of
    agg_cases first, the rest of the requested groups / rows V1; every case's rows are shuffled."""
    rng = np.random.default_rng(seed)
    if vset == "V3":
        sg, sv, sc = AC.special_rows()
        n_groups = max(n_groups, N_SPECIAL)
        n_fill = max(n_rows - len(sg), n_groups - N_SPECIAL)
        fill = AC.assign_groups(rng, n_fill, n_groups - N_SPECIAL) + N_SPECIAL if n_groups > N_SPECIAL else np.zeros(0, np.int64)
        gid = np.concatenate([sg, fill])
        vals = np.concatenate([sv, AC.v1_values(rng, len(fill))])
        codes = np.concatenate([sc, np.zeros(len(fill), np.int8)])
        p = rng.permutation(len(gid))
        gid, vals, codes = gid[p], vals[p], codes[p]
    else:
        gid = AC.assign_groups(rng, n_rows, n_groups)
        vals = AC.v1_values(rng, n_rows) if vset == "V1" else AC.v2_values(rng, gid)
        codes = np.zeros(n_rows, np.int8)
    n = len(gid)
    vals2 = AC.v2_values(rng, gid) if n else np.zeros(0)  # a second value column
    ids, num, isn = AC.encode(np.concatenate([vals, vals2]), np.concatenate([codes, np.zeros(n, np.int8)]), base=4)
    n_groups = max(n_groups, 1)
    if n_key_cols == 1:
        edge = (c.KB_ID_NONE, 0, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE) if key_none else (0, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE)
        keys = AC.group_keys(rng, n_groups, edge)[:, None]
    else:
        # the last column tells the groups apart; the first repeats a few edge and random ids across groups, the others are random
        first = AC.group_keys(rng, n_groups // 3 + 1)[np.arange(n_groups) % (n_groups // 3 + 1)]
        mid = [rng.integers(0, 1 << 32, n_groups, dtype=np.uint64).astype(np.uint32) for _ in range(n_key_cols - 2)]
        keys = np.stack([first] + mid + [AC.group_keys(rng, n_groups, ())], axis=1)
    rows = np.concatenate([keys[gid], ids[:n, None], ids[n:, None]], axis=1).astype(np.uint32)
    return rows, num, isn


def e1_cases():
    out = [(n, 7, v) for n in (0, 1, 31, 32, 33, 1023, 1024, 1025, PASS_E1 - 1, PASS_E1 + 1) for v in ("V1", "V2")]
    out += [(max(8 * g, 4000), g, v) for g in (1, 63, 64, 65, 4096, 4097) for v in ("V1", "V2", "V3")]
    out += [(300_000, 70_000, "V2"), (300_000, 70_000, "V3"), (3_000_000, 4097, "V1")]
    return out


@pytest.mark.parametrize("n_rows,n_groups,vset", e1_cases())
def test_group_aggregate_one_key(ctx, n_rows, n_groups, vset):
    """E1: group1_kernel for every aggregate kind, with KB_ID_NONE (its free-slot marker) among the keys"""
    f = Failures()
    rows, num, isn = make_rows(n_rows * 7 + n_groups, n_rows, n_groups, vset, key_none=True)
    ctx.dict_numeric_load(num, isn)
    rel = ctx.rel_from_host([0, 1, 2], [rows[:, 0], rows[:, 1], rows[:, 2]])
    for aggs in [[]] + [[(k, 1)] for k in KINDS] + [[(R.SUM, 0)], [(R.MIN, 0)]]:  # the key itself aggregated
        g = ctx.group_aggregate(rel, [0], aggs)
        f.check(g, rows, num, [0], aggs, f"E1 {vset} rows={n_rows} groups={n_groups} aggs={aggs}")
    rel.free()
    f.done()


ALL8 = [(R.COUNT, 0), (R.SUM, "v"), (R.MIN, "v"), (R.MAX, "v"), (R.AVG, "v"), (R.SUM, 0), (R.MIN, "w"), (R.MAX, "w")]


def e2_cases():
    out = [(n, 5, v, 2) for n in (0, 1, 31, 32, 33, 1023, 1024, 1025, PASS_E2 - 1, PASS_E2 + 1) for v in ("V1", "V2")]
    out += [(max(8 * g, 4000), g, v, k) for g in (1, 63, 64, 65, 4096, 4097) for v in ("V1", "V3") for k in (2, 4)]
    out += [(300_000, 70_000, "V3", 3)]
    return out


@pytest.mark.parametrize("n_rows,n_groups,vset,n_keys", e2_cases())
def test_group_aggregate_multi_key_all_aggregates(ctx, n_rows, n_groups, vset, n_keys):
    """E2: group_kernel with 2-4 key columns and all 8 aggregates at once (a key column also aggregated), and one key with two
    aggregates"""
    f = Failures()
    rows, num, isn = make_rows(n_rows * 3 + n_groups + n_keys, n_rows, n_groups, vset, n_key_cols=n_keys)
    ctx.dict_numeric_load(num, isn)
    slots = list(range(n_keys + 2))
    rel = ctx.rel_from_host(slots, [rows[:, j] for j in slots])
    col = {"v": n_keys, "w": n_keys + 1}
    aggs = [(k, col.get(s, s)) for k, s in ALL8]
    g = ctx.group_aggregate(rel, list(range(n_keys)), aggs)
    f.check(g, rows, num, list(range(n_keys)), aggs, f"E2 {vset} rows={n_rows} groups={n_groups} keys={n_keys}")
    for a2 in ([(R.MIN, n_keys), (R.SUM, n_keys)], [(R.AVG, n_keys), (R.MAX, n_keys)]):
        g = ctx.group_aggregate(rel, [0], a2)
        f.check(g, rows, num, [0], a2, f"E2 one key, two aggregates {vset} rows={n_rows} groups={n_groups}")
    rel.free()
    f.done()


def test_group_kernel_warp_hash_collision(ctx):
    """two distinct 2-column keys whose in-warp match hash collides, interleaved in the same 32-row chunks: group_kernel's
    'odd lanes go alone' branch must keep them apart (it once left the key comparison early, skipping a shuffle the other lanes of
    the match group waited for: the warp deadlocked)"""
    f = Failures()
    (a0, a1), (b0, b1) = AC.colliding_pair()
    assert AC.warp_hash([[a0], [a1]])[0] == AC.warp_hash([[b0], [b1]])[0]
    for vset in ("V1", "V3"):
        rows, num, isn = make_rows(99, 4096, 8, vset, n_key_cols=2)
        n = len(rows)
        first = np.arange(n) % 32 < 16  # half of every warp's rows -> the two colliding keys, alternating
        pick = np.arange(n) % 2 == 0
        rows[first & pick, 0], rows[first & pick, 1] = a0, a1
        rows[first & ~pick, 0], rows[first & ~pick, 1] = b0, b1
        ctx.dict_numeric_load(num, isn)
        rel = ctx.rel_from_host([0, 1, 2, 3], [rows[:, j] for j in range(4)])
        aggs = [(k, 2) for k in KINDS] + [(R.SUM, 3)]
        g = ctx.group_aggregate(rel, [0, 1], aggs)
        f.check(g, rows, num, [0, 1], aggs, f"warp hash collision {vset}")
        rel.free()
    f.done()


# ---- star joins: (?e P_key ?k) . (?e P_val ?v) [. (?e P_z ?z)], both predicates functional and subject-dense
P_KEY, P_VAL, P_Z = 0x7FFFFF01, 0x7FFFFF02, 0x7FFFFF03
E, K, V, Z = 0, 1, 2, 3
A_PAT = c.pattern(c.V(E), c.K(P_KEY), c.V(K))
B_PAT = c.pattern(c.V(E), c.K(P_VAL), c.V(V))
Z_PAT = c.pattern(c.V(E), c.K(P_Z), c.V(Z))
# which pattern probes: the first of equal-size slices — key on the probe side / value on the probe side / both looked up
ORDERS = {"key probes": [A_PAT, B_PAT], "value probes": [B_PAT, A_PAT], "both looked up": [Z_PAT, A_PAT, B_PAT]}


def load_star(ctx, rows, num, isn, index=True):
    n = len(rows)
    e = (np.uint32(1 << 24) + np.arange(n, dtype=np.uint32)).astype(np.uint32)
    s = np.concatenate([e, e, e])
    p = np.concatenate([np.full(n, P_KEY, np.uint32), np.full(n, P_VAL, np.uint32), np.full(n, P_Z, np.uint32)])
    o = np.concatenate([rows[:, 0], rows[:, 1], e])
    ctx.store_load(s, p, o)
    ctx.dict_numeric_load(num, isn)
    if index:
        ctx.build_index()


STAR_CASES = [(n, 5, "V1") for n in (1, 31, 33, 1025)] + [(max(8 * g, 4000), g, v) for g in (1, 63, 64, 65, 4096) for v in ("V1", "V2", "V3")]


@pytest.mark.parametrize("n_rows,n_groups,vset", STAR_CASES)
def test_star_join_aggregate_fused(ctx, n_rows, n_groups, vset):
    """E3: the GROUP BY folded into the index probe kernel (asserted: one probe launch + the table init), group and aggregated
    variables on the probe side and on looked-up sides, the key itself aggregated"""
    f = Failures()
    rows, num, isn = make_rows(n_rows + n_groups * 11, n_rows, n_groups, vset)
    load_star(ctx, rows, num, isn)
    for what, pats in ORDERS.items():
        for aggs in [[]] + [[(k, V)] for k in KINDS] + [[(R.MAX, K)]]:
            n0 = ctx.get_stats()["kernel_launches"]
            g, n_joined = ctx.star_join_aggregate(E, pats, None, [K], aggs)
            assert ctx.get_stats()["kernel_launches"] - n0 <= 2, f"fused path not taken ({what}, {aggs})"
            assert n_joined == len(rows)
            f.check(g, rows[:, :2], num, [0], [(k, 1 if s == V else 0) for k, s in aggs],
                                  f"E3 {what} {vset} rows={n_rows} groups={n_groups} aggs={aggs}")
    f.done()


@pytest.mark.parametrize("n_rows,n_groups,vset", [(20_000, 65, "V3"), (40_000, 4097, "V3"), (300_000, 70_000, "V2"), (20_000, 64, "V1")])
def test_star_join_aggregate_unfused(ctx, n_rows, n_groups, vset):
    """E4: no index (join, then group), two aggregates (join + group_kernel), and more groups than the fused 4096-slot table"""
    f = Failures()
    rows, num, isn = make_rows(n_rows + 5, n_rows, n_groups, vset)
    for index in (False, True):
        load_star(ctx, rows, num, isn, index=index)
        for aggs in [[(k, V)] for k in KINDS] + [[(R.SUM, V), (R.MIN, V)], [(R.COUNT, 0), (R.MAX, V)]]:
            g, n_joined = ctx.star_join_aggregate(E, ORDERS["key probes"], None, [K], aggs)
            assert n_joined == len(rows)
            f.check(g, rows[:, :2], num, [0], [(k, 1 if s == V else 0) for k, s in aggs],
                                  f"E4 index={index} {vset} rows={n_rows} groups={n_groups} aggs={aggs}")
    f.done()


@pytest.mark.parametrize("n_groups,vset", [(1, "V1"), (64, "V2"), (65, "V3"), (4096, "V3"), (4096, "V1")])
def test_prepared_group_plan(ctx, n_groups, vset):
    """E5: grouped prepared plans, ring of 2, several submits in flight"""
    f = Failures()
    rows, num, isn = make_rows(n_groups * 3, max(8 * n_groups, 4000), n_groups, vset)
    load_star(ctx, rows, num, isn)
    for aggs in [[]] + [[(k, V)] for k in KINDS]:
        plan = ctx.prepare_star_join(E, ORDERS["value probes"], None, group_slots=[K], aggs=aggs, ring=2)
        assert plan.grouped
        want = [(k, 1 if s == V else 0) for k, s in aggs]
        tickets = []
        for rep in range(5):
            tickets.append(plan.submit())
            if len(tickets) == 2:
                g, n_joined = plan.collect_groups(tickets.pop(0))
                assert n_joined == len(rows)
                f.check(g, rows[:, :2], num, [0], want, f"E5 {vset} groups={n_groups} aggs={aggs} submit {rep}")
        g, _ = plan.collect_groups(tickets.pop(0))
        f.check(g, rows[:, :2], num, [0], want, f"E5 {vset} groups={n_groups} aggs={aggs} last")
        plan.free()
    f.done()


def test_prepared_group_plan_limit(ctx):
    """E5: one group more than the plan's 4096-slot table is KB_E_LIMIT at collect, never a truncated result"""
    rows, num, isn = make_rows(4097, 40_000, 4097, "V3")
    load_star(ctx, rows, num, isn)
    plan = ctx.prepare_star_join(E, ORDERS["key probes"], None, group_slots=[K], aggs=[(R.SUM, V)], ring=2)
    for _ in range(2):
        t = plan.submit()
        with pytest.raises(c.KolibrieError) as e:
            plan.collect_groups(t)
        assert e.value.status == c.KB_E_LIMIT
    plan.free()


def packed_group(ctx, rel, group_slots, aggs):
    """kb_group_aggregate's result in its transport form (kb_groups_pack)"""
    gs = (C.c_uint32 * len(group_slots))(*group_slots)
    ag = (c.KbAgg * max(len(aggs), 1))(*[c.KbAgg(k, s) for k, s in aggs])
    g = C.c_void_p()
    ctx._check(c.lib().kb_group_aggregate(ctx.h, rel.h, gs, len(group_slots), ag, len(aggs), C.byref(g)))
    try:
        return ctx._groups_pack(g)
    finally:
        c.lib().kb_groups_free(g)


def split_rows(seed, n_parts):
    """V3 rows plus groups split across shards so that one shard's part is all NaN or all -0.0 and another's is not; returns
    (rows, num, isn, shard of every row)"""
    rows, num, isn = make_rows(seed, 6000, 200, "V3")
    rng = np.random.default_rng(seed)
    shard = rng.integers(0, n_parts, len(rows))
    # appended groups: key 1000+j; shard 0 holds the special part, shard 1 (or every other shard) the rest
    parts = [([AC.NAN] * 3, [4.0, -1.5]), ([-0.0] * 3, [2.5]), ([-0.0] * 2, [-0.0] * 3), ([AC.NAN] * 2, [AC.NAN]), ([AC.NAN], [-0.0, -0.0]),
             ([-0.0], [0.0])]
    extra = [(1000 + j, v, 0) for j, (a, _) in enumerate(parts) for v in a]
    extra += [(1000 + j, v, 1 + i % (n_parts - 1)) for j, (_, b) in enumerate(parts) for i, v in enumerate(b)]
    extra_k, extra_v, extra_s = (list(x) for x in zip(*extra))
    base = len(num)
    num = np.concatenate([num, np.array(extra_v)])
    isn = np.concatenate([isn, np.ones(len(extra_v), np.uint8)])
    ids = (base + np.arange(len(extra_v))).astype(np.uint32)
    extra = np.stack([np.array(extra_k, np.uint32), ids, ids], axis=1)
    return np.concatenate([rows, extra]), num, isn, np.concatenate([shard, np.array(extra_s)])


@pytest.mark.parametrize("n_parts", [2, 3, 8])
def test_groups_merge_of_row_shards(ctx, n_parts):
    """E6: partials of 2, 3 and 8 row shards -> kb_groups_pack -> kb_groups_merge (group_merge_kernel) equal the GROUP BY of all rows"""
    f = Failures()
    rows, num, isn, shard = split_rows(40 + n_parts, n_parts)
    ctx.dict_numeric_load(num, isn)
    for gcols, aggs in [([0], [(k, 1) for k in KINDS]), ([0], [(R.MIN, 1)]), ([0], [(R.SUM, 1)]), ([0], [(R.MAX, 1)]), ([0], [(R.AVG, 1)]),
                        ([0, 2], [(R.COUNT, 0), (R.SUM, 1), (R.MIN, 1), (R.MAX, 1), (R.AVG, 1), (R.SUM, 0), (R.MIN, 2), (R.MAX, 2)])]:
        parts = []
        for r in range(n_parts):
            m = shard == r
            rel = ctx.rel_from_host([0, 1, 2], [rows[m, 0], rows[m, 1], rows[m, 2]])
            parts.append(packed_group(ctx, rel, gcols, aggs))
            rel.free()
        g = ctx.groups_merge(parts)
        f.check(g, rows, num, gcols, aggs, f"E6 {n_parts} shards, keys {gcols}, aggs {aggs}")
    f.done()


@pytest.mark.parametrize("n_groups,vset", [(65, "V3"), (4096, "V3"), (64, "V2")])
def test_peer_merged_group_plan_world_of_one(ctx, n_groups, vset):
    """E7: kb_plan_attach_peers in a world of one: join+group -> barrier -> group_merge_peers_kernel -> compaction"""
    f = Failures()
    import torch

    rows, num, isn = make_rows(n_groups + 77, max(8 * n_groups, 4000), n_groups, vset)
    load_star(ctx, rows, num, isn)
    dev = torch.device("cuda", ctx.device)
    for aggs in [[(k, V)] for k in KINDS]:
        plan = ctx.prepare_star_join(E, ORDERS["both looked up"], None, group_slots=[K], aggs=aggs, ring=2)
        scratch = torch.zeros((plan.peer_scratch_bytes() + 3) // 4, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        plan.attach_peers(0, 1, [scratch.data_ptr()], keep=scratch)
        want = [(k, 1 if s == V else 0) for k, s in aggs]
        tickets = []
        for rep in range(4):
            tickets.append(plan.submit())
            if len(tickets) == 2:
                g, n_joined = plan.collect_groups(tickets.pop(0))
                assert n_joined == len(rows)
                f.check(g, rows[:, :2], num, [0], want, f"E7 {vset} groups={n_groups} aggs={aggs} submit {rep}")
        plan.collect_groups(tickets.pop(0))
        plan.free()
    f.done()
