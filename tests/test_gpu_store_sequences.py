"""GPU: seeded sequences of every store mutation (tests/store_sequences.py), with the store read after every step through the readers
that trust the maintained index: the table-mode probe with its rank filter and codes (star S1), an object-keyed star (S2), a star
without a filter (S3), constant-subject and constant-object scans, the bind join and kb_bgp_execute; every 5 steps also the fused
GROUP BY, prepared plans (fresh and stale) and the store statistics. Each answer is compared as a bag with the CPU oracle over the
model's rows. A failure names the seed, mode, step, reader and the ops up to that step; store_sequences.replay re-runs them.

Modes: the index built after the first slides and maintained from then on; never built; built but switched off
(kb_set_use_index(0)); a subject-sharded context (kb_set_sharding(1, 2)) with occasional foreign subjects."""
import tempfile

import numpy as np
import pytest

from kolibrie_b200 import capi as c
from tests import helpers as H
from tests import oracle_api as O
from tests import stats_reference as R
from tests import store_sequences as S

pytestmark = pytest.mark.gpu

X, V, CC, NN, A, B, Y = 0, 1, 2, 3, 4, 5, 6
S1 = [c.pattern(c.V(X), c.K(S.F), c.V(V)), c.pattern(c.V(X), c.K(S.C), c.V(CC)), c.pattern(c.V(X), c.K(S.N), c.V(NN))]
S2 = [c.pattern(c.V(A), c.K(S.I), c.V(X)), c.pattern(c.V(B), c.K(S.M), c.V(X))]
S3 = [c.pattern(c.V(X), c.K(S.M), c.V(Y)), c.pattern(c.V(X), c.K(S.F), c.V(V))]
CHAIN = [c.pattern(c.V(A), c.K(S.I), c.V(X)), c.pattern(c.V(X), c.K(S.F), c.V(V)), c.pattern(c.V(X), c.K(S.M), c.V(Y))]
CMPS = [c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE, c.CMP_EQ, c.CMP_NE]


@pytest.fixture(scope="module")
def ctx():
    """a context of this module's own: the sequences load dictionaries, numeric tables and sharding no other test should inherit"""
    x = c.Context(0)
    yield x
    x.close()


@pytest.fixture(scope="module")
def dict_strings():
    return S.strings()


def rows(rel, order):
    out = rel.to_numpy(order) if rel.n_rows else np.empty((0, len(order)), np.uint32)
    if isinstance(rel, c.Relation):
        rel.free()
    return out


def filt(cmp, value):
    return [c.fop(c.F_CMP_NUM, slot=V, cmp=cmp, value=value)]


class Run:
    def __init__(self, ctx, seed, mode, dict_strings):
        self.ctx, self.seed, self.mode = ctx, seed, mode
        self.log, _ = S.generate(seed, mode)
        self.model = S.Model(self.log[0][1]["family"])
        S.setup_device(ctx, mode, self.model, dict_strings)
        self.plan = None
        self.plan_versioned = 0
        self.live_reads = 0       # S1 reads answered from an index maintained across at least one mutation

    def where(self, step, reader):
        return S.report(self.seed, self.mode, step, reader, self.log[:step + 1])

    def same(self, step, reader, got, want):
        try:
            H.assert_same_bag(got, want, reader)
        except AssertionError as e:
            raise AssertionError(f"{e}\n{self.where(step, reader)}") from None

    def step(self, i, tmp, keep):
        op = self.log[i]
        want = S.apply_model(self.model, op)
        try:
            S.apply_device(self.ctx, op, self.model, want, tmp, keep)
        except (c.KolibrieError, AssertionError) as e:
            raise AssertionError(f"{e}\n{self.where(i, op[0])}") from None

    def read(self, i):
        cx, m = self.ctx, self.model
        want_rows = m.rows()
        self.same(i, "store_download", np.stack(cx.store_download(), axis=1), want_rows)
        db = O.Db(want_rows[:, 0], want_rows[:, 1], want_rows[:, 2], m.num, m.isn)
        consts = S.filter_constants(m) or [("present", 0.0)]
        # S1: the table-mode probe, its rank filter and the subject codes
        for k, (cls, value) in enumerate(consts):
            f = filt(CMPS[(i + k) % len(CMPS)], value)
            n0 = cx.get_stats()["index_joins"]
            got = rows(cx.star_join(X, S1, f), [X, V, CC, NN])
            if self.mode == "maintained" and m.use_index and m.built and m.since_build and cx.get_stats()["index_joins"] > n0:
                self.live_reads += 1
            self.same(i, f"S1 filter {cls} {value}", got, rows(db.bgp(S1, f), [X, V, CC, NN]))
        # S1 without a FILTER: the smallest slice probes, so F's subject table is looked up instead of streamed
        self.same(i, "S1 without a filter", rows(cx.star_join(X, S1), [X, V, CC, NN]), rows(db.bgp(S1), [X, V, CC, NN]))
        self.same(i, "S2 keyed on the object", rows(cx.star_join(X, S2), [X, A, B]), rows(db.bgp(S2), [X, A, B]))
        self.same(i, "S3", rows(cx.star_join(X, S3), [X, Y, V]), rows(db.bgp(S3), [X, Y, V]))
        # constant subjects and objects: live ones and one absent
        rng = np.random.default_rng(i)
        pats = []
        for p in (S.F, S.M, S.I):
            live = want_rows[want_rows[:, 1] == p]
            pick = live[rng.integers(0, len(live), 3)] if len(live) else np.empty((0, 3), np.uint32)
            for s_ in pick[:, 0].tolist() + [S.S_BASE - 5]:
                pats.append((c.pattern(c.K(s_), c.K(p), c.V(1)), [1]))
            for o_ in pick[:, 2].tolist() + [S.S_BASE - 5]:
                pats.append((c.pattern(c.V(0), c.K(p), c.K(o_)), [0]))
        got = [rel for k in range(0, len(pats), 8) for rel in cx.scan([pt for pt, _ in pats[k:k + 8]])]  # (a scan takes 1..8 patterns)
        for rel, (pt, order) in zip(got, pats):
            self.same(i, f"scan ({pt.s.value if not pt.s.is_var else '?'} {pt.p.value} {pt.o.value if not pt.o.is_var else '?'})",
                      rows(rel, order), rows(db.scan(pt), order))
        # the bind join of live subjects and an absent one with (?x M ?y)
        live = want_rows[want_rows[:, 1] == S.M, 0]
        xs = np.unique(np.concatenate([live[rng.integers(0, len(live), 50)] if len(live) else [], [S.S_BASE - 5]]).astype(np.uint32))
        left = cx.rel_from_host([X], [xs])
        got = rows(cx.bind_join(left, c.pattern(c.V(X), c.K(S.M), c.V(Y))), [X, Y])
        left.free()
        want = O.hash_join(O.rel_from_host([X], [xs]), db.scan(c.pattern(c.V(X), c.K(S.M), c.V(Y))))
        self.same(i, "bind_join (?x M ?y)", got, rows(want, [X, Y]))
        # kb_bgp_execute of a chain with a FILTER
        f = filt(CMPS[i % len(CMPS)], consts[0][1])
        self.same(i, "bgp_execute chain", rows(cx.bgp_execute(CHAIN, f), [A, X, V, Y]), rows(db.bgp(CHAIN, f), [A, X, V, Y]))
        if i % 5 == 0:
            self.read_every_5(i, db, consts)

    def read_every_5(self, i, db, consts):
        cx, m = self.ctx, self.model
        f = filt(c.CMP_GE, consts[0][1])
        aggs = [(c.AGG_SUM, V)]
        got, n = cx.star_join_aggregate(X, S1, f, [CC], aggs)
        ref = db.bgp(S1, f)
        want = db.group(ref, [CC], aggs)
        o1, o2 = np.argsort(got["keys"][0]), np.argsort(want["keys"][0])
        try:
            assert n == ref.n_rows, (n, ref.n_rows)
            assert np.array_equal(got["keys"][0][o1], want["keys"][0][o2])
            assert np.array_equal(got["counts"][o1], want["counts"][o2])
            assert np.array_equal(got["values"][0][o1], want["values"][0][o2])  # (integer-valued: the SUM is exact)
        except AssertionError as e:
            raise AssertionError(f"{e}\n{self.where(i, 'star_join_aggregate COUNT/SUM by ?c')}") from None
        # the plan prepared at the last check is stale once the store, its index or the numeric table moved
        if self.plan is not None:
            if m.versioned != self.plan_versioned:
                with pytest.raises(c.KolibrieError) as e:
                    self.plan.submit()
                assert e.value.status == c.KB_E_INVALID and "stale" in e.value.message, self.where(i, "stale plan")
            self.plan.free()
            self.plan = None
        try:
            self.plan = cx.prepare_star_join(X, S1, f, ring=2)
        except c.KolibrieError as e:
            assert e.status == c.KB_E_UNSUPPORTED, f"{e}\n{self.where(i, 'prepare')}"  # not on the one-kernel index path
        if self.plan is not None:
            self.plan_versioned = m.versioned
            assert self.plan.collect(self.plan.submit()) == ref.n_rows, self.where(i, "prepared plan count")
        # DatabaseStats::gather_stats_fast over every distinct triple
        st = cx.store_gather_stats(0)
        want = R.gather_stats_numpy(m.rows(), 0, 0)
        for k in ("total_triples", "take", "step"):
            assert st[k] == want[k], f"{k}: {st[k]} vs {want[k]}\n{self.where(i, 'store_gather_stats')}"
        for k in ("subject", "predicate", "object"):
            ok = np.array_equal(st[k][0], want[k][0]) and np.array_equal(st[k][1], want[k][1])
            assert ok, self.where(i, f"store_gather_stats {k}")

    def run(self):
        keep = []
        with tempfile.TemporaryDirectory() as tmp:
            for i in range(1, len(self.log)):
                self.step(i, tmp, keep)
                self.read(i)
                keep.clear()
        if self.plan is not None:
            self.plan.free()


@pytest.mark.parametrize("mode", S.MODES)
@pytest.mark.parametrize("seed", S.SEEDS)
def test_store_sequence_matches_the_oracle(ctx, dict_strings, seed, mode):
    run = Run(ctx, seed, mode, dict_strings)
    run.run()
    if mode == "maintained":
        assert run.live_reads > 0, f"seed {seed}: no S1 read was answered from an index maintained across a mutation"
