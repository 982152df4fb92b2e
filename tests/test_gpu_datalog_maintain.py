"""GPU: kb_datalog_maintain (delete-and-rederive of the inferred segment across a window slide) against the oracle's closure from scratch
over the new base B'. After every call: the inferred facts equal closure(B') \\ B' (each once), the store is the live base segments plus
them, and the reported differences are I \\ I' and I' \\ I."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import helpers as H
from tests import sharded_cases as SC
from tests.window_oracle import as_rows, rows_set

pytestmark = pytest.mark.gpu

CASES = {"taxonomy": lambda: SC.taxonomy_case(3, 4, 3000), "family": lambda: SC.family_case(), "chain": lambda: SC.chain_case()}


def rel_rows(r):
    return r.to_numpy([0, 1, 2]) if r.n_rows else np.empty((0, 3), np.uint32)


class Window:
    """a tagged segment store on the device and the same on the host; check() compares them after each call"""

    def __init__(self, cx, rules, numeric=None):
        self.cx, self.rules, self.numeric = cx, rules, numeric
        self.segs = {}
        cx.store_clear()
        if numeric is not None:
            cx.dict_numeric_load(*numeric)

    def append(self, tag, rows):
        rows = np.asarray(rows, np.uint32).reshape(-1, 3)
        self.cx.store_append(rows[:, 0], rows[:, 1], rows[:, 2], tag)
        self.segs[tag] = rows

    def base(self):
        return set().union(*[rows_set(r) for r in self.segs.values()]) if self.segs else set()

    def closure(self):
        st, inf = SC.closure_of(as_rows(self.base()), self.rules, self.numeric)
        assert st == 0
        return rows_set(inf) - self.base()

    def fixpoint(self, strategy=c.SEMI_NAIVE):
        rel, st = self.cx.datalog_fixpoint(self.rules, strategy)
        self.inferred = rows_set(rel_rows(rel))
        assert self.inferred == self.closure()
        return st

    def maintain(self, evict, add_rows, add_tag, strategy=c.SEMI_NAIVE, label=""):
        add = None if add_rows is None else np.asarray(add_rows, np.uint32).reshape(-1, 3)
        gone, new, st = self.cx.datalog_maintain(self.rules, evict, add, add_tag, strategy)
        for t in evict:
            del self.segs[t]
        if add is not None:
            self.segs[add_tag] = add
        want = self.closure()
        g, n = rel_rows(gone), rel_rows(new)
        assert len(rows_set(g)) == len(g) and len(rows_set(n)) == len(n), f"{label}: a difference holds a fact twice"
        assert rows_set(g) == self.inferred - want, f"{label}: inferred_removed"
        assert rows_set(n) == want - self.inferred, f"{label}: inferred_added"
        assert st.inferred_removed == len(g) and st.inferred_added == len(n)
        self.inferred = want
        s, p, o = self.cx.store_download()
        live = np.concatenate(list(self.segs.values()) + [as_rows(want)], axis=0) if self.segs else as_rows(want)
        H.assert_same_bag(np.stack([s, p, o], axis=1), live, f"{label}: store")
        return g, n, st


def chunks_of(rows, k, seed):
    order = np.random.default_rng(seed).permutation(len(rows))
    return [rows[order[i::k]] for i in range(k)]


def run_sequence(cx, name, strategy, seed=3, firings=10):
    rows, rules, numeric, _ = CASES[name]()
    w = Window(cx, rules, numeric)
    ch = chunks_of(rows, 16, seed)
    for i in range(8):
        w.append(i + 1, ch[i])
    w.fixpoint()
    rng = np.random.default_rng(seed)
    nxt, trace = 8, []
    for f in range(firings):
        live = sorted(w.segs)
        evict = [int(t) for t in rng.choice(live, size=min(len(live), int(rng.integers(1, 3))), replace=False)]
        add = ch[nxt % len(ch)]
        nxt += 1
        g, n, st = w.maintain(evict, add, 100 + f, strategy, f"{name} firing {f}")
        trace.append((canon(g), canon(n)))
    return trace


def canon(a):
    return H.canon(a).tobytes()


@pytest.mark.parametrize("name", sorted(CASES))
def test_sliding_sequences_match_the_closure_from_scratch(ctx, monkeypatch, name):
    """10 firings, each evicting 1-2 of the live chunks and adding one; every hash-join strategy (KB_NAIVE shares the closure and is
    maintained from the delta), with the kept state and with a rebuild from the store every call: answers identical call by call"""
    traces = []
    for strategy in (c.SEMI_NAIVE, c.SEMI_NAIVE_OLD_DELTA, c.NAIVE):
        for state in ("1", "0"):
            monkeypatch.setenv("KOLIBRIE_FIX_STATE", state)
            traces.append(run_sequence(ctx, name, strategy))
    assert all(t == traces[0] for t in traces)


def test_fuzzed_rule_sets(ctx):
    ran = 0
    for seed in range(40):
        rows, rules, numeric, _ = SC.fuzz_case(seed)
        if len(rows) < 8:
            continue
        st, _ = SC.closure_of(rows, rules, numeric)
        if st != 0:
            continue
        w = Window(ctx, rules, numeric)
        ch = chunks_of(rows, 6, seed)
        for i in range(4):
            w.append(i + 1, ch[i])
        try:
            w.fixpoint()
        except c.KolibrieError as e:
            assert e.status == c.KB_E_UNSUPPORTED
            continue
        rng = np.random.default_rng(seed)
        for f in range(4):
            live = sorted(w.segs)
            evict = [int(t) for t in rng.choice(live, size=min(len(live), int(rng.integers(0, 3))), replace=False)]
            add = ch[(4 + f) % 6] if rng.random() < 0.8 else None
            w.maintain(evict, add, 50 + f, label=f"fuzz {seed} firing {f}")
        ran += 1
    assert ran >= 10, ran


def ancestor(cx):
    PAR, ANC = 1, 2
    rules = [{"premise": [c.pattern(c.V(0), c.K(PAR), c.V(1))], "conclusion": [c.pattern(c.V(0), c.K(ANC), c.V(1))], "filters": []},
             {"premise": [c.pattern(c.V(0), c.K(PAR), c.V(1)), c.pattern(c.V(1), c.K(ANC), c.V(2))], "conclusion": [c.pattern(c.V(0), c.K(ANC), c.V(2))],
              "filters": []}]
    return Window(cx, rules), PAR, ANC


def test_diamond_overdeletes_and_rederives(ctx):
    """A->B, A->C, B->D, C->D with the ancestor rules; evicting A->B over-deletes anc(A,B) and anc(A,D); anc(A,D) comes back through C"""
    w, PAR, ANC = ancestor(ctx)
    A, B, C_, D = 10, 11, 12, 13
    w.append(1, [[A, PAR, B]])
    w.append(2, [[A, PAR, C_], [B, PAR, D], [C_, PAR, D]])
    w.fixpoint()
    g, n, st = w.maintain([1], None, 0, label="diamond")
    assert st.base_removed == 1 and st.base_added == 0
    assert st.overdeleted == 2 and st.rederived == 1
    assert rows_set(g) == {(A, ANC, B)} and len(n) == 0
    assert st.inferred_removed == 1 and st.inferred_added == 0


def test_still_derivable_base_fact_becomes_inferred(ctx):
    w, PAR, ANC = ancestor(ctx)
    w.append(1, [[1, PAR, 2], [2, PAR, 3]])
    w.append(2, [[1, ANC, 3]])  # a base fact the rules also derive
    w.fixpoint()
    assert (1, ANC, 3) not in w.inferred
    g, n, st = w.maintain([2], None, 0, label="still derivable")
    assert st.base_removed == 1 and rows_set(n) == {(1, ANC, 3)} and len(g) == 0


def test_inferred_fact_added_as_base_moves_to_the_base(ctx):
    w, PAR, ANC = ancestor(ctx)
    w.append(1, [[1, PAR, 2], [2, PAR, 3]])
    w.fixpoint()
    assert (1, ANC, 3) in w.inferred
    g, n, st = w.maintain([], [[1, ANC, 3]], 7, label="inferred added")
    assert st.base_added == 1 and rows_set(g) == {(1, ANC, 3)} and len(n) == 0
    s, p, o = ctx.store_download()
    assert list(map(tuple, np.stack([s, p, o], 1).tolist())).count((1, ANC, 3)) == 1


def test_fact_in_two_segments_is_not_removed(ctx):
    w, PAR, ANC = ancestor(ctx)
    w.append(1, [[1, PAR, 2], [2, PAR, 3]])
    w.append(2, [[1, PAR, 2]])
    w.fixpoint()
    g, n, st = w.maintain([2], None, 0, label="two segments")
    assert st.base_removed == 0 and st.overdeleted == 0 and len(g) == 0 and len(n) == 0


def taxonomy_stream(n_instances=20000, n_slides=10):
    t = datagen.taxonomy_dataset(fanout=3, depth=4, n_instances=n_instances)
    rows = np.stack([t.s, t.p, t.o], axis=1).astype(np.uint32)
    tbox, abox = rows[rows[:, 1] == t.ids["rdfs:subClassOf"]], rows[rows[:, 1] == t.ids["rdf:type"]]
    return tbox, np.array_split(abox, 2 * n_slides), datagen.taxonomy_rules(t)


def test_reference_firing_protocol_is_proportional_to_the_slide(ctx):
    """every firing evicts the WHOLE previous window and re-adds the whole current one (rsp_engine.rs:94-104): base_removed and
    base_added are still the slide difference, and the work is far below a closure from scratch"""
    tbox, slides, rules = taxonomy_stream()
    w = Window(ctx, rules)
    w.append(1000, tbox)
    w.append(1, np.concatenate(slides[0:10]))
    w.fixpoint()
    scratch = c.Context(0)
    try:
        for f in range(1, 5):
            cur = np.concatenate(slides[f:f + 10])
            g, n, st = w.maintain([f], cur, f + 1, label=f"protocol {f}")
            assert st.base_removed == len(rows_set(slides[f - 1])) and st.base_added == len(rows_set(slides[f + 9]))
            scratch.store_load(*(np.concatenate([tbox, cur])[:, k].copy() for k in range(3)))
            _, full = scratch.datalog_fixpoint(rules)
            assert st.derivations * 2 < full.derivations, (st.derivations, full.derivations)
    finally:
        scratch.close()


def test_q11_streamed_triple_equal_to_a_derived_fact_stays(ctx):
    """SimpleR2R::materialize deletes the previous firing's derived triples after the firing's adds (simple_r2r.rs:103-108): the
    reference loses such a streamed triple for one firing; the device keeps it"""
    w, PAR, ANC = ancestor(ctx)
    w.append(1, [[1, PAR, 2], [2, PAR, 3]])
    w.fixpoint()
    w.maintain([1], [[1, PAR, 2], [1, ANC, 3]], 2, label="q11")  # the whole window again, plus a triple derived last firing
    s, p, o = ctx.store_download()
    assert (1, ANC, 3) in set(map(tuple, np.stack([s, p, o], 1).tolist()))


def test_index_stays_valid_and_on_the_index_path(ctx):
    """the index built before the first maintenance stays valid: a star join over a functional rule head predicate (a label copied
    by a rule) and the label itself keeps the one-kernel index path after every call"""
    from tests import oracle_api as O

    LABEL, LABEL2 = 1 << 24, (1 << 24) + 1
    tbox, slides, rules = taxonomy_stream(6000, 6)
    rules = rules + [{"premise": [c.pattern(c.V(0), c.K(LABEL), c.V(1))], "conclusion": [c.pattern(c.V(0), c.K(LABEL2), c.V(1))], "filters": []}]
    lab = lambda r: np.stack([r[:, 0], np.full(len(r), LABEL, np.uint32), r[:, 0] + (1 << 25)], axis=1).astype(np.uint32)
    w = Window(ctx, rules)
    w.append(1000, tbox)
    for i in range(6):
        w.append(i + 1, np.concatenate([slides[i], lab(slides[i])]))
    w.fixpoint()
    ctx.build_index()
    pats = [c.pattern(c.V(0), c.K(LABEL2), c.V(1)), c.pattern(c.V(0), c.K(LABEL), c.V(2))]

    def query(label):
        n0 = ctx.get_stats()["index_joins"]
        got = ctx.star_join(0, pats)
        assert ctx.get_stats()["index_joins"] == n0 + 1, f"{label}: the query left the index path"
        allr = np.concatenate(list(w.segs.values()) + [as_rows(w.inferred)])
        want = O.Db(allr[:, 0], allr[:, 1], allr[:, 2]).bgp(pats, None)
        H.assert_same_bag(got.to_numpy(sorted(got.slots)), want.to_numpy(sorted(want.slots)), label)

    query("before the first maintenance")
    for f in range(5):
        w.maintain([f + 1], np.concatenate([slides[6 + f], lab(slides[6 + f])]), 10 + f, label=f"index {f}")
        query(f"firing {f}")


def test_refusals_leave_the_store_unchanged(ctx):
    w, PAR, ANC = ancestor(ctx)
    w.append(1, [[1, PAR, 2], [2, PAR, 3]])
    w.append(2, [[3, PAR, 4]])
    w.fixpoint()
    before = H.canon(np.stack(ctx.store_download(), axis=1))

    def refused(status, **kw):
        args = dict(rules=w.rules, evict_tags=[], add=None, add_tag=9, strategy=c.SEMI_NAIVE)
        args.update(kw)
        with pytest.raises(c.KolibrieError) as e:
            ctx.datalog_maintain(**args)
        assert e.value.status == status, (kw, e.value)
        assert np.array_equal(H.canon(np.stack(ctx.store_download(), axis=1)), before)

    refused(c.KB_E_NOT_FOUND, evict_tags=[77])
    refused(c.KB_E_INVALID, evict_tags=[c.KB_TAG_INFERRED])
    refused(c.KB_E_INVALID, add=np.array([[5, PAR, 6]], np.uint32), add_tag=c.KB_TAG_INFERRED)
    refused(c.KB_E_INVALID, add=ctx.rel_from_host([0, 1], [np.array([5], np.uint32), np.array([PAR], np.uint32)]))
    refused(c.KB_E_UNSUPPORTED, evict_tags=[2], strategy=c.SEMI_NAIVE_PARALLEL)
    refused(c.KB_E_INVALID, rules=w.rules[:1], evict_tags=[2])  # other rules
    w.maintain([2], [[4, PAR, 5]], 3, label="after the refusals")  # the next valid call is right
    # stale tokens: an append in between, kb_datalog_fixpoint_seed
    w.append(4, [[5, PAR, 6]])
    before = H.canon(np.stack(ctx.store_download(), axis=1))
    refused(c.KB_E_INVALID, evict_tags=[4])
    ctx.store_evict(c.KB_TAG_INFERRED)
    w.fixpoint()
    w.maintain([4], None, 0, label="after a new fixpoint")
    seed = ctx.rel_from_host([0, 1, 2], [np.array([7], np.uint32), np.array([PAR], np.uint32), np.array([8], np.uint32)])
    ctx.datalog_fixpoint_seed(w.rules, seed)
    before = H.canon(np.stack(ctx.store_download(), axis=1))
    refused(c.KB_E_INVALID, evict_tags=[3])


def test_no_op(ctx):
    w, PAR, ANC = ancestor(ctx)
    w.append(1, [[1, PAR, 2], [2, PAR, 3]])
    w.fixpoint()
    before = H.canon(np.stack(ctx.store_download(), axis=1))
    g, n, st = ctx.datalog_maintain(w.rules, [], None, 0)
    assert g.n_rows == 0 and n.n_rows == 0 and st.derivations == 0 and st.base_removed == 0
    assert np.array_equal(H.canon(np.stack(ctx.store_download(), axis=1)), before)
    w.maintain([1], [[1, PAR, 2]], 2, label="after the no-op")


def test_partitioned_dedup(monkeypatch):
    monkeypatch.setenv("KOLIBRIE_DERIVE_PART", "1")
    monkeypatch.setenv("KOLIBRIE_DERIVE_SLICE", "2048")
    monkeypatch.setenv("KOLIBRIE_DERIVE_MIN_ROWS", "16")
    cx = c.Context(0)
    try:
        part = run_sequence(cx, "taxonomy", c.SEMI_NAIVE, firings=6)
    finally:
        cx.close()
    monkeypatch.setenv("KOLIBRIE_DERIVE_PART", "0")
    cx = c.Context(0)
    try:
        assert run_sequence(cx, "taxonomy", c.SEMI_NAIVE, firings=6) == part
    finally:
        cx.close()


def test_stats_layout():
    import ctypes as C

    assert C.sizeof(c.KbMaintainStats) == 7 * 8 + 2 * 4 + 8


def test_engine_simple_r2r_mirror_on_the_device(ctx):
    from kolibrie_b200.engine import Constant, Rule, SimpleR2R, Variable, compile_rule

    tbox, slides, _ = taxonomy_stream(3000, 6)
    x, y, z = Variable("x"), Variable("y"), Variable("z")
    rules = [Rule(premise=[(x, Constant(0), y), (y, Constant(0), z)], conclusion=[(x, Constant(0), z)]),
             Rule(premise=[(x, Constant(1), y), (y, Constant(0), z)], conclusion=[(x, Constant(1), z)])]
    r2r = SimpleR2R(ctx=ctx)
    r2r.add_reasoning_rules(rules)
    ctx.store_clear()
    prev = []
    for f in range(6):
        window = [tuple(t) for t in tbox.tolist()] + [tuple(t) for t in np.concatenate(slides[f:f + 6]).tolist()]
        for t in prev:
            r2r.remove(t)
        for t in window:
            r2r.add(t)
        got = r2r.materialize()
        st, inf = SC.closure_of(as_rows(set(window)), [compile_rule(r) for r in rules])
        assert set(got) == rows_set(inf) - set(window), f"firing {f}"
        assert r2r.last_mode == ("fixpoint" if f == 0 else "maintain")
        prev = window


def test_base_count_table_stays_bounded_over_a_long_window(ctx, monkeypatch, capfd):
    """the reference's firing protocol re-adds the whole window every firing: over 50 firings the base count tables must follow the
    live facts, not the rows the window has seen (their size comes from the KOLIBRIE_TRACE line of every call)"""
    import re

    tbox, slides, rules = taxonomy_stream(4000, 10)
    w = Window(ctx, rules)
    w.append(1000, tbox)
    width = 6
    w.append(0, np.concatenate(slides[0:width]))
    w.fixpoint()
    monkeypatch.setenv("KOLIBRIE_TRACE", "1")
    sizes = []
    for f in range(1, 51):
        cur = np.concatenate([slides[(f + k) % len(slides)] for k in range(width)])
        capfd.readouterr()
        ctx.datalog_maintain(rules, [f - 1], cur, f)
        err = capfd.readouterr().err
        sizes.append(int(re.search(r"maintain: base count slots\s+\S+ ms\s+rows=(\d+)", err).group(1)))
        del w.segs[f - 1]
        w.segs[f] = cur
    monkeypatch.delenv("KOLIBRIE_TRACE")
    live = len(tbox) + width * max(len(x) for x in slides)
    assert max(sizes[20:]) <= max(sizes[:10]), sizes
    assert max(sizes) <= 16 * live + 4 * 4096, (max(sizes), live)
    # and the window is still right after all of it
    s, p, o = ctx.store_download()
    H.assert_same_bag(np.stack([s, p, o], axis=1), np.concatenate(list(w.segs.values()) + [as_rows(w.closure())], axis=0), "after 50 firings")


def test_numeric_table_voids_the_token_only_for_rules_that_compare_numbers(ctx):
    w, PAR, ANC = ancestor(ctx)
    w.append(1, [[1, PAR, 2], [2, PAR, 3]])
    w.fixpoint()
    ctx.dict_numeric_load(np.arange(16, dtype=np.float64), np.ones(16, np.uint8))  # e.g. the dictionary grew by a streamed literal
    w.maintain([], [[3, PAR, 4]], 2, label="numeric table reloaded, no numeric filter")
    numeric = [dict(r, filters=[c.KbRuleFilter(0, c.CMP_GT, 0, 0, 1.0)]) for r in w.rules]
    ctx.store_evict(c.KB_TAG_INFERRED)
    w.rules = numeric
    w.numeric = (np.arange(16, dtype=np.float64), np.ones(16, np.uint8))
    w.fixpoint()
    ctx.dict_numeric_load(*w.numeric)
    with pytest.raises(c.KolibrieError) as e:
        ctx.datalog_maintain(numeric, [], np.array([[4, PAR, 5]], np.uint32), 3)
    assert e.value.status == c.KB_E_INVALID
