"""CPU: the host logic of engine.SimpleR2R (a sliding window with rules) over the oracle-backed kb_datalog_maintain contract
(tests/window_oracle.py): segment and tag bookkeeping, the fixpoint-then-maintain switch, the fallback after a rule change."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200.engine import Constant, Rule, SimpleR2R, Variable
from tests.sharded_cases import closure_of
from tests.window_oracle import WindowOracleCtx, as_rows, rows_set


def taxonomy_window():
    t = datagen.taxonomy_dataset(fanout=3, depth=3, n_instances=300)
    rows = np.stack([t.s, t.p, t.o], axis=1).astype(np.uint32)
    sub, typ = t.ids["rdfs:subClassOf"], t.ids["rdf:type"]
    x, y, z = Variable("x"), Variable("y"), Variable("z")
    rules = [Rule(premise=[(x, Constant(sub), y), (y, Constant(sub), z)], conclusion=[(x, Constant(sub), z)]),
             Rule(premise=[(x, Constant(typ), y), (y, Constant(sub), z)], conclusion=[(x, Constant(typ), z)])]
    return rows[rows[:, 1] == sub], rows[rows[:, 1] == typ], rules


def make_r2r(rules):
    r = SimpleR2R(ctx=WindowOracleCtx())
    d = r.item.dictionary
    for i in range(64):  # the numeric table covers the small ids the tests use
        d.encode(f"t{i}")
    r.add_reasoning_rules(rules)
    return r


def expected_inferred(rows, r2r):
    from kolibrie_b200.engine import compile_rule

    st, inf = closure_of(as_rows(rows_set(rows)), [compile_rule(x) for x in r2r.rules])
    assert st == 0
    return rows_set(inf) - rows_set(rows)


def test_sliding_window_firings_switch_from_fixpoint_to_maintain():
    tbox, abox, rules = taxonomy_window()
    r2r = make_r2r(rules)
    ctx = r2r.ctx
    slide, width = 30, 5
    prev = []
    for f in range(8):
        window = [tuple(x) for x in tbox.tolist()] + [tuple(x) for x in abox[f * slide:(f + width) * slide].tolist()]
        for t in prev:  # the reference's firing protocol: the whole previous window leaves, the current one arrives
            r2r.remove(t)
        for t in window:
            r2r.add(t)
        got = r2r.materialize()
        assert set(got) == expected_inferred(np.array(window, np.uint32), r2r), f"firing {f}"
        assert r2r.last_mode == ("fixpoint" if f == 0 else "maintain")
        # the store: the window's triples once each (in their segments) plus the inferred segment
        s, p, o = ctx.store_download()
        store = np.stack([s, p, o], axis=1)
        assert len(store) == len(set(window)) + len(got)
        assert rows_set(store) == set(window) | set(got)
        prev = window
    # every segment tag is a live firing (or the inferred segment): slides that left were evicted
    tags = {t for t, _ in ctx.segs} - {c.KB_TAG_INFERRED}
    assert tags == set(r2r._live)
    assert all(n > 0 for n in r2r._live.values())


def test_segment_bookkeeping_evicts_a_slide_only_when_all_of_it_left():
    tbox, abox, rules = taxonomy_window()
    r2r = make_r2r(rules)
    a, b = [tuple(x) for x in abox[:10].tolist()], [tuple(x) for x in abox[10:20].tolist()]
    for t in a:
        r2r.add(t)
    r2r.materialize()
    for t in b:
        r2r.add(t)
    r2r.materialize()
    assert set(r2r._live) == {1, 2}
    for t in a[:9]:
        r2r.remove(t)
    r2r.materialize()
    assert r2r.ctx.calls[-1] == ("maintain", ([], None, 3)) and 1 in r2r._live  # (the next firing's tag: no adds took it yet)
    r2r.remove(a[9])
    r2r.materialize()
    assert r2r.ctx.calls[-1] == ("maintain", ([1], None, 3)) and set(r2r._live) == {2}
    # a triple added twice in one firing, or again while its slide is live, is one triple of one segment
    r2r.add(a[0]); r2r.add(a[0]); r2r.add(b[0])
    r2r.materialize()
    assert r2r.ctx.calls[-1] == ("maintain", ([], 1, 3)) and r2r._live == {2: 10, 3: 1}


def test_rule_change_falls_back_to_the_fixpoint():
    tbox, abox, rules = taxonomy_window()
    r2r = make_r2r(rules[:1])
    for t in tbox.tolist() + abox[:50].tolist():
        r2r.add(tuple(t))
    r2r.materialize()
    assert r2r.last_mode == "fixpoint"
    r2r.add(tuple(abox[50].tolist()))
    r2r.materialize()
    assert r2r.last_mode == "maintain"
    r2r.add_reasoning_rules(rules[1:])  # other rules: the store is not closed under them
    got = r2r.materialize()
    assert r2r.last_mode == "fixpoint"
    window = np.concatenate([tbox, abox[:51]], axis=0)
    assert set(got) == expected_inferred(window, r2r)
    r2r.remove(tuple(abox[0].tolist()))
    r2r.materialize()
    assert r2r.last_mode == "maintain"


def test_a_plain_store_change_voids_the_token():
    tbox, abox, rules = taxonomy_window()
    r2r = make_r2r(rules)
    for t in tbox.tolist() + abox[:40].tolist():
        r2r.add(tuple(t))
    r2r.materialize()
    r2r.ctx.store_append([1], [2], [3], 777)  # outside the window object
    with pytest.raises(c.KolibrieError) as e:
        r2r.ctx.datalog_maintain([], [], None, 0)
    assert e.value.status == c.KB_E_INVALID


def test_oracle_contract_on_the_corner_cases():
    """the CPU restatement itself: a fact in two segments does not move; a removed but derivable base fact becomes inferred; an
    inferred fact that is added becomes a base fact and is stored once"""
    from tests.sharded_cases import chain_case

    _, rules, _, ids = chain_case(n=10)
    E = ids["edge"]
    ctx = WindowOracleCtx()
    ctx.store_append([1, 2, 1], [E, E, E], [2, 3, 3], 1)  # 1->2, 2->3, 1->3 (1->3 also derivable)
    ctx.store_append([1], [E], [2], 2)                    # 1->2 in a second segment
    ctx.datalog_fixpoint(rules)
    assert ctx.inferred() == set()
    rem, new, st = ctx.datalog_maintain(rules, [2], None, 0)  # 1->2 still in segment 1: nothing moves
    assert st.base_removed == 0 and rem.n_rows == 0 and new.n_rows == 0
    rem, new, st = ctx.datalog_maintain(rules, [1], np.array([[1, E, 2], [2, E, 3]], np.uint32), 3)  # 1->3 leaves the base, derivable
    assert st.base_removed == 1 and rows_set(new.to_numpy([0, 1, 2])) == {(1, E, 3)}
    rem, new, st = ctx.datalog_maintain(rules, [], np.array([[1, E, 3]], np.uint32), 4)  # the inferred fact becomes base
    assert rows_set(rem.to_numpy([0, 1, 2])) == {(1, E, 3)} and ctx.inferred() == set()
    s, p, o = ctx.store_download()
    assert sorted(map(tuple, np.stack([s, p, o], 1).tolist())).count((1, E, 3)) == 1


def test_oracle_base_counts_cover_the_rule_predicates_only():
    """as the header states: a triple of a predicate no rule mentions takes no part in the closure and is not counted"""
    from tests.sharded_cases import chain_case

    _, rules, _, ids = chain_case(n=10)
    E, OTHER = ids["edge"], 99
    ctx = WindowOracleCtx()
    ctx.store_append([1, 2, 5], [E, E, OTHER], [2, 3, 6], 1)
    ctx.datalog_fixpoint(rules)
    rem, new, st = ctx.datalog_maintain(rules, [1], np.array([[2, E, 3], [7, OTHER, 8]], np.uint32), 2)
    assert st.base_removed == 1 and st.base_added == 0  # 1->2 left; (5 OTHER 6) left and (7 OTHER 8) arrived, uncounted


def test_numeric_table_voids_the_token_only_for_rules_that_compare_numbers():
    from tests.sharded_cases import chain_case

    _, rules, _, ids = chain_case(n=10)
    E = ids["edge"]
    ctx = WindowOracleCtx()
    ctx.store_append([1, 2], [E, E], [2, 3], 1)
    ctx.datalog_fixpoint(rules)
    ctx.dict_numeric_load(np.zeros(8), np.zeros(8, np.uint8))
    ctx.datalog_maintain(rules, [], np.array([[3, E, 4]], np.uint32), 2)  # no rule filter: still closed
    numeric = [dict(r, filters=[c.KbRuleFilter(0, c.CMP_GT, 0, 0, 1.0)]) for r in rules]
    ctx.store_evict(c.KB_TAG_INFERRED)
    ctx.datalog_fixpoint(numeric)
    ctx.dict_numeric_load(np.zeros(9), np.zeros(9, np.uint8))
    with pytest.raises(c.KolibrieError) as e:
        ctx.datalog_maintain(numeric, [], np.array([[4, E, 5]], np.uint32), 3)
    assert e.value.status == c.KB_E_INVALID
