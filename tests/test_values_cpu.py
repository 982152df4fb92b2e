"""CPU: the restatement of VALUES and of the joins above it (tests/values_reference.py) on hand-worked cases, and the planner mirror's
Values leaf (cost, cardinality, the join operator it picks)."""
import pytest

from kolibrie_b200 import engine as E
from kolibrie_b200 import planner as PL
from tests import values_reference as V


def enc():
    d = E.Dictionary()
    d.encode("<pre>")  # id 0 exists before the block
    return d


def test_encode_order_repeats_and_new_strings():
    d = enc()
    rows = V.values(["?a", "?b"], [["x", "<pre>"], ["y", "x"], ["<pre>", "z"]], d.encode)
    assert d.id_to_string == ["<pre>", "x", "y", "z"]  # row-major, first-seen order; "<pre>" keeps id 0
    assert rows == [{"a": 1, "b": 0}, {"a": 2, "b": 1}, {"a": 0, "b": 3}]


def test_verbatim_terms():
    d = E.Dictionary()
    V.values(["?a"], [["ex:thing"], ["<http://x>"], ['"5"']], d.encode)
    assert d.id_to_string == ["ex:thing", "<http://x>", '"5"']  # no prefix resolution, no bracket stripping


def test_all_undef_rows_are_dropped_and_encode_nothing():
    d = enc()
    rows = V.values(["?a", "?b"], [[None, None], ["q", None], [None, None], [None, "r"]], d.encode)
    assert rows == [{"a": 1}, {"b": 2}]
    assert d.id_to_string == ["<pre>", "q", "r"]


def test_repeated_header_variable_later_defined_cell_wins():
    d = enc()
    rows = V.values(["?a", "?b", "?a"], [["p", "q", "r"], ["s", "t", None], [None, "u", "v"]], d.encode)
    assert d.id_to_string == ["<pre>", "p", "q", "r", "s", "t", "u", "v"]  # both cells of ?a are encoded
    assert rows == [{"a": 3, "b": 2}, {"a": 4, "b": 5}, {"a": 7, "b": 6}]


def test_short_rows_are_undef_at_the_end():
    d = enc()
    rows = V.values(["?a", "?b", "?c"], [["p"], ["q", "r"], []], d.encode)
    assert rows == [{"a": 1}, {"a": 2, "b": 3}]


def test_key_is_read_from_row_zero():
    left = [{"x": 1}, {"x": 2, "y": 7}]
    right = [{"x": 1, "y": 9}, {"x": 2, "y": 8}]
    assert V.common_vars(left, right) == ["x"]  # ?y is shared, but row 0 of the left side lacks it
    # ?y is not compared: (x=2, y=7) pairs with (x=2, y=8); HashJoin keeps the left cell
    assert V.bag(V.hash_join(left, right)) == V.bag([{"x": 1, "y": 9}, {"x": 2, "y": 7}])
    assert V.bag(V.nested_loop_join(left, right)) == V.bag([{"x": 1, "y": 9}])  # compatible mappings only


def test_a_later_row_lacking_the_key_panics():
    left = [{"x": 1, "y": 2}, {"y": 3}]
    right = [{"x": 1}]
    for j in (V.hash_join, V.optimized_hash_join, V.merge_join, V.parallel_join):
        with pytest.raises(V.Panic):
            j(left, right)
    assert V.bag(V.nested_loop_join(left, right)) == V.bag([{"x": 1, "y": 2}, {"x": 1, "y": 3}])


@pytest.mark.parametrize("n_left", [1, 2, 3])
def test_every_merge_policy(n_left):
    """key ?x (row 0 of the left side lacks ?y); ?y shared outside the key, bound on both sides with different values"""
    left = [{"x": 9}] + [{"x": 1, "y": 10 + i} for i in range(n_left)]
    right = [{"x": 1, "y": 20}, {"x": 1, "y": 21}]
    lf = V.bag([{"x": 1, "y": l["y"]} for l in left[1:] for _ in right])
    rf = V.bag([{"x": 1, "y": r["y"]} for _ in left[1:] for r in right])
    assert V.bag(V.hash_join(left, right)) == lf
    assert V.bag(V.merge_join(left, right)) == lf
    assert V.bag(V.parallel_join(left, right)) == lf
    # OptimizedHashJoin: build = the smaller side (left on ties), the probe row wins
    assert V.bag(V.optimized_hash_join(left, right)) == (rf if len(left) <= len(right) else lf)


def test_cartesian_product_is_right_first():
    left = [{"y": 5}, {"x": 1}]
    right = [{"x": 2}]
    assert V.common_vars(left, right) == []
    want = V.bag([{"y": 5, "x": 2}, {"x": 2}])
    for j in (V.hash_join, V.optimized_hash_join, V.parallel_join):
        assert V.bag(j(left, right)) == want


def test_empty_sides():
    for j in V.JOINS.values():
        assert j([], [{"x": 1}]) == [] and j([{"x": 1}], []) == []


def test_bind_join_leaves_unbound_variables_free():
    triples = [(1, 100, 5), (2, 100, 6)]
    left = [{"x": 1}, {"y": 6}]
    got = V.bind_join(left, ("?x", 100, "?y"), triples)
    assert V.bag(got) == V.bag([{"x": 1, "y": 5}, {"x": 2, "y": 6}])
    assert V.bag(got) == V.bag(V.nested_loop_join(left, V.scan(("?x", 100, "?y"), triples)))


def planner(total=1000, pc=None):
    return PL.Streamertail(PL.DatabaseStats.from_counts(total, pc or {100: total}), gpu=True)


def test_planner_values_cost_and_cardinality():
    st = planner()
    v = E.Values(["?x"], [["a"], ["b"], [None]])
    assert st.cost.estimate_cost(v) == 3 and st.cost.estimate_output_cardinality(v) == 3
    plan = st.find_best_plan(PL.LValues(["?x"], [["a"]]))
    assert plan == E.Values(["?x"], [["a"]])


def test_planner_joins_values_with_the_reference_candidates_only():
    st = planner()
    lv = PL.LValues(["?x"], [["a"], ["b"]])
    plan = st.find_best_plan(PL.build_logical_plan([(E.Variable("x"), E.Constant(100), E.Variable("y"))], values=lv))
    assert isinstance(plan, (E.HashJoin, E.OptimizedHashJoin, E.NestedLoopJoin, E.ParallelJoin))
    assert plan.left == E.Values(["?x"], [["a"], ["b"]])  # the cheaper side goes left
    assert not PL.uses_device(plan)
    costs = {type(p).__name__: st.cost.estimate_cost(p) for p in (E.OptimizedHashJoin(plan.left, plan.right), E.HashJoin(plan.left, plan.right),
                                                                   E.ParallelJoin(plan.left, plan.right), E.NestedLoopJoin(plan.left, plan.right))}
    assert st.cost.estimate_cost(plan) == min(costs.values())


def test_planner_star_detection_ignores_the_values_block():
    """collect_patterns skips Values (optimizer.rs:178): three patterns on one variable make a star, built from the patterns alone"""
    st = planner()
    pats = [(E.Variable("x"), E.Constant(100 + k), E.Variable("o%d" % k)) for k in range(3)]
    plan = st.find_best_plan(PL.build_logical_plan(pats, values=PL.LValues(["?x"], [["a"]])))
    assert "Values" not in repr(plan)


def test_planner_orders_and_gates_joins_above_values_as_the_reference():
    """VALUES (?s ?w) {10 rows} . ?s p ?o . ?s q ?w with |p| = 100, |q| = 105 of 205 triples, worked by hand from optimizer.rs:
    inner Join(Values, p): cost 10 <= 100, no swap; card max(int(min(10, 100) * 100/205), 1) = 4; cost 10 + 100 + int(10 * 100 * 100/205) = 597.
    top Join(inner, q): 597 > 105, so the q scan goes left; both cardinalities (105, 4) are below 1000, so NestedLoopJoin is a candidate."""
    st = planner(205, {100: 100, 101: 105})
    s, o, w = E.Variable("s"), E.Variable("o"), E.Variable("w")
    pp, pq = (s, E.Constant(100), o), (s, E.Constant(101), w)
    lv = PL.LValues(["?s", "?w"], [["a%d" % k, "b"] for k in range(10)])
    logical = PL.build_logical_plan([pp, pq], values=lv)
    inner = logical.left
    assert st._ref_logical_cost(lv) == 10 and st._ref_logical_card(inner) == 4 and st._ref_logical_cost(inner) == 597
    plan = st.find_best_plan(logical)
    assert plan.left.pattern == pq and plan.right.left == E.Values(lv.variables, lv.values) and plan.right.right.pattern == pp
    cands = [E.OptimizedHashJoin(plan.left, plan.right), E.HashJoin(plan.left, plan.right), E.ParallelJoin(plan.left, plan.right),
             E.NestedLoopJoin(plan.left, plan.right)]
    assert st.cost.estimate_cost(plan) == min(st.cost.estimate_cost(p) for p in cands)
    # without VALUES the mirror's ordering is unchanged: the larger pattern stays right
    plain = st.find_best_plan(PL.build_logical_plan([pp, pq]))
    assert plain.left.pattern == pp
