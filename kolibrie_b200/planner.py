"""Planner hook: the part of Streamertail (kolibrie/src/streamertail_optimizer) that decides WHICH physical operator runs, mirrored for
the hot path and extended by the device operators, so that the optimizer *chooses* device plans by cost instead of a shim pattern-matching
CPU plans after the fact (SURVEY.md §8 (f)3).

Mirrored (paths relative to kolibrie/src/streamertail_optimizer of the Kolibrie checkout):
* `LogicalOperator::{Scan, Selection, Projection, Join, Values}` operators/logical.rs
* `DatabaseStats` (predicate / subject / object cardinalities)  stats.rs, consumed by cost/estimator.rs:193-255
* `CostConstants`, `CostEstimator::estimate_cost`               cost/estimator.rs:17-29, 43-191 (the hot-path variants)
* `Streamertail::find_best_plan`                                optimizer.rs:60-62, 84-152 (star detection), 192-300 (candidates),
                                                                400-480 (star construction), 482-501 (scan choice)

Added: `GpuStarJoin`, `GpuHashJoin`, `GpuBindJoin`, `GpuIndexScan` physical operators and `GpuCostConstants`. The reference's cost unit
is "one row touched by the CPU index scan" (COST_PER_ROW_INDEX_SCAN = 1), taken as ~0.1 us of host time. The device constants are
expressed in the same unit: a device operator costs a fixed ~25 us (launch + the stream synchronisation that hands the row count back:
250 units; bench.py's sync_path minus its device time is ~34 us per query on an H100, result allocation included) and then one unit per
~16 000 probed rows (~6 ps per row; the H100 probes 16.7 M rows in 0.158 ms, ~9.5 ps) and per ~3 000 scanned triples (~33 ps; the
H100 scans and builds over 100 M triples in 0.68 ms). The constants only rank device plans against CPU plans whose costs differ by orders of
magnitude, so factors of two between GPUs do not change a choice. A device plan therefore wins
as soon as a query touches more than a few hundred rows and loses for point lookups — which is what the candidates' costs say.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

from . import engine as E


# ---------------------------------------------------------------------------------------------------------------------
# logical operators (operators/logical.rs)
@dataclass
class Scan:
    pattern: E.TriplePattern


@dataclass
class Selection:
    predicate: object
    condition: E.Condition


@dataclass
class LProjection:
    predicate: object
    variables: List[str]


@dataclass
class Join:
    left: object
    right: object


@dataclass
class LValues:
    """LogicalOperator::Values: a VALUES block, rows of terms in header order, None for UNDEF"""
    variables: List[str]
    values: List[List[Optional[str]]]


def build_logical_plan(patterns: Sequence[E.TriplePattern], condition: Optional[E.Condition] = None, variables: Optional[List[str]] = None,
                       values: Optional[LValues] = None):
    """build_logical_plan (utils.rs:101-191): left-deep joins in textual order, then the selection, then the projection. A VALUES
    block is the base of the chain and every pattern is joined onto it (utils.rs:110-171)."""
    plan = values if values is not None else Scan(patterns[0])
    for p in patterns[0 if values is not None else 1:]:
        plan = Join(plan, Scan(p))
    if condition is not None:
        plan = Selection(plan, condition)
    if variables is not None:
        plan = LProjection(plan, variables)
    return plan


# ---------------------------------------------------------------------------------------------------------------------
# device physical operators (next to engine.TableScan / IndexScan / StarJoin / HashJoin ...)
@dataclass
class GpuStarJoin:
    join_var: str
    patterns: List[E.TriplePattern]


@dataclass
class GpuHashJoin:
    left: object
    right: object


@dataclass
class GpuBindJoin:  # left relation joined with one store pattern through the index's persistent table (kb_bind_join)
    left: object
    pattern: E.TriplePattern


@dataclass
class GpuIndexScan:
    pattern: E.TriplePattern


class DatabaseStats:
    """stats.rs: what the estimator reads — total triples and per-term cardinalities by position"""

    def __init__(self, triples):
        self.total_triples = 0
        self.predicate_card: Dict[int, int] = {}
        self.subject_card: Dict[int, int] = {}
        self.object_card: Dict[int, int] = {}
        self.quoted_triple_count = 0
        for s, p, o in triples:
            self.total_triples += 1
            self.subject_card[s] = self.subject_card.get(s, 0) + 1
            self.predicate_card[p] = self.predicate_card.get(p, 0) + 1
            self.object_card[o] = self.object_card.get(o, 0) + 1

    @classmethod
    def from_counts(cls, total: int, predicate_card: Dict[int, int], subject_card=None, object_card=None, quoted_triple_count: int = 0):
        st = cls(())
        st.total_triples = total
        st.predicate_card = dict(predicate_card)
        st.subject_card = dict(subject_card or {})
        st.object_card = dict(object_card or {})
        st.quoted_triple_count = quoted_triple_count
        return st

    def get_predicate_cardinality(self, p):
        return self.predicate_card.get(p, 0)

    def get_subject_cardinality(self, s):
        return self.subject_card.get(s, 0)

    def get_object_cardinality(self, o):
        return self.object_card.get(o, 0)


class CostConstants:  # cost/estimator.rs:17-29, verbatim values
    COST_PER_ROW_SCAN = 100
    COST_PER_ROW_INDEX_SCAN = 1
    COST_PER_FILTER = 1
    COST_PER_ROW_JOIN = 2
    COST_PER_ROW_NESTED_LOOP = 10
    COST_PER_PROJECTION = 1
    COST_PER_ROW_OPTIMIZED_JOIN = 1
    TUPLE_COST = 1


class GpuCostConstants:
    """same unit as CostConstants (one CPU index-scan row ~ 0.1 us); derivation in the module docstring"""
    LAUNCH = 250              # one device operator: launch + synchronisation + row count back (~25 us)
    ROWS_PER_UNIT_PROBE = 16000   # probe / index-scan rows per cost unit (~6 ps each; probe_index_kernel on the H100: ~9.5 ps)
    ROWS_PER_UNIT_SCAN = 3000     # store-scanning rows per cost unit (~33 ps each; scan_star_kernel on the H100: ~6.8 ps)
    ROWS_PER_UNIT_JOIN = 4000     # build + probe of a materialised join (~25 ps per input row; not timed on the H100)


def _is_const(t) -> bool:
    return isinstance(t, E.Constant)


class CostEstimator:
    def __init__(self, stats: DatabaseStats, indexed: bool = True):
        self.stats = stats
        self.indexed = indexed  # the device store has its predicate index (kb_store_build_index)

    # ---- cardinalities (estimator.rs:193-255)
    def estimate_cardinality(self, pattern) -> int:
        s, p, o = pattern
        cs, cp, co = _is_const(s), _is_const(p), _is_const(o)
        st = self.stats
        if any(isinstance(t, E.QuotedTriple) for t in pattern):
            bound = sum(1 for t in pattern if _is_const(t))
            qt = max(st.quoted_triple_count, 1)
            return [min(qt, st.total_triples), max(qt // 5, 1), max(qt // 10, 1), 1][min(bound, 3)]
        if cs and cp and co:
            return 1
        if cs and cp:
            return max(min(st.get_subject_cardinality(s.id), st.get_predicate_cardinality(p.id)), 1)
        if cs and co:
            return max(min(st.get_subject_cardinality(s.id), st.get_object_cardinality(o.id)), 1)
        if cp and co:
            return max(min(st.get_predicate_cardinality(p.id), st.get_object_cardinality(o.id)), 1)
        if cs:
            return max(st.get_subject_cardinality(s.id), 1)
        if cp:
            return max(st.get_predicate_cardinality(p.id), 1)
        if co:
            return max(st.get_object_cardinality(o.id), 1)
        return st.total_triples

    @staticmethod
    def count_bound_variables(pattern) -> int:
        return sum(1 for t in pattern if _is_const(t))

    # ---- selectivities (estimator.rs:257-311)
    def estimate_selectivity(self, condition: E.Condition) -> float:
        def rec(e) -> float:
            if isinstance(e, E.Comparison):
                return {"=": 0.05, "!=": 0.95, ">": 0.25, "<": 0.25, ">=": 0.30, "<=": 0.30}.get(e.op, 0.5)
            if isinstance(e, E.And):
                return rec(e.left) * rec(e.right)
            if isinstance(e, E.Or):
                a, b = rec(e.left), rec(e.right)
                return a + b - a * b
            if isinstance(e, E.Not):
                return 1.0 - rec(e.inner)
            if isinstance(e, E.FunctionCall):
                return 0.1 if e.name == "isTRIPLE" else 0.5
            return 0.5

        return rec(condition.expression)

    def estimate_output_cardinality(self, plan) -> int:
        if isinstance(plan, (E.TableScan, E.IndexScan, GpuIndexScan)):
            return self.estimate_cardinality(plan.pattern)
        if isinstance(plan, E.Filter):
            return int(self.estimate_output_cardinality(plan.input) * self.estimate_selectivity(plan.condition))
        if isinstance(plan, E.Projection):
            return self.estimate_output_cardinality(plan.input)
        if isinstance(plan, (E.StarJoin, GpuStarJoin)):
            return min(self.estimate_cardinality(p) for p in plan.patterns)
        if isinstance(plan, GpuBindJoin):
            return self.estimate_output_cardinality(plan.left)
        if isinstance(plan, (E.HashJoin, E.OptimizedHashJoin, E.NestedLoopJoin, E.ParallelJoin, GpuHashJoin)):
            return max(self.estimate_output_cardinality(plan.left), self.estimate_output_cardinality(plan.right))
        if isinstance(plan, E.InMemoryBuffer):
            return len(plan.content)
        if isinstance(plan, E.Values):  # estimator.rs:399-402
            return len(plan.values)
        return 1

    # ---- costs (estimator.rs:43-191) + the device operators
    def estimate_cost(self, plan) -> int:
        C, G = CostConstants, GpuCostConstants
        if isinstance(plan, E.TableScan):
            return self.estimate_cardinality(plan.pattern) * C.COST_PER_ROW_SCAN
        if isinstance(plan, E.IndexScan):
            card = self.estimate_cardinality(plan.pattern)
            discount = {0: 1, 1: 10, 2: 100, 3: 1000}.get(self.count_bound_variables(plan.pattern), 1)
            return (card * C.COST_PER_ROW_INDEX_SCAN) // discount
        if isinstance(plan, GpuIndexScan):
            # with the store index a constant-predicate pattern reads its slice (or one table slot / one directory run); otherwise the store is scanned
            if self.indexed and _is_const(plan.pattern[1]):
                return G.LAUNCH + self.estimate_cardinality(plan.pattern) // G.ROWS_PER_UNIT_PROBE
            return G.LAUNCH + self.stats.total_triples // G.ROWS_PER_UNIT_SCAN
        if isinstance(plan, E.Filter):
            return int(self.estimate_cost(plan.input) * self.estimate_selectivity(plan.condition)) + C.COST_PER_FILTER
        if isinstance(plan, E.OptimizedHashJoin):
            return (self.estimate_cost(plan.left) + self.estimate_cost(plan.right)
                    + (self.estimate_output_cardinality(plan.left) + self.estimate_output_cardinality(plan.right)) * C.COST_PER_ROW_OPTIMIZED_JOIN)
        if isinstance(plan, E.HashJoin):
            return (self.estimate_cost(plan.left) + self.estimate_cost(plan.right)
                    + (self.estimate_output_cardinality(plan.left) + self.estimate_output_cardinality(plan.right)) * C.COST_PER_ROW_JOIN)
        if isinstance(plan, E.NestedLoopJoin):
            return (self.estimate_cost(plan.left) + self.estimate_cost(plan.right)
                    + self.estimate_output_cardinality(plan.left) * self.estimate_output_cardinality(plan.right) * C.COST_PER_ROW_NESTED_LOOP)
        if isinstance(plan, E.ParallelJoin):
            if isinstance(plan.right, (E.TableScan, E.IndexScan)):  # can_use_efficient_join: the right side is a scan -> bind join
                return self.estimate_cost(plan.left) + self.estimate_output_cardinality(plan.left) * C.COST_PER_ROW_JOIN // 20
            return (self.estimate_cost(plan.left) + self.estimate_cost(plan.right)
                    + (self.estimate_output_cardinality(plan.left) + self.estimate_output_cardinality(plan.right)) * C.COST_PER_ROW_JOIN // 2)
        if isinstance(plan, E.Projection):
            return self.estimate_cost(plan.input) + C.COST_PER_PROJECTION
        if isinstance(plan, E.StarJoin):
            costs = sorted(self.estimate_cardinality(p) for p in plan.patterns)
            return costs[0] * C.COST_PER_ROW_INDEX_SCAN + sum(costs[1:]) * C.COST_PER_ROW_INDEX_SCAN // 10
        if isinstance(plan, GpuStarJoin):
            # ONE kernel: the most selective slice is the probe stream, every other pattern a table lookup per probe row
            cards = sorted(self.estimate_cardinality(p) for p in plan.patterns)
            if self.indexed and all(_is_const(p[1]) and not _is_const(p[0]) and not _is_const(p[2]) for p in plan.patterns):
                return G.LAUNCH + cards[0] * len(cards) // G.ROWS_PER_UNIT_PROBE
            return 2 * G.LAUNCH + self.stats.total_triples // G.ROWS_PER_UNIT_SCAN + cards[-1] * len(cards) // G.ROWS_PER_UNIT_PROBE
        if isinstance(plan, GpuBindJoin):
            return self.estimate_cost(plan.left) + G.LAUNCH + self.estimate_output_cardinality(plan.left) // G.ROWS_PER_UNIT_PROBE
        if isinstance(plan, GpuHashJoin):
            return (self.estimate_cost(plan.left) + self.estimate_cost(plan.right) + 2 * G.LAUNCH
                    + (self.estimate_output_cardinality(plan.left) + self.estimate_output_cardinality(plan.right)) // G.ROWS_PER_UNIT_JOIN)
        if isinstance(plan, E.InMemoryBuffer):
            return 0
        if isinstance(plan, E.Values):  # estimator.rs:169-173
            return len(plan.values) * C.TUPLE_COST
        raise TypeError(plan)


class Streamertail:
    """optimizer.rs: find_best_plan over the hot-path logical operators. gpu=True adds the device candidates; the cheapest wins."""

    def __init__(self, stats: DatabaseStats, gpu: bool = True, indexed: bool = True):
        self.stats = stats
        self.gpu = gpu
        self.cost = CostEstimator(stats, indexed)

    # ---- star detection (optimizer.rs:84-152)
    def collect_patterns(self, plan, out):
        if isinstance(plan, Scan):
            out.append(plan.pattern)
        elif isinstance(plan, Join):
            self.collect_patterns(plan.left, out)
            self.collect_patterns(plan.right, out)
        elif isinstance(plan, (Selection, LProjection)):
            self.collect_patterns(plan.predicate, out)

    def is_star_query(self, plan):
        patterns: List[E.TriplePattern] = []
        self.collect_patterns(plan, patterns)
        if len(patterns) < 3:
            return None
        var_counts: Dict[str, List[int]] = {}
        for idx, pat in enumerate(patterns):
            for t in pat:
                if isinstance(t, E.Variable):
                    var_counts.setdefault(t.name, []).append(idx)
        star_vars = sorted(((v, ix) for v, ix in sorted(var_counts.items()) if len(ix) >= 2), key=lambda x: -len(x[1]))  # BTreeMap order, stable sort
        used, stars = set(), []
        for var, ix in star_vars:
            avail = [i for i in ix if i not in used]
            if len(avail) >= 2:
                used.update(avail)
                stars.append((var, [patterns[i] for i in avail]))
        return stars or None

    def _star_op(self, var, pats):
        cpu = E.StarJoin(var, pats)
        if not self.gpu:
            return cpu
        dev = GpuStarJoin(var, pats)
        return dev if self.cost.estimate_cost(dev) <= self.cost.estimate_cost(cpu) else cpu

    def _bind(self, left, pattern):
        """ParallelJoin(result, IndexScan(pattern)) (optimizer.rs:441-451) or its device counterpart"""
        cpu = E.ParallelJoin(left, E.IndexScan(pattern))
        if not self.gpu:
            return cpu
        dev = GpuBindJoin(left, pattern)
        return dev if self.cost.estimate_cost(dev) <= self.cost.estimate_cost(cpu) else cpu

    def build_star_join_from_patterns(self, stars, logical_plan):
        allp: List[E.TriplePattern] = []
        self.collect_patterns(logical_plan, allp)
        used = set()
        for _, sp in stars:
            for p in sp:
                if p in allp:
                    used.add(allp.index(p))
        if len(stars) > 1:
            ordered = sorted(stars, key=lambda s_: -sum(1 for p in s_[1] if any(_is_const(t) for t in p)))
            var, pats = ordered[0]
            result = self._star_op(var, pats)
            for _, pats in ordered[1:]:
                for p in pats:
                    result = self._bind(result, p)
        else:
            var, pats = stars[0]
            result = self._star_op(var, pats)
        for i, p in enumerate(allp):
            if i not in used:
                result = self._bind(result, p)
        return result

    # ---- scans (optimizer.rs:482-501)
    def choose_best_scan(self, pattern):
        bound = self.cost.count_bound_variables(pattern)
        size = self.cost.estimate_cardinality(pattern)
        cpu = E.IndexScan(pattern) if bound >= 2 or (bound == 1 and size < 10000) else E.TableScan(pattern)
        if not self.gpu or any(isinstance(t, E.QuotedTriple) for t in pattern):
            return cpu
        dev = GpuIndexScan(pattern)
        return dev if self.cost.estimate_cost(dev) <= self.cost.estimate_cost(cpu) else cpu

    def _logical_card(self, plan) -> int:
        if isinstance(plan, Scan):
            return self.cost.estimate_cardinality(plan.pattern)
        if isinstance(plan, Join):
            return max(self._logical_card(plan.left), self._logical_card(plan.right))
        if isinstance(plan, Selection):
            return int(self._logical_card(plan.predicate) * self.cost.estimate_selectivity(plan.condition))
        if isinstance(plan, LProjection):
            return self._logical_card(plan.predicate)
        if isinstance(plan, LValues):  # optimizer.rs:762-764
            return len(plan.values)
        return 1

    # ---- the logical estimates of optimizer.rs:643-757, used to order and gate the joins of a plan with a VALUES block: over UNDEF
    # cells the join operators answer differently, so the side order and the operator must be the reference's
    def _join_selectivity(self, l, r) -> float:  # estimate_join_selectivity (optimizer.rs:698-709), database_stats.rs:129-152
        def pred(plan):  # extract_predicate_from_plan (optimizer.rs:712-730)
            if isinstance(plan, Scan):
                return plan.pattern[1].id if _is_const(plan.pattern[1]) else None
            if isinstance(plan, Join):
                return pred(plan.left)
            if isinstance(plan, (Selection, LProjection)):
                return pred(plan.predicate)
            return None
        p = pred(l)
        if p is None:
            p = pred(r)
        if p is None or self.stats.total_triples <= 0:
            return 0.1
        return self.stats.get_predicate_cardinality(p) / self.stats.total_triples

    def _ref_logical_card(self, plan) -> int:  # estimate_output_cardinality_from_logical (optimizer.rs:733-768)
        if isinstance(plan, Scan):
            return self.cost.estimate_cardinality(plan.pattern)
        if isinstance(plan, Selection):
            return max(int(self._ref_logical_card(plan.predicate) * self.cost.estimate_selectivity(plan.condition)), 1)
        if isinstance(plan, LProjection):
            return self._ref_logical_card(plan.predicate)
        if isinstance(plan, Join):
            lc, rc = self._ref_logical_card(plan.left), self._ref_logical_card(plan.right)
            return max(int(min(lc, rc) * self._join_selectivity(plan.left, plan.right)), 1)
        if isinstance(plan, LValues):
            return len(plan.values)
        raise TypeError(plan)

    def _ref_logical_cost(self, plan) -> int:  # estimate_logical_cost (optimizer.rs:643-695)
        if isinstance(plan, Scan):
            return self.cost.estimate_cardinality(plan.pattern)
        if isinstance(plan, Join):
            lcard, rcard = self._ref_logical_card(plan.left), self._ref_logical_card(plan.right)
            return (self._ref_logical_cost(plan.left) + self._ref_logical_cost(plan.right)
                    + int(lcard * rcard * self._join_selectivity(plan.left, plan.right)))
        if isinstance(plan, Selection):
            return int(self._ref_logical_cost(plan.predicate) * self.cost.estimate_selectivity(plan.condition))
        if isinstance(plan, LProjection):
            return self._ref_logical_cost(plan.predicate)
        if isinstance(plan, LValues):
            return len(plan.values)
        raise TypeError(plan)

    def find_best_plan(self, plan):
        # star shapes first (optimizer.rs:200-232)
        if isinstance(plan, LProjection) and isinstance(plan.predicate, Selection):
            stars = self.is_star_query(plan.predicate.predicate)
            if stars:
                return E.Projection(E.Filter(self.build_star_join_from_patterns(stars, plan.predicate.predicate), plan.predicate.condition), plan.variables)
        if isinstance(plan, Selection):
            stars = self.is_star_query(plan.predicate)
            if stars:
                return E.Filter(self.build_star_join_from_patterns(stars, plan.predicate), plan.condition)
        if not isinstance(plan, (Selection, LProjection)):
            stars = self.is_star_query(plan)
            if stars:
                return self.build_star_join_from_patterns(stars, plan)
        cands = []
        if isinstance(plan, Scan):
            cands.append(self.choose_best_scan(plan.pattern))
        elif isinstance(plan, LValues):  # a leaf (optimizer.rs:325-330)
            cands.append(E.Values(plan.variables, plan.values))
        elif isinstance(plan, Selection):
            cands.append(E.Filter(self.find_best_plan(plan.predicate), plan.condition))
        elif isinstance(plan, LProjection):
            cands.append(E.Projection(self.find_best_plan(plan.predicate), plan.variables))
        elif isinstance(plan, Join):
            l, r = plan.left, plan.right
            values = _has_values(l) or _has_values(r)
            cost = self._ref_logical_cost if values else self._logical_card
            card = self._ref_logical_card if values else self._logical_card
            if cost(l) > cost(r):  # cheaper side first (optimizer.rs:254-262)
                l, r = r, l
            bl, br = self.find_best_plan(l), self.find_best_plan(r)
            cands += [E.OptimizedHashJoin(bl, br), E.HashJoin(bl, br), E.ParallelJoin(bl, br)]
            if card(l) < 1000 and card(r) < 1000:  # optimizer.rs:276-285
                cands.append(E.NestedLoopJoin(bl, br))
            # over a VALUES block the join operators differ in what they do with UNDEF cells (ExecutionEngine._join): only the
            # reference's own candidates, so that the mirror picks the operator the reference picks
            if self.gpu and not values:
                cands.append(GpuHashJoin(bl, br))
                if isinstance(r, Scan) and not any(isinstance(t, E.QuotedTriple) for t in r.pattern):
                    cands.append(GpuBindJoin(bl, r.pattern))
        else:
            raise TypeError(plan)
        return min(cands, key=self.cost.estimate_cost)


def _has_values(plan) -> bool:
    if isinstance(plan, LValues):
        return True
    return any(_has_values(getattr(plan, a)) for a in ("left", "right", "predicate") if hasattr(plan, a))


def uses_device(plan) -> bool:
    if isinstance(plan, (GpuStarJoin, GpuHashJoin, GpuBindJoin, GpuIndexScan)):
        return True
    for attr in ("input", "left", "right"):
        if hasattr(plan, attr) and uses_device(getattr(plan, attr)):
            return True
    return False


def lower_to_engine(plan):
    """the device operators as the operators kolibrie_b200.engine.ExecutionEngine runs (every engine operator executes on the device:
    the distinction matters to the reference's optimizer, which also has the CPU executor to choose from)"""
    if isinstance(plan, GpuStarJoin):
        return E.StarJoin(plan.join_var, plan.patterns)
    if isinstance(plan, GpuHashJoin):
        return E.HashJoin(lower_to_engine(plan.left), lower_to_engine(plan.right))
    if isinstance(plan, GpuBindJoin):
        return E.ParallelJoin(lower_to_engine(plan.left), E.IndexScan(plan.pattern))
    if isinstance(plan, GpuIndexScan):
        return E.IndexScan(plan.pattern)
    if isinstance(plan, E.Filter):
        return E.Filter(lower_to_engine(plan.input), plan.condition)
    if isinstance(plan, E.Projection):
        return E.Projection(lower_to_engine(plan.input), plan.variables)
    if isinstance(plan, (E.HashJoin, E.OptimizedHashJoin, E.NestedLoopJoin, E.ParallelJoin)):
        return type(plan)(lower_to_engine(plan.left), lower_to_engine(plan.right))
    return plan
