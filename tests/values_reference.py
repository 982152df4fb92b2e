"""An exact restatement of `PhysicalOperator::Values` and of the joins above it over rows that may leave variables unbound, transcribed
from the reference (paths relative to the root of the Kolibrie checkout). A row is a dict {variable name without '?': id}; a variable the
row does not bind is not a key. What kb_values and kb_hash_join_keyed / kb_natural_join compute on the device is tested against this.

* values                  kolibrie/src/streamertail_optimizer/execution/engine.rs:279-308
* optimized_hash_join     engine.rs:710-763   (build = the smaller side, left on ties; the build row extended by the probe row)
* hash_join               engine.rs:766-811   (build = left; the right row adds only the keys the left row lacks)
* nested_loop_join        engine.rs:814-837   with can_join_with_ids, engine.rs:1042-1051
* bind_join               engine.rs:840-923   (bind_pattern, then `entry().or_insert`; quirk Q1's caps are left off)
* parallel_join           engine.rs:926-950   (a scan on the right -> bind join; else merge join when can_use_merge_join, else hash join)
* merge_join              engine.rs:970-1039
* cartesian_product_join  engine.rs:1054-1071 (the left row extended by the right row: right-first)

Where the reference panics (`tuple[var]` of a key variable a later row lacks, in both hash joins) the restatement raises Panic. Where its
merge join builds keys of different shapes from rows lacking a key variable (`filter_map`, over a HashSet whose order is unspecified)
the restatement raises Panic too: the result is not determined by the rows alone, and the device refuses both."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

Row = Dict[str, int]


class Panic(Exception):
    """the reference panics here, or its result depends on more than the rows"""


def strip(v: str) -> str:
    return v[1:] if v.startswith("?") else v


def values(variables: Sequence[str], rows: Sequence[Sequence[Optional[str]]], encode) -> List[Row]:
    """engine.rs:279-308: rows in order, variables in header order, every defined cell encoded verbatim (`encode` is Dictionary::encode);
    a missing trailing cell is UNDEF (`value_row.get(i)`); a repeated variable keeps its later defined cell; an empty row is dropped"""
    names = [strip(v) for v in variables]
    out = []
    for value_row in rows:
        row: Row = {}
        for i, var in enumerate(names):
            if i < len(value_row) and value_row[i] is not None:
                row[var] = encode(value_row[i])
        if row:
            out.append(row)
    return out


def common_vars(left: List[Row], right: List[Row]) -> List[str]:
    """the shared keys of row 0 of each side"""
    return sorted(set(left[0]) & set(right[0]))


def _key(row: Row, vars_: List[str]) -> Tuple[int, ...]:
    try:
        return tuple(row[v] for v in vars_)  # tuple[var]
    except KeyError as e:
        raise Panic(f"row lacks key variable {e.args[0]!r}")


def cartesian_product_join(left: List[Row], right: List[Row]) -> List[Row]:
    return [{**l, **r} for l in left for r in right]


def optimized_hash_join(left: List[Row], right: List[Row]) -> List[Row]:
    if not left or not right:
        return []
    cv = common_vars(left, right)
    if not cv:
        return cartesian_product_join(left, right)
    build, probe = (left, right) if len(left) <= len(right) else (right, left)
    table: Dict[Tuple[int, ...], List[Row]] = {}
    for t in build:
        table.setdefault(_key(t, cv), []).append(t)
    out = []
    for p in probe:
        for b in table.get(_key(p, cv), []):
            out.append({**b, **p})  # result.extend(probe_tuple): the probe row overwrites
    return out


def hash_join(left: List[Row], right: List[Row]) -> List[Row]:
    if not left or not right:
        return []
    cv = common_vars(left, right)
    if not cv:
        return cartesian_product_join(left, right)
    table: Dict[Tuple[int, ...], List[Row]] = {}
    for t in left:
        table.setdefault(_key(t, cv), []).append(t)
    out = []
    for r in right:
        for l in table.get(_key(r, cv), []):
            out.append({**r, **l})  # only the keys the left row lacks come from the right row
    return out


def can_join(l: Row, r: Row) -> bool:
    return all(r[k] == v for k, v in l.items() if k in r)


def nested_loop_join(left: List[Row], right: List[Row]) -> List[Row]:
    return [{**r, **l} for l in left for r in right if can_join(l, r)]


def merge_join(left: List[Row], right: List[Row]) -> List[Row]:
    if not left or not right:
        return []
    cv = common_vars(left, right)
    if not cv:
        return cartesian_product_join(left, right)
    for row in left + right:
        if any(v not in row for v in cv):  # filter_map: a key of another shape
            raise Panic("merge-join key changes shape")
    index: Dict[Tuple[int, ...], List[Row]] = {}
    for r in right:
        index.setdefault(_key(r, cv), []).append(r)
    return [{**r, **l} for l in left for r in index.get(_key(l, cv), [])]


def can_use_merge_join(left: List[Row], right: List[Row]) -> bool:
    if not left or not right:
        return False
    return 1 <= len(common_vars(left, right)) <= 2


def parallel_join(left: List[Row], right: List[Row]) -> List[Row]:
    """ParallelJoin whose right side is not a scan"""
    return merge_join(left, right) if can_use_merge_join(left, right) else hash_join(left, right)


def scan(pattern: Tuple[object, object, object], triples) -> List[Row]:
    """the matches of a pattern of ('?x' variables or int constants) over (s, p, o) id triples; a repeated variable must be equal"""
    out = []
    for t in triples:
        row: Row = {}
        ok = True
        for term, v in zip(pattern, t):
            if isinstance(term, str):
                k = strip(term)
                if row.get(k, v) != v:
                    ok = False
                row[k] = v
            elif term != v:
                ok = False
        if ok:
            out.append(row)
    return out


def bind_join(left: List[Row], pattern: Tuple[object, object, object], triples) -> List[Row]:
    """ParallelJoin with a scan on the right: every left row binds the pattern (bind_pattern leaves a variable the row lacks free) and
    keeps its own cells (`entry().or_insert`)"""
    out = []
    for l in left:
        bound = tuple(l.get(strip(t), t) if isinstance(t, str) else t for t in pattern)
        for r in scan(bound, triples):
            out.append({**r, **l})
    return out


JOINS = {"HashJoin": hash_join, "OptimizedHashJoin": optimized_hash_join, "NestedLoopJoin": nested_loop_join, "ParallelJoin": parallel_join}


def bag(rows: Sequence[Row]) -> List[Tuple[Tuple[str, int], ...]]:
    return sorted(tuple(sorted(r.items())) for r in rows)
