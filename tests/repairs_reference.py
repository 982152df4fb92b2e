"""Host restatements of Reasoner::query_with_repairs (datalog/src/reasoning/repairs.rs:10-43) and what kb_datalog_query_repairs answers.

Terms: a string starting with "?" is a variable, an int a constant id. A fact is an (s, p, o) tuple of ids, a premise or a query an
(s, p, o) tuple of terms, a constraint a list of premises (its filters and conclusion are never read).

  (a) transcribe: compute_repairs (datalog/src/reasoning.rs:111-150) and query_with_repairs as written. Rust's HashSet iterates a set
      and every clone of it with an element removed in one order, fixed per process; here that order is an explicit permutation of
      the store (`order`), and `seen` holds sets, which is what its vectors in that order stand for.
  (b) brute_force: the intersection of all maximal consistent subsets of the store.
  (c) iar: the store minus every fact of a minimal conflict. Polynomial; (b) == (c) because the constraints are monotone.
An answer is the set of distinct bindings of the query's variables, each a tuple in s, p, o first-appearance order (kb_scan's column
order); a ground query's answer is {()} or set().
"""
from itertools import combinations


def is_var(t):
    return isinstance(t, str)


def match(pattern, fact, binding):
    """matches_rule_pattern (datalog/src/reasoning/rules.rs:9-72): the extended binding, or None"""
    b = dict(binding)
    for t, v in zip(pattern, fact):
        if is_var(t):
            if b.setdefault(t, v) != v:
                return None
        elif t != v:
            return None
    return b


def matches(premises, facts):
    """every binding of the premises over `facts` (each premise matched against every fact, in premise order)"""
    out = [{}]
    for pr in premises:
        out = [b2 for b in out for f in facts for b2 in [match(pr, f, b)] if b2 is not None]
        if not out:
            break
    return out


def violates(constraints, facts):
    """violates_constraints (reasoning.rs:100-108): join_rule over the set is non-empty iff the premises match inside it; a constraint
    without premises gives no binding"""
    return any(c and matches(c, facts) for c in constraints)


def query_vars(query):
    out = []
    for t in query:
        if is_var(t) and t not in out:
            out.append(t)
    return out


def answer(query, facts):
    names = query_vars(query)
    return {tuple(b[n] for n in names) for f in facts for b in [match(query, f, {})] if b is not None}


# ---- (a) the reference's algorithm
def compute_repairs(facts, constraints, order):
    """compute_repairs as written: a depth-first search from the whole store that removes one fact at a time from every inconsistent
    set, keeping a consistent set unless a set kept earlier strictly contains it. Exponential in the store's size."""
    rank = {f: i for i, f in enumerate(order)}
    it = lambda s: sorted(s, key=rank.__getitem__)  # noqa: E731  (the process's iteration order)
    repairs, work, seen = [], [frozenset(facts)], set()
    while work:
        cur = work.pop()
        if cur in seen:
            continue
        seen.add(cur)
        if not violates(constraints, cur):
            if all(not (r >= cur) or r == cur for r in repairs):
                repairs.append(cur)
        else:
            for f in it(cur):
                new = cur - {f}
                if new not in seen:
                    work.append(new)
    return repairs


def transcribe(facts, constraints, query, order):
    """query_with_repairs as written: the bindings of the first kept set, retained when every other kept set has a fact binding the
    same map. Returns (answer, kept sets)."""
    repairs = compute_repairs(facts, constraints, order)
    if not repairs:
        return set(), repairs
    names = query_vars(query)
    rank = {f: i for i, f in enumerate(order)}
    results = [b for f in sorted(repairs[0], key=rank.__getitem__) for b in [match(query, f, {})] if b is not None]
    results = [b for b in results if all(any(match(query, f, {}) == b for f in r) for r in repairs[1:])]
    return {tuple(b[n] for n in names) for b in results}, repairs


# ---- (b) brute force
def maximal_repairs(facts, constraints):
    facts = sorted(set(facts))
    consistent = [frozenset(s) for k in range(len(facts) + 1) for s in combinations(facts, k) if not violates(constraints, s)]
    return [s for s in consistent if not any(s < t for t in consistent)]


def brute_force(facts, constraints, query):
    reps = maximal_repairs(facts, constraints)
    kept = frozenset.intersection(*reps) if reps else frozenset()
    return answer(query, kept)


# ---- (c) the polynomial rule (what the device computes)
def conflicts(facts, constraints):
    """the distinct conflicts: per match of a constraint's premises, the set of distinct facts it instantiates"""
    facts = sorted(set(facts))
    out = set()
    for c in constraints:
        if not c:
            continue
        for b in matches(c, facts):
            out.add(frozenset(tuple(b[t] if is_var(t) else t for t in pr) for pr in c))
    return out


def minimal_conflicts(cs):
    return {c for c in cs if not any(o < c for o in cs)}


def conflicted_facts(facts, constraints):
    return frozenset().union(*minimal_conflicts(conflicts(facts, constraints)))


def iar(facts, constraints, query):
    bad = conflicted_facts(facts, constraints)
    return answer(query, [f for f in set(facts) if f not in bad])


def stats(facts, constraints):
    """what kb_repair_stats counts, without the match count (a bag: the device's joins count duplicate segments)"""
    cs = conflicts(facts, constraints)
    mins = minimal_conflicts(cs)
    sizes = {len(c) for c in cs}
    return {"constraints": sum(1 for c in constraints if c), "conflicts": len(cs), "minimal_conflicts": len(mins),
            "conflicted_facts": len(frozenset().union(*mins)), "subsets_probed": int(len(sizes) > 1)}
