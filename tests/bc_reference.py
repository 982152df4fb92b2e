"""Host restatements of Reasoner::backward_chaining (datalog/src/reasoning/backward_chaining.rs:165-259) that the device's
kb_datalog_query is held to:

- `sld`: the reference's SLD resolution transcribed literally (unify_terms, resolve_term, substitute, rename_rule_variables with its
  shared counter, MAX_DEPTH), with a budget on helper calls because its cost grows exponentially with the depth;
- `bounded_closure`: T^depth, the facts with a proof of height <= depth (premise constants enforced, rule filters ignored);
- `demand`: the demand patterns of a query and the rules they make relevant, and `restricted_closure`, the bounded closure over the
  demanded facts only.

Terms are engine.Variable / engine.Constant; facts are (s, p, o) id tuples; a rule is (premises, conclusions), lists of term triples."""
from typing import Dict, List, Optional, Sequence, Set, Tuple

from kolibrie_b200.engine import Constant, Variable

ANY = None
MAX_DEPTH = 10


class BudgetExceeded(Exception):
    pass


# ---- SLD resolution, literally
def _resolve(t, b):
    while isinstance(t, Variable) and t.name in b:
        t = b[t.name]
    return t


def _unify_terms(t1, t2, b) -> bool:
    t1, t2 = _resolve(t1, b), _resolve(t2, b)
    if isinstance(t1, Constant) and isinstance(t2, Constant):
        return t1.id == t2.id
    if isinstance(t1, Variable) and isinstance(t2, Constant):
        b[t1.name] = t2
        return True
    if isinstance(t1, Constant) and isinstance(t2, Variable):
        b[t2.name] = t1
        return True
    if t1.name != t2.name:
        b[t1.name] = t2
    return True


def _unify(p1, p2, b) -> Optional[dict]:
    nb = dict(b)
    for a, c in zip(p1, p2):
        if not _unify_terms(a, c, nb):
            return None
    return nb


def _substitute(p, b):
    def st(t):
        if isinstance(t, Variable) and t.name in b:
            return st(b[t.name])
        return t
    return tuple(st(t) for t in p)


def _rename(rule, counter: List[int]):
    vm: Dict[str, str] = {}

    def rn(t):
        if isinstance(t, Variable):
            if t.name not in vm:
                vm[t.name] = f"v{counter[0]}"
                counter[0] += 1
            return Variable(vm[t.name])
        return t
    prem = [tuple(rn(t) for t in p) for p in rule[0]]
    conc = [tuple(rn(t) for t in p) for p in rule[1]]
    return prem, conc


def sld(facts: Sequence[Tuple[int, int, int]], rules, query, max_depth: int = MAX_DEPTH, budget: int = 200_000) -> List[dict]:
    """backward_chaining(query) with MAX_DEPTH = max_depth: one binding map per derivation, as the reference returns them"""
    fact_pats = [tuple(Constant(x) for x in f) for f in facts]
    counter, calls = [0], [0]

    def helper(q, b, depth):
        calls[0] += 1
        if calls[0] > budget:
            raise BudgetExceeded()
        if depth > max_depth:
            return []
        sub = _substitute(q, b)
        res = []
        for f in fact_pats:
            nb = _unify(sub, f, b)
            if nb is not None:
                res.append(nb)
        for rule in rules:
            prem, conc = _rename(rule, counter)
            for c in conc:
                rb = _unify(c, sub, b)
                if rb is None:
                    continue
                pr = [rb]
                for p in prem:
                    nxt = []
                    for x in pr:
                        nxt.extend(helper(p, x, depth + 1))
                    pr = nxt
                res.extend(pr)
        return res

    return helper(tuple(query), {}, 0)


def query_vars(query) -> List[str]:
    out = []
    for t in query:
        if isinstance(t, Variable) and t.name not in out:
            out.append(t.name)
    return out


def project_sld(results: List[dict], query) -> Set[tuple]:
    """the distinct bindings of the query's own variables in the reference's maps (variable chains followed by resolve_term)"""
    names = query_vars(query)
    out = set()
    for b in results:
        vals = tuple(_resolve(Variable(n), b) for n in names)
        if all(isinstance(v, Constant) for v in vals):
            out.add(tuple(v.id for v in vals))
    return out


# ---- bounded closure
def _match(pat, fact, b) -> Optional[dict]:
    nb = dict(b)
    for t, v in zip(pat, fact):
        if isinstance(t, Constant):
            if t.id != v:
                return None
        elif t.name in nb:
            if nb[t.name] != v:
                return None
        else:
            nb[t.name] = v
    return nb


def _bindings(prem, facts) -> List[dict]:
    """every binding of the premises' variables over `facts`; a premise is matched against the facts of its predicate that hold its
    bound subject (or object), found through an index built on first use (the match itself decides)"""
    by_p: Dict[object, list] = {}
    for f in facts:
        by_p.setdefault(f[1], []).append(f)
    idx: Dict[tuple, dict] = {}

    def val(t, b):
        return t.id if isinstance(t, Constant) else b.get(t.name)

    def candidates(p, b):
        pv = val(p[1], b)
        if pv is None:
            return facts
        for pos in (0, 2):
            v = val(p[pos], b)
            if v is not None:
                if (pv, pos) not in idx:
                    d: Dict[int, list] = {}
                    for f in by_p.get(pv, []):
                        d.setdefault(f[pos], []).append(f)
                    idx[(pv, pos)] = d
                return idx[(pv, pos)].get(v, [])
        return by_p.get(pv, [])

    bs = [{}]
    for p in prem:
        bs = [nb for b in bs for f in candidates(p, b) for nb in [_match(p, f, b)] if nb is not None]
        if not bs:
            break
    return bs


def _heads(rule, facts, keep=None) -> Set[tuple]:
    out = set()
    for b in _bindings(rule[0], facts):
        for c in rule[1]:
            h = tuple(t.id if isinstance(t, Constant) else b[t.name] for t in c)
            if keep is None or keep(h):
                out.add(h)
    return out


def bounded_closure(facts, rules, depth: int, keep=None) -> Tuple[Set[tuple], int]:
    """(T^depth, rounds run): rounds stop early at a fixpoint. keep: the facts a round may add (demand restriction)"""
    t = set(map(tuple, facts)) if keep is None else {f for f in map(tuple, facts) if keep(f)}
    rounds = 0
    for _ in range(depth):
        new = set()
        for r in rules:
            new |= _heads(r, t, keep)
        rounds += 1
        if new <= t:
            break
        t |= new
    return t, rounds


def answers(facts: Set[tuple], query) -> Set[tuple]:
    names = query_vars(query)
    out = set()
    for f in facts:
        b = _match(query, f, {})
        if b is not None:
            out.add(tuple(b[n] for n in names))
    return out


# ---- demand
def _subsumes(a, b) -> bool:
    return (a[0] is ANY or a[0] == b[0]) and (a[1] is ANY or a[1] == b[1])


def demand(rules, query) -> Tuple[Set[int], Dict[object, List[tuple]]]:
    """(relevant rule indices, predicate -> demand patterns (s, o) with ANY): the query's own pattern, then every premise of a rule whose
    head unifies with a demand pattern, with its constants and the head variables the demand binds, until nothing new appears. A
    variable predicate in the query demands its pattern of every head predicate; a repeated query variable demands any value."""
    pats: Dict[object, List[tuple]] = {}
    work = []

    def add(p, x):
        v = pats.setdefault(p, [])
        if any(_subsumes(e, x) for e in v):
            return
        v[:] = [e for e in v if not _subsumes(x, e)]
        v.append(x)
        work.append((p, x))

    q0 = tuple(t.id if isinstance(t, Constant) else ANY for t in (query[0], query[2]))
    if isinstance(query[1], Constant):
        add(query[1].id, q0)
    else:
        for r in rules:
            for c in r[1]:
                add(c[1].id, q0)
    relevant = set()
    while work:
        p, x = work.pop(0)
        for i, r in enumerate(rules):
            for c in r[1]:
                if c[1].id != p:
                    continue
                bind, ok = {}, True
                for t, v in ((c[0], x[0]), (c[2], x[1])):
                    if v is ANY:
                        continue
                    if isinstance(t, Constant):
                        ok = ok and t.id == v
                    elif t.name in bind:
                        ok = ok and bind[t.name] == v
                    else:
                        bind[t.name] = v
                if not ok:
                    continue
                relevant.add(i)

                def term(t):
                    return t.id if isinstance(t, Constant) else bind.get(t.name, ANY)
                for pr in r[0]:
                    add(pr[1].id, (term(pr[0]), term(pr[2])))
    return relevant, pats


def restricted_closure(facts, rules, query, depth: int) -> Tuple[Set[tuple], int]:
    relevant, pats = demand(rules, query)

    def keep(f):
        return any(_subsumes(x, (f[0], f[2])) for x in pats.get(f[1], []))
    rel_rules = [r for i, r in enumerate(rules) if i in relevant]
    if isinstance(query[1], Variable):  # every stored fact can answer a variable predicate: the store is kept whole
        t, rounds = bounded_closure([f for f in facts if keep(f)], rel_rules, depth, keep)
        return t | set(map(tuple, facts)), rounds
    return bounded_closure(facts, rel_rules, depth, keep)


def device_answers(facts, rules, query, depth: int = MAX_DEPTH) -> Set[tuple]:
    """what kb_datalog_query returns, as a set of binding tuples (query-variable order)"""
    return answers(bounded_closure(facts, rules, depth)[0], query)
