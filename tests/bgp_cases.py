"""Random BGPs for kb_bgp_execute's component route and the independent oracle the GPU tests compare it with: every pattern scanned
(ko_scan), joined inside its connected component in a BFS order of the test's own (ko_hash_join), the components cross-joined, then
FILTER (ko_filter) and projection (ko_project) — none of the library's planning."""
import numpy as np

from kolibrie_b200 import capi as c
from tests import oracle_api as O

CROSS_LIMIT = 1 << 28  # kb_bgp_execute's cartesian limit (only a cross join between components can reach it)


def pattern_vars(p):
    out = []
    for t in (p.s, p.p, p.o):
        if t.is_var and int(t.value) not in out:
            out.append(int(t.value))
    return out


def components(pv):
    comp, out = [-1] * len(pv), []
    for s in range(len(pv)):
        if comp[s] >= 0:
            continue
        comp[s], todo, members = len(out), [s], []
        while todo:
            k = todo.pop()
            members.append(k)
            for j in range(len(pv)):
                if comp[j] < 0 and set(pv[k]) & set(pv[j]):
                    comp[j] = len(out)
                    todo.append(j)
        out.append(sorted(members))
    return out


def bfs_order(pv, members):
    """textual BFS: start at the first pattern, then always the first pattern that shares a variable with those joined"""
    order, held = [members[0]], set(pv[members[0]])
    while len(order) < len(members):
        k = next(k for k in members if k not in order and held & set(pv[k]))
        order.append(k)
        held |= set(pv[k])
    return order


def columns(pats, project=None):
    if project is not None:
        return list(project)
    out = []
    for p in pats:
        out += [v for v in pattern_vars(p) if v not in out]
    return out


def oracle(db, pats, filt=None, project=None, max_rows=5_000_000):
    """(relation, component row counts) or (None, why): 'cross' when the components' product passes CROSS_LIMIT (the device must
    decline with KB_E_LIMIT), 'big' when a component's rows pass max_rows (the case is skipped)"""
    pv = [pattern_vars(p) for p in pats]
    comps = components(pv)
    results = []
    for members in comps:
        order = bfs_order(pv, members)
        cur = db.scan(pats[order[0]])
        for k in order[1:]:
            cur = O.hash_join(cur, db.scan(pats[k]))
            if cur.n_rows > max_rows:
                return None, "big"
        results.append(cur)
    sizes = [r.n_rows for r in results]
    if 0 not in sizes and int(np.prod([float(x) for x in sizes])) > CROSS_LIMIT and len(sizes) > 1:
        return None, "cross"
    cur = results[0]
    for r in results[1:]:
        cur = O.hash_join(cur, r)
    if filt:
        cur = db.filter(cur, filt)
    if project is not None:
        cur = O.project(cur, project)
    return cur, sizes


def random_bgp(seed):
    """a random store and a BGP of 2-16 patterns: trees, cycles, several components, constants, repeated variables, variable
    predicates, patterns without variables, FILTER and projection"""
    rng = np.random.default_rng(77_000 + seed)
    n_terms = int(rng.choice([30, 80, 200]))
    n_preds = int(rng.integers(3, 7))
    n = int(rng.choice([0, 50, 600, 3000]))
    tr = np.stack([rng.integers(0, n_terms, n), rng.integers(100, 100 + n_preds, n), rng.integers(0, n_terms, n)], axis=1).astype(np.uint32)
    tr = np.unique(tr, axis=0) if n else tr
    num = np.zeros(n_terms + 200)
    isn = np.zeros(n_terms + 200, np.uint8)
    numeric = rng.random(n_terms) < 0.6
    num[:n_terms][numeric] = np.round(rng.normal(50, 40, int(numeric.sum())), 1)
    isn[:n_terms][numeric] = 1
    n_pats = int(rng.integers(2, 17))
    pred = lambda: c.K(int(rng.integers(100, 100 + n_preds)))
    pats, nxt = [], 0
    while len(pats) < n_pats:
        kind = rng.choice(["tree", "cycle", "const", "repeat", "varpred", "triple"], p=[0.45, 0.2, 0.08, 0.07, 0.1, 0.1])
        if kind == "tree":  # a fresh variable hung off an existing one (or a new root)
            a = int(rng.integers(0, nxt)) if nxt and rng.random() < 0.8 else nxt
            nxt = max(nxt, a + 1)
            b, nxt = nxt, nxt + 1
            s_, o_ = (c.V(a), c.V(b)) if rng.random() < 0.6 else (c.V(b), c.V(a))
            if rng.random() < 0.1:
                o_ = c.K(int(rng.integers(0, n_terms)))
            pats.append(c.pattern(s_, pred(), o_))
        elif kind == "cycle" and nxt >= 2:  # an edge between two existing variables
            a, b = (int(x) for x in rng.choice(nxt, 2, replace=False))
            pats.append(c.pattern(c.V(a), pred(), c.V(b)))
        elif kind == "const":  # no variable: a component of its own
            t = tr[int(rng.integers(0, len(tr)))] if len(tr) and rng.random() < 0.7 else np.array([0, 100, 1], np.uint32)
            pats.append(c.pattern(c.K(int(t[0])), c.K(int(t[1])), c.K(int(t[2]))))
        elif kind == "repeat" and nxt:  # ?x P ?x (quirk Q4: enforced)
            a = int(rng.integers(0, nxt))
            pats.append(c.pattern(c.V(a), pred(), c.V(a)))
        elif kind == "varpred" and nxt:  # a variable predicate (its own variable, shared with nothing)
            a = int(rng.integers(0, nxt))
            pats.append(c.pattern(c.V(a), c.V(12 + int(rng.integers(0, 2))), c.K(int(rng.integers(0, n_terms)))))
        elif kind == "triple" and nxt >= 2:  # three variables: a hyperedge that can cover a triangle
            a, b = (int(x) for x in rng.choice(nxt, 2, replace=False))
            pats.append(c.pattern(c.V(a), c.V(14), c.V(b)))
        if nxt >= 11:
            nxt = 11  # at most 16 variables in all (slots 0-11, 12-13 predicates, 14)
    bound = sorted({v for p in pats for v in pattern_vars(p)})
    filt = None
    if bound and rng.random() < 0.4:
        ops = []
        for q in range(int(rng.integers(1, 3))):
            slot = int(rng.choice(bound))
            if rng.random() < 0.6:
                ops.append(c.fop(c.F_CMP_NUM, slot=slot, cmp=int(rng.choice([c.CMP_GT, c.CMP_LT])), value=float(rng.normal(50, 30))))
            else:
                ops.append(c.fop(c.F_NE_ID, slot=slot, id=int(rng.integers(0, n_terms))))
            if q:
                ops.append(c.fop(c.F_AND if rng.random() < 0.7 else c.F_OR))
        filt = ops
    project = None
    if bound and rng.random() < 0.3:
        project = [int(x) for x in rng.choice(bound, int(rng.integers(1, len(bound) + 1)), replace=False)]
    return tr, num, isn, pats, filt, project
