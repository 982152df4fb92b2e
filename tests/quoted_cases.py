"""Seeded RDF-star stores and patterns, and the literal restatements the quoted-triple tests hold the mirror and the device to:
resolve_quoted_triple_scan (kolibrie/src/streamertail_optimizer/execution/engine.rs:1111-1188) with match_term (engine.rs:1088-1107),
and Dictionary::decode_term (shared/src/dictionary.rs:60-72) with the "unknown" of engine.rs:42-43."""
from collections import Counter
from typing import Dict, List

import numpy as np

from kolibrie_b200 import engine as E

QBIT = E.QUOTED_TRIPLE_ID_BIT
VARS = ("a", "b", "c", "x")


def _match_term(term, value: int, b: Dict[str, int]) -> bool:  # engine.rs:1088-1107
    if isinstance(term, E.Constant):
        return term.id == value
    if isinstance(term, E.Variable):
        name = term.name.lstrip("?")
        if name in b:
            return b[name] == value
        b[name] = value
        return True
    return (value & QBIT) != 0


def brute_quoted_scan(db: E.SparqlDatabase, pattern) -> List[Dict[str, int]]:
    """engine.rs:1111-1188, entry by entry: match the quoted term(s), substitute the entry's id, scan the store for the concrete pattern
    (a repeated variable is enforced inside it, as kb_scan enforces it), merge the bindings and drop conflicting rows"""
    qs, qo = isinstance(pattern[0], E.QuotedTriple), isinstance(pattern[2], E.QuotedTriple)
    out = []
    for qid, (s, p, o) in db.quoted_triple_store.id_to_components.items():
        inner: Dict[str, int] = {}
        ok = True
        for q in ([pattern[0]] if qs else []) + ([pattern[2]] if qo else []):
            ok = ok and _match_term(q.s, s, inner) and _match_term(q.p, p, inner) and _match_term(q.o, o, inner)
        if not ok:
            continue
        concrete = (E.Constant(qid) if qs else pattern[0], pattern[1], E.Constant(qid) if qo else pattern[2])
        for t in db.triples:
            row: Dict[str, int] = {}
            if not all(_match_term(term, v, row) for term, v in zip(concrete, t)):
                continue
            merged, conflict = dict(inner), False
            for k, v in row.items():
                if k in merged and merged[k] != v:
                    conflict = True
                    break
                merged[k] = v
            if not conflict:
                out.append(merged)
    return out


def bag(rows) -> Counter:
    return Counter(tuple(sorted(r.items())) for r in rows)


def decode_term_ref(db: E.SparqlDatabase, i: int) -> str:
    """dictionary.rs:60-72 with the `?` of each step, then engine.rs:42-43's "unknown" for None"""
    def rec(x):
        if x & QBIT:
            comp = db.quoted_triple_store.id_to_components.get(x)
            if comp is None:
                return None
            parts = []
            for c in comp:
                r = rec(c)
                if r is None:
                    return None
                parts.append(r)
            return "<< %s %s %s >>" % tuple(parts)
        return db.dictionary.id_to_string[x] if x < len(db.dictionary.id_to_string) else None

    r = rec(i)
    return "unknown" if r is None else r


def random_store(db: E.SparqlDatabase, rng, n_terms=12, n_quoted=40, n_triples=120, max_depth=3):
    """a small RDF-star store: terms t0.., quoted triples (components may be earlier quoted ids: nesting up to max_depth), and triples
    with quoted subjects and objects next to plain ones. Returns the quoted ids."""
    terms = [db.dictionary.encode("t%d" % k) for k in range(n_terms)]
    depth = {}
    qids = []
    for _ in range(n_quoted):
        comp = []
        for pos in range(3):
            if pos != 1 and qids and rng.random() < 0.25:
                q = qids[int(rng.integers(len(qids)))]
                if depth[q] < max_depth:
                    comp.append(q)
                    continue
            comp.append(terms[int(rng.integers(min(n_terms, 5 if pos == 1 else n_terms)))])
        q = db.quoted_triple_store.encode(*comp)
        depth.setdefault(q, 1 + max((depth.get(c, 0) for c in comp), default=0))
        qids.append(q)
    preds = terms[:4]
    for _ in range(n_triples):
        s = qids[int(rng.integers(len(qids)))] if rng.random() < 0.5 else terms[int(rng.integers(n_terms))]
        o = qids[int(rng.integers(len(qids)))] if rng.random() < 0.3 else terms[int(rng.integers(n_terms))]
        db.add_triple((int(s), int(preds[int(rng.integers(len(preds)))]), int(o)))
    return qids


def random_pattern(db: E.SparqlDatabase, rng):
    """a pattern with a quoted subject, object or both; inner terms are variables (shared names, so repeats within and across the
    inner and outer terms occur), constants (some absent from the store) or nested quoted terms"""
    d = db.dictionary

    def var():
        return E.Variable("?" + VARS[int(rng.integers(len(VARS)))])

    def const():
        return E.Constant(d.encode("t%d" % int(rng.integers(14))))  # t12, t13: never in a triple

    def inner_term(pos):
        r = rng.random()
        if r < 0.55:
            return var()
        if r < 0.85 or pos == 1:
            return const()
        return E.QuotedTriple(var(), var(), var())

    def quoted():
        return E.QuotedTriple(inner_term(0), inner_term(1), inner_term(2))

    kind = int(rng.integers(3))
    s = quoted() if kind in (0, 2) else (var() if rng.random() < 0.8 else const())
    o = quoted() if kind in (1, 2) else (var() if rng.random() < 0.8 else const())
    p = var() if rng.random() < 0.3 else E.Constant(d.encode("t%d" % int(rng.integers(4))))
    return (s, p, o)


def holey_store(db: E.SparqlDatabase, rng, n_entries: int, n_terms: int = 50, max_depth: int = 4):
    """n_entries quoted triples under ids with holes (ids never handed out) inserted in a permuted order, components nested up to
    max_depth; plus one annotation triple per entry. Vectorised: sizes up to a few 100 K."""
    terms = np.array([db.dictionary.encode("w%d" % k) for k in range(n_terms)], dtype=np.int64)
    idx = np.sort(rng.choice(np.arange(3 * max(n_entries, 1)), size=n_entries, replace=False)).astype(np.int64)
    ids = (QBIT + idx).astype(np.int64)
    comp = terms[rng.integers(0, n_terms, size=(n_entries, 3))]
    depth = np.ones(n_entries, dtype=np.int64)
    # nesting: an entry may take an EARLIER entry as subject / object, as QuotedTripleStore::encode requires
    for pos in (0, 2):
        pick = rng.random(n_entries) < 0.3
        for i in np.nonzero(pick)[0]:
            if i == 0:
                continue
            j = int(rng.integers(i))
            if depth[j] < max_depth:
                comp[i, pos] = ids[j]
                depth[i] = max(depth[i], depth[j] + 1)
    qts = db.quoted_triple_store
    for i in rng.permutation(n_entries):
        key = (int(comp[i, 0]), int(comp[i, 1]), int(comp[i, 2]))
        if key in qts.components_to_id:
            continue
        qts.id_to_components[int(ids[i])] = key
        qts.components_to_id[key] = int(ids[i])
    qts.next_qt_id = int(QBIT + 3 * max(n_entries, 1))
    live = np.array(sorted(qts.id_to_components), dtype=np.int64)
    ann, src = db.dictionary.encode("ex:source"), db.dictionary.encode("ex:src")
    for q in live.tolist():
        db.triples.add((q, ann, src if q % 3 else int(terms[q % n_terms])))
    db._version += 1
    return live
