"""The 20 WatDiv-shaped queries (tests/golden/watdiv/queries.json) as kb_pattern lists over a datagen.watdiv store."""
from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import helpers as H

QUERIES = H.load("watdiv/queries.json")["queries"]
STAR = {"C3", "L3", "L4", "S2", "S3", "S4", "S5", "S6", "S7"}  # one variable in every pattern, at most 8 patterns


def compile_query(d: datagen.WatDivData, q):
    """(patterns, projection slots): ?vN is slot N; an IRI the store does not hold -> KeyError"""
    def term(t):
        return c.V(int(t[2:])) if t.startswith("?") else c.K(d.ids[t])
    pats = [c.pattern(*(term(t) for t in p)) for p in q["patterns"]]
    return pats, [int(v[2:]) for v in q["select"]]
