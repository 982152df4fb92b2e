"""A Python restatement of the Relation-to-Stream operator (kolibrie/src/rsp/r2s.rs:24-58) with the order contract of kb_r2s_eval
(include/kolibrie_b200.h): ISTREAM emits the new rows in response order, duplicates kept; DSTREAM emits the rows that left once each,
in the order of their first occurrence in the response that set the state. Rows are hashable tuples."""
from typing import Hashable, List, Sequence

RSTREAM, ISTREAM, DSTREAM = 0, 1, 2
NAMES = {"RSTREAM": RSTREAM, "ISTREAM": ISTREAM, "DSTREAM": DSTREAM}


class Relation2Stream:
    def __init__(self, stream_operator):
        self.stream_operator = NAMES.get(stream_operator, stream_operator)
        self.last: List[Hashable] = []  # distinct rows of the previous evaluation, first-occurrence order
        self._last_set = set()

    def eval(self, new_response: Sequence[Hashable]) -> list:
        if self.stream_operator == RSTREAM:  # r2s.rs:39
            return list(new_response)
        distinct = list(dict.fromkeys(new_response))
        new_set = set(distinct)
        if self.stream_operator == ISTREAM:  # r2s.rs:40-47
            emitted = [r for r in new_response if r not in self._last_set]
        else:  # r2s.rs:48-56
            emitted = [r for r in self.last if r not in new_set]
        self.last, self._last_set = distinct, new_set
        return emitted


def window_rows(window, pattern, select):
    """the answers of one triple pattern (terms as strings, variables start with '?') over a window's triples, in window order,
    projected on `select` (names without '?')"""
    rows = []
    for t in window:
        b = {}
        ok = True
        for term, value in zip(pattern, t):
            if term.startswith("?"):
                if b.setdefault(term[1:], value) != value:
                    ok = False
            elif term != value:
                ok = False
        if ok:
            rows.append(tuple(b[v] for v in select))
    return rows
