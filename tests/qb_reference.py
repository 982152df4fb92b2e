"""A transcription of QueryBuilder's triple queries (kolibrie/src/query_builder.rs:355-643) over a set of (s, p, o) id triples and the
dictionary's id -> string list: the reference the device path (kb_qb_triples / kb_qb_terms) and the engine's QueryBuilder are held to.

Dictionary::decode(id) is id_to_string[id] for an id the list holds and None otherwise: a quoted-triple id (bit 31) and an id past the
list do not decode (shared/src/dictionary.rs:49-51). Filters are ("Exact" | "Contains" | "StartsWith" | "EndsWith", text) or
("Custom", fn); join conditions "OnSubject", "OnPredicate", "OnObject" or a callable (JoinCondition::Custom). Where the reference panics
(an offset past the rows: a slice start past its end) this raises IndexError."""
from typing import Callable, List, Optional, Sequence, Tuple

Triple = Tuple[int, int, int]


class Ref:
    def __init__(self, triples, strings: Sequence[str], right=None):
        self.triples = set(map(tuple, triples))
        self.strings = list(strings)
        self.right = None if right is None else set(map(tuple, right))  # join(other): the other database's triples
        self.subject_filter = self.predicate_filter = self.object_filter = None
        self.custom_filter: Optional[Callable] = None
        self.join_conditions: List = []
        self.distinct_results = False
        self.sort_key: Optional[Callable] = None
        self.descending = False
        self.limit: Optional[int] = None
        self.offset: Optional[int] = None

    def decode(self, i: int) -> Optional[str]:
        return self.strings[i] if 0 <= i < len(self.strings) else None

    @staticmethod
    def apply_filter(f, value: str) -> bool:  # :571-579
        kind, arg = f
        if kind == "Exact":
            return value == arg
        if kind == "Contains":
            return arg in value
        if kind == "StartsWith":
            return value.startswith(arg)
        if kind == "EndsWith":
            return value.endswith(arg)
        return bool(arg(value))

    def apply_filters(self) -> List[Triple]:  # :486-568, the BTreeSet as a sorted list
        results = set()
        for t in sorted(self.triples):
            matches = True
            for f, x in zip((self.subject_filter, self.predicate_filter, self.object_filter), t):
                if matches and f is not None:
                    v = self.decode(x)
                    matches = v is not None and self.apply_filter(f, v)
            if matches and self.custom_filter is not None:
                matches = bool(self.custom_filter(t))
            if matches:
                results.add(t)
        if self.right is not None and self.join_conditions:  # :537-541
            results = self.apply_join(sorted(results))
        if self.sort_key is not None:  # :544-551: sorted, then collected back into a BTreeSet
            results = set(sorted(results, key=self.sort_key, reverse=self.descending))
        rows = sorted(results)
        if self.offset is not None or self.limit is not None:  # :554-564
            off = self.offset or 0
            if off > len(rows):
                raise IndexError("slice index starts past the end")
            end = len(rows) if self.limit is None else min(off + self.limit, len(rows))
            rows = rows[off:end]
        return rows

    def apply_join(self, left: List[Triple]) -> set:  # :582-643
        out = set()
        for cond in self.join_conditions:
            for l in left:
                for r in sorted(self.right):
                    if cond == "OnSubject" and l[0] == r[0]:
                        out.add((l[0], l[1], r[2]))
                    elif cond == "OnPredicate" and l[1] == r[1]:
                        out.add((l[0], l[1], r[2]))
                    elif cond == "OnObject" and l[2] == r[2]:
                        out.add((l[0], r[1], r[2]))
                    elif callable(cond) and cond(l, r):
                        out.add((l[0], r[1], r[2]))
        return out

    # ---- results (:355-466)
    def get_triples(self) -> List[Triple]:
        return self.apply_filters()

    def count(self) -> int:
        return len(self.apply_filters())

    def get_decoded_triples(self) -> List[Tuple[str, str, str]]:
        return [tuple(self.decode(x) or "" for x in t) for t in self.apply_filters()]

    def terms(self, col: int) -> List[str]:  # get_subjects / get_predicates / get_objects
        out = [v for v in (self.decode(t[col]) for t in self.apply_filters()) if v is not None]
        if self.distinct_results:
            out = sorted(set(out), key=lambda s: s.encode("utf-8"))  # String's Ord: byte order
        return out

    def get_subjects(self) -> List[str]:
        return self.terms(0)

    def get_predicates(self) -> List[str]:
        return self.terms(1)

    def get_objects(self) -> List[str]:
        return self.terms(2)


# ---- the fixture's queries (tests/golden/querybuilder/querybuilder.json) on this transcription and on kolibrie_b200.engine.QueryBuilder
def ref_query(triples, strings, q, right=None) -> Ref:
    r = Ref(triples, strings, right)
    r.subject_filter, r.predicate_filter, r.object_filter = [None if f is None else tuple(f) for f in q["filters"]]
    r.join_conditions = list(q["join"])
    r.distinct_results = q["distinct"]
    r.offset, r.limit = q["offset"], q["limit"]
    if q["order_by"]:
        r.sort_key = lambda t: r.decode(t[2]) or ""
        r.descending = q["order_by"] == "desc"
    return r


def engine_query(db, q, right_db=None):
    b = db.query()
    for pos, f in zip(("subject", "predicate", "object"), q["filters"]):
        if f is not None:
            suffix = {"Exact": "", "Contains": "_like", "StartsWith": "_starting", "EndsWith": "_ending"}[f[0]]
            b = getattr(b, f"with_{pos}{suffix}")(f[1])
    if right_db is not None:
        b = b.join(right_db)
    for j in q["join"]:
        b = getattr(b, {"OnSubject": "join_on_subject", "OnPredicate": "join_on_predicate", "OnObject": "join_on_object"}[j])()
    if q["distinct"]:
        b = b.distinct()
    if q["order_by"]:
        b = b.order_by(lambda t: str(t[2]))
        b = b.desc() if q["order_by"] == "desc" else b.asc()
    if q["offset"] is not None:
        b = b.offset(q["offset"])
    if q["limit"] is not None:
        b = b.limit(q["limit"])
    return b


def results(make, kind):
    """one result method of a fresh builder from make(): 'triples' sorted as lists, the others as the method returns them"""
    b = make()
    if kind == "triples":
        return [list(t) for t in sorted(b.get_triples())]
    if kind == "count":
        return b.count()
    if kind == "decoded":
        return [list(t) for t in b.get_decoded_triples()]
    return {"subjects": b.get_subjects, "predicates": b.get_predicates, "objects": b.get_objects}[kind]()


def assert_expect(make, expect, all_rows=None):
    """every entry of a fixture case's "expect" holds for the builders make() returns"""
    import pytest

    for k, v in expect.items():
        if k == "error":
            with pytest.raises(IndexError):
                results(make, "triples")
        elif k.endswith("_len"):
            assert len(results(make, k[:-4])) == v, k
        elif k.endswith("_contain"):
            assert v in results(make, k[: -len("_contain")]), k
        elif k == "first_is_all_at":
            assert results(make, "triples")[0] == all_rows[v]
        else:
            assert results(make, k) == v, k
