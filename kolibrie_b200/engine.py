"""Python mirror of the reference's host-side interfaces for the hot path, on top of the C ABI.

Same names, argument meaning and error behaviour as the reference (paths relative to the root of the Kolibrie checkout):

* `Dictionary`            — shared/src/dictionary.rs:17-51 (ids dense from 0 in first-seen order)
* `Term`/`TriplePattern`  — shared/src/terms.rs:13-23
* `PhysicalOperator`      — kolibrie/src/streamertail_optimizer/operators/physical.rs:16-76 (the operators on the hot path, and Values)
* `ExecutionEngine`       — kolibrie/src/streamertail_optimizer/execution/engine.rs:27,54 (`execute`, `execute_with_ids`)
* `Condition`             — kolibrie/src/streamertail_optimizer/types.rs:110-186 (FILTER expressions)
* `SparqlDatabase`        — kolibrie/src/sparql_database.rs:49-60,215-258,3364-3394 (triples + dictionary + build_all_indexes)
* `QueryBuilder`          — kolibrie/src/query_builder.rs:39-643 without its streaming half (a host restatement runs only for Python
                            callables, which cannot cross the C ABI, and for contexts without the device query)
* `Rule`/`FilterCondition`/`Reasoner` — shared/src/rule.rs:14-25, datalog/src/reasoning.rs:31-38,60-100,
                            datalog/src/reasoning/materialisation/semi_naive.rs:89, my_naive.rs:74

The canonical C++ mirror (the reference is compiled code) is kolibrie_b200/host/kolibrie_host.hpp; this module exists because
pytest, bench.py and torch.distributed live in Python. All work is done by libkolibrie_b200.so — there is no CPU path here.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import capi as c

# ---------------------------------------------------------------------------------------------------------------------
_RUST_F64 = re.compile(r"[+-]?(?:(?:inf|infinity|nan)|(?:(?:[0-9]+\.?[0-9]*|\.[0-9]+)(?:[eE][+-]?[0-9]+)?))", re.IGNORECASE)
_RUST_F64_SPECIAL = re.compile(r"[+-]?(?:inf|infinity|nan)", re.IGNORECASE)


def rust_parse_f64(s: str) -> Optional[float]:
    """`str::parse::<f64>()` acceptance of Rust (no whitespace, no '_', no hex; inf/infinity/nan in any case; '5.', '.5', '1e5')."""
    if not isinstance(s, str) or not s.isascii() or not _RUST_F64.fullmatch(s):
        return None
    if _RUST_F64_SPECIAL.fullmatch(s):
        return float(s)  # Python accepts the same special spellings
    return float(s)


class Dictionary:
    def __init__(self):
        self.string_to_id: Dict[str, int] = {}
        self.id_to_string: List[str] = []

    def encode(self, value: str) -> int:
        i = self.string_to_id.get(value)
        if i is None:
            i = len(self.id_to_string)
            assert i < 0x8000_0000, "Dictionary ID space exhausted"  # dictionary.rs:36-40
            self.string_to_id[value] = i
            self.id_to_string.append(value)
        return i

    def encode_bulk(self, ctx, terms: Sequence[str]) -> np.ndarray:
        """the load-time encode of a whole batch (sparql_database.rs:1000-1013 calls encode once per term) on the device: kb_dict_encode
        hands out the ids the sequential loop would, and this dictionary learns the new strings from the positions that introduced them.
        The device dictionary must mirror this one (it does when every string entered through encode_bulk / dict_strings_load)."""
        n_dev, _ = ctx.dict_strings_info()
        if n_dev != len(self.id_to_string):
            ctx.dict_strings_load(self.id_to_string)
        ids, first = ctx.dict_encode(terms)
        for pos in first:
            t = terms[int(pos)]
            assert len(self.id_to_string) < 0x8000_0000, "Dictionary ID space exhausted"  # dictionary.rs:36-40
            self.string_to_id[t] = len(self.id_to_string)
            self.id_to_string.append(t)
        return ids

    def lookup(self, value: str) -> Optional[int]:
        return self.string_to_id.get(value)

    def decode(self, i: int) -> Optional[str]:
        return self.id_to_string[i] if 0 <= i < len(self.id_to_string) else None

    def numeric_table(self) -> Tuple[np.ndarray, np.ndarray]:
        n = len(self.id_to_string)
        num = np.zeros(n, dtype=np.float64)
        isn = np.zeros(n, dtype=np.uint8)
        for i, s in enumerate(self.id_to_string):
            v = rust_parse_f64(s)
            if v is not None:
                num[i] = v
                isn[i] = 1
        return num, isn


def _push_new_strings(ctx, dictionary: Dictionary, synced: int) -> bool:
    """the device dictionary takes the host strings it lacks. When it still holds the `synced` strings this mirror put there, only
    id_to_string[synced:] go up (kb_dict_encode, which must hand them the ids synced.. in order); otherwise, or when the ids differ, the
    whole dictionary is reloaded. Returns True when the device kept its earlier strings (a numeric table over them stays valid)."""
    n = len(dictionary.id_to_string)
    n_dev, _ = ctx.dict_strings_info()
    if synced >= 0 and n_dev == synced <= n:
        if n == synced:
            return True
        ids, _ = ctx.dict_encode(dictionary.id_to_string[synced:])
        if np.array_equal(ids, np.arange(synced, n, dtype=np.uint32)):
            return True
    ctx.dict_strings_load(dictionary.id_to_string)
    return False


def _derive_numeric(ctx, first_id: int = c.NUMERIC_APPEND):
    """kb_dict_numeric_derive of the f64 table from first_id (default: the ids it lacks); a table the call cannot extend (it holds more
    ids than the device dictionary: another dictionary's) is derived whole"""
    try:
        ctx.dict_numeric_derive(c.NUMERIC_F64, first_id)
    except c.KolibrieError as e:
        if e.status != c.KB_E_INVALID or first_id == 0:
            raise
        ctx.dict_numeric_derive(c.NUMERIC_F64, 0)


# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Variable:
    name: str


@dataclass(frozen=True)
class Constant:
    id: int


@dataclass(frozen=True)
class QuotedTriple:
    """Term::QuotedTriple(Box<(Term, Term, Term)>) (shared/src/terms.rs:19): an RDF-star pattern `<< s p o >>` in subject or object position"""
    s: object
    p: object
    o: object


Term = Union[Variable, Constant, QuotedTriple]
TriplePattern = Tuple[Term, Term, Term]

QUOTED_TRIPLE_ID_BIT = 0x8000_0000  # shared/src/quoted_triple_store.rs:17


def is_quoted_triple_id(i: int) -> bool:
    return (i & QUOTED_TRIPLE_ID_BIT) != 0


class QuotedTripleStore:
    """shared/src/quoted_triple_store.rs:28-80: quoted triples as u32 ids with bit 31 set, bidirectional, deduplicating; components
    may themselves be quoted-triple ids (nesting)."""

    def __init__(self):
        self.id_to_components: Dict[int, Tuple[int, int, int]] = {}
        self.components_to_id: Dict[Tuple[int, int, int], int] = {}
        self.next_qt_id = QUOTED_TRIPLE_ID_BIT

    def encode(self, subject: int, predicate: int, obj: int) -> int:
        key = (int(subject), int(predicate), int(obj))
        i = self.components_to_id.get(key)
        if i is not None:
            return i
        i = self.next_qt_id
        self.next_qt_id += 1
        self.id_to_components[i] = key
        self.components_to_id[key] = i
        return i

    def decode(self, i: int) -> Optional[Tuple[int, int, int]]:
        return self.id_to_components.get(int(i))

    def __len__(self):
        return len(self.id_to_components)

    def is_empty(self) -> bool:
        return not self.id_to_components

    def merge(self, other: "QuotedTripleStore"):
        for i, comp in other.id_to_components.items():
            self.id_to_components.setdefault(i, comp)
            self.components_to_id.setdefault(comp, i)
        self.next_qt_id = max(self.next_qt_id, other.next_qt_id)


def _clean_term(t: str) -> str:
    """the plain-term branch of encode_term_star (sparql_database.rs:96-106) on a trimmed term"""
    if t.startswith("<") and t.endswith(">"):
        return t[1:-1]
    if t.startswith('"'):
        close = t[1:].find('"')
        return t[1:close + 1] if close >= 0 else t.strip('"')
    return t


def _split_quoted_content(content: str) -> Tuple[str, str, str]:
    """split_quoted_triple_content (sparql_database.rs:125-190): `s p o` split at top-level whitespace, outside IRIs, literals and
    nested `<< >>`; parts past the third are joined into the object, missing ones are empty"""
    parts: List[str] = []
    cur = ""
    depth = 0
    in_uri = in_lit = esc = False
    for ch in content:
        if esc:
            cur += ch
            esc = False
        elif ch == "\\" and in_lit:
            cur += ch
            esc = True
        elif ch == '"' and not in_uri:
            in_lit = not in_lit
            cur += ch
        elif ch == "<" and not in_lit:
            cur += ch
            if cur.endswith("<<"):
                depth += 1
            elif depth == 0:
                in_uri = True
        elif ch == ">" and not in_lit:
            cur += ch
            if in_uri:
                in_uri = False
            elif cur.endswith(">>") and depth > 0:
                depth -= 1
        elif ch in " \t\n\r" and depth == 0 and not in_uri and not in_lit:
            if cur.strip():
                parts.append(cur.strip())
                cur = ""
        else:
            cur += ch
    if cur.strip():
        parts.append(cur.strip())
    if len(parts) >= 3:
        return parts[0], parts[1], " ".join(parts[2:])
    parts += [""] * (3 - len(parts))
    return parts[0], parts[1], parts[2]


def _strip(v: str) -> str:
    return v[1:] if v.startswith("?") else v  # engine.rs strips '?' from variable names everywhere


class SlotMap:
    """variable name <-> integer slot (variables never reach the device as strings)"""

    def __init__(self):
        self.slot: Dict[str, int] = {}
        self.names: List[str] = []
        self.bind_out: set = set()   # slots a Bind wrote: a KB_ID_NONE there is an unbound variable (left out of result rows)
        self.bind_only: set = set()  # Bind outputs no device operator may read (unbound rows, or strings the numeric table lacks)
        self.ragged: set = set()     # slots a VALUES block binds: a KB_ID_NONE there is an UNDEF cell, which each join treats its own way

    def of(self, name: str) -> int:
        name = _strip(name)
        if name not in self.slot:
            self.slot[name] = len(self.names)
            self.names.append(name)
        return self.slot[name]

    def term(self, t: Term) -> c.KbTerm:
        if isinstance(t, QuotedTriple):
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, "a quoted-triple term must be resolved on the host first (ExecutionEngine._scan_quoted)")
        return c.V(self.of(t.name)) if isinstance(t, Variable) else c.K(t.id)

    def pattern(self, p: TriplePattern) -> c.KbPattern:
        return c.pattern(self.term(p[0]), self.term(p[1]), self.term(p[2]))

    def quoted_pattern(self, p: TriplePattern) -> c.KbQuotedPattern:
        """kb_quoted_pattern of a pattern with a `<< s p o >>` subject and/or object: inside it, a nested quoted term is KB_TERM_QUOTED
        ("any quoted-triple id", engine.rs:1100-1105)"""
        def inner(t) -> c.KbTerm:
            return c.KbTerm(c.KB_TERM_QUOTED, 0) if isinstance(t, QuotedTriple) else self.term(t)

        def position(t):
            if isinstance(t, QuotedTriple):
                return c.KbTerm(c.KB_TERM_QUOTED, 0), c.pattern(inner(t.s), inner(t.p), inner(t.o))
            return self.term(t), c.KbPattern()

        if isinstance(p[1], QuotedTriple):
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, "quoted triple in predicate position")
        s, inner_s = position(p[0])
        pt = self.term(p[1])
        o, inner_o = position(p[2])
        return c.KbQuotedPattern(c.pattern(s, pt, o), inner_s, inner_o)


# ---------------------------------------------------------------------------------------------------------------------
# FILTER expressions (shared/src/query.rs:15-57) and their evaluation contract (types.rs:110-186)
@dataclass
class Comparison:
    var: str
    op: str
    value: str


@dataclass
class And:
    left: object
    right: object


@dataclass
class Or:
    left: object
    right: object


@dataclass
class Not:
    inner: object


@dataclass
class Arith:
    """ArithmeticExpression: ('op', l, r) trees with str operands; truthy when != 0"""
    expr: object


@dataclass
class FunctionCall:
    name: str
    args: List[str]


_CMP = {">": c.CMP_GT, ">=": c.CMP_GE, "<": c.CMP_LT, "<=": c.CMP_LE}
_SLOT_OPS = {c.F_CMP_NUM, c.F_EQ_ID, c.F_NE_ID, c.F_PUSH_VAR, c.F_IS_TRIPLE, c.F_CMP_LEGACY}  # filter ops that read row[slot]


class Condition:
    def __init__(self, expression):
        self.expression = expression

    def compile(self, slots: SlotMap, dictionary: Dictionary) -> List[c.KbFilterOp]:
        ops: List[c.KbFilterOp] = []

        def arith(e):
            if isinstance(e, str):
                if e.startswith("?"):
                    ops.append(c.fop(c.F_PUSH_VAR, slot=slots.of(e)))
                else:
                    v = rust_parse_f64(e)
                    if v is None:
                        raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"arithmetic operand {e!r} is not a number (the reference evaluates the filter to false)")
                    ops.append(c.fop(c.F_PUSH_CONST, value=v))
                return
            kind, l, r = e
            arith(l)
            arith(r)
            ops.append(c.fop({"+": c.F_ADD, "-": c.F_SUB, "*": c.F_MUL, "/": c.F_DIV}[kind]))

        def rec(e):
            if isinstance(e, Comparison):
                slot = slots.of(e.var)
                if e.op in ("=", "!="):
                    # decoded == literal  <=>  id == encode(literal) when the literal is in the dictionary (types.rs:131-132)
                    lit = dictionary.lookup(e.value)
                    ops.append(c.fop(c.F_EQ_ID if e.op == "=" else c.F_NE_ID, slot=slot, id=c.KB_ID_NONE if lit is None else lit))
                elif e.op in _CMP:
                    v = rust_parse_f64(e.value)  # types.rs:133-148: value.parse::<f64>().unwrap_or(0.0) — also for "?other" (quirk Q10)
                    ops.append(c.fop(c.F_CMP_NUM, slot=slot, cmp=_CMP[e.op], value=0.0 if v is None else v))
                else:
                    raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"operator {e.op!r}: the reference evaluates it to false")
            elif isinstance(e, And):
                rec(e.left); rec(e.right); ops.append(c.fop(c.F_AND))
            elif isinstance(e, Or):
                rec(e.left); rec(e.right); ops.append(c.fop(c.F_OR))
            elif isinstance(e, Not):
                rec(e.inner); ops.append(c.fop(c.F_NOT))
            elif isinstance(e, Arith):
                arith(e.expr); ops.append(c.fop(c.F_TRUTHY))
            elif isinstance(e, FunctionCall):
                if e.name == "isTRIPLE" and e.args:
                    ops.append(c.fop(c.F_IS_TRIPLE, slot=slots.of(e.args[0])))
                else:
                    raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"function {e.name!r}: the reference evaluates it to false")
            else:
                raise TypeError(e)

        rec(self.expression)
        return ops


# ---------------------------------------------------------------------------------------------------------------------
# PhysicalOperator (operators/physical.rs:16-76) — the variants on the hot path
@dataclass
class TableScan:
    pattern: TriplePattern


@dataclass
class IndexScan:
    pattern: TriplePattern


@dataclass
class Filter:
    input: object
    condition: Condition


@dataclass
class Projection:
    input: object
    variables: List[str]


@dataclass
class HashJoin:
    left: object
    right: object


@dataclass
class OptimizedHashJoin:
    left: object
    right: object


@dataclass
class NestedLoopJoin:
    left: object
    right: object


@dataclass
class ParallelJoin:
    left: object
    right: object


@dataclass
class StarJoin:
    join_var: str
    patterns: List[TriplePattern]


@dataclass
class InMemoryBuffer:
    content: List[Dict[str, int]]


@dataclass
class Bind:
    """PhysicalOperator::Bind (operators/physical.rs; engine.rs:144-277): a built-in function of the input's rows into
    output_variable. Arguments are strings as in the reference: "?x" a variable, anything else a constant."""
    input: object
    function_name: str
    arguments: List[str]
    output_variable: str


@dataclass
class Values:
    """PhysicalOperator::Values (operators/physical.rs; engine.rs:279-308): the rows of a VALUES block, each a list of terms in header
    order, None for UNDEF (a row may be shorter than the header)"""
    variables: List[str]
    values: List[List[Optional[str]]]


_BIND_FUNCTIONS = {"SUBJECT": c.BIND_SUBJECT, "PREDICATE": c.BIND_PREDICATE, "OBJECT": c.BIND_OBJECT, "isTRIPLE": c.BIND_IS_TRIPLE,
                   "TRIPLE": c.BIND_TRIPLE, "CONCAT": c.BIND_CONCAT}


class SparqlDatabase:
    """triples (set semantics, iteration in (s,p,o) order like the reference's BTreeSet) + dictionary + the device store."""

    def __init__(self, ctx: Optional[c.Context] = None, device: int = 0):
        self.dictionary = Dictionary()
        self.quoted_triple_store = QuotedTripleStore()  # sparql_database.rs:58
        self.triples: set = set()
        self.ctx = ctx or c.Context(device)
        self._uploaded_version = -1
        self._version = 0
        self._uploaded_quoted = -1  # size of the quoted-triple store the context's table was loaded from
        self.prefixes: List[Tuple[str, str]] = []  # sparql_database.rs:54, ordered: the Turtle header lists them in this order
        self.cached_stats = None  # sparql_database.rs:58: get_or_build_stats fills it, invalidate_stats_cache empties it

    def encode_term(self, t) -> int:
        """a term given as a string, or as a nested (s, p, o) tuple for a quoted triple `<< s p o >>` (components encoded first, in
        s, p, o order, then the quoted triple itself: sparql_database.rs encode_quoted_triple)"""
        if isinstance(t, (tuple, list)):
            s, p, o = (self.encode_term(x) for x in t)
            return self.quoted_triple_store.encode(s, p, o)
        return self.dictionary.encode(t)

    def decode_term(self, i: int) -> Optional[str]:
        """Dictionary::decode_term (dictionary.rs:58-68): quoted-triple ids decode recursively to `<< s p o >>`"""
        if is_quoted_triple_id(i):
            comp = self.quoted_triple_store.decode(i)
            if comp is None:
                return None
            parts = [self.decode_term(x) for x in comp]
            if any(x is None for x in parts):
                return None
            return "<< " + " ".join(parts) + " >>"
        return self.dictionary.decode(i)

    def set_prefixes(self, prefixes):
        """SparqlDatabase::set_prefixes (sparql_database.rs:193-195) with an ORDER: (name, uri) pairs, or a dict in its iteration order.
        The reference keeps a HashMap, so the order of its Turtle header is unspecified; here it is this order."""
        self.prefixes = [(str(k), str(v)) for k, v in (prefixes.items() if isinstance(prefixes, dict) else prefixes)]

    def generate_ntriples(self) -> str:
        """SparqlDatabase::generate_ntriples (sparql_database.rs:301-322): the store as N-Triples-star, rendered on the device"""
        return self._serialize(c.SER_NTRIPLES)

    def generate_turtle(self) -> str:
        """SparqlDatabase::generate_turtle (sparql_database.rs:324-382): the store as Turtle-star with this database's prefixes"""
        return self._serialize(c.SER_TURTLE)

    def _serialize(self, fmt: int) -> str:
        if hasattr(self.ctx, "serialize"):  # sorted, grouped and written on the device (kb_serialize_begin / _next)
            self._sync()
            return b"".join(self.ctx.serialize(fmt, self.prefixes)).decode("utf-8")
        # contexts without it (the oracle): the reference's loops over the triple set, decode_any(..).unwrap_or_default()
        text = lambda i: self.decode_term(i) or ""
        subj = lambda t: t if t.startswith("<<") else f"<{t}>"
        obj = lambda t: t if t.startswith("<<") else f"<{t}>" if t.startswith(("http://", "https://")) else f'"{t}"'
        rows = [tuple(text(x) for x in t) for t in sorted(self.triples)]
        if fmt == c.SER_NTRIPLES:
            return "".join(f"{subj(s)} <{p}> {obj(o)} .\n" for s, p, o in rows)
        out = [f"@prefix {k}: <{v}> .\n" for k, v in self.prefixes] + (["\n"] if self.prefixes else [])
        groups: Dict[str, Dict[str, List[str]]] = {}
        for s, p, o in rows:
            groups.setdefault(s, {}).setdefault(p, []).append(o)
        for s in sorted(groups):  # str order = UTF-8 byte order (Rust String)
            preds = groups[s]
            out.append(subj(s) + " ;\n    ".join(f" <{p}>"[i > 0:] + " ,".join(" " + obj(o) for o in preds[p]) for i, p in enumerate(sorted(preds))) + " .\n")
        return "".join(out)

    def get_or_build_stats(self):
        """SparqlDatabase::get_or_build_stats (sparql_database.rs:197-205): the cached planner.DatabaseStats, or a new one from
        DatabaseStats::gather_stats_fast, gathered on the device (kb_store_gather_stats) and cached. As in the reference, a later change
        to the triples does not refresh the cache: call invalidate_stats_cache() after one, as the reference's INSERT / DELETE do."""
        if self.cached_stats is None:
            from . import planner

            if hasattr(self.ctx, "store_gather_stats"):
                self._sync()
                g = self.ctx.store_gather_stats(c.GATHER_STATS_FAST)
                maps = [dict(zip(g[k][0].tolist(), g[k][1].tolist())) for k in ("subject", "predicate", "object")]
                total, quoted = g["total_triples"], g["quoted_triple_count"]
            else:  # contexts without it (the oracle): gather_stats_fast over the host set
                total, quoted = len(self.triples), len(self.quoted_triple_store)
                maps = _gather_stats_fast(sorted(self.triples), c.GATHER_STATS_FAST)
            self.cached_stats = planner.DatabaseStats.from_counts(total, maps[1], maps[0], maps[2], quoted_triple_count=quoted)
        return self.cached_stats

    def invalidate_stats_cache(self):
        """SparqlDatabase::invalidate_stats_cache (sparql_database.rs:207-209): the next get_or_build_stats gathers again"""
        self.cached_stats = None

    def query(self) -> "QueryBuilder":
        """SparqlDatabase::query (sparql_database.rs): the fluent QueryBuilder over this database"""
        return QueryBuilder(self)

    def add_statement(self, s, p, o):
        """add one triple whose terms are strings or nested tuples (quoted triples)"""
        self.add_triple((self.encode_term(s), self.encode_term(p), self.encode_term(o)))

    def add_triple_parts(self, s: str, p: str, o: str):
        t = (self.dictionary.encode(s), self.dictionary.encode(p), self.dictionary.encode(o))
        self.add_triple(t)

    def add_triples_bulk(self, statements: Sequence[Tuple[str, str, str]]):
        """bulk load of parsed (s, p, o) STRING triples (what parse_ntriples / parse_rdf hand to the per-term encode loop,
        sparql_database.rs:1000-1013): one device encode of all 3n terms in s, p, o order per triple — the ids are those of the
        sequential loop (dictionary.rs:32-48) — then the triples join the set"""
        terms = [t for st in statements for t in st]
        ids = self.dictionary.encode_bulk(self.ctx, terms).reshape(-1, 3)
        for row in ids:
            self.add_triple((int(row[0]), int(row[1]), int(row[2])))

    def add_triple(self, t: Tuple[int, int, int]):  # sparql_database.rs:215-226
        if t not in self.triples:
            self.triples.add(t)
            self._version += 1

    def delete_triple(self, t: Tuple[int, int, int]) -> bool:  # sparql_database.rs:229-242
        if t in self.triples:
            self.triples.remove(t)
            self._version += 1
            return True
        return False

    def insert_triples(self, ids) -> List[bool]:
        """add_triple of each (s, p, o) id triple in order, applied to this set and to the device store together (kb_store_insert):
        result[i] is whether triple i was new. The device store is left current, so the next query uploads nothing; it keeps the new
        triples in a segment of their own, in batch order, rather than in the set's order."""
        return self._write(ids, insert=True)

    def delete_triples(self, ids) -> List[bool]:
        """delete_triple of each (s, p, o) id triple in order, on this set and on the device store together (kb_store_remove):
        result[i] is whether triple i was there to remove"""
        return self._write(ids, insert=False)

    def _write(self, ids, insert: bool) -> List[bool]:
        arr = np.asarray(ids, dtype=np.uint32).reshape(-1, 3)
        if len(arr) == 0:
            return []
        self._sync()  # the device store holds this set before the batch applies to both
        if insert:
            dev = self.ctx.store_insert(arr[:, 0], arr[:, 1], arr[:, 2])
        else:
            dev = self.ctx.store_remove(arr[:, 0], arr[:, 1], arr[:, 2])
        flags = []
        for row in arr:
            t = (int(row[0]), int(row[1]), int(row[2]))
            flags.append(t not in self.triples if insert else t in self.triples)
            if insert:
                self.triples.add(t)
            else:
                self.triples.discard(t)
        if flags != [bool(f) for f in dev]:
            raise RuntimeError("the device store and the host set disagree on a batch write")
        if any(flags):
            self._version += 1
            self._uploaded_version = self._version
        # the device dictionary and its numeric side table take the strings the batch's terms added (encode_bulk has put them in the
        # device dictionary already; terms encoded on the host have not)
        n_dev, _ = self.ctx.dict_strings_info()
        kept = n_dev == len(self.dictionary.id_to_string) or _push_new_strings(self.ctx, self.dictionary, n_dev)
        _derive_numeric(self.ctx, c.NUMERIC_APPEND if kept else 0)
        self._sync_quoted()
        return flags

    def encode_terms_star(self, terms: Sequence[str]) -> List[int]:
        """encode_term_star (sparql_database.rs:82-109) of each term in order: a `<< s p o >>` term is split
        (split_quoted_triple_content, :125-190), its components encoded first and the triple then; a plain term is trimmed and
        cleaned (<iri> loses its brackets, a literal keeps what lies between its first two quotes). All plain terms go through one
        device encode (Dictionary.encode_bulk) in the order the reference's recursion meets them, so they get the same ids."""
        self._sync()  # the device dictionary mirrors this one before the batch encode (a shared context may hold another's)
        plain: List[str] = []

        def walk(term: str):  # -> a plan: ("d", position in plain) or ("q", plan_s, plan_p, plan_o)
            t = term.strip()
            if t.startswith("<<") and t.endswith(">>"):
                return ("q",) + tuple(walk(x) for x in _split_quoted_content(t[2:-2].strip()))
            plain.append(_clean_term(t))
            return ("d", len(plain) - 1)

        plans = [walk(t) for t in terms]
        ids = self.dictionary.encode_bulk(self.ctx, plain) if plain else np.empty(0, np.uint32)

        def resolve(plan) -> int:
            if plan[0] == "d":
                return int(ids[plan[1]])
            return self.quoted_triple_store.encode(resolve(plan[1]), resolve(plan[2]), resolve(plan[3]))

        return [resolve(pl) for pl in plans]

    def handle_update(self, kind: str, triples: Sequence[Tuple[str, str, str]]) -> str:
        """SparqlDatabase::handle_update (sparql_database.rs:3091-3117) given what parse_insert / parse_delete yield: the kind
        ("INSERT" or "DELETE") and the term strings of each triple. Every term is encoded with encode_term_star, then the triples are
        inserted or removed as one batch on the host set and the device store. Returns the reference's strings."""
        if kind not in ("INSERT", "DELETE"):
            return "Update Failed"
        ids = self.encode_terms_star([x for t in triples for x in t])
        if kind == "INSERT":
            self.insert_triples(ids)
        else:
            self.delete_triples(ids)
        return "Update Successful"

    def execute_delete_where(self, delete_template: Sequence[Tuple[str, str, str]], where_patterns: Sequence[Tuple[str, str, str]],
                             insert_template: Optional[Sequence[Tuple[str, str, str]]] = None) -> int:
        """DELETE { delete_template } WHERE { where_patterns } [INSERT { insert_template }] as execute_query_rayon_parallel2_volcano runs
        it (execute_query.rs:354-413). Terms are the parser's strings ("?x", "<iri>", "\\"literal\\"", "<< s p o >>" in a template).
        The WHERE runs on the device (kb_bgp_execute); kb_store_remove_template then fills the template from its rows and removes the
        result from the device store, and the host set loses the same triples. Where the device refuses a binding (one that
        encode_term_star would not map back to its own id, or a template variable the WHERE leaves unbound) the reference's loop runs
        instead: every row decoded, every filled term encoded with encode_term_star, the triples removed as one batch. Returns the
        triples removed. The reference's quirks are kept:
          - the WHERE is its patterns only: the reference rebuilds the query from them, so a FILTER in it has no effect;
          - the INSERT template is inserted as written (process_insert_clause, execute_query.rs:758-773), so "?x" in it is a term;
          - the template's constants are encoded for the first WHERE row, so a DELETE of unknown terms adds them to the dictionary.
        A WHERE constant is looked up in the dictionary (one it lacks matches nothing); a quoted term in the WHERE is refused
        (ValueError)."""
        self._sync()
        slots = SlotMap()
        pats, matches = [], True
        for tp in where_patterns:
            terms = []
            for x in tp:
                if x.startswith("?"):
                    terms.append(c.V(slots.of(x)))
                    continue
                t = x.strip()
                if t.startswith("<<") and t.endswith(">>"):
                    raise ValueError("a quoted term in the WHERE of a DELETE WHERE is not supported")
                i = self.dictionary.lookup(_clean_term(t))
                matches = matches and i is not None
                terms.append(c.K(0 if i is None else i))
            pats.append(c.pattern(*terms))
        removed = 0
        rel = self.ctx.bgp_execute(pats) if pats and matches else None
        try:
            if rel is not None and rel.n_rows:
                removed = self._remove_template(rel, slots, delete_template)
        finally:
            if rel is not None:
                rel.free()
        if insert_template:
            self.handle_update("INSERT", insert_template)
        return removed

    def _remove_template(self, rel: c.Relation, slots: SlotMap, template: Sequence[Tuple[str, str, str]]) -> int:
        consts = [x for tp in template for x in tp if not x.startswith("?")]
        ids = iter(self.encode_terms_star(consts))  # what the first row's encode_term_star calls add, in their order
        _derive_numeric(self.ctx)
        tmpl = [c.pattern(*[c.V(slots.of(x)) if x.startswith("?") else c.K(next(ids)) for x in tp]) for tp in template]
        self._sync_quoted()
        rel_slots = rel.slots
        rows = rel.to_numpy(rel_slots)
        try:
            n = self.ctx.store_remove_template(rel, tmpl)
        except c.KolibrieError as e:
            if e.status != c.KB_E_UNSUPPORTED:
                raise
            # the reference's loop: each row's bindings as text, the filled terms encoded with encode_term_star, one remove batch
            col = {name: rel_slots.index(s) for name, s in slots.slot.items() if s in rel_slots}
            terms = []
            for row in rows:
                for tp in template:
                    for x in tp:
                        j = col.get(_strip(x)) if x.startswith("?") else None
                        v = self.decode_term(int(row[j])) if j is not None and int(row[j]) != c.KB_ID_NONE else None
                        terms.append(x if v is None else v)
            return sum(self.delete_triples(self.encode_terms_star(terms)))
        # the device removed the filled triples; the host set loses the same ones
        col = [[rel_slots.index(t.value) if t.is_var else None for t in (p.s, p.p, p.o)] for p in tmpl]
        const = [[t.value for t in (p.s, p.p, p.o)] for p in tmpl]
        gone = 0
        for row in rows:
            for cj, cv in zip(col, const):
                t = tuple(int(row[j]) if j is not None else v for j, v in zip(cj, cv))
                if t in self.triples:
                    self.triples.remove(t)
                    gone += 1
        if gone != n:
            raise RuntimeError("the device store and the host set disagree on a DELETE WHERE")
        if n:
            self._version += 1
            self._uploaded_version = self._version
        return n

    def union(self, other: "SparqlDatabase") -> "SparqlDatabase":
        """SparqlDatabase::union (sparql_database.rs:1874-1933): a new database on a new context on this one's device. Its dictionary is
        a clone of this one's extended with other's strings in the order the reference re-encodes other's triples (ascending (s, p, o)
        of other's ids, s, p, o of each); its triples are this set together with other's re-encoded set; it shares this database's
        quoted-triple store and prefixes, and has no index, cached statistics or stream log. On the device (kb_store_union) the new
        context's store, dictionary strings and quoted table are built there and the triple set and new strings are downloaded; the host
        restatement runs for contexts without the entry point and for an `other` that shares this context (one context holds one store).
        An id of other's triples that other's dictionary does not map (a quoted id, an id past it: the reference's decode(..).unwrap()
        panics) raises ValueError and changes nothing."""
        if self._device_pair(other, "store_union"):
            self._sync_strings()
            other._sync_strings()
            out = SparqlDatabase(ctx=c.Context(self.ctx.device))
            try:
                info = out.ctx.store_union(self.ctx, other.ctx)
            except c.KolibrieError as e:
                out.ctx.close()
                if e.status == c.KB_E_INVALID:
                    raise ValueError(str(e)) from e
                if e.status != c.KB_E_UNSUPPORTED:
                    raise
            else:
                out.dictionary = self._clone_dictionary()
                for t in out.ctx.dict_strings_download(info["dict_first"], info["dict_new"]):
                    out.dictionary.encode(t)
                self.last_union_info = info
                return self._device_result(out)
        merged = self._clone_dictionary()
        re_encoded = set()
        for t in sorted(other.triples):
            ids = []
            for x in t:
                v = other.dictionary.decode(x)
                if v is None:
                    raise ValueError(f"id {x} of other's triple {t} has no string in other's dictionary (the reference's decode(..).unwrap() panics)")
                ids.append(merged.encode(v))
            re_encoded.add(tuple(ids))
        out = SparqlDatabase(ctx=self._new_context())
        out.dictionary = merged
        for t in sorted(self.triples | re_encoded):
            out.add_triple(t)
        return self._host_result(out)

    def par_join(self, other: "SparqlDatabase", predicate: str) -> "SparqlDatabase":
        """SparqlDatabase::par_join (sparql_database.rs:1935-2005): `predicate` is encoded in this dictionary (which may add it); with A
        this set's triples with that id and B other's (ids compared raw), the new database holds (s, p, y) for (s,p,o) in A and (o,p,y)
        in B, and (s, p, o) for (s,p,o) in A whose o is the object of a triple of B. It shares this database's dictionary and
        quoted-triple store, on a new context on this one's device (kb_store_par_join; the host restatement as for union)."""
        pid = self.dictionary.encode(predicate)
        if self._device_pair(other, "store_par_join"):
            self._sync_strings()
            other._sync()
            out = SparqlDatabase(ctx=c.Context(self.ctx.device))
            try:
                info = out.ctx.store_par_join(self.ctx, other.ctx, pid)
            except c.KolibrieError as e:
                out.ctx.close()
                if e.status != c.KB_E_UNSUPPORTED:
                    raise
            else:
                out.dictionary = self.dictionary
                self.last_par_join_info = info
                return self._device_result(out)
        keyed: Dict[int, List[Tuple[int, int, int]]] = {}
        for t in other.triples:
            if t[1] == pid:
                keyed.setdefault(t[0], []).append(t)
                keyed.setdefault(t[2], []).append(t)
        out = SparqlDatabase(ctx=self._new_context())
        out.dictionary = self.dictionary
        for t in sorted({(s, q[1], q[2]) for s, p, o in self.triples if p == pid for q in keyed.get(o, ())}):
            out.add_triple(t)
        return self._host_result(out)

    def _device_pair(self, other: "SparqlDatabase", entry: str) -> bool:
        """whether union / par_join run on the device: the context has the entry point and `other` is this database or has a context
        of its own on the same device"""
        return hasattr(self.ctx, entry) and (other is self or (other.ctx is not self.ctx and getattr(other.ctx, "device", None) == self.ctx.device))

    def _new_context(self):
        return c.Context(self.ctx.device) if isinstance(self.ctx, c.Context) else type(self.ctx)()

    def _clone_dictionary(self) -> Dictionary:
        d = Dictionary()
        d.string_to_id = dict(self.dictionary.string_to_id)
        d.id_to_string = list(self.dictionary.id_to_string)
        return d

    def _host_result(self, out: "SparqlDatabase") -> "SparqlDatabase":
        out.quoted_triple_store = self.quoted_triple_store  # Arc::clone(&self.quoted_triple_store)
        out.prefixes = list(self.prefixes)
        return out

    def _device_result(self, out: "SparqlDatabase") -> "SparqlDatabase":
        """the new context holds the result: its triple set is downloaded and marked uploaded, its numeric side table derived"""
        s, p, o = out.ctx.store_download()
        out.triples = set(zip(s.tolist(), p.tolist(), o.tolist()))
        out._uploaded_version = out._version
        out.quoted_triple_store = self.quoted_triple_store
        out._uploaded_quoted = len(out.quoted_triple_store)  # the new context's table is a copy of this one's
        out.prefixes = list(self.prefixes)
        out.ctx.dict_numeric_derive(c.NUMERIC_F64, 0)
        return out

    def _sync_strings(self):
        """the store, and the device dictionary holding every string of this dictionary (strings encoded since the last upload go up)"""
        self._sync()
        n_dev, _ = self.ctx.dict_strings_info()
        if n_dev != len(self.dictionary.id_to_string):
            kept = _push_new_strings(self.ctx, self.dictionary, n_dev)
            _derive_numeric(self.ctx, c.NUMERIC_APPEND if kept else 0)

    def build_all_indexes(self):
        """The reference builds its six hash indexes here (sparql_database.rs:3364-3394); the device store is (re)uploaded and
        partitioned by predicate (kb_store_build_index)."""
        self._sync()
        self.ctx.build_index()

    def _sync(self):
        self._sync_quoted()
        if self._uploaded_version == self._version:
            return
        arr = np.array(sorted(self.triples), dtype=np.uint32).reshape(-1, 3)  # (s,p,o) order: the reference's BTreeSet iteration
        self.ctx.store_load(arr[:, 0], arr[:, 1], arr[:, 2])
        if hasattr(self.ctx, "dict_numeric_derive"):  # the numeric side table parsed on the device from the strings
            self.ctx.dict_strings_load(self.dictionary.id_to_string)  # the final id -> string step runs on the device too
            self.ctx.dict_numeric_derive(c.NUMERIC_F64, 0)
        else:
            num, isn = self.dictionary.numeric_table()
            self.ctx.dict_numeric_load(num, isn)
            self.ctx.dict_strings_load(self.dictionary.id_to_string)
        self._uploaded_version = self._version

    def _sync_quoted(self):
        """the quoted-triple table on the device (kb_quoted_load) whenever the store's size changed (it only grows: encode never
        removes an entry); an empty store CLEARS the table, so that a context shared with another database never keeps that one's table"""
        qts = self.quoted_triple_store
        if len(qts) == self._uploaded_quoted or not hasattr(self.ctx, "quoted_load"):
            return
        ids = np.fromiter(qts.id_to_components.keys(), dtype=np.uint32, count=len(qts))
        comp = np.array(list(qts.id_to_components.values()), dtype=np.uint32).reshape(-1, 3)
        self.ctx.quoted_load(ids, comp[:, 0], comp[:, 1], comp[:, 2])
        self._uploaded_quoted = len(qts)


_QB_TEXT = {"Contains": c.QB_CONTAINS, "StartsWith": c.QB_STARTS, "EndsWith": c.QB_ENDS}
_QB_JOIN = {"OnSubject": c.QB_ON_SUBJECT, "OnPredicate": c.QB_ON_PREDICATE, "OnObject": c.QB_ON_OBJECT}


class QueryBuilder:
    """QueryBuilder (query_builder.rs:39-643) without its streaming half: the same builder methods and results, answered on the device
    (kb_qb_triples / kb_qb_terms) whenever no Python callable is involved. A position filter is a TripleFilter as a tuple: ("Exact" |
    "Contains" | "StartsWith" | "EndsWith", text) or ("Custom", callable on the decoded string); the with_* methods set them, and
    subject_filter / predicate_filter / object_filter may be set to a ("Custom", fn) directly, as the reference's enum allows. Results:
    get_triples() a set of (s, p, o) id tuples (sorted() gives the BTreeSet order), get_decoded_triples() a list of string triples,
    get_subjects() / get_predicates() / get_objects() lists of strings, count() an int, group_by() a dict in key order.
    The host restatement runs instead for filter(fn), a ("Custom", fn) position filter or join_with(fn) (a Python callable cannot cross
    the C ABI), for contexts without the device query or without device dictionary strings, and for a join with another database that
    shares this one's context. `last_path` records which ran ("device" or "host"). order_by / asc / desc have no effect, as in the
    reference: it collects the sorted rows back into a BTreeSet. An offset past the rows raises IndexError, where the reference panics."""

    def __init__(self, db: SparqlDatabase):
        self.db = db
        self.subject_filter = self.predicate_filter = self.object_filter = None
        self.custom_filter = None
        self.join_conditions: List = []
        self.join_db: Optional[SparqlDatabase] = None
        self.distinct_results = False
        self.sort_key = None
        self.descending = False
        self._limit: Optional[int] = None
        self._offset: Optional[int] = None
        self.last_path: Optional[str] = None

    def _set(self, attr, kind, text):
        setattr(self, attr, (kind, text))
        return self

    def with_subject(self, v): return self._set("subject_filter", "Exact", v)
    def with_subject_like(self, v): return self._set("subject_filter", "Contains", v)
    def with_subject_starting(self, v): return self._set("subject_filter", "StartsWith", v)
    def with_subject_ending(self, v): return self._set("subject_filter", "EndsWith", v)
    def with_predicate(self, v): return self._set("predicate_filter", "Exact", v)
    def with_predicate_like(self, v): return self._set("predicate_filter", "Contains", v)
    def with_predicate_starting(self, v): return self._set("predicate_filter", "StartsWith", v)
    def with_predicate_ending(self, v): return self._set("predicate_filter", "EndsWith", v)
    def with_object(self, v): return self._set("object_filter", "Exact", v)
    def with_object_like(self, v): return self._set("object_filter", "Contains", v)
    def with_object_starting(self, v): return self._set("object_filter", "StartsWith", v)
    def with_object_ending(self, v): return self._set("object_filter", "EndsWith", v)

    def filter(self, fn):
        self.custom_filter = fn
        return self

    def join(self, other: SparqlDatabase):
        self.join_db = other
        return self

    def join_on_subject(self):
        self.join_conditions.append("OnSubject")
        return self

    def join_on_predicate(self):
        self.join_conditions.append("OnPredicate")
        return self

    def join_on_object(self):
        self.join_conditions.append("OnObject")
        return self

    def join_with(self, fn):
        self.join_conditions.append(fn)
        return self

    def distinct(self):
        self.distinct_results = True
        return self

    def order_by(self, key):
        self.sort_key = key
        return self

    def desc(self):
        self.descending = True
        return self

    def asc(self):
        self.descending = False
        return self

    def limit(self, n: int):
        self._limit = n
        return self

    def offset(self, n: int):
        self._offset = n
        return self

    # ---- results
    def get_triples(self) -> set:
        return set(self._rows())

    def count(self) -> int:
        n = self._device(count_only=True)
        return len(self._host_rows()) if n is None else n

    def get_decoded_triples(self) -> List[Tuple[str, str, str]]:
        rel = self._device()
        if rel is not None:
            try:
                cols = [self.db.ctx.qb_terms(rel, k, c.QB_TERMS_EMPTY) for k in range(3)]
            finally:
                rel.free()
            return list(zip(*cols))
        d = self.db.dictionary.decode
        return [tuple(d(x) or "" for x in t) for t in self._host_rows()]

    def get_subjects(self) -> List[str]:
        return self._terms(0)

    def get_predicates(self) -> List[str]:
        return self._terms(1)

    def get_objects(self) -> List[str]:
        return self._terms(2)

    def group_by(self, key_fn) -> dict:
        """get_triples, then the key function on the host in set order; the groups in key order (a BTreeMap)"""
        groups: dict = {}
        for t in sorted(self.get_triples()):
            groups.setdefault(key_fn(t), []).append(t)
        return {k: groups[k] for k in sorted(groups)}

    def _terms(self, col: int) -> List[str]:
        rel = self._device()
        if rel is not None:
            try:
                return self.db.ctx.qb_terms(rel, col, c.QB_TERMS_DISTINCT if self.distinct_results else c.QB_TERMS_DROP)
            finally:
                rel.free()
        d = self.db.dictionary.decode
        out = [d(t[col]) for t in self._host_rows()]
        out = [x for x in out if x is not None]
        return sorted(set(out), key=lambda x: x.encode("utf-8")) if self.distinct_results else out

    def _joins(self) -> bool:
        return self.join_db is not None and bool(self.join_conditions)

    def _device(self, count_only: bool = False):
        """the relation of the rows (or their count), or None when the host restatement must run"""
        db, right = self.db, self.join_db if self._joins() else None
        filters = (self.subject_filter, self.predicate_filter, self.object_filter)
        if (self.custom_filter is not None or any(f is not None and f[0] == "Custom" for f in filters)
                or any(callable(j) for j in self.join_conditions) or not hasattr(db.ctx, "qb_triples")
                or (right is not None and right is not db and right.ctx is db.ctx)):
            self.last_path = "host"
            return None
        spec = []
        for f in filters:
            if f is None:
                spec.append(None)
            elif f[0] == "Exact":
                i = db.dictionary.lookup(f[1])
                spec.append((c.QB_EXACT, c.KB_ID_NONE if i is None else i))
            else:
                spec.append((_QB_TEXT[f[0]], f[1]))
        join = 0
        for j in self.join_conditions:
            join |= _QB_JOIN[j]
        db._sync()
        if right is not None:
            right._sync()
        try:
            rel, info = db.ctx.qb_triples(spec, join if right is not None else 0, right.ctx if right is not None else None, self._offset or 0,
                                       self._limit, count_only=count_only)
        except c.KolibrieError as e:
            if e.status == c.KB_E_UNSUPPORTED:
                self.last_path = "host"
                return None
            if e.status == c.KB_E_INVALID and self._offset:
                raise IndexError(str(e)) from e
            raise
        self.last_path = "device"
        return info["n_rows"] if count_only else rel

    def _rows(self) -> List[Tuple[int, int, int]]:
        """apply_filters (query_builder.rs:486-568): the rows in set order, on the device or by the host restatement"""
        rel = self._device()
        if rel is not None:
            try:
                return [tuple(int(x) for x in r) for r in rel.to_numpy()]
            finally:
                rel.free()
        return self._host_rows()

    def _host_rows(self) -> List[Tuple[int, int, int]]:
        """the host restatement of apply_filters and apply_join"""
        d = self.db.dictionary.decode

        def ok(f, tid):
            if f is None:
                return True
            v = d(tid)
            if v is None:
                return False
            kind, arg = f
            return (v == arg if kind == "Exact" else arg in v if kind == "Contains" else v.startswith(arg) if kind == "StartsWith"
                    else v.endswith(arg) if kind == "EndsWith" else bool(arg(v)))

        filters = (self.subject_filter, self.predicate_filter, self.object_filter)
        rows = sorted(t for t in self.db.triples if all(ok(f, x) for f, x in zip(filters, t))
                      and (self.custom_filter is None or self.custom_filter(t)))
        if self._joins():
            out = set()
            right = self.join_db.triples
            for j in self.join_conditions:
                for l in rows:
                    for r in right:
                        if j == "OnSubject" and l[0] == r[0] or j == "OnPredicate" and l[1] == r[1]:
                            out.add((l[0], l[1], r[2]))
                        elif (j == "OnObject" and l[2] == r[2]) or (callable(j) and j(l, r)):
                            out.add((l[0], r[1], r[2]))
            rows = sorted(out)
        if self._offset is not None or self._limit is not None:
            off = self._offset or 0
            if off > len(rows):
                raise IndexError(f"offset {off} past the {len(rows)} rows")
            rows = rows[off:] if self._limit is None else rows[off:off + self._limit]
        return rows


def _gather_stats_fast(triples, max_sample: int):
    """DatabaseStats::gather_stats_fast's counts (database_stats.rs:43-92) over `triples` in (s, p, o) order: every step-th of the first
    take * step triples, each counted `step` times; max_sample 0 counts every triple. Returns the subject, predicate and object maps."""
    total = len(triples)
    take = min(total, max_sample) if max_sample else total
    step = total // take if max_sample and total > max_sample else 1
    maps = ({}, {}, {})
    for t in triples[: take * step: step]:
        for m, x in zip(maps, t):
            m[x] = m.get(x, 0) + step
    return maps


class ExecutionEngine:
    """engine.rs:24-143 — static functions on a unit struct."""

    @staticmethod
    def _run(op, db: SparqlDatabase, slots: SlotMap) -> c.Relation:
        ctx = db.ctx
        if isinstance(op, (TableScan, IndexScan)):
            if any(isinstance(t, QuotedTriple) for t in op.pattern):
                if hasattr(ctx, "scan_quoted"):  # matched, joined and merged on the device (kb_scan_quoted)
                    return ctx.scan_quoted(slots.quoted_pattern(op.pattern))
                return ExecutionEngine._scan_quoted(op.pattern, db, slots)
            return ctx.scan([slots.pattern(op.pattern)])[0]
        if isinstance(op, Filter):
            # Selection directly over a star / scan: let the fused operator push conjuncts into its scans
            if isinstance(op.input, StarJoin):
                return ctx.star_join(slots.of(op.input.join_var), [slots.pattern(p) for p in op.input.patterns],
                                     op.condition.compile(slots, db.dictionary))
            rel = ExecutionEngine._run(op.input, db, slots)
            prog = op.condition.compile(slots, db.dictionary)
            ExecutionEngine._check_reads(slots, {o.slot for o in prog if o.op in _SLOT_OPS}, "a FILTER")
            return ctx.filter(rel, prog)
        if isinstance(op, Projection):
            rel = ExecutionEngine._run(op.input, db, slots)
            return ctx.project(rel, [slots.of(v) for v in op.variables])
        if isinstance(op, (HashJoin, OptimizedHashJoin, NestedLoopJoin)):
            return ExecutionEngine._join(ctx, slots, ExecutionEngine._run(op.left, db, slots), ExecutionEngine._run(op.right, db, slots), type(op).__name__)
        if isinstance(op, ParallelJoin):
            # right side a scan -> bind join (engine.rs:935-937) == natural join of left with the pattern's matches: kb_bind_join looks the
            # pattern up in the index's persistent tables when it can, and scans + joins otherwise
            if isinstance(op.right, (TableScan, IndexScan)) and not any(isinstance(t, QuotedTriple) for t in op.right.pattern) and hasattr(ctx, "bind_join"):
                left = ExecutionEngine._run(op.left, db, slots)
                pat = slots.pattern(op.right.pattern)
                shared = set(left.slots) & {t.value for t in (pat.s, pat.p, pat.o) if t.is_var}
                ExecutionEngine._check_reads(slots, shared, "a join")
                if shared & slots.ragged:  # bind_pattern leaves a variable the row lacks free: the join of mappings
                    return ctx.natural_join(left, ctx.scan([pat])[0])
                return ctx.bind_join(left, pat)
            return ExecutionEngine._join(ctx, slots, ExecutionEngine._run(op.left, db, slots), ExecutionEngine._run(op.right, db, slots), "ParallelJoin")
        if isinstance(op, StarJoin):
            return ctx.star_join(slots.of(op.join_var), [slots.pattern(p) for p in op.patterns])
        if isinstance(op, InMemoryBuffer):
            names = sorted({k for row in op.content for k in row})
            cols = [np.array([row[k] for row in op.content], dtype=np.uint32) for k in names]
            return ctx.rel_from_host([slots.of(k) for k in names], cols)
        if isinstance(op, Values):
            return ExecutionEngine._values(op, db, slots)
        if isinstance(op, Bind):
            rel = ExecutionEngine._run(op.input, db, slots)
            if hasattr(ctx, "bind"):  # on the device (kb_bind)
                return ExecutionEngine._bind_device(op, rel, db, slots)
            return ExecutionEngine._bind_rel(op, rel, db, slots)
        raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"operator {type(op).__name__} stays on the reference's CPU path")

    @staticmethod
    def _check_reads(slots: SlotMap, read: set, what: str):
        """the reference's plan builder puts Bind above every join and filter (utils.rs:101-191); a plan that reads a Bind output
        with unbound rows, or a CONCAT / isTRIPLE string the device's numeric table does not know, below that is refused"""
        bad = read & slots.bind_only
        if bad:
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"{what} reads the BIND output ?{slots.names[min(bad)]}: the reference's CPU path")

    @staticmethod
    def _join(ctx, slots: SlotMap, left: c.Relation, right: c.Relation, kind: str = "HashJoin") -> c.Relation:
        """the join operator `kind` over device relations. Without an UNDEF cell in a shared column every operator is the natural join
        (kb_hash_join). Over VALUES rows they differ (engine.rs:710-1071): NestedLoopJoin is the join of mappings (kb_natural_join); the
        hash joins and the merge join pair rows on the shared variables bound in row 0 of both sides and coalesce the other shared
        variables left-first, except OptimizedHashJoin whose probe side (the larger, right on ties) wins and the cartesian product,
        whose right side wins (kb_hash_join_keyed; a key cell a row lacks raises KB_E_UNSUPPORTED where the reference panics).
        Row 0 is the device relation's row 0. That is the reference's row 0 where the relation lies in the reference's order (a VALUES
        block, a scan); above a join it lies in device order, while the reference's row 0 there is hash-iteration order (after its merge
        join's unstable sort, not even fixed). So above a join the key can differ from the reference's: the device may refuse where
        the reference answers, or answer where it panics, depending on the row order. Where both answer, the answers agree."""
        shared = set(left.slots) & set(right.slots)
        ExecutionEngine._check_reads(slots, shared, "a join")
        if not shared & slots.ragged:
            return ctx.hash_join(left, right)
        if kind == "NestedLoopJoin":
            return ctx.natural_join(left, right)
        (nl, lslots), (nr, rslots) = left.info(), right.info()
        key = []
        if nl and nr:  # row 0 of each side: a one-row view, 4 bytes a shared column
            l0, r0 = ctx.order_by(left, [], 1)[0], ctx.order_by(right, [], 1)[0]
            key = [s_ for s_ in sorted(shared) if l0.column(lslots.index(s_))[0] != c.KB_ID_NONE and r0.column(rslots.index(s_))[0] != c.KB_ID_NONE]
        right_first = not key or (kind == "OptimizedHashJoin" and nl <= nr)
        return ctx.hash_join_keyed(left, right, key, c.MERGE_RIGHT_FIRST if right_first else c.MERGE_LEFT_FIRST)

    @staticmethod
    def _values(op: "Values", db: SparqlDatabase, slots: SlotMap) -> c.Relation:
        """kb_values, then the host Dictionary takes the new strings in the order the device created them"""
        ctx = db.ctx
        n_dev, _ = ctx.dict_strings_info()
        reloaded = n_dev != len(db.dictionary.id_to_string)
        if reloaded:
            ctx.dict_strings_load(db.dictionary.id_to_string)
        sl = [slots.of(v) for v in op.variables]
        rel, info = ctx.values(sl, op.values)
        d = db.dictionary
        for t in ctx.dict_strings_download(info["dict_first"], info["dict_new"]):
            d.string_to_id[t] = len(d.id_to_string)
            d.id_to_string.append(t)
        if reloaded:  # kb_values extended the numeric table of the strings the device held before the reload
            _derive_numeric(ctx, 0)
        slots.ragged.update(sl)
        slots.bind_out.update(sl)  # an UNDEF cell is a variable the row does not bind
        return rel

    @staticmethod
    def _bind_host(function_name: str, arguments: Sequence[str], cols: Dict[str, np.ndarray], n: int, old: Optional[np.ndarray],
                   dictionary: Dictionary, qts: QuotedTripleStore) -> np.ndarray:
        """Bind (engine.rs:144-277) restated on the host over columns: `cols` maps a variable name (no '?') to its ids, KB_ID_NONE where
        the row lacks it; `old` is the output variable's column when the input binds it already. Returns the output column (KB_ID_NONE
        where the reference inserts nothing and `old` has nothing) and makes the encodes the reference makes, in its order, in
        `dictionary` and `qts`. What kb_bind computes on the device, kept for contexts without it (the oracle) and as the reference
        the device is tested against."""
        NONE = c.KB_ID_NONE
        out = np.full(n, NONE, dtype=np.uint32) if old is None else np.array(old, dtype=np.uint32)
        if n == 0:
            return out

        def arg_col(arg: str) -> np.ndarray:  # row.get(arg.strip_prefix('?')): a missing key is KB_ID_NONE
            col = cols.get(_strip(arg))
            return np.full(n, NONE, dtype=np.uint32) if col is None else np.asarray(col, dtype=np.uint32)

        if function_name == "CONCAT":  # engine.rs:148-182: Dictionary::decode (not decode_term), "" when it gives None
            parts = []
            for arg in arguments:
                if arg.startswith("?"):
                    ids = arg_col(arg)
                    uniq, inv = np.unique(ids, return_inverse=True)
                    text = np.array([dictionary.decode(int(i)) or "" for i in uniq], dtype=object)
                    parts.append(text[inv.reshape(-1)])
                else:
                    parts.append(np.full(n, arg.strip('"'), dtype=object))  # trim_matches('"'): every leading and trailing quote
            joined = ["".join(p[i] for p in parts) for i in range(n)] if parts else [""] * n
            for i, t in enumerate(joined):
                out[i] = dictionary.encode(t)
            return out
        if function_name in ("SUBJECT", "PREDICATE", "OBJECT"):  # engine.rs:218-239
            if not arguments:
                return out
            k = ("SUBJECT", "PREDICATE", "OBJECT").index(function_name)
            ids = arg_col(arguments[0])
            q = ((ids & QUOTED_TRIPLE_ID_BIT) != 0) & (ids != NONE)
            uniq, inv = np.unique(ids[q], return_inverse=True)
            comp = np.array([(qts.decode(int(i)) or (NONE, NONE, NONE))[k] for i in uniq], dtype=np.uint32)
            val = comp[inv.reshape(-1)] if len(uniq) else np.empty(0, np.uint32)
            hit = val != NONE
            rows = np.nonzero(q)[0][hit]
            out[rows] = val[hit]
            return out
        if function_name == "TRIPLE":  # engine.rs:240-259
            if len(arguments) != 3:
                return out
            vals = []
            for arg in arguments:  # a constant is encoded inside the row loop: at the first row, in argument order
                vals.append(arg_col(arg) if arg.startswith("?") else np.full(n, dictionary.encode(arg), dtype=np.uint32))
            s, p, o = vals
            bound = np.nonzero((s != NONE) & (p != NONE) & (o != NONE))[0]
            key = (s[bound].astype(np.uint64) << np.uint64(32) | p[bound].astype(np.uint64), o[bound])
            order = np.lexsort((bound, key[1], key[0]))  # rows grouped by triple, each group in row order
            ks, ko = key[0][order], key[1][order]
            start = np.ones(len(order), dtype=bool)
            start[1:] = (ks[1:] != ks[:-1]) | (ko[1:] != ko[:-1])
            firsts = order[start]
            group = np.cumsum(start) - 1
            ids = np.empty(len(firsts), dtype=np.uint32)
            for g in np.argsort(bound[firsts], kind="stable"):  # encode in the order of each triple's first row
                r = bound[firsts[g]]
                ids[g] = qts.encode(int(s[r]), int(p[r]), int(o[r]))
            res = np.empty(len(bound), dtype=np.uint32)
            res[order] = ids[group]
            out[bound] = res
            return out
        if function_name == "isTRIPLE":  # engine.rs:260-273: "true" / "false" encoded when a row first needs them
            if not arguments:
                return out
            ids = arg_col(arguments[0])
            bound = ids != NONE
            quoted = bound & ((ids & QUOTED_TRIPLE_ID_BIT) != 0)
            plain = bound & ~quoted
            need = sorted((int(np.argmax(m)), t) for m, t in ((quoted, "true"), (plain, "false")) if m.any())
            tid = {t: dictionary.encode(t) for _, t in need}
            if "true" in tid:
                out[quoted] = tid["true"]
            if "false" in tid:
                out[plain] = tid["false"]
            return out
        return out  # "Function ... not found": the rows as they were (engine.rs:274-276)

    @staticmethod
    def _bind_rel(op: "Bind", rel: c.Relation, db: SparqlDatabase, slots: SlotMap) -> c.Relation:
        """Bind through the host restatement: download, _bind_host, upload"""
        n, rslots = rel.info()
        cols = {slots.names[sl]: rel.column(i) for i, sl in enumerate(rslots)}
        out_name = _strip(op.output_variable)
        out_slot = slots.of(out_name)
        n_ids = len(db.dictionary.id_to_string)
        col = ExecutionEngine._bind_host(op.function_name, op.arguments, cols, n, cols.get(out_name), db.dictionary, db.quoted_triple_store)
        if len(db.dictionary.id_to_string) != n_ids and hasattr(db.ctx, "dict_strings_load"):
            db.ctx.dict_strings_load(db.dictionary.id_to_string)  # the final decode reads the new strings on the device
        db._sync_quoted()
        cols[out_name] = col
        ExecutionEngine._mark_bind(slots, out_slot, op.function_name, bool((col == c.KB_ID_NONE).any()), False)
        names = list(cols)
        return db.ctx.rel_from_host([slots.of(k) for k in names], [cols[k] for k in names])

    @staticmethod
    def _mark_bind(slots: SlotMap, out_slot: int, function_name: str, has_unbound: bool, derived: bool):
        """derived: the numeric side table covers the strings the BIND created (kb_dict_numeric_derive ran after it)"""
        slots.bind_out.add(out_slot)
        if has_unbound or (function_name in ("CONCAT", "isTRIPLE") and not derived):
            slots.bind_only.add(out_slot)
        else:
            slots.bind_only.discard(out_slot)

    @staticmethod
    def _bind_device(op: "Bind", rel: c.Relation, db: SparqlDatabase, slots: SlotMap) -> c.Relation:
        """kb_bind, then the host Dictionary and QuotedTripleStore take the new entries in the order the device created them"""
        ctx = db.ctx
        fn = _BIND_FUNCTIONS.get(op.function_name)
        if fn is None:
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"BIND function {op.function_name!r}: the reference's CPU path (UDFs stay there)")
        n, rslots = rel.info()

        def var(arg: str) -> c.KbTerm:
            sl = slots.slot.get(_strip(arg))
            if sl is None or sl not in rslots:
                raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"BIND argument {arg!r} is not a variable of its input: the reference's CPU path")
            return c.V(sl)

        args: List[c.KbTerm] = []
        consts: List[bytes] = []
        if fn == c.BIND_CONCAT:
            for arg in op.arguments:
                sl = slots.slot.get(_strip(arg)) if arg.startswith("?") else None
                if sl is not None and sl in rslots:
                    args.append(c.V(sl))
                else:  # a constant, or a variable the rows lack (it contributes "")
                    args.append(c.K(len(consts)))
                    consts.append(b"" if arg.startswith("?") else arg.strip('"').encode("utf-8"))
        elif fn == c.BIND_TRIPLE:
            if len(op.arguments) != 3:
                raise c.KolibrieError(c.KB_E_UNSUPPORTED, "TRIPLE takes 3 arguments")
            const = [a for a in op.arguments if not a.startswith("?")]
            ids = iter(db.dictionary.encode_bulk(ctx, const) if (const and n) else [0] * len(const))  # encoded at the first row only
            args = [var(a) if a.startswith("?") else c.K(int(next(ids))) for a in op.arguments]
        else:
            if len(op.arguments) != 1:
                raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"{op.function_name} takes 1 argument")
            args = [var(op.arguments[0])]
        n_dev, _ = ctx.dict_strings_info()
        reloaded = n_dev != len(db.dictionary.id_to_string)
        if reloaded:
            ctx.dict_strings_load(db.dictionary.id_to_string)
        out_slot = slots.of(_strip(op.output_variable))
        qts = db.quoted_triple_store
        res, info = ctx.bind(rel, fn, args, out_slot, qts.next_qt_id if fn == c.BIND_TRIPLE else 0, consts)
        d = db.dictionary
        for t in ctx.dict_strings_download(info["dict_first"], info["dict_new"]):
            d.string_to_id[t] = len(d.id_to_string)
            d.id_to_string.append(t)
        if info["quoted_new"]:
            first = info["quoted_first"]
            qs, qp, qo = ctx.quoted_download(first, info["quoted_new"])
            for k in range(info["quoted_new"]):
                key = (int(qs[k]), int(qp[k]), int(qo[k]))
                qts.id_to_components[first + k] = key
                qts.components_to_id[key] = first + k
            qts.next_qt_id = first + info["quoted_new"]
            db._uploaded_quoted = len(qts)  # the device table holds them already: no reload (it would drop the reverse index)
        derived = hasattr(ctx, "dict_numeric_derive")
        if derived and (info["dict_new"] or reloaded):  # the numeric side table learns the strings CONCAT / isTRIPLE created, on the device
            _derive_numeric(ctx, 0 if reloaded else c.NUMERIC_APPEND)
        ExecutionEngine._mark_bind(slots, out_slot, op.function_name, info["n_unbound"] > 0, derived)
        return res

    @staticmethod
    def _scan_quoted(pattern: TriplePattern, db: SparqlDatabase, slots: SlotMap):
        """resolve_quoted_triple_scan (engine.rs:1111-1188) restated on the host: what kb_scan_quoted does on the device, kept for
        contexts without it (the oracle) and as the reference the device is tested against. Its entries are matched against the
        `<< s p o >>` term(s) on the host (match_term, engine.rs:1088-1107: constants by id, variables bound on first use and compared
        afterwards, a nested quoted term only requires a quoted-triple id), which yields one row (quoted id, inner bindings) per
        matching entry. The reference then runs one index scan per entry with the id substituted and merges the bindings, dropping
        conflicts; relationally that is the natural join of those rows with ONE scan of the pattern whose quoted position is a fresh
        variable (scan + rel_from_host + hash_join)."""
        ctx = db.ctx
        qt_s, qt_o = isinstance(pattern[0], QuotedTriple), isinstance(pattern[2], QuotedTriple)
        if isinstance(pattern[1], QuotedTriple):
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, "quoted triple in predicate position")
        rows: List[Dict[str, int]] = []
        for qid, comp in db.quoted_triple_store.id_to_components.items():
            b: Dict[str, int] = {}

            def match(term, value) -> bool:
                if isinstance(term, Constant):
                    return term.id == value
                if isinstance(term, Variable):
                    name = _strip(term.name)
                    if name in b:
                        return b[name] == value
                    b[name] = value
                    return True
                return is_quoted_triple_id(value)  # nested quoted pattern: engine.rs:1100-1105

            ok = True
            for term in ([pattern[0]] if qt_s else []) + ([pattern[2]] if qt_o else []):  # the SAME entry serves both positions (engine.rs:1135-1150)
                ok = ok and match(term.s, comp[0]) and match(term.p, comp[1]) and match(term.o, comp[2])
            if ok:
                b["__qt"] = qid
                rows.append(b)
        qslot = slots.of("__qt_%d" % len(slots.names))
        names = sorted({k for r in rows for k in r if k != "__qt"})
        # the outer pattern with the quoted position(s) replaced by the fresh variable
        outer = (Variable(slots.names[qslot]) if qt_s else pattern[0], pattern[1], Variable(slots.names[qslot]) if qt_o else pattern[2])
        outer_rel = ctx.scan([slots.pattern(outer)])[0]
        cols = [np.array([r["__qt"] for r in rows], dtype=np.uint32)] + [np.array([r[k] for r in rows], dtype=np.uint32) for k in names]
        inner_rel = ctx.rel_from_host([qslot] + [slots.of(k) for k in names], cols)
        joined = ctx.hash_join(inner_rel, outer_rel)
        _, jslots = joined.info()
        return ctx.project(joined, [s_ for s_ in jslots if s_ != qslot])

    @staticmethod
    def execute_with_ids(op, db: SparqlDatabase) -> List[Dict[str, int]]:
        db._sync()
        slots = SlotMap()
        rel = ExecutionEngine._run(op, db, slots)
        n, rslots = rel.info()
        cols = [rel.column(i) for i in range(len(rslots))]
        names = [slots.names[s] for s in rslots]
        if slots.bind_out:  # a variable a BIND left unbound is not a key of the row (the reference does not insert it)
            return [{names[j]: int(cols[j][i]) for j in range(len(names)) if not (rslots[j] in slots.bind_out and cols[j][i] == c.KB_ID_NONE)}
                    for i in range(n)]
        return [{names[j]: int(cols[j][i]) for j in range(len(names))} for i in range(n)]

    @staticmethod
    def execute(op, db: SparqlDatabase, order_by: Sequence["OrderCondition"] = (), limit: int = 0) -> List[Dict[str, str]]:
        # engine.rs:33-49: ids are turned into strings only at the very end — here by kb_rel_decode, column by column, on the device.
        # order_by / limit: apply_order_by and the LIMIT cut that follow it (execute_query.rs:693-699), run by kb_order_by before the
        # decode so that only the rows kept are decoded; a key column the device refuses (KB_E_UNSUPPORTED) is sorted here after the decode
        db._sync()
        slots = SlotMap()
        rel = ExecutionEngine._run(op, db, slots)
        host_order = False
        if order_by or limit > 0:
            keys = [(slots.slot[_strip(o.variable)], o.direction == SortDirection.DESC) for o in order_by if _strip(o.variable) in slots.slot]
            try:
                rel, _ = db.ctx.order_by(rel, keys, limit)
            except c.KolibrieError as e:
                if e.status != c.KB_E_UNSUPPORTED:
                    raise
                host_order = True
        rows = ExecutionEngine._decode_rows(rel, db, slots)
        if host_order:
            rows = apply_order_by(rows, order_by)
            if limit > 0:
                rows = rows[:limit]
        return rows

    @staticmethod
    def _decode_rows(rel: c.Relation, db: SparqlDatabase, slots: SlotMap) -> List[Dict[str, str]]:
        n, rslots = rel.info()
        cols = []
        for i in range(len(rslots)):
            try:
                cols.append(rel.decode_strings(i))
            except c.KolibrieError as e:  # no quoted-triple table, or a term nested too deep: decoded on the host (dictionary.rs:60-72)
                if e.status not in (c.KB_E_UNSUPPORTED, c.KB_E_LIMIT):
                    raise
                cols.append([db.decode_term(int(x)) or "unknown" for x in rel.column(i)])
        names = [slots.names[s] for s in rslots]
        unbound = {j: rel.column(j) == c.KB_ID_NONE for j in range(len(rslots)) if rslots[j] in slots.bind_out}
        if unbound:
            return [{names[j]: cols[j][i] for j in range(len(names)) if not (j in unbound and unbound[j][i])} for i in range(n)]
        return [{names[j]: cols[j][i] for j in range(len(names))} for i in range(n)]


class SortDirection:  # shared/src/query.rs:234-237
    ASC = "ASC"
    DESC = "DESC"


@dataclass(frozen=True)
class OrderCondition:  # shared/src/query.rs:240-243
    variable: str
    direction: str = SortDirection.ASC


def _order_cmp(a: str, b: str) -> int:
    x, y = rust_parse_f64(a), rust_parse_f64(b)
    if x is not None and y is not None:  # partial_cmp, NaN -> Equal
        return -1 if x < y else 1 if x > y else 0
    ab, bb = a.encode("utf-8"), b.encode("utf-8")  # str::cmp: byte order, a proper prefix first
    return -1 if ab < bb else 1 if ab > bb else 0


def apply_order_by(rows: List[Dict[str, str]], conditions: Sequence[OrderCondition]) -> List[Dict[str, str]]:
    """apply_order_by (execute_query.rs:113-149) on decoded rows: a stable sort (`sort_by`) where a missing variable is "". Where the
    comparison is not an order (a mixed column) the result depends on the sort algorithm, as the reference's does."""
    import functools

    if not conditions:
        return rows

    def cmp(ra, rb):
        for o in conditions:
            v = _strip(o.variable)
            r = _order_cmp(ra.get(v, ""), rb.get(v, ""))
            if o.direction == SortDirection.DESC:
                r = -r
            if r:
                return r
        return 0

    return sorted(rows, key=functools.cmp_to_key(cmp))


# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class FilterCondition:  # shared/src/rule.rs:14-18
    variable: str
    operator: str
    value: str


@dataclass
class Rule:  # shared/src/rule.rs:21-25
    premise: List[TriplePattern]
    conclusion: List[TriplePattern]
    filters: List[FilterCondition] = field(default_factory=list)


_RULE_CMP = {">": c.CMP_GT, ">=": c.CMP_GE, "<": c.CMP_LT, "<=": c.CMP_LE, "=": c.CMP_EQ, "!=": c.CMP_NE}


def compile_rule(rule: Rule) -> dict:
    slots = SlotMap()
    prem = [slots.pattern(p) for p in rule.premise]
    conc = [slots.pattern(p) for p in rule.conclusion]
    fl = []
    for f in rule.filters:
        cmp = _RULE_CMP.get(f.operator, 0)  # e.g. "OR:>" is a no-op in the reference (rules.rs:133-165)
        name = _strip(f.variable)
        if name not in slots.slot:
            continue  # unbound lhs: the reference skips the filter (rules.rs:139)
        rhs_name = _strip(f.value)
        if rhs_name in slots.slot:
            fl.append(c.KbRuleFilter(slots.slot[name], cmp, 1, slots.slot[rhs_name], 0.0))
        else:
            v = rust_parse_f64(f.value)
            fl.append(c.KbRuleFilter(slots.slot[name], cmp, 0, 0, 0.0 if v is None else v))
    return {"premise": prem, "conclusion": conc, "filters": fl}


class Reasoner:
    """datalog/src/reasoning.rs:31-100. Facts live in the device store; rules are compiled to slot form per call."""

    def __init__(self, ctx: Optional[c.Context] = None, device: int = 0):
        self.dictionary = Dictionary()
        self.rules: List[Rule] = []
        self.constraints: List[Rule] = []
        self.ctx = ctx or c.Context(device)
        self._facts: List[Tuple[int, int, int]] = []
        self._fact_set: set = set()
        self._dirty = True
        self.last_stats = None
        self._n_in_store: Optional[int] = None  # facts of self._facts the device store holds, once a fixpoint has closed it
        self._closed_rules = -1                 # len(self.rules) at that fixpoint
        self._strings_ids = -1                  # dictionary strings this reasoner put on the device

    def add_abox_triple(self, subject: str, predicate: str, obj: str):
        t = (self.dictionary.encode(subject), self.dictionary.encode(predicate), self.dictionary.encode(obj))
        if t not in self._fact_set:  # index_manager.insert dedups (index_manager.rs:41-57)
            self._fact_set.add(t)
            self._facts.append(t)
            self._dirty = True

    def add_rule(self, rule: Rule):
        self.rules.append(rule)

    def add_constraint(self, constraint: Rule):
        """reasoning.rs:95-98: a denial constraint; only its premises are read (its filters and conclusion are ignored)"""
        self.constraints.append(constraint)

    def _sync(self):
        if self._dirty:
            arr = np.array(self._facts, dtype=np.uint32).reshape(-1, 3)
            self.ctx.store_load(arr[:, 0], arr[:, 1], arr[:, 2])
            self._dirty = False
            if self._n_in_store is not None and self._n_in_store != len(self._facts):
                self._n_in_store = None  # the reloaded store holds triples no fixpoint has seen: it is not a closed store plus a seed
        self._load_numeric()

    def _load_numeric(self):
        """the numeric side table the rule filters read: on the device, the strings added since the last call go up and the table is
        extended over their ids (kb_dict_numeric_derive); the host loop for contexts without it"""
        if hasattr(self.ctx, "dict_numeric_derive"):
            kept = _push_new_strings(self.ctx, self.dictionary, self._strings_ids)
            self._strings_ids = len(self.dictionary.id_to_string)
            _derive_numeric(self.ctx, c.NUMERIC_APPEND if kept else 0)
        else:
            num, isn = self.dictionary.numeric_table()
            self.ctx.dict_numeric_load(num, isn)

    def _infer(self, strategy: int) -> List[Tuple[int, int, int]]:
        self._sync()
        rel, st = self.ctx.datalog_fixpoint([compile_rule(r) for r in self.rules], strategy)
        self.last_stats = st
        rows = rel.to_numpy([0, 1, 2])
        out = [tuple(int(x) for x in r) for r in rows]
        for t in out:  # the device already appended them to its store (infer_generic.rs:46)
            self._fact_set.add(t)
            self._facts.append(t)
        self._n_in_store, self._closed_rules = len(self._facts), len(self.rules)
        return out

    def infer_new_facts_incremental(self, strategy: int = c.SEMI_NAIVE):
        """`add_abox_triple` after a fixpoint, then infer again WITHOUT starting over (the reference starts over: semi_naive.rs:89 sets
        the delta to every fact): the triples added since the last fixpoint are the seed of kb_datalog_fixpoint_seed — they alone are
        the first delta, the closed store is OLD. Returns the facts inferred from them, the same set a fresh
        infer_new_facts_semi_naive() would add. Falls back to the full fixpoint when there is no closed store to extend."""
        if self._n_in_store is None or self._closed_rules != len(self.rules) or self._n_in_store > len(self._facts):
            return self._infer(strategy)
        rules = [compile_rule(r) for r in self.rules]
        rule_preds = {int(x.p.value) for r in rules for x in list(r["premise"]) + list(r["conclusion"]) if not x.p.is_var}
        added = np.array(self._facts[self._n_in_store:], dtype=np.uint32).reshape(-1, 3)
        self._load_numeric()
        in_rules = np.isin(added[:, 1], np.fromiter(rule_preds, np.uint32, len(rule_preds))) if len(added) else np.zeros(0, bool)
        other = added[~in_rules]
        if len(other):  # predicates no rule mentions: plain store rows
            self.ctx.store_append(other[:, 0], other[:, 1], other[:, 2], 0)
        sd = added[in_rules]
        seed = self.ctx.rel_from_host([0, 1, 2], [np.ascontiguousarray(sd[:, k]) for k in range(3)])
        rel, n_new, st = self.ctx.datalog_fixpoint_seed(rules, seed, strategy)
        self.last_stats = st
        rows = rel.to_numpy([0, 1, 2])[n_new:]
        out = [tuple(int(x) for x in r) for r in rows]
        for t in out:
            self._fact_set.add(t)
            self._facts.append(t)
        self._n_in_store, self._dirty = len(self._facts), False
        return out

    def infer_new_facts_semi_naive(self):
        return self._infer(c.SEMI_NAIVE)

    def infer_new_facts_naive(self):
        return self._infer(c.NAIVE)

    def infer_new_facts_semi_naive_parallel(self):
        return self._infer(c.SEMI_NAIVE_PARALLEL)  # semi_naive_parallel.rs:11: 1-2 premise rules, no filters, constants enforced

    def infer_new_facts(self):
        return self.infer_new_facts_naive()  # my_naive.rs:78-80 "for backward compatibility"

    def backward_chaining(self, query: TriplePattern, max_depth: int = c.BC_MAX_DEPTH) -> List[Dict[str, Term]]:
        """backward_chaining.rs:165-171 on the device (kb_datalog_query): the bindings of the query's variables over the facts with a
        proof of height <= max_depth. Each distinct binding of the query's own variables comes once, without the renamed rule variables
        the reference's per-derivation maps carry (quirk Q12). A ground query gives [{}] when it holds and [] when it does not. The
        store is only read."""
        self._sync()
        slots = SlotMap()
        q = slots.pattern(query)
        rel, st = self.ctx.datalog_query([compile_rule(r) for r in self.rules], q, max_depth)
        self.last_stats = st
        n, sl = rel.info()
        if not sl:
            return [{}] if n else []
        cols = [rel.column(i) for i in range(len(sl))]
        return [{slots.names[s]: Constant(int(cols[j][i])) for j, s in enumerate(sl)} for i in range(n)]

    def query_with_repairs(self, query: TriplePattern) -> List[Dict[str, int]]:
        """repairs.rs:10-43 on the device (kb_datalog_query_repairs), under IAR semantics: the query's bindings over the facts that lie
        in no minimal conflict of the constraints. Each distinct binding comes once, as ids (the reference's u32 values). The
        reference's answer can be a strict subset of this one when its search keeps a non-maximal repair (quirk Q13). A ground query
        gives [{}] when it holds and [] when it does not. The store is only read."""
        self._sync()
        slots = SlotMap()
        q = slots.pattern(query)
        rel, st = self.ctx.datalog_query_repairs([compile_rule(r) for r in self.constraints], q)
        self.last_stats = st
        n, sl = rel.info()
        if not sl:
            return [{}] if n else []
        cols = [rel.column(i) for i in range(len(sl))]
        return [{slots.names[s]: int(cols[j][i]) for j, s in enumerate(sl)} for i in range(n)]

    def query_abox(self, subject: Optional[str], predicate: Optional[str], obj: Optional[str]):
        """reasoning.rs:79-93 — note: like the reference, querying ENCODES unknown strings (they simply match nothing)."""
        self._sync()
        ts = []
        for k, v in enumerate((subject, predicate, obj)):
            ts.append(c.V(k) if v is None else c.K(self.dictionary.encode(v)))
        rel = self.ctx.scan([c.pattern(*ts)])[0]
        n, slots = rel.info()
        cols = {s: rel.column(i) for i, s in enumerate(slots)}
        fixed = [None if v is None else self.dictionary.encode(v) for v in (subject, predicate, obj)]
        return [tuple(int(cols[k][i]) if fixed[k] is None else fixed[k] for k in range(3)) for i in range(n)]


class SimpleR2R:
    """rsp/simple_r2r.rs over the device store, the host-side window a stream engine drives: a firing is remove(previous window) +
    add(current window) + materialize() + execute_query(op) (rsp_engine.rs:94-109). The adds of one firing become ONE store segment tagged
    with the firing number; a segment is evicted when all of its triples have left the window (so the store index is maintained, not
    rebuilt). materialize(): the first time, and whenever the rules changed or the store was changed outside it, the inferred segment is
    evicted and kb_datalog_fixpoint closes the window; from then on ONE kb_datalog_maintain per firing moves the closure by the slide
    (delete-and-rederive) instead of recomputing it. Triples are dictionary id tuples (s, p, o) of `item.dictionary`.

    Divergence from the reference (quirk Q11): SimpleR2R::materialize deletes the previous firing's derived triples AFTER the firing's
    adds (simple_r2r.rs:103-108), so a streamed triple equal to a previously derived one is missing from that firing's store; here it is
    kept (the relational answer)."""

    def __init__(self, ctx: Optional[c.Context] = None, device: int = 0, strategy: int = c.SEMI_NAIVE):
        self.item = SparqlDatabase(ctx, device)  # the window's base triples (host set) + dictionary; the device store holds segments
        self.ctx = self.item.ctx
        self.rules: List[Rule] = []
        self.strategy = strategy
        self.derived: set = set()       # the inferred segment, mirrored on the host
        self.last_stats = None          # KbFixpointStats or KbMaintainStats of the last materialize()
        self.last_mode: Optional[str] = None  # "fixpoint" / "maintain"
        self._pending: List[Tuple[int, int, int]] = []  # adds of the current firing, not on the device yet
        self._pending_set: set = set()
        self._evicted: List[int] = []   # segments whose triples all left the window, not evicted on the device yet
        self._firing = 1
        self._tag_of: Dict[Tuple[int, int, int], int] = {}
        self._live: Dict[int, int] = {}  # tag -> triples of that segment still in the window
        self._closed_sig: Optional[str] = None  # the rules the device store is closed under (None: not closed)
        self._numeric_ids = -1          # dictionary size of the numeric table on the device
        self._strings_ids = -1

    def add_reasoning_rules(self, rules: Sequence[Rule]):
        self.rules.extend(rules)

    def add(self, t: Tuple[int, int, int]):
        t = tuple(int(x) for x in t)
        self.item.add_triple(t)
        if t in self._tag_of or t in self._pending_set:  # already in the window (the reference's store is a set)
            return
        self._pending.append(t)
        self._pending_set.add(t)

    def remove(self, t: Tuple[int, int, int]):
        t = tuple(int(x) for x in t)
        self.item.delete_triple(t)
        if t in self._pending_set:
            self._pending_set.discard(t)
            self._pending.remove(t)
            return
        tag = self._tag_of.pop(t, None)
        if tag is None:
            return
        self._live[tag] -= 1
        if self._live[tag] == 0:  # the whole slide left the window
            del self._live[tag]
            self._evicted.append(tag)

    def _commit_pending(self):
        if self._pending:
            self._live[self._firing] = len(self._pending)
            for t in self._pending:
                self._tag_of[t] = self._firing
        self._pending, self._pending_set = [], set()
        self._firing += 1

    def _flush(self):
        """the window's changes as plain segment operations (no rules involved): the store is no longer closed"""
        for tag in self._evicted:
            self.ctx.store_evict(tag)
            self._closed_sig = None
        self._evicted = []
        if self._pending:
            a = np.array(self._pending, dtype=np.uint32).reshape(-1, 3)
            self.ctx.store_append(a[:, 0], a[:, 1], a[:, 2], self._firing)
            self._commit_pending()
            self._closed_sig = None

    def _signature(self) -> str:
        return repr([(r.premise, r.conclusion, r.filters) for r in self.rules])

    def _load_tables(self):
        """the dictionary's numeric and string tables on the device when it grew (FILTERs of rules and queries read the first; loading
        it voids the closed token only when a rule filter compares numbers)"""
        d = self.item.dictionary
        n = len(d.id_to_string)
        if not hasattr(self.ctx, "dict_numeric_derive"):
            if n != self._numeric_ids:
                num, isn = d.numeric_table()
                self.ctx.dict_numeric_load(num, isn)
                self._numeric_ids = n
            if n != self._strings_ids:
                self.ctx.dict_strings_load(d.id_to_string)
                self._strings_ids = n
            return
        # incremental: a firing uploads the strings it added and the device parses them (host work and bytes ~ the slide, not the dictionary)
        kept = True
        if n != self._strings_ids:
            kept = _push_new_strings(self.ctx, d, self._strings_ids)
            self._strings_ids = n
        if n != self._numeric_ids:
            _derive_numeric(self.ctx, c.NUMERIC_APPEND if kept and self._numeric_ids >= 0 else 0)
            self._numeric_ids = n

    def materialize(self) -> List[Tuple[int, int, int]]:
        """the closure of the current window's triples beyond them (simple_r2r.rs:103-128), sorted"""
        if not self.rules:
            self._flush()
            return []
        self._load_tables()
        rules = [compile_rule(r) for r in self.rules]
        sig = self._signature()
        done = False
        if self._closed_sig == sig:
            add = np.array(self._pending, dtype=np.uint32).reshape(-1, 3) if self._pending else None
            try:
                gone, new, st = self.ctx.datalog_maintain(rules, list(self._evicted), add, self._firing, self.strategy)
                done = True
            except c.KolibrieError as e:
                if e.status != c.KB_E_INVALID:  # (INVALID: the token is void — a numeric table that a rule filter reads was reloaded)
                    raise
                self._closed_sig = None
        if done:
            self._evicted = []
            if self._pending:
                self._commit_pending()
            self.derived.difference_update(map(tuple, gone.to_numpy([0, 1, 2]).tolist()))
            self.derived.update(map(tuple, new.to_numpy([0, 1, 2]).tolist()))
            self.last_mode = "maintain"
        else:
            self._flush()
            try:
                self.ctx.store_evict(c.KB_TAG_INFERRED)
            except c.KolibrieError as e:
                if e.status != c.KB_E_NOT_FOUND:
                    raise
            rel, st = self.ctx.datalog_fixpoint(rules, self.strategy)
            self.derived = set(map(tuple, rel.to_numpy([0, 1, 2]).tolist()))
            self._closed_sig = sig
            self.last_mode = "fixpoint"
        self.last_stats = st
        return sorted(self.derived)

    def _device_ready(self):
        self._flush()
        self._load_tables()
        self.item._uploaded_version = self.item._version  # the device store is maintained segment by segment, never reloaded from the set

    def execute_query(self, op) -> List[Dict[str, str]]:
        """ExecutionEngine over the window (its base triples and, after materialize(), the inferred ones)"""
        self._device_ready()
        return ExecutionEngine.execute(op, self.item)

    def execute_query_rel(self, op, slots: Optional[SlotMap] = None) -> c.Relation:
        """execute_query without the download and the decode: the firing's result as a device relation, what
        Relation2StreamOperator.eval takes. `slot_names[s]` is the name of the variable in slot s (the same for every firing of op).
        `slots`: a map shared with other plans (every window plan and the static plan of one WindowJoin), else a fresh one."""
        self._device_ready()
        slots = slots if slots is not None else SlotMap()
        rel = ExecutionEngine._run(op, self.item, slots)
        self.slot_names = list(slots.names)
        return rel


_STREAM_OPS = {"RSTREAM": c.RSTREAM, "ISTREAM": c.ISTREAM, "DSTREAM": c.DSTREAM}


class Relation2StreamOperator:
    """rsp/r2s.rs:24-58 on device relations (kb_r2s_eval): eval(response, ts) returns the emitted rows as a device relation. The
    previous evaluation's distinct rows stay in device memory, so an ISTREAM / DSTREAM firing downloads only what it emits. Rows compare
    by their ids (the dictionary is a bijection), with the columns in slot order; ISTREAM keeps the response's order and duplicates,
    DSTREAM emits the rows that left in the order they first appeared (r2s.rs:50 leaves that order to a HashSet)."""

    def __init__(self, ctx: c.Context, stream_operator: Union[int, str] = c.RSTREAM, _start_time: int = 0):
        self.ctx = ctx
        self.stream_operator = _STREAM_OPS.get(stream_operator, stream_operator)
        self._op: Optional[c.StreamOperator] = None  # created at the first response: its variables fix the row shape

    def eval(self, new_response: c.Relation, _ts: int = 0) -> c.Relation:
        if self._op is None:
            self._op = self.ctx.r2s(self.stream_operator, sorted(new_response.slots))
        return self._op.eval(new_response)

    def last_rows(self) -> int:
        """distinct rows of the previous ISTREAM / DSTREAM evaluation"""
        return self._op.info()[0] if self._op is not None else 0

    def free(self):
        if self._op is not None:
            self._op.free()
            self._op = None


class WindowJoin:
    """The emit step of a query over several windows, or over windows and static data (rsp_engine.rs:647-681), on device relations:
    the latest result of every window is natural-joined (kb_natural_join) in the order `windows` lists them — the join is commutative and
    associative on bags, so the order does not change the answer —, then joined with the static plan's result, then passed through
    Relation2StreamOperator and decoded. Around it, the two emit rules of the reference:
      * single thread (process_single_thread_window_results, rsp_engine.rs:549-593): put() queues results, process_single_thread()
        drains them; it emits once every window has a result, then Wait and Timeout clear the results and Steal keeps them;
      * coordinator (rsp_engine.rs:387-508) without its thread: receive(batch, now) is a result plus those that arrived with it, tick(now)
        the deadline of Timeout{Steal, Drop} expiring. The clock is the caller's (seconds).
    policy: "wait", "steal" or ("timeout", seconds, "steal" | "drop").

    Every window plan and the static plan must run through `slots` (one SlotMap), so that a variable has one slot everywhere. The static
    data lives in its own SparqlDatabase on a second context of the same device, sharing the windows' Dictionary object
    (rsp_engine.rs:238-243): static triples are invisible to window queries. Its result is copied device to device into the window
    context and kept while the static store and the dictionary are unchanged (the reference recomputes it per emit; the answer is the same).
    An emitted row is its bound variables as (name, value) pairs sorted by name; a variable left unbound (KB_ID_NONE) is not in it."""

    def __init__(self, ctx: c.Context, windows: Sequence[str], slots: SlotMap, stream_operator: Union[int, str] = c.RSTREAM, policy="wait",
                 static_db: Optional[SparqlDatabase] = None, static_plan=None):
        self.ctx, self.windows, self.slots, self.policy = ctx, list(windows), slots, policy
        self.r2s = Relation2StreamOperator(ctx, stream_operator)
        self.static_db, self.static_plan = static_db, static_plan
        self.last: Dict[str, c.Relation] = {}
        self._pending: List[Tuple[str, c.Relation, int]] = []
        self._static: Optional[c.Relation] = None
        self._static_key = None
        self._triggered: set = set()
        self._cycle_start: Optional[float] = None
        self._max_ts = 0

    def _store(self, window_iri: str, rel: c.Relation):
        if window_iri not in self.windows:
            raise ValueError(f"unknown window {window_iri}")
        old = self.last.get(window_iri)
        self.last[window_iri] = rel
        if old is not None and old is not rel:
            old.free()

    def _clear(self):
        for r in self.last.values():
            r.free()
        self.last = {}

    def put(self, window_iri: str, rel: c.Relation, ts: int):
        """a window's firing result (single thread): queued until process_single_thread(); it then replaces (and frees) the window's
        previous result"""
        self._pending.append((window_iri, rel, ts))

    def process_single_thread(self) -> Optional[List[List[Tuple[str, str]]]]:
        """rsp_engine.rs:549-593: the emitted rows, or None when nothing was emitted"""
        if not self._pending:
            return None
        max_ts = 0
        for iri, rel, ts in self._pending:
            max_ts = max(max_ts, ts)
            self._store(iri, rel)
        self._pending = []
        if len(self.last) != len(self.windows):
            return None
        rows = self.emit(max_ts)
        if self.policy != "steal":  # Wait, and Timeout (no wall clock in a single thread)
            self._clear()
        return rows

    def _reset_cycle(self):
        self._triggered.clear()
        self._cycle_start = None
        self._max_ts = 0

    def tick(self, now: float) -> List[List[List[Tuple[str, str]]]]:
        """Timeout's deadline (rsp_engine.rs:421-440): past it, Steal emits with what it has and Drop discards the cycle"""
        out = []
        if not isinstance(self.policy, tuple) or self._cycle_start is None or now - self._cycle_start < self.policy[1]:
            return out
        if self._triggered:
            if self.policy[2] == "steal" and len(self.last) == len(self.windows):
                out.append(self.emit(self._max_ts))
            self._reset_cycle()
        return out

    def receive(self, batch: Sequence[Tuple[str, c.Relation, int]], now: float) -> List[List[List[Tuple[str, str]]]]:
        """rsp_engine.rs:450-503: batch[0] is the result received, the rest arrived with it; returns the emits (a deadline that passed
        before `now` fires first)"""
        out = self.tick(now)
        for k, (iri, rel, ts) in enumerate(batch):
            self._max_ts = max(self._max_ts, ts)
            self._store(iri, rel)
            if k == 0 and not self._triggered:
                self._cycle_start = now
            self._triggered.add(iri)
        if len(self._triggered) == len(self.windows):
            out.append(self.emit(self._max_ts))
            self._reset_cycle()
        elif self.policy == "steal":
            if len(self.last) == len(self.windows):
                out.append(self.emit(self._max_ts))
            self._reset_cycle()
        return out

    def static_relation(self) -> Optional[c.Relation]:
        """the static plan's result in the window context, recomputed when the static store or the dictionary changed"""
        if self.static_plan is None:
            return None
        db = self.static_db
        key = (db._version, len(db.dictionary.id_to_string))
        if self._static is None or self._static_key != key:
            db._sync()
            rel = ExecutionEngine._run(self.static_plan, db, self.slots)
            db.ctx.synchronize()  # the copy below runs on the window context's stream
            n, rslots = rel.info()
            copy = self.ctx.rel_from_device(rslots, [rel.device_ptr(i) for i in range(len(rslots))], n)
            self.ctx.synchronize()  # the source's columns go back to the static context's pool: the copy must have read them
            rel.free()
            if self._static is not None:
                self._static.free()
            self._static, self._static_key = copy, key
        return self._static

    def join(self) -> c.Relation:
        """the natural join of every window's latest result and the static result (kb_natural_join), before R2S"""
        joined = None
        for iri in self.windows:
            rel = self.last[iri]
            nxt = rel if joined is None else self.ctx.natural_join(joined, rel)
            if joined is not None and joined is not self.last[self.windows[0]]:
                joined.free()
            joined = nxt
        static = self.static_relation()
        if static is not None:
            nxt = self.ctx.natural_join(joined, static)
            if joined is not self.last[self.windows[0]]:
                joined.free()
            joined = nxt
        return joined

    def emit(self, ts: int = 0) -> List[List[Tuple[str, str]]]:
        """emit_results (rsp_engine.rs:647-681): join, R2S, decode"""
        joined = self.join()
        emitted = self.r2s.eval(joined, ts)
        if joined is not self.last[self.windows[0]]:
            joined.free()
        n, rslots = emitted.info()
        names = [self.slots.names[s] for s in rslots]
        ids = [emitted.column(j) for j in range(len(rslots))]
        vals = [emitted.decode_strings(j) if n else [] for j in range(len(rslots))]
        emitted.free()
        order = sorted(range(len(rslots)), key=lambda j: names[j])
        return [[(names[j], vals[j][i]) for j in order if ids[j][i] != c.KB_ID_NONE] for i in range(n)]

    def free(self):
        self._clear()
        for _, rel, _ in self._pending:
            rel.free()
        self._pending = []
        if self._static is not None:
            self._static.free()
            self._static = None
        self.r2s.free()


# ---------------------------------------------------------------------------------------------------------------------
# The LEGACY executor's BGP + FILTER stage (kolibrie/src/execute_query.rs:151-341 — the path `execute_query` takes: CLI, criterion bench,
# README): patterns are joined one by one by perform_join_par_simd_with_strict_filter_1 (sparql_database.rs:2056-2213) over rows of
# STRING bindings, then apply_filters_simd (sparql_database.rs:1381-1669). Its quirks, kept here because they decide the answer:
#   * a pattern's predicate is compared as a string: a variable predicate ("?p") equals no predicate, the pattern matches nothing;
#   * a constant SUBJECT is not enforced: the constant's text is used as a binding NAME, so it behaves like a variable (that joins with
#     other occurrences of the same constant); a constant OBJECT is enforced (literal_filter) and bound under its own text as well;
#   * FILTER comparison at the top level: i32 comparison when the bound term and the constant both parse as i32, byte-wise string
#     = / != otherwise; the same comparison nested under AND / OR / NOT parses f64 instead (evaluate_filter_expression);
#   * an operand containing + - * / goes to the reference's arithmetic-expression parser: not evaluated on the device (UNSUPPORTED).
_I32 = re.compile(r"[+-]?[0-9]+")


def rust_parse_i32(s: str) -> Optional[int]:
    """`str::parse::<i32>()` acceptance: optional sign, ASCII digits, in range; nothing else"""
    if not isinstance(s, str) or not _I32.fullmatch(s):
        return None
    v = int(s)
    return v if -(1 << 31) <= v < (1 << 31) else None


def _has_arith(s: str) -> bool:
    return any(ch in s for ch in "+-*/")


class LegacyExecutor:
    def __init__(self, db: "SparqlDatabase"):
        self.db = db
        self._i32_loaded = -1

    def _sync(self):
        db = self.db
        db._sync()
        n = len(db.dictionary.id_to_string)
        if n != self._i32_loaded and hasattr(db.ctx, "dict_numeric_derive"):  # parsed on the device from the dictionary's strings
            if db.ctx.dict_strings_info()[0] != n:
                db.ctx.dict_strings_load(db.dictionary.id_to_string)
            db.ctx.dict_numeric_derive(c.NUMERIC_I32, 0)
            self._i32_loaded = n
        elif n != self._i32_loaded and hasattr(db.ctx, "dict_legacy_i32_load"):
            val = np.zeros(n, dtype=np.int32)
            isi = np.zeros(n, dtype=np.uint8)
            for i, st in enumerate(db.dictionary.id_to_string):
                v = rust_parse_i32(st)
                if v is not None:
                    val[i] = v
                    isi[i] = 1
            db.ctx.dict_legacy_i32_load(val, isi)
            self._i32_loaded = n

    def _compile_filter(self, e, slots: SlotMap, nested: bool, ops: List[c.KbFilterOp]):
        d = self.db.dictionary
        if isinstance(e, Comparison):
            if _has_arith(e.var) or _has_arith(e.value):
                raise c.KolibrieError(c.KB_E_UNSUPPORTED, "operands with + - * / go through the reference's arithmetic-expression parser")
            if not e.var.startswith("?") or e.value.startswith("?"):
                raise c.KolibrieError(c.KB_E_UNSUPPORTED, "legacy FILTER: variable <op> constant only")
            cmpc = {">": c.CMP_GT, ">=": c.CMP_GE, "<": c.CMP_LT, "<=": c.CMP_LE, "=": c.CMP_EQ, "!=": c.CMP_NE}.get(e.op)
            if cmpc is None:
                raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"operator {e.op!r}: the reference evaluates it to false")
            name = _strip(e.var)
            if name not in slots.slot:
                raise c.KolibrieError(c.KB_E_UNSUPPORTED, "FILTER on an unbound variable: the reference evaluates it to false")
            lit = d.lookup(e.value)
            num = rust_parse_f64(e.value) if nested else rust_parse_i32(e.value)
            flags = (c.LEGACY_CONST_IS_I32 if num is not None else 0) | (c.LEGACY_NESTED_F64 if nested else 0)
            ops.append(c.fop(c.F_CMP_LEGACY, slot=slots.slot[name], cmp=cmpc | flags, id=c.KB_ID_NONE if lit is None else lit, value=float(num) if num is not None else 0.0))
        elif isinstance(e, And):
            self._compile_filter(e.left, slots, True, ops); self._compile_filter(e.right, slots, True, ops); ops.append(c.fop(c.F_AND))
        elif isinstance(e, Or):
            self._compile_filter(e.left, slots, True, ops); self._compile_filter(e.right, slots, True, ops); ops.append(c.fop(c.F_OR))
        elif isinstance(e, Not):
            self._compile_filter(e.inner, slots, True, ops); ops.append(c.fop(c.F_NOT))
        elif isinstance(e, FunctionCall) and e.name == "isTRIPLE" and e.args and e.args[0].startswith("?") and _strip(e.args[0]) in slots.slot:
            ops.append(c.fop(c.F_IS_TRIPLE, slot=slots.slot[_strip(e.args[0])]))
        else:
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, f"legacy FILTER construct {type(e).__name__}")

    def execute_bgp(self, patterns: Sequence[Tuple[str, str, str]], filters: Sequence[object] = (), select: Optional[Sequence[str]] = None) -> List[Dict[str, str]]:
        """patterns: (subject, predicate, object) as RESOLVED strings, variables start with '?'. Returns rows of string bindings for the
        variables (pseudo-bindings named after constants are dropped unless selected)."""
        db = self.db
        self._sync()
        d = db.dictionary
        slots = SlotMap()
        pats, eqs = [], []
        for s_, p_, o_ in patterns:
            if p_.startswith("?"):
                return []  # the predicate string "?p" equals no predicate (sparql_database.rs:2136)
            pid = d.lookup(p_)
            if pid is None:
                return []
            # a constant subject / object is a binding NAME in the legacy join: one slot per distinct text
            st = c.V(slots.of(s_ if s_.startswith("?") else "?\x00" + s_))  # "\x00<text>": a name no variable can have
            ot = c.V(slots.of(o_ if o_.startswith("?") else "?\x00" + o_))
            if not o_.startswith("?"):  # literal_filter: the object string must equal the constant
                oid = d.lookup(o_)
                if oid is None:
                    return []
                eqs.append(c.fop(c.F_EQ_ID, slot=ot.value, id=oid))
            pats.append(c.pattern(st, c.K(pid), ot))
        ops: List[c.KbFilterOp] = []
        for i, e in enumerate(eqs):
            ops.append(e)
            if i:
                ops.append(c.fop(c.F_AND))
        for f in filters:  # filters.iter().all(...): a conjunction of top-level expressions
            had = bool(ops)
            self._compile_filter(f, slots, False, ops)
            if had:
                ops.append(c.fop(c.F_AND))
        rel = db.ctx.bgp_execute(pats, ops or None)
        n, rslots = rel.info()
        names = [slots.names[s_] for s_ in rslots]
        keep = [j for j, nm in enumerate(names) if (select is None and any(nm == _strip(t) for pt in patterns for t in (pt[0], pt[2]) if t.startswith("?")))
                or (select is not None and ("?" + nm) in select)]
        cols = {j: rel.column(j) for j in keep}
        return [{"?" + names[j]: db.decode_term(int(cols[j][i])) for j in keep} for i in range(n)]
