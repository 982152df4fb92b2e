"""TEST INFRASTRUCTURE: a literal restatement of the reference's serializers, SparqlDatabase::generate_ntriples
(kolibrie/src/sparql_database.rs:301-322) and generate_turtle (sparql_database.rs:324-382), with decode_any (sparql_database.rs:111-121)
and Dictionary::decode_term (shared/src/dictionary.rs:60-72), over the reference's state:

* triples    — any iterable of (s, p, o) u32 ids, taken as the BTreeSet<Triple> (shared/src/triple.rs:13-18): a set, iterated in
               ascending (s, p, o) order;
* strings    — the Dictionary's id_to_string: a list (id i -> strings[i]) or a dict;
* quoted     — the QuotedTripleStore's id_to_components: a dict id -> (s, p, o);
* prefixes   — (name, uri) pairs in the order the Turtle header lists them (the reference's HashMap order is unspecified).

What the device's kb_serialize_begin / kb_serialize_next are compared against, byte for byte."""
from typing import Dict, Iterable, Optional, Sequence, Tuple, Union

QUOTED_BIT = 0x8000_0000


def _decode(strings, i: int) -> Optional[str]:
    if isinstance(strings, dict):
        return strings.get(i)
    return strings[i] if 0 <= i < len(strings) else None


def decode_any(i: int, strings: Union[Sequence[str], Dict[int, str]], quoted: Dict[int, Tuple[int, int, int]]) -> Optional[str]:
    """decode_any: a quoted id renders as `<< s p o >>` with every component decoded the same way; None when any id on the way is held
    by neither table"""
    if i & QUOTED_BIT:
        comp = quoted.get(i)
        if comp is None:
            return None
        parts = []
        for c in comp:
            x = decode_any(c, strings, quoted)
            if x is None:
                return None
            parts.append(x)
        return "<< " + parts[0] + " " + parts[1] + " " + parts[2] + " >>"
    return _decode(strings, i)


def _texts(strings, quoted):
    """decode_any(id).unwrap_or_default() of every id asked for (decode_any is a pure function of the tables: each id is decoded once)"""
    memo = {}

    def text(i: int) -> str:
        x = memo.get(i)
        if x is None:
            x = decode_any(i, strings, quoted)
            x = memo[i] = "" if x is None else x  # unwrap_or_default
        return x

    return text


def _subject(s: str) -> str:
    return s if s.startswith("<<") else "<" + s + ">"


def _object(o: str) -> str:
    if o.startswith("<<"):
        return o
    if o.startswith("http://") or o.startswith("https://"):
        return "<" + o + ">"
    return '"' + o + '"'


def generate_ntriples(triples: Iterable[Tuple[int, int, int]], strings, quoted) -> str:
    out = []
    text = _texts(strings, quoted)
    for s, p, o in sorted(set(map(tuple, triples))):
        S, P, O = text(s), text(p), text(o)
        out.append(_subject(S) + " " + "<" + P + ">" + " " + _object(O) + " .\n")
    return "".join(out)


def generate_turtle(triples: Iterable[Tuple[int, int, int]], strings, quoted, prefixes: Sequence[Tuple[str, str]] = ()) -> str:
    out = []
    for prefix, uri in prefixes:
        out.append("@prefix " + prefix + ": <" + uri + "> .\n")
    if prefixes:
        out.append("\n")
    subjects: Dict[str, Dict[str, list]] = {}  # BTreeMap<String, BTreeMap<String, Vec<String>>>: iterated in String (UTF-8 byte) order
    text = _texts(strings, quoted)
    for s, p, o in sorted(set(map(tuple, triples))):
        S, P, O = text(s), text(p), text(o)
        subjects.setdefault(S, {}).setdefault(P, []).append(O)
    key = lambda t: t.encode("utf-8")
    for subject in sorted(subjects, key=key):
        predicates = subjects[subject]
        out.append(_subject(subject))
        names = sorted(predicates, key=key)
        for i, predicate in enumerate(names):
            out.append(" " if i == 0 else " ;\n    ")
            out.append("<" + predicate + ">")
            for j, obj in enumerate(predicates[predicate]):
                if j > 0:
                    out.append(" ,")
                out.append(" ")
                out.append(_object(obj))
            if i == len(names) - 1:
                out.append(" .\n")
    return "".join(out)
