"""A restatement of the reference's writes to the store, over a Python set: SparqlDatabase::add_triple / delete_triple
(kolibrie/src/sparql_database.rs:215-226, a BTreeSet), encode_term_star with split_quoted_triple_content (:82-190), handle_update
(:3091-3117) and the DELETE { template } WHERE branch of execute_query_rayon_parallel2_volcano (kolibrie/src/execute_query.rs:354-413).
The tests hold the device and the engine to it."""
from typing import Dict, List, Optional, Sequence, Tuple

QUOTED_BIT = 0x8000_0000


class RefDb:
    def __init__(self):
        self.triples = set()
        self.string_to_id: Dict[str, int] = {}
        self.id_to_string: List[str] = []
        self.qt_to_id: Dict[Tuple[int, int, int], int] = {}
        self.id_to_qt: Dict[int, Tuple[int, int, int]] = {}

    # ---- dictionary.rs:32-48 and quoted_triple_store.rs:28-55
    def encode(self, s: str) -> int:
        i = self.string_to_id.get(s)
        if i is None:
            i = len(self.id_to_string)
            self.string_to_id[s] = i
            self.id_to_string.append(s)
        return i

    def encode_qt(self, s: int, p: int, o: int) -> int:
        k = (s, p, o)
        if k not in self.qt_to_id:
            i = QUOTED_BIT + len(self.qt_to_id)
            self.qt_to_id[k] = i
            self.id_to_qt[i] = k
        return self.qt_to_id[k]

    # ---- sparql_database.rs:82-109
    def encode_term_star(self, term: str) -> int:
        t = term.strip()
        if t.startswith("<<") and t.endswith(">>"):
            s, p, o = split_quoted_triple_content(t[2:-2].strip())
            si, pi, oi = self.encode_term_star(s), self.encode_term_star(p), self.encode_term_star(o)
            return self.encode_qt(si, pi, oi)
        return self.encode(clean_term(t))

    # ---- sparql_database.rs:215-226
    def add_triple(self, t: Tuple[int, int, int]) -> bool:
        if t in self.triples:
            return False
        self.triples.add(t)
        return True

    def delete_triple(self, t: Tuple[int, int, int]) -> bool:
        if t in self.triples:
            self.triples.remove(t)
            return True
        return False

    # ---- sparql_database.rs:3091-3117, with the parser's output (parse_insert / parse_delete) as input
    def handle_update(self, kind: str, triples: Sequence[Tuple[str, str, str]]) -> str:
        if kind not in ("INSERT", "DELETE"):
            return "Update Failed"
        for s, p, o in triples:
            t = (self.encode_term_star(s), self.encode_term_star(p), self.encode_term_star(o))
            if kind == "INSERT":
                self.add_triple(t)
            else:
                self.delete_triple(t)
        return "Update Successful"

    # ---- execute_query.rs:354-413: every WHERE row (variable name -> the decoded binding) fills every template pattern; the filled
    # strings are encoded with encode_term_star and deleted; an INSERT template is then inserted as written (process_insert_clause,
    # :758-773), so a variable in it is the term "?x"
    def execute_delete_where(self, template, where, insert_template=None):
        self.delete_where(template, self.where_rows(where), insert_template)

    @property
    def quoted_triple_store(self):
        return self.id_to_qt

    def delete_where(self, template: Sequence[Tuple[str, str, str]], rows: Sequence[Dict[str, str]],
                     insert_template: Optional[Sequence[Tuple[str, str, str]]] = None):
        for row in rows:
            for pat in template:
                filled = [row.get(x, x) if x.startswith("?") else x for x in pat]
                self.delete_triple(tuple(self.encode_term_star(x) for x in filled))
        if insert_template:
            self.handle_update("INSERT", insert_template)

    # ---- the rows the WHERE's SELECT returns: its patterns only, matched against the set (variable name -> decoded term)
    def where_rows(self, patterns: Sequence[Tuple[str, str, str]]) -> List[Dict[str, str]]:
        rows: List[Dict[str, int]] = [{}]
        for pat in patterns:
            want = [None if x.startswith("?") else self.string_to_id.get(clean_term(x.strip()), -1) for x in pat]
            nxt = []
            for row in rows:
                for t in sorted(self.triples):
                    b = dict(row)
                    ok = True
                    for x, w, v in zip(pat, want, t):
                        if w is not None:
                            ok = ok and v == w
                        elif b.setdefault(x, v) != v:
                            ok = False
                    if ok:
                        nxt.append(b)
            rows = nxt
        return [{k: self.decode(v) for k, v in r.items()} for r in rows]

    def decode(self, i: int) -> str:
        if i & QUOTED_BIT:
            return "<< " + " ".join(self.decode(x) for x in self.id_to_qt[i]) + " >>"
        return self.id_to_string[i]

    # ---- parse_ntriples_and_add of a fixture's data: a nested [s, p, o] list is a quoted triple, components first
    def load(self, data) -> None:
        def enc(x):
            return self.encode_qt(*[enc(y) for y in x]) if isinstance(x, list) else self.encode(x)
        for s, p, o in data:
            self.add_triple((enc(s), enc(p), enc(o)))


def run_fixture_case(db, case) -> None:
    """a fixture case's steps on db (RefDb, or the engine's SparqlDatabase through the same method names), with its assertions"""
    for step in case["steps"]:
        if step["kind"] == "DELETE_WHERE":
            db.execute_delete_where(step["template"], step["where"], step.get("insert"))
        else:
            r = db.handle_update(step["kind"], step["triples"])
            if "result" in step:
                assert r == step["result"], (case["name"], r)
    assert len(db.triples) == case["triples"], (case["name"], len(db.triples))
    if case.get("quoted_nonempty"):
        assert len(db.quoted_triple_store) > 0, case["name"]


def clean_term(t: str) -> str:
    """the plain-term branch of encode_term_star on a trimmed term: <iri> loses its brackets, a literal keeps what lies between its
    first two quotes (or loses its quotes when it has one)"""
    if t.startswith("<") and t.endswith(">"):
        return t[1:-1]
    if t.startswith('"'):
        close = t[1:].find('"')
        return t[1:close + 1] if close >= 0 else t.strip('"')
    return t


def split_quoted_triple_content(content: str) -> Tuple[str, str, str]:
    """sparql_database.rs:125-190"""
    parts: List[str] = []
    cur = ""
    depth = 0
    in_uri = in_lit = esc = False
    for ch in content:
        if esc:
            cur += ch
            esc = False
            continue
        if ch == "\\" and in_lit:
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


def batch_insert(store: set, batch: Sequence[Tuple[int, int, int]]) -> List[bool]:
    """kb_store_insert's flags: BTreeSet::insert in batch order"""
    out = []
    for t in batch:
        out.append(t not in store)
        store.add(t)
    return out


def batch_remove(store: set, batch: Sequence[Tuple[int, int, int]]) -> List[bool]:
    """kb_store_remove's flags: BTreeSet::remove in batch order"""
    out = []
    for t in batch:
        out.append(t in store)
        store.discard(t)
    return out
