"""A literal transcription of SparqlDatabase::union and SparqlDatabase::par_join (kolibrie/src/sparql_database.rs:1874-2005) and of
Dictionary::encode / decode (shared/src/dictionary.rs:32-52), loop for loop: the reference the device entry points (kb_store_union /
kb_store_par_join) and the engine's SparqlDatabase.union / par_join are held to.

A database is its triple set, its Dictionary and its quoted-triple ids (the entries of the QuotedTripleStore it shares). Where the
reference panics (`decode(..).unwrap()` on an id without a string, encode's assert on next_id) this raises Panic. The timestamped
`streams` log is not modelled."""
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

Triple = Tuple[int, int, int]
QUOTED_TRIPLE_ID_BIT = 0x8000_0000  # shared/src/quoted_triple_store.rs:17


class Panic(Exception):
    """the reference panics here"""


class Dictionary:
    def __init__(self, strings: Iterable[str] = ()):
        self.string_to_id: Dict[str, int] = {}
        self.id_to_string: Dict[int, str] = {}
        self.next_id = 0
        for s in strings:
            self.encode(s)

    def clone(self) -> "Dictionary":
        d = Dictionary()
        d.string_to_id = dict(self.string_to_id)
        d.id_to_string = dict(self.id_to_string)
        d.next_id = self.next_id
        return d

    def encode(self, value: str) -> int:  # dictionary.rs:32-48
        if value in self.string_to_id:
            return self.string_to_id[value]
        if not self.next_id < QUOTED_TRIPLE_ID_BIT:
            raise Panic(f"Dictionary ID space exhausted: next_id {self.next_id} would collide with quoted triple ID range")
        i = self.next_id
        self.string_to_id[value] = i
        self.id_to_string[i] = value
        self.next_id += 1
        return i

    def decode(self, i: int) -> Optional[str]:  # dictionary.rs:50-52
        return self.id_to_string.get(i)

    def strings(self) -> List[str]:
        """id_to_string as the list of ids 0 .. next_id (the dictionaries here are dense)"""
        return [self.id_to_string[i] for i in range(self.next_id)]


class Db:
    def __init__(self, triples: Iterable[Triple] = (), dictionary: Optional[Dictionary] = None, quoted: Sequence[int] = ()):
        self.triples = set(map(tuple, triples))
        self.dictionary = dictionary if dictionary is not None else Dictionary()
        self.quoted = quoted  # shared: Arc::clone(&self.quoted_triple_store)


def _unwrap(v: Optional[str]) -> str:
    if v is None:
        raise Panic("called `Option::unwrap()` on a `None` value")
    return v


def union(self: Db, other: Db) -> Db:  # sparql_database.rs:1874-1933
    self_dict = self.dictionary
    other_dict = other.dictionary
    merged_dictionary = self_dict.clone()
    re_encoded_triples = set()
    for triple in sorted(other.triples):  # for triple in &other.triples: BTreeSet order
        subject = merged_dictionary.encode(_unwrap(other_dict.decode(triple[0])))
        predicate = merged_dictionary.encode(_unwrap(other_dict.decode(triple[1])))
        obj = merged_dictionary.encode(_unwrap(other_dict.decode(triple[2])))
        re_encoded_triples.add((subject, predicate, obj))
    union_triples = self.triples | re_encoded_triples
    return Db(union_triples, merged_dictionary, self.quoted)


def par_join(self: Db, other: Db, predicate: str) -> Db:  # sparql_database.rs:1935-2005
    predicate_id = self.dictionary.encode(predicate)
    other_map: Dict[int, List[Triple]] = {}
    for other_triple in sorted(other.triples):
        if other_triple[1] != predicate_id:
            continue
        for key in (other_triple[0], other_triple[2]):
            other_map.setdefault(key, []).append(other_triple)
    joined_triples = set()
    for triple in sorted(self.triples):
        if triple[1] != predicate_id:
            continue
        for other_triple in other_map.get(triple[2], []):
            joined_triples.add((triple[0], other_triple[1], other_triple[2]))
    return Db(joined_triples, self.dictionary, self.quoted)  # Arc::clone(&self.dictionary)
