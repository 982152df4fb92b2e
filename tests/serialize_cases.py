"""Hand-worked stores and the texts generate_ntriples / generate_turtle (sparql_database.rs:301-382) write for them, shared by the CPU
test of the restatement (tests/test_serialize_cpu.py) and the device test (tests/test_gpu_serialize.py). A case: strings (the
dictionary, id i -> strings[i]), quoted (quoted id -> (s, p, o)), triples (ids), prefixes, and the expected `nt` / `ttl` texts."""
Q = 0x8000_0000

CASES = [
    # ids 7 is past the dictionary: its text is "" wherever it stands (<> as a subject or predicate, "" as an object)
    dict(name="missing_plain_id", strings=["http://x/a", "http://x/p", "lit"], quoted={}, prefixes=[],
         triples=[(0, 1, 2), (0, 1, 7), (7, 1, 0), (0, 7, 2)],
         nt='<http://x/a> <http://x/p> "lit" .\n<http://x/a> <http://x/p> "" .\n<http://x/a> <> "lit" .\n<> <http://x/p> <http://x/a> .\n',
         ttl='<> <http://x/p> <http://x/a> .\n<http://x/a> <> "lit" ;\n    <http://x/p> "lit" , "" .\n'),
    # a quoted id with a missing component, and one the table does not hold: the whole term is ""
    dict(name="quoted_missing_component", strings=["s", "p", "o", "http://x/q"], quoted={Q: (0, 1, 9), Q + 1: (0, 1, 2)}, prefixes=[],
         triples=[(Q, 3, 2), (Q + 1, 3, Q), (0, 3, Q + 2)],
         nt='<s> <http://x/q> "" .\n<> <http://x/q> "o" .\n<< s p o >> <http://x/q> "" .\n',
         ttl='<> <http://x/q> "o" .\n<< s p o >> <http://x/q> "" .\n<s> <http://x/q> "" .\n'),
    # a plain string equal to a quoted rendering: written raw (it starts with "<<"), and ONE Turtle group with the quoted id
    dict(name="plain_equals_quoted", strings=["a", "b", "c", "<< a b c >>", "http://x/p", "http://x/o1", "http://x/o2"], quoted={Q: (0, 1, 2)},
         prefixes=[], triples=[(3, 4, 6), (Q, 4, 5)],
         nt="<< a b c >> <http://x/p> <http://x/o2> .\n<< a b c >> <http://x/p> <http://x/o1> .\n",
         ttl="<< a b c >> <http://x/p> <http://x/o2> , <http://x/o1> .\n"),
    # object classes: http:// and https:// in brackets, "<<" raw, everything else (empty, near misses) quoted
    dict(name="object_classes", strings=["http://x/s", "http://x/p", "http://x/o", "https://x/o", "ftp://x/o", "", "http:/x", "Http://x", "<<raw"],
         quoted={}, prefixes=[("x", "http://x/")], triples=[(0, 1, k) for k in range(2, 9)],
         nt="".join("<http://x/s> <http://x/p> " + o + " .\n" for o in ["<http://x/o>", "<https://x/o>", '"ftp://x/o"', '""', '"http:/x"', '"Http://x"', "<<raw"]),
         ttl='@prefix x: <http://x/> .\n\n<http://x/s> <http://x/p> <http://x/o> , <https://x/o> , "ftp://x/o" , "" , "http:/x" , "Http://x" , <<raw .\n'),
    # a quoted predicate is bracketed like any other
    dict(name="quoted_predicate", strings=["http://x/s", "http://x/p", "http://x/o", "lit"], quoted={Q: (0, 1, 2)}, prefixes=[],
         triples=[(0, Q, 3), (0, 1, 3)],
         nt='<http://x/s> <http://x/p> "lit" .\n<http://x/s> <<< http://x/s http://x/p http://x/o >>> "lit" .\n',
         ttl='<http://x/s> <<< http://x/s http://x/p http://x/o >>> "lit" ;\n    <http://x/p> "lit" .\n'),
    # nesting, as subject and object
    dict(name="nested", strings=["a", "b", "c", "http://x/said", "http://x/who"], quoted={Q: (0, 1, 2), Q + 1: (Q, 3, 4), Q + 2: (4, 3, Q + 1)}, prefixes=[],
         triples=[(Q + 1, 3, Q), (4, 3, Q + 2), (Q, 3, Q + 1)],
         nt="<http://x/who> <http://x/said> << http://x/who http://x/said << << a b c >> http://x/said http://x/who >> >> .\n"
            "<< a b c >> <http://x/said> << << a b c >> http://x/said http://x/who >> .\n"
            "<< << a b c >> http://x/said http://x/who >> <http://x/said> << a b c >> .\n",
         ttl="<< << a b c >> http://x/said http://x/who >> <http://x/said> << a b c >> .\n"
             "<< a b c >> <http://x/said> << << a b c >> http://x/said http://x/who >> .\n"
             "<http://x/who> <http://x/said> << http://x/who http://x/said << << a b c >> http://x/said http://x/who >> >> .\n"),
    # Turtle groups in UTF-8 byte order (a proper prefix first); N-Triples in id order
    dict(name="utf8_order", strings=["http://x/é", "http://x/z", "http://x/p", "ü", "http://x/\U0001F600", "http://x/ſ", "http://x/zz"],
         quoted={}, prefixes=[], triples=[(k, 2, 3) for k in (0, 1, 4, 5, 6)],
         nt="".join("<http://x/" + s + '> <http://x/p> "ü" .\n' for s in ["é", "z", "\U0001F600", "ſ", "zz"]),
         ttl="".join("<http://x/" + s + '> <http://x/p> "ü" .\n' for s in ["z", "zz", "é", "ſ", "\U0001F600"])),
    dict(name="empty", strings=[], quoted={}, prefixes=[], triples=[], nt="", ttl=""),
    dict(name="empty_with_prefixes", strings=[], quoted={}, prefixes=[("ex", "http://example.org/"), ("foaf", "http://xmlns.com/foaf/0.1/")], triples=[],
         nt="", ttl="@prefix ex: <http://example.org/> .\n@prefix foaf: <http://xmlns.com/foaf/0.1/> .\n\n"),
]
