"""Writes queries.json in this directory: a hand transcription of the 20 WatDiv basic graph patterns and SELECT lists of the
reference's WatDiv harness (the "source" field cites file and lines, by path inside the Kolibrie checkout), for the WatDiv-shaped
workload (kolibrie_b200/datagen.py: watdiv). Run: python tests/golden/watdiv/make_queries.py"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def dump(name, doc):
    with open(os.path.join(HERE, name), "w") as f:
        json.dump(doc, f, indent=1)


WSDBM = "http://db.uwaterloo.ca/~galuc/wsdbm/"
WATDIV_NS = {"wsdbm": WSDBM, "sorg": "http://schema.org/", "dc": "http://purl.org/dc/terms/", "foaf": "http://xmlns.com/foaf/",
             "gr": "http://purl.org/goodrelations/", "gn": "http://www.geonames.org/ontology#", "mo": "http://purl.org/ontology/mo/",
             "og": "http://ogp.me/ns#", "rev": "http://purl.org/stuff/rev#", "rdf": "http://www.w3.org/1999/02/22-rdf-syntax-ns#"}


def watdiv(name, line, select, body):
    """one query: `body` is the WHERE clause as written in the harness, one pattern per line, prefixed names expanded"""
    def term(t):
        if t.startswith("?") or t.startswith("<"):
            return t
        pre, local = t.split(":", 1)
        return "<" + WATDIV_NS[pre] + local + ">"
    pats = [[term(x) for x in ln.split()] for ln in body.strip().split("\n")]
    return {"name": name, "line": line, "select": select.split(), "patterns": pats}


dump("queries.json", {
    "source": "kolibrie/examples/sparql_syntax/n_triples_data/n_triple_10M.rs:104-570",
    "note": "The 20 WatDiv basic graph patterns (C1-C3, F1-F5, L1-L5, S1-S7) and their SELECT lists, transcribed pattern by pattern, prefixed "
            "names expanded with WatDiv's namespaces. rdf: is http://www.w3.org/1999/02/22-rdf-syntax-ns# throughout: the harness binds "
            "rdf: to an RDF Schema IRI in several queries, which would make every rdf:type pattern match nothing on WatDiv data.",
    "queries": [
        watdiv("C1", 107, "?v0 ?v4 ?v6 ?v7", """
?v0 sorg:caption ?v1
?v0 sorg:text ?v2
?v0 sorg:contentRating ?v3
?v0 rev:hasReview ?v4
?v4 rev:title ?v5
?v4 rev:reviewer ?v6
?v7 sorg:actor ?v6
?v7 sorg:language ?v8"""),
        watdiv("C2", 134, "?v0 ?v3 ?v4 ?v8", """
?v0 sorg:legalName ?v1
?v0 gr:offers ?v2
?v2 sorg:eligibleRegion wsdbm:Country5
?v2 gr:includes ?v3
?v4 sorg:jobTitle ?v5
?v4 foaf:homepage ?v6
?v4 wsdbm:makesPurchase ?v7
?v7 wsdbm:purchaseFor ?v3
?v3 rev:hasReview ?v8
?v8 rev:totalVotes ?v9"""),
        watdiv("C3", 162, "?v0", """
?v0 wsdbm:likes ?v1
?v0 wsdbm:friendOf ?v2
?v0 dc:Location ?v3
?v0 foaf:age ?v4
?v0 wsdbm:gender ?v5
?v0 foaf:givenName ?v6"""),
        watdiv("F1", 187, "?v0 ?v2 ?v3 ?v4 ?v5", """
?v0 og:tag wsdbm:Topic7
?v0 rdf:type ?v2
?v3 sorg:trailer ?v4
?v3 sorg:keywords ?v5
?v3 wsdbm:hasGenre ?v0
?v3 rdf:type wsdbm:ProductCategory2"""),
        watdiv("F2", 211, "?v0 ?v1 ?v2 ?v4 ?v5 ?v6 ?v7", """
?v0 foaf:homepage ?v1
?v0 og:title ?v2
?v0 rdf:type ?v3
?v0 sorg:caption ?v4
?v0 sorg:description ?v5
?v1 sorg:url ?v6
?v1 wsdbm:hits ?v7
?v0 wsdbm:hasGenre wsdbm:SubGenre1"""),
        watdiv("F3", 237, "?v0 ?v1 ?v2 ?v4 ?v5 ?v6", """
?v0 sorg:contentRating ?v1
?v0 sorg:contentSize ?v2
?v0 wsdbm:hasGenre wsdbm:SubGenre5
?v4 wsdbm:makesPurchase ?v5
?v5 wsdbm:purchaseDate ?v6
?v5 wsdbm:purchaseFor ?v0"""),
        watdiv("F4", 261, "?v0 ?v1 ?v2 ?v4 ?v5 ?v6 ?v7 ?v8", """
?v0 foaf:homepage ?v1
?v2 gr:includes ?v0
?v0 og:tag wsdbm:Topic1
?v0 sorg:description ?v4
?v0 sorg:contentSize ?v8
?v1 sorg:url ?v5
?v1 wsdbm:hits ?v6
?v1 sorg:language wsdbm:Language0
?v7 wsdbm:likes ?v0"""),
        watdiv("F5", 288, "?v0 ?v1 ?v3 ?v4 ?v5 ?v6", """
?v0 gr:includes ?v1
wsdbm:Retailer1 gr:offers ?v0
?v0 gr:price ?v3
?v0 gr:validThrough ?v4
?v1 og:title ?v5
?v1 rdf:type ?v6"""),
        watdiv("L1", 312, "?v0 ?v2 ?v3", """
?v0 wsdbm:subscribes wsdbm:Website546
?v2 sorg:caption ?v3
?v0 wsdbm:likes ?v2"""),
        watdiv("L2", 333, "?v1 ?v2", """
wsdbm:City0 gn:parentCountry ?v1
?v2 wsdbm:likes wsdbm:Product0
?v2 sorg:nationality ?v1"""),
        watdiv("L3", 354, "?v0 ?v1", """
?v0 wsdbm:likes ?v1
?v0 wsdbm:subscribes wsdbm:Website546"""),
        watdiv("L4", 374, "?v0 ?v2", """
?v0 og:tag wsdbm:Topic10
?v0 sorg:caption ?v2"""),
        watdiv("L5", 394, "?v0 ?v1 ?v3", """
?v0 sorg:jobTitle ?v1
wsdbm:City0 gn:parentCountry ?v3
?v0 sorg:nationality ?v3"""),
        watdiv("S1", 415, "?v0 ?v1 ?v3 ?v4 ?v5 ?v6 ?v7 ?v8 ?v9", """
?v0 gr:includes ?v1
wsdbm:Retailer0 gr:offers ?v0
?v0 gr:price ?v3
?v0 gr:serialNumber ?v4
?v0 gr:validFrom ?v5
?v0 gr:validThrough ?v6
?v0 sorg:eligibleQuantity ?v7
?v0 sorg:eligibleRegion ?v8
?v0 sorg:priceValidUntil ?v9"""),
        watdiv("S2", 442, "?v0 ?v1 ?v3", """
?v0 dc:Location ?v1
?v0 sorg:nationality wsdbm:Country6
?v0 wsdbm:gender ?v3
?v0 rdf:type wsdbm:Role2"""),
        watdiv("S3", 464, "?v0 ?v2 ?v3 ?v4", """
?v0 rdf:type wsdbm:ProductCategory4
?v0 sorg:caption ?v2
?v0 wsdbm:hasGenre ?v3
?v0 sorg:publisher ?v4"""),
        watdiv("S4", 486, "?v0 ?v2 ?v3", """
?v0 foaf:age wsdbm:AgeGroup4
?v0 foaf:familyName ?v2
?v3 mo:artist ?v0
?v0 sorg:nationality wsdbm:Country1"""),
        watdiv("S5", 508, "?v0 ?v2 ?v3", """
?v0 rdf:type wsdbm:ProductCategory2
?v0 sorg:description ?v2
?v0 sorg:keywords ?v3
?v0 sorg:language wsdbm:Language0"""),
        watdiv("S6", 530, "?v0 ?v1 ?v2", """
?v0 mo:conductor ?v1
?v0 rdf:type ?v2
?v0 wsdbm:hasGenre wsdbm:SubGenre26"""),
        watdiv("S7", 551, "?v0 ?v1 ?v2", """
?v0 rdf:type ?v1
?v0 sorg:text ?v2
wsdbm:User7 wsdbm:likes ?v0"""),
    ]})
