"""Seeded synthetic inputs in the reference's shapes (SURVEY.md §8d / BASELINE.md §4).

The reference's generator (kolibrie/examples/synthetic_data/gen_data.rs:100-150) draws from an OS-seeded RNG and its
datasets are Git-LFS pointers, so the shapes are regenerated here deterministically:

* employee shape — 6 triples per employee in document order (gen_data.rs:116-143): foaf:name (= the employee IRI string, so
  it gets the SAME dictionary id as the subject), foaf:title in {Manager, Developer, Salesperson}, foaf:workplaceHomepage
  (one company), ds:full_or_part_time "F", ds:salary_or_hourly "SALARY", ds:annual_salary in [30000, 150000).
  PRNG = splitmix64, seed 42, two draws per employee (title, salary). Dictionary ids are assigned in first-seen order,
  subject, predicate, object per triple (kolibrie/src/sparql_database.rs:668-673; shared/src/dictionary.rs:32-48).
* taxonomy shape (config 4) — complete `fanout`-ary class tree + rdf:type facts on random classes, seed 43.

Everything is vectorised numpy so the 100 M-triple shape generates in seconds; ids come out exactly as a sequential
Dictionary::encode pass would assign them (checked against a literal sequential encoder in tests/test_datagen.py).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, Optional

import numpy as np

POSITIONS = ("Manager", "Developer", "Salesperson")  # gen_data.rs:22-24
_GAMMA = np.uint64(0x9E3779B97F4A7C15)
_M1 = np.uint64(0xBF58476D1CE4E5B9)
_M2 = np.uint64(0x94D049BB133111EB)


def splitmix64_at(seed: int, k: np.ndarray) -> np.ndarray:
    """k-th output (0-based) of a splitmix64 stream seeded with `seed` (state advances by GAMMA per draw)."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (k.astype(np.uint64) + np.uint64(1)) * _GAMMA
        z = (z ^ (z >> np.uint64(30))) * _M1
        z = (z ^ (z >> np.uint64(27))) * _M2
        return z ^ (z >> np.uint64(31))


@dataclass
class EmployeeData:
    s: np.ndarray
    p: np.ndarray
    o: np.ndarray
    n_ids: int
    ids: Dict[str, int]          # named constants: predicates, titles, company, "F", "SALARY"
    num_or0: np.ndarray          # float64[n_ids]  parse::<f64>().unwrap_or(0.0) of every term
    is_num: np.ndarray           # uint8[n_ids]
    n_employees: int
    salary_of_employee: np.ndarray = field(repr=False, default=None)
    title_of_employee: np.ndarray = field(repr=False, default=None)
    sal_id_by_value: np.ndarray = field(repr=False, default=None)    # id of the literal str(30000+k), -1 if never drawn
    title_id_by_value: np.ndarray = field(repr=False, default=None)  # id of POSITIONS[k], -1 if never drawn
    # closed form of the GLOBAL dataset this shard was cut from (employee_subject_ids): subject ids of its first `len(subj_prefix)`
    # employees; every later employee i has id prefix_ids + (i - len(subj_prefix))
    subj_prefix: np.ndarray = field(repr=False, default=None)
    prefix_ids: int = 0
    n_total: int = 0
    seed: int = 42

    @property
    def n_triples(self) -> int:
        return len(self.s)


def employee_dataset(n_employees: int, seed: int = 42, first: int = 1, global_ids: bool = True) -> EmployeeData:
    """Employees first..first+n-1 of the seeded stream. With first=1 the ids are those of a fresh dictionary."""
    E = int(n_employees)
    assert E >= 1 and first == 1, "sub-ranges are produced by employee_shard()"
    i = np.arange(E, dtype=np.uint64)
    r_title = splitmix64_at(seed, 2 * i)
    r_sal = splitmix64_at(seed, 2 * i + 1)
    title_idx = (r_title % np.uint64(3)).astype(np.int64)
    salary = (np.uint64(30000) + r_sal % np.uint64(120000)).astype(np.int64)

    # first-seen flags
    new_title = np.zeros(E, dtype=bool)
    _, first_t = np.unique(title_idx, return_index=True)
    new_title[first_t] = True
    new_sal = np.zeros(E, dtype=bool)
    uniq_sal, first_s = np.unique(salary, return_index=True)
    new_sal[first_s] = True

    # ids consumed by each employee: employee 0 also introduces 6 predicates, the company, "F" and "SALARY"
    consumed = 1 + new_title.astype(np.int64) + new_sal.astype(np.int64)
    consumed[0] += 9
    start = np.concatenate(([0], np.cumsum(consumed)[:-1]))  # id of each employee's subject
    n_ids = int(start[-1] + consumed[-1])
    subj = start.copy()

    # constants (document order inside employee 0: s, name, [name obj = s], title, TITLE, wh, company, fpt, F, soh, SALARY, sal, SALVAL)
    ids = {
        "foaf:name": 1, "foaf:title": 2, "foaf:workplaceHomepage": 4, "company": 5, "ds:full_or_part_time": 6, "F": 7,
        "ds:salary_or_hourly": 8, "SALARY": 9, "ds:annual_salary": 10,
    }
    # id of a new title introduced by employee e: right after the title predicate for e=0, right after the subject otherwise
    title_id_by_value = np.zeros(3, dtype=np.int64)
    for t in range(3):
        hits = np.nonzero(new_title & (title_idx == t))[0]
        if len(hits):
            e = int(hits[0])
            title_id_by_value[t] = 3 if e == 0 else subj[e] + 1
        else:
            title_id_by_value[t] = -1
    for t, name in enumerate(POSITIONS):
        if title_id_by_value[t] >= 0:
            ids[name] = int(title_id_by_value[t])
    # id of a new salary literal introduced by employee e
    sal_new_id = subj + 1 + new_title.astype(np.int64)
    sal_new_id[0] = 11
    sal_id_by_value = np.full(120000, -1, dtype=np.int64)
    sal_id_by_value[uniq_sal - 30000] = sal_new_id[first_s]

    title_obj = title_id_by_value[title_idx]
    sal_obj = sal_id_by_value[salary - 30000]

    s = np.repeat(subj, 6).astype(np.uint32)
    p = np.tile(np.array([1, 2, 4, 6, 8, 10], dtype=np.uint32), E)
    o = np.empty(6 * E, dtype=np.uint32)
    o[0::6] = subj
    o[1::6] = title_obj
    o[2::6] = 5
    o[3::6] = 7
    o[4::6] = 9
    o[5::6] = sal_obj

    num = np.zeros(n_ids, dtype=np.float64)
    isn = np.zeros(n_ids, dtype=np.uint8)
    num[sal_new_id[first_s]] = uniq_sal.astype(np.float64)
    isn[sal_new_id[first_s]] = 1
    return EmployeeData(s, p, o, n_ids, ids, num, isn, E, salary_of_employee=salary, title_of_employee=title_idx,
                        sal_id_by_value=sal_id_by_value, title_id_by_value=title_id_by_value,
                        subj_prefix=subj.astype(np.uint32), prefix_ids=n_ids, n_total=E, seed=seed)


SHARD_BLOCK_BITS = 10  # == KB_SHARD_BLOCK_BITS


def shard_of_np(keys: np.ndarray, world: int) -> np.ndarray:
    """kb_shard_of on an array: block-cyclic on the dense dictionary id, (key >> 10) % world"""
    return ((np.asarray(keys, dtype=np.uint32) >> np.uint32(SHARD_BLOCK_BITS)) % np.uint32(world)).astype(np.int64)


def mix32_np(x: np.ndarray) -> np.ndarray:
    """kb_shard_of's hash (murmur3 finaliser) on a uint32 array"""
    with np.errstate(over="ignore"):
        x = x.astype(np.uint32).copy()
        x ^= x >> np.uint32(16)
        x *= np.uint32(0x85EBCA6B)
        x ^= x >> np.uint32(13)
        x *= np.uint32(0xC2B2AE35)
        x ^= x >> np.uint32(16)
    return x


def employee_shard(n_total: int, rank: int, world: int, seed: int = 42, prefix: int = 4_000_000) -> EmployeeData:
    """The triples of the GLOBAL n_total-employee dataset whose subject id belongs to `rank` (kb_shard_of(subject, world)), in global
    document order — i.e. one GPU's shard under hash(subject) sharding (SURVEY.md §8e). Ids are those of the global dictionary:
    once every title and salary literal has been seen (a few million employees) each further employee consumes exactly one id,
    so the tail is closed-form and a rank never materialises the other ranks' rows."""
    if world == 1:
        return employee_dataset(n_total, seed)
    P = min(prefix, n_total)
    while True:
        head = employee_dataset(P, seed)
        complete = (head.sal_id_by_value >= 0).all() and (head.title_id_by_value >= 0).all()
        if complete or P == n_total:
            break
        P = min(P * 2, n_total)
    subj_head = head.s[0::6]
    keep = shard_of_np(subj_head, world) == rank
    rows = np.repeat(keep, 6)
    S, Pp, Oo = [head.s[rows]], [head.p[rows]], [head.o[rows]]
    n_emp = int(keep.sum())
    chunk = 8_000_000
    preds = np.array([1, 2, 4, 6, 8, 10], dtype=np.uint32)
    for a in range(P, n_total, chunk):
        b = min(a + chunk, n_total)
        i = np.arange(a, b, dtype=np.uint64)
        subj = (np.uint64(head.n_ids) + (i - np.uint64(P))).astype(np.uint32)
        k = shard_of_np(subj, world) == rank
        i, subj = i[k], subj[k]
        r_title = splitmix64_at(seed, 2 * i)
        r_sal = splitmix64_at(seed, 2 * i + 1)
        t_obj = head.title_id_by_value[(r_title % np.uint64(3)).astype(np.int64)]
        s_obj = head.sal_id_by_value[(r_sal % np.uint64(120000)).astype(np.int64)]
        m = len(subj)
        o = np.empty(6 * m, dtype=np.uint32)
        o[0::6] = subj; o[1::6] = t_obj; o[2::6] = 5; o[3::6] = 7; o[4::6] = 9; o[5::6] = s_obj
        S.append(np.repeat(subj, 6)); Pp.append(np.tile(preds, m)); Oo.append(o)
        n_emp += m
    n_ids = head.n_ids + (n_total - P)
    return EmployeeData(np.concatenate(S), np.concatenate(Pp), np.concatenate(Oo), n_ids, head.ids, head.num_or0, head.is_num, n_emp,
                        sal_id_by_value=head.sal_id_by_value, title_id_by_value=head.title_id_by_value,
                        subj_prefix=subj_head.astype(np.uint32), prefix_ids=head.n_ids, n_total=n_total, seed=seed)


def employee_subject_ids(d: EmployeeData, index: np.ndarray) -> np.ndarray:
    """dictionary id of the subject of global employee number `index` (0-based) of the dataset `d` was cut from"""
    index = np.asarray(index, dtype=np.int64)
    P = len(d.subj_prefix)
    out = (np.int64(d.prefix_ids) + (index - P)).astype(np.uint32)
    head = index < P
    out[head] = d.subj_prefix[index[head]]
    return out


def employee_strings(d: EmployeeData) -> list:
    """a dictionary text for every id of `d`: "http://example.org/employee<k>" for employee k's subject, the named constants by their
    names (predicates, titles, "F", "SALARY", ...), the numeric literals as their integer text, "http://example.org/term<id>" otherwise"""
    out = np.array(["http://example.org/term%d" % i for i in range(d.n_ids)], dtype=object)
    for name, i in d.ids.items():
        out[i] = name
    k = np.arange(d.n_employees)
    out[employee_subject_ids(d, k)] = ["http://example.org/employee%d" % i for i in k.tolist()]
    num = np.nonzero(d.is_num)[0]
    out[num] = [str(int(v)) for v in d.num_or0[num]]
    return out.tolist()


def employee_title_ids(d: EmployeeData, index: np.ndarray) -> np.ndarray:
    """dictionary id of the foaf:title object of global employee number `index` (closed form: first draw of the employee's pair)"""
    r = splitmix64_at(d.seed, 2 * np.asarray(index, dtype=np.uint64))
    return d.title_id_by_value[(r % np.uint64(3)).astype(np.int64)].astype(np.uint32)


def employee_indices_of_shard(d: EmployeeData, rank: int, world: int) -> np.ndarray:
    """global employee numbers whose subject belongs to shard `rank` (the employees of employee_shard(n_total, rank, world)), in order"""
    if world == 1:
        return np.arange(d.n_total, dtype=np.int64)
    P = len(d.subj_prefix)
    head = np.nonzero(shard_of_np(d.subj_prefix, world) == rank)[0].astype(np.int64)
    tail_i = np.arange(P, d.n_total, dtype=np.int64)
    tail_ids = (np.int64(d.prefix_ids) + (tail_i - P)).astype(np.uint32)
    return np.concatenate([head, tail_i[shard_of_np(tail_ids, world) == rank]])


def reports_to_relation(d: EmployeeData, rank: int, world: int, seed: int = 77):
    """A path-join companion of the employee shape (bench.py's shuffle leg): (?e ds:reports_to ?m) for the employees of this shard,
    ?m = a pseudo-random employee of the GLOBAL dataset — the rows live with ?e but join with (?m foaf:title ?t), which lives on the
    owner of ?m: a non-subject-key join. Returns (e ids, m ids, closed-form title id of m)."""
    idx = employee_indices_of_shard(d, rank, world)
    m_idx = (splitmix64_at(seed, idx.astype(np.uint64)) % np.uint64(d.n_total)).astype(np.int64)
    return employee_subject_ids(d, idx), employee_subject_ids(d, m_idx), employee_title_ids(d, m_idx)


def employee_queries(d: EmployeeData):
    """The BASELINE.md §4 queries on this dataset as (join_slot, patterns, filter) in capi terms. Slots: e=0 t=1 s=2 n=3 c=4."""
    from . import capi as c

    ids = d.ids
    e, t, s, n, co = 0, 1, 2, 3, 4
    q = {
        # cfg1: ?p foaf:workplaceHomepage ?c . ?p foaf:name ?n
        "cfg1": (e, [c.pattern(c.V(e), c.K(ids["foaf:workplaceHomepage"]), c.V(co)), c.pattern(c.V(e), c.K(ids["foaf:name"]), c.V(n))], []),
        # cfg2: ?e foaf:title ?t . ?e ds:annual_salary ?s . ?e foaf:name ?n FILTER(?s > 100000)
        "cfg2": (e, [c.pattern(c.V(e), c.K(ids["foaf:title"]), c.V(t)), c.pattern(c.V(e), c.K(ids["ds:annual_salary"]), c.V(s)),
                     c.pattern(c.V(e), c.K(ids["foaf:name"]), c.V(n))], [c.fop(c.F_CMP_NUM, slot=s, cmp=c.CMP_GT, value=100000.0)]),
        # cfg3: cfg2's patterns + ?e foaf:workplaceHomepage ?c (GROUP BY ?t COUNT is applied by the caller)
        "cfg3": (e, [c.pattern(c.V(e), c.K(ids["foaf:title"]), c.V(t)), c.pattern(c.V(e), c.K(ids["ds:annual_salary"]), c.V(s)),
                     c.pattern(c.V(e), c.K(ids["foaf:name"]), c.V(n)), c.pattern(c.V(e), c.K(ids["foaf:workplaceHomepage"]), c.V(co))], []),
    }
    q["star3"] = (e, q["cfg2"][1], [])  # the 3-pattern star without FILTER (SURVEY §8d worked numbers)
    return q


@dataclass
class TaxonomyData:
    s: np.ndarray
    p: np.ndarray
    o: np.ndarray
    n_ids: int
    ids: Dict[str, int]
    n_classes: int
    n_instances: int


def taxonomy_dataset(fanout: int = 10, depth: int = 6, n_instances: int = 48_888_890, seed: int = 43, first_instance: int = 0) -> TaxonomyData:
    """Complete `fanout`-ary class tree of `depth` levels below the root (subClassOf child->parent) + `x rdf:type C` facts.
    ids: rdfs:subClassOf = 0, rdf:type = 1, classes 2..2+n_classes-1 (breadth-first, root first), instances after."""
    n_classes = sum(fanout ** k for k in range(depth + 1))
    SC, TYPE, C0 = 0, 1, 2
    child = np.arange(1, n_classes, dtype=np.int64)
    parent = (child - 1) // fanout
    X0 = C0 + n_classes
    j = np.arange(first_instance, first_instance + n_instances, dtype=np.uint64)  # a rank's slice of the global instance range
    cls = (splitmix64_at(seed, j) % np.uint64(n_classes)).astype(np.int64)
    s = np.concatenate([child + C0, j.astype(np.int64) + X0]).astype(np.uint32)
    p = np.concatenate([np.full(len(child), SC), np.full(n_instances, TYPE)]).astype(np.uint32)
    o = np.concatenate([parent + C0, cls + C0]).astype(np.uint32)
    return TaxonomyData(s, p, o, int(X0 + first_instance + n_instances), {"rdfs:subClassOf": SC, "rdf:type": TYPE}, n_classes, n_instances)


def taxonomy_rules(d: TaxonomyData):
    """R1 (?a sc ?b),(?b sc ?c)->(?a sc ?c); R2 (?x type ?a),(?a sc ?b)->(?x type ?b) (R2 = deep_taxonomy.rs:70-91)."""
    from . import capi as c

    sc, ty = d.ids["rdfs:subClassOf"], d.ids["rdf:type"]
    a, b, cc, x = 0, 1, 2, 3
    r1 = {"premise": [c.pattern(c.V(a), c.K(sc), c.V(b)), c.pattern(c.V(b), c.K(sc), c.V(cc))], "conclusion": [c.pattern(c.V(a), c.K(sc), c.V(cc))]}
    r2 = {"premise": [c.pattern(c.V(x), c.K(ty), c.V(a)), c.pattern(c.V(a), c.K(sc), c.V(b))], "conclusion": [c.pattern(c.V(x), c.K(ty), c.V(b))]}
    return [r1, r2]


def taxonomy_conflicts(d: TaxonomyData, fanout: int = 10, depth: int = 6, frac: float = 0.01, seed: int = 47):
    """Inconsistency for the taxonomy shape: a second, seeded leaf type for `frac` of the instances, and `disjointWith` (id d.n_ids)
    between every ordered pair of the `fanout` level-1 classes. Returns (s, p, o) of the added facts, the disjointWith id and the
    level-1 class ids. An instance whose two leaves lie under different level-1 classes violates
    (?x type ?a), (?x type ?b), (?a disjointWith ?b) once the types are closed under subClassOf."""
    g = np.random.default_rng(seed)
    X0 = 2 + d.n_classes
    n_leaves = fanout ** depth
    xs = np.unique(g.integers(0, d.n_instances, max(1, int(d.n_instances * frac)))) + X0
    leaves = 2 + d.n_classes - n_leaves + g.integers(0, n_leaves, len(xs))
    dw = d.n_ids
    level1 = np.arange(3, 3 + fanout, dtype=np.int64)
    a, b = np.meshgrid(level1, level1, indexing="ij")
    keep = a != b
    s = np.concatenate([xs, a[keep]]).astype(np.uint32)
    p = np.concatenate([np.full(len(xs), d.ids["rdf:type"]), np.full(int(keep.sum()), dw)]).astype(np.uint32)
    o = np.concatenate([leaves, b[keep]]).astype(np.uint32)
    return (s, p, o), dw, level1.astype(np.uint32)


@dataclass
class AnnotatedSalaries:
    """The employee shape plus one RDF-star annotation per salary triple: `<< e ds:annual_salary s >> ex:source src_k`."""
    d: EmployeeData
    s: np.ndarray            # the store: the employee triples, then the annotation triples
    p: np.ndarray
    o: np.ndarray
    qt_ids: np.ndarray       # quoted-triple table (QuotedTripleStore::id_to_components): id -> (e, ds:annual_salary, s)
    qt_s: np.ndarray
    qt_p: np.ndarray
    qt_o: np.ndarray
    source: int              # id of ex:source
    src_of_employee: np.ndarray  # id of the source annotating employee i's salary triple
    n_ids: int
    num_or0: np.ndarray
    is_num: np.ndarray


def annotated_salary_dataset(n_employees: int, n_sources: int = 64, seed: int = 42, src_seed: int = 7) -> AnnotatedSalaries:
    """employee_dataset(n_employees) plus, for employee i, the quoted triple 0x80000000 + i = << e_i ds:annual_salary s_i >> (the ids
    QuotedTripleStore::encode hands out in that order) and the triple (that id, ex:source, src_k), k = splitmix64(src_seed, i) mod
    n_sources. ex:source and src_0..src_{n_sources-1} take the next dictionary ids."""
    d = employee_dataset(n_employees, seed=seed)
    E = d.n_employees
    sal = d.o[5::6]
    subj = d.s[5::6]
    source = d.n_ids
    srcs = np.arange(d.n_ids + 1, d.n_ids + 1 + n_sources, dtype=np.uint32)
    k = (splitmix64_at(src_seed, np.arange(E, dtype=np.uint64)) % np.uint64(n_sources)).astype(np.int64)
    src_of = srcs[k]
    qt_ids = (np.uint32(0x80000000) + np.arange(E, dtype=np.uint32)).astype(np.uint32)
    n_ids = d.n_ids + 1 + n_sources
    num = np.zeros(n_ids, dtype=np.float64)
    isn = np.zeros(n_ids, dtype=np.uint8)
    num[: d.n_ids], isn[: d.n_ids] = d.num_or0, d.is_num
    return AnnotatedSalaries(d, np.concatenate([d.s, qt_ids]), np.concatenate([d.p, np.full(E, source, np.uint32)]), np.concatenate([d.o, src_of]),
                             qt_ids, subj.copy(), np.full(E, d.ids["ds:annual_salary"], np.uint32), sal.copy(), source, src_of, n_ids, num, isn)


def annotated_salary_answer(a: AnnotatedSalaries, threshold: float = 100000.0) -> np.ndarray:
    """closed form of `<< ?e ds:annual_salary ?s >> ex:source ?src FILTER(?s > threshold)`: rows (e, s, src)"""
    keep = a.d.salary_of_employee > threshold
    return np.stack([a.qt_s[keep], a.qt_o[keep], a.src_of_employee[keep]], axis=1).astype(np.uint32)


def canonical_rows(a: np.ndarray) -> np.ndarray:
    """rows sorted lexicographically — the canonical form parity is judged on (the reference's row order is hash order)."""
    a = np.ascontiguousarray(a, dtype=np.uint32)
    if a.ndim == 1:
        a = a.reshape(-1, 1)
    if a.shape[0] == 0 or a.shape[1] == 0:
        return a
    order = np.lexsort(tuple(a[:, k] for k in range(a.shape[1] - 1, -1, -1)))
    return a[order]


def row_checksums(a: np.ndarray):
    """(row count, sum of mix64(row) mod 2^64, xor of mix64(row)) — order-independent digest for results too large to sort-compare."""
    a = np.ascontiguousarray(a, dtype=np.uint32)
    if a.ndim == 1:
        a = a.reshape(-1, 1)
    with np.errstate(over="ignore"):
        h = np.full(a.shape[0], 0x243F6A8885A308D3, dtype=np.uint64)
        for k in range(a.shape[1]):
            h = h ^ a[:, k].astype(np.uint64)
            h ^= h >> np.uint64(33)
            h *= np.uint64(0xFF51AFD7ED558CCD)
            h ^= h >> np.uint64(33)
            h *= np.uint64(0xC4CEB9FE1A85EC53)
            h ^= h >> np.uint64(33)
        return int(a.shape[0]), int(h.sum(dtype=np.uint64)), int(np.bitwise_xor.reduce(h)) if len(h) else 0


def permuted_dataset(d: EmployeeData, seed: int = 5):
    """The same dataset under a random relabelling of ALL dictionary ids and a random order of the triples: what a store looks like
    whose dictionary was not filled in document order (ids of one employee's terms far apart, subjects in no order). Returns
    (s, p, o, num_or0, is_num, pi) with pi[old id] = new id."""
    rng = np.random.default_rng(seed)
    pi = rng.permutation(d.n_ids).astype(np.uint32)
    order = rng.permutation(d.n_triples)
    num = np.zeros_like(d.num_or0)
    isn = np.zeros_like(d.is_num)
    num[pi] = d.num_or0
    isn[pi] = d.is_num
    return pi[d.s][order], pi[d.p][order], pi[d.o][order], num, isn, pi


def multivalued_dataset(n_subjects: int, per_subject: int = 3, seed: int = 9):
    """A store with one MULTI-VALUED predicate: subject k (id 100 + k) has `per_subject` distinct `tag` objects, one functional
    `score` literal and one functional `name`. ids: tag = 1, score = 2, name = 3; tag objects 10 .. 10 + 50; subjects from 100; score
    literals after the subjects (value v has id lit0 + v, v in [0, 1000)). Returns (s, p, o, num_or0, is_num, meta)."""
    n = int(n_subjects)
    subj = (np.arange(n, dtype=np.uint32) + np.uint32(100))
    k = np.arange(n, dtype=np.uint64)
    lit0 = 100 + n
    score = (splitmix64_at(seed, k) % np.uint64(1000)).astype(np.uint32)
    tag0 = (splitmix64_at(seed + 1, k) % np.uint64(50)).astype(np.uint32)
    assert 1 <= per_subject <= 7  # (tag0 + 7 j) mod 50 are distinct for j < 50 / 7
    tags = [tag0 + np.uint32(10)] + [((tag0 + np.uint32(j * 7)) % np.uint32(50)) + np.uint32(10) for j in range(1, per_subject)]
    s = np.concatenate([np.repeat(subj, per_subject), subj, subj])
    p = np.concatenate([np.full(n * per_subject, 1, np.uint32), np.full(n, 2, np.uint32), np.full(n, 3, np.uint32)])
    o = np.concatenate([np.stack(tags, axis=1).reshape(-1), score + np.uint32(lit0), subj])
    n_ids = lit0 + 1000
    num = np.zeros(n_ids, dtype=np.float64)
    isn = np.zeros(n_ids, dtype=np.uint8)
    num[lit0:] = np.arange(1000, dtype=np.float64)
    isn[lit0:] = 1
    return s.astype(np.uint32), p, o.astype(np.uint32), num, isn, {"subj": subj, "score": score, "tags": tags, "lit0": lit0, "per_subject": per_subject}


# ---------------------------------------------------------------------------------------------------------------------------------
# WatDiv-shaped workload: the entity classes, predicates and named constants of the 20 WatDiv queries of the reference's harness
# (kolibrie/examples/sparql_syntax/n_triples_data/n_triple_10M.rs:104-570; tests/golden/watdiv/queries.json). It is WatDiv-SHAPED,
# not WatDiv: its numbers are not comparable with the reference's WatDiv latencies.
WATDIV_NS = {"wsdbm": "http://db.uwaterloo.ca/~galuc/wsdbm/", "sorg": "http://schema.org/", "dc": "http://purl.org/dc/terms/",
             "foaf": "http://xmlns.com/foaf/", "gr": "http://purl.org/goodrelations/", "gn": "http://www.geonames.org/ontology#",
             "mo": "http://purl.org/ontology/mo/", "og": "http://ogp.me/ns#", "rev": "http://purl.org/stuff/rev#",
             "rdf": "http://www.w3.org/1999/02/22-rdf-syntax-ns#"}
# entity classes (IRI wsdbm:<Class><i>) and, per scale unit s, how many of each; fixed-size classes hold every named constant
WATDIV_CLASSES = ("User", "Product", "Review", "Offer", "Retailer", "Purchase", "Website", "City", "Country", "Topic", "SubGenre",
                  "ProductCategory", "Role", "AgeGroup", "Language", "Genre")
_WD_LIT = len(WATDIV_CLASSES)  # literal terms: class id _WD_LIT, sub = predicate


def watdiv_sizes(n_triples: int) -> Dict[str, int]:
    s = max(1, n_triples // 462)  # ~462 triples per scale unit
    return {"User": 10 * s, "Product": 10 * s, "Review": 15 * s, "Offer": 10 * s, "Retailer": 10 + s // 10, "Purchase": 15 * s,
            "Website": 600 + s, "City": 50 + s // 20, "Country": 25, "Topic": 100, "SubGenre": 150, "ProductCategory": 5, "Role": 3,
            "AgeGroup": 9, "Language": 25, "Genre": 1}


# (predicate, subject class, object: a class name, "lit" (a literal per subject), "lit:<k>" (one of k literals); every subject
# carries it when `every` == 1, else the subjects i with i % every == 0; `per` objects per subject)
WATDIV_PREDICATES = (
    ("wsdbm:likes", "User", "Product", 1, 2), ("wsdbm:friendOf", "User", "User", 1, 2), ("dc:Location", "User", "City", 1, 1),
    ("foaf:age", "User", "AgeGroup", 1, 1), ("wsdbm:gender", "User", "lit:2", 1, 1), ("foaf:givenName", "User", "lit", 1, 1),
    ("foaf:familyName", "User", "lit", 1, 1), ("wsdbm:subscribes", "User", "Website", 1, 1), ("sorg:nationality", "User", "Country", 1, 1),
    ("rdf:type", "User", "Role", 1, 1), ("foaf:homepage", "User", "Website", 2, 1), ("sorg:jobTitle", "User", "lit:50", 3, 1),
    ("sorg:caption", "Product", "lit", 1, 1), ("sorg:text", "Product", "lit", 1, 1), ("sorg:contentRating", "Product", "lit:10", 1, 1),
    ("og:tag", "Product", "Topic", 1, 1), ("rdf:type", "Product", "ProductCategory", 1, 1), ("wsdbm:hasGenre", "Product", "SubGenre", 1, 1),
    ("sorg:keywords", "Product", "lit", 1, 1), ("foaf:homepage", "Product", "Website", 1, 1), ("og:title", "Product", "lit", 1, 1),
    ("sorg:description", "Product", "lit", 1, 1), ("sorg:contentSize", "Product", "lit:1000", 1, 1), ("sorg:language", "Product", "Language", 1, 1),
    ("sorg:trailer", "Product", "lit", 4, 1), ("mo:conductor", "Product", "User", 5, 1), ("sorg:actor", "Product", "User", 3, 1),
    ("mo:artist", "Product", "User", 5, 1), ("sorg:publisher", "Product", "lit:200", 2, 1),
    ("rev:hasReview", "Review", "Product", 1, 1),  # (stored reversed: product rev:hasReview review)
    ("rev:title", "Review", "lit", 1, 1), ("rev:reviewer", "Review", "User", 1, 1), ("rev:totalVotes", "Review", "lit:100", 1, 1),
    ("gr:includes", "Offer", "Product", 1, 1), ("sorg:eligibleRegion", "Offer", "Country", 1, 1), ("gr:price", "Offer", "lit:1000", 1, 1),
    ("gr:serialNumber", "Offer", "lit", 1, 1), ("gr:validFrom", "Offer", "lit:365", 1, 1), ("gr:validThrough", "Offer", "lit:365", 1, 1),
    ("sorg:eligibleQuantity", "Offer", "lit:20", 1, 1), ("sorg:priceValidUntil", "Offer", "lit:365", 1, 1),
    ("gr:offers", "Offer", "Retailer", 1, 1),  # (stored reversed: retailer gr:offers offer)
    ("sorg:legalName", "Retailer", "lit", 1, 1),
    ("wsdbm:makesPurchase", "Purchase", "User", 1, 1),  # (stored reversed: user wsdbm:makesPurchase purchase)
    ("wsdbm:purchaseFor", "Purchase", "Product", 1, 1), ("wsdbm:purchaseDate", "Purchase", "lit:365", 1, 1),
    ("sorg:url", "Website", "lit", 1, 1), ("wsdbm:hits", "Website", "lit:1000", 1, 1), ("sorg:language", "Website", "Language", 1, 1),
    ("gn:parentCountry", "City", "Country", 1, 1),
    ("og:tag", "SubGenre", "Topic", 1, 1), ("rdf:type", "SubGenre", "Genre", 1, 1),
)
_WD_REVERSED = {"rev:hasReview", "gr:offers", "wsdbm:makesPurchase"}
# the constants the queries name, drawn most often (rank 0, 1, ...) by the popularity law below
WATDIV_POPULAR = {"Country": (1, 5, 6), "Topic": (1, 7, 10), "SubGenre": (1, 5, 26), "Retailer": (0, 1), "Website": (546,), "City": (0,),
                  "Product": (0,), "User": (7,), "ProductCategory": (2, 4), "Role": (2,), "AgeGroup": (4,), "Language": (0,)}


def watdiv_iri(prefixed: str) -> str:
    pre, local = prefixed.split(":", 1)
    return "<" + WATDIV_NS[pre] + local + ">"


def watdiv_predicate_counts(n_triples: int) -> Dict[str, int]:
    """closed form: rows per predicate IRI"""
    sz, out = watdiv_sizes(n_triples), {}
    for p, cls, _, every, per in WATDIV_PREDICATES:
        out[watdiv_iri(p)] = out.get(watdiv_iri(p), 0) + ((sz[cls] + every - 1) // every) * per
    return out


@dataclass
class WatDivData:
    s: np.ndarray
    p: np.ndarray
    o: np.ndarray
    n_ids: int
    ids: Dict[str, int]  # IRI (<...>) of every predicate and of every entity a query names -> dictionary id
    sizes: Dict[str, int]


def watdiv(n_triples: int, seed: int = 11) -> WatDivData:
    """A seeded WatDiv-shaped store of about n_triples triples (splitmix64 draws). Objects of entity-valued predicates follow a
    Zipf-like popularity law over a rank order whose first ranks are the named constants (rank r of m drawn with probability about
    1 / (2 sqrt(m r))), so every query has answers at ~100 K triples already while the most popular entity keeps a share of 1/sqrt(m). Dictionary ids are assigned in first-seen order over (s, p, o) per triple."""
    sz = watdiv_sizes(n_triples)
    cls_id = {c: i for i, c in enumerate(WATDIV_CLASSES)}
    preds = []
    for p, *_ in WATDIV_PREDICATES:
        if p not in preds:
            preds.append(p)
    S, P, O = [], [], []
    key = lambda c, sub, idx: (np.uint64(c) << np.uint64(56)) | (np.uint64(sub) << np.uint64(32)) | idx.astype(np.uint64)
    PRED_CLASS = _WD_LIT + 1
    for j, (p, cls, obj, every, per) in enumerate(WATDIV_PREDICATES):
        subj = np.arange(0, sz[cls], every, dtype=np.uint64)
        subj = np.repeat(subj, per)
        r = splitmix64_at(seed + 1000 * j, np.arange(len(subj), dtype=np.uint64))
        if obj.startswith("lit"):
            k = int(obj.split(":")[1]) if ":" in obj else 0
            val = (r % np.uint64(k)) if k else subj
            o = key(_WD_LIT, j, val)
        else:
            m = sz[obj]
            u = (r >> np.uint64(11)).astype(np.float64) / float(1 << 53)
            rank = np.minimum((float(m) * u * u).astype(np.int64), m - 1)  # P(rank r) ~ 1 / (2 sqrt(m r)): rank 0 gets 1/sqrt(m)
            named = list(WATDIV_POPULAR.get(obj, ()))
            order = np.concatenate([np.array(named, np.int64), np.setdiff1d(np.arange(m, dtype=np.int64), named)])
            o = key(cls_id[obj], 0, order[rank].astype(np.uint64))
        s = key(cls_id[cls], 0, subj)
        if p in _WD_REVERSED:
            s, o = o, s
        S.append(s)
        P.append(np.full(len(s), (np.uint64(PRED_CLASS) << np.uint64(56)) | np.uint64(preds.index(p)), np.uint64))
        O.append(o)
    S, P, O = np.concatenate(S), np.concatenate(P), np.concatenate(O)
    # interleave the triples' terms -> ids in first-seen order
    allk = np.stack([S, P, O], axis=1).reshape(-1)
    uniq, first, inv = np.unique(allk, return_index=True, return_inverse=True)
    rank_of = np.empty(len(uniq), np.int64)
    rank_of[np.argsort(first, kind="stable")] = np.arange(len(uniq))
    ids_all = rank_of[inv].astype(np.uint32).reshape(-1, 3)
    ids: Dict[str, int] = {}
    for i, p in enumerate(preds):
        k = (np.uint64(PRED_CLASS) << np.uint64(56)) | np.uint64(i)
        ids[watdiv_iri(p)] = int(rank_of[np.searchsorted(uniq, k)])
    for c, named in WATDIV_POPULAR.items():
        for x in named:
            k = key(cls_id[c], 0, np.array([x]))[0]
            at = np.searchsorted(uniq, k)
            if at < len(uniq) and uniq[at] == k:
                ids[watdiv_iri("wsdbm:" + c + str(x))] = int(rank_of[at])
    return WatDivData(ids_all[:, 0].copy(), ids_all[:, 1].copy(), ids_all[:, 2].copy(), int(len(uniq)), ids, sz)
