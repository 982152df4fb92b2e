"""Term ids at the edges of the u32 domain, for the join, scan, index and Datalog routes (no GPU, no reference checkout).

Remaps: seeded injective maps f of a workload's ids. Every family maps KB_ID_NONE to itself and nothing onto it, and fixes the ids the
numeric side table marks numeric (FILTER reads num[id], and no table reaches 2^31). Predicates and rule constants are remapped too.

  identity    the control
  top_plain   id -> 0x7FFFFFFF - id: the top of the plain range, order reversed
  quoted      id -> 0x80000000 | id: quoted-triple ids (bit 31), table index below 2^28
  straddle    the ids in rank order, half just below 2^31 and half from 2^31 up
  extremes    five ids moved to 0, 1, 0x7FFFFFFF, 0x80000000 and 0xFFFFFFFE (whoever held those takes their place), the rest dense
  scatter     id * odd constant mod 2^32, an image that lands on KB_ID_NONE or a fixed id drawn again

Threshold builders: for each id-range threshold of a route, the inputs at the threshold (range equal to it) and one id past it, and
the route each must take. `n` is kept small so that the density side of each max() binds.
"""
import numpy as np

from kolibrie_b200 import capi as c

NONE = 0xFFFFFFFF
QUOTED_LIMIT = 1 << 28  # quoted-triple table indices (id & 0x7FFFFFFF) stay below it
FAMILIES = ("identity", "top_plain", "quoted", "straddle", "extremes", "scatter")
EXTREMES = (0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE)
SCATTER_MUL = 0x9E3779B1


class Remap:
    """an injective map of the u32 ids `domain` (NONE excluded); ids in `fixed` map to themselves"""

    def __init__(self, family, domain, fixed=(), seed=0):
        domain = np.unique(np.asarray(domain, dtype=np.uint64))
        domain = domain[domain != NONE]
        fixed = set(int(x) for x in fixed)
        free = [int(x) for x in domain if int(x) not in fixed]
        img = {x: x for x in fixed}
        g = np.random.default_rng(seed)
        if family == "identity":
            img.update({x: x for x in free})
        elif family == "top_plain":
            assert all(x < 0x7FFFFFFF for x in free)
            img.update({x: 0x7FFFFFFF - x for x in free})
        elif family == "quoted":
            assert all(x < QUOTED_LIMIT for x in free)
            img.update({x: 0x80000000 | x for x in free})
        elif family == "straddle":
            base = 0x80000000 - len(free) // 2
            img.update({x: base + i for i, x in enumerate(sorted(free))})
        elif family == "extremes":
            img.update({x: x for x in free})
            inv = {v: k for k, v in img.items()}
            movers = g.choice(free, size=min(len(EXTREMES), len(free)), replace=False)
            for x, t in zip(movers.tolist(), EXTREMES):
                assert t not in fixed, f"{t:#x} is a numeric id"
                y = inv.get(t)  # the id whose image is t now, if any: it takes x's image
                img[x], old = t, img[x]
                if y is not None and y != x:
                    img[y] = old
                inv = {v: k for k, v in img.items()}
        elif family == "scatter":
            used = set(fixed)
            for x in free:
                v = (x * SCATTER_MUL) & 0xFFFFFFFF
                while v == NONE or v in used:
                    v = (v * SCATTER_MUL + 1) & 0xFFFFFFFF
                used.add(v)
                img[x] = v
        else:
            raise ValueError(family)
        self.family = family
        self.keys = np.array(sorted(img), dtype=np.uint64)
        self.vals = np.array([img[int(k)] for k in self.keys], dtype=np.uint64)

    def __call__(self, a):
        """f applied to every cell of `a` (NONE stays NONE); an id outside the domain is an error"""
        a = np.asarray(a)
        flat = a.astype(np.uint64).ravel()
        out = flat.copy()
        live = flat != NONE
        i = np.searchsorted(self.keys, flat[live])
        assert np.all(i < len(self.keys)) and np.array_equal(self.keys[i], flat[live]), "id outside the remap's domain"
        out[live] = self.vals[i]
        return out.reshape(a.shape).astype(np.uint32)

    def id(self, x):
        return int(self(np.array([x], dtype=np.uint32))[0])

    def term(self, t):
        return t if t.is_var else c.K(self.id(int(t.value)))

    def pattern(self, p):
        return c.pattern(self.term(p.s), self.term(p.p), self.term(p.o))

    def rule(self, r):
        return {"premise": [self.pattern(p) for p in r["premise"]], "conclusion": [self.pattern(p) for p in r["conclusion"]],
                "filters": list(r.get("filters", []))}

    def filt(self, ops):
        """a FILTER program with its id constants remapped (comparisons against f64 constants are untouched)"""
        out = []
        for op in ops or []:
            o = c.KbFilterOp()
            for f, _ in c.KbFilterOp._fields_:
                setattr(o, f, getattr(op, f))
            if op.op in (c.F_EQ_ID, c.F_NE_ID) and op.id != NONE:
                o.id = self.id(int(op.id))
            out.append(o)
        return out


# ---------------------------------------------------------------- workloads
# predicates; numeric literals are the ids [NUM_LO, NUM_HI), all below 2^8; ids 0 and 1 are plain (the extremes remap moves ids there)
P_NAME, P_AGE, P_DEPT, P_KNOWS, P_LINK, P_REACH, P_TAG = 10, 11, 12, 13, 14, 15, 16
NUM_LO, NUM_HI = 32, 96


def numeric_table():
    """(num_or0, is_num) for ids below NUM_HI: id -> id / 2 - 20 for the numeric ids"""
    ids = np.arange(NUM_HI)
    is_num = ((ids >= NUM_LO) & (ids < NUM_HI)).astype(np.uint8)
    return np.where(is_num == 1, ids / 2.0 - 20.0, 0.0), is_num


def star_store(seed=0, n_subj=600):
    """a star-shaped store: every subject has one name and one age (numeric) and one dept; knows is 1:N; link forms chains for the
    fixpoint; tag holds plain ids 0 and 1 as objects"""
    g = np.random.default_rng(seed)
    subj = 1000 + np.sort(g.choice(20 * n_subj, n_subj, replace=False))
    rows = [np.stack([subj, np.full(n_subj, P_NAME), 200000 + np.arange(n_subj)], axis=1),
            np.stack([subj, np.full(n_subj, P_AGE), g.integers(NUM_LO, NUM_HI, n_subj)], axis=1),
            np.stack([subj, np.full(n_subj, P_DEPT), 300000 + g.integers(0, 40, n_subj)], axis=1)]
    k = 3 * n_subj
    rows.append(np.stack([subj[g.integers(0, n_subj, k)], np.full(k, P_KNOWS), subj[g.integers(0, n_subj, k)]], axis=1))
    chain = subj[g.permutation(n_subj)[: n_subj // 4]]
    cut = (np.arange(1, len(chain)) % 25) != 0  # chains of 25: the closure takes fewer rounds than kb_fixpoint_stats records
    rows.append(np.stack([chain[:-1][cut], np.full(int(cut.sum()), P_LINK), chain[1:][cut]], axis=1))
    t = n_subj // 3
    rows.append(np.stack([subj[:t], np.full(t, P_TAG), g.integers(0, 2, t)], axis=1))
    tr = np.unique(np.concatenate(rows).astype(np.uint32), axis=0)
    return tr[g.permutation(len(tr))]


def star_queries():
    """name -> (join slot, patterns, FILTER) over star_store"""
    V, K = c.V, c.K
    age_gt = [c.fop(c.F_CMP_NUM, slot=2, cmp=c.CMP_GT, value=5.0)]
    return {
        "name_age_dept": (0, [c.pattern(V(0), K(P_NAME), V(1)), c.pattern(V(0), K(P_AGE), V(2)), c.pattern(V(0), K(P_DEPT), V(3))], age_gt),
        "name_dept": (0, [c.pattern(V(0), K(P_NAME), V(1)), c.pattern(V(0), K(P_DEPT), V(3))], []),
        "knows_dept": (0, [c.pattern(V(0), K(P_KNOWS), V(1)), c.pattern(V(0), K(P_DEPT), V(3))], []),
    }


def store_rules():
    """transitive reachability over P_LINK, and a rule with constant object 1 (moved by the extremes remap)"""
    V, K = c.V, c.K
    return [{"premise": [c.pattern(V(0), K(P_LINK), V(1))], "conclusion": [c.pattern(V(0), K(P_REACH), V(1))], "filters": []},
            {"premise": [c.pattern(V(0), K(P_REACH), V(1)), c.pattern(V(1), K(P_LINK), V(2))], "conclusion": [c.pattern(V(0), K(P_REACH), V(2))],
             "filters": []},
            {"premise": [c.pattern(V(0), K(P_TAG), K(1)), c.pattern(V(0), K(P_LINK), V(1))], "conclusion": [c.pattern(V(1), K(P_TAG), K(1))],
             "filters": []}]


def domain_of(rows, extra=()):
    """every id of a workload: its cells, the predicates and constants its queries and rules name, the numeric range"""
    return np.unique(np.concatenate([np.asarray(rows, np.uint64).ravel(), np.asarray(list(extra), np.uint64),
                                     np.arange(NUM_HI, dtype=np.uint64), np.arange(P_NAME, P_TAG + 1, dtype=np.uint64)]))


def remaps(rows, seed=0):
    fixed = range(NUM_LO, NUM_HI)
    dom = domain_of(rows)
    return {f: Remap(f, dom, fixed, seed) for f in FAMILIES}


def bgp_chain():
    """a non-star BGP over star_store: ?a knows ?b . ?b link ?c . ?c dept ?d"""
    V, K = c.V, c.K
    return [c.pattern(V(0), K(P_KNOWS), V(1)), c.pattern(V(1), K(P_LINK), V(2)), c.pattern(V(2), K(P_DEPT), V(3))]


# ---------------------------------------------------------------- threshold builders
def spread(g, lo, hi, n):
    """n distinct ids in [lo, hi], both ends included"""
    assert hi - lo + 1 >= n >= 2
    mid = lo + 1 + g.choice(hi - lo - 1, n - 2, replace=False) if n > 2 else np.empty(0, np.int64)
    return np.sort(np.concatenate([[lo, hi], mid]).astype(np.uint64)).astype(np.uint32)


GROUPED_MIN = 1 << 20  # kb_join.cu join_grouped: range <= max(16 * build rows, 2^20) and < 2^31 -> key-grouped directory


def grouped_pair(hi, past, n_build=1000, n_probe=5000, seed=0):
    """kb_hash_join sides whose build (smaller) side's key range is 2^20 (grouped) or 2^20 + 1 (chained), ending at `hi`.
    Returns ((slots, cols) left, (slots, cols) right, route) with route 'grouped' or 'chained'."""
    g = np.random.default_rng(seed)
    rng_ = GROUPED_MIN + (1 if past else 0)
    keys = spread(g, hi - rng_ + 1, hi, n_build)
    lk = keys[g.integers(0, n_build, n_probe)]
    left = ([0, 1], [lk, g.integers(0, 1000, n_probe).astype(np.uint32)])
    right = ([0, 2], [g.permutation(keys), g.integers(0, 1000, n_build).astype(np.uint32)])
    return left, right, "chained" if past else "grouped"


PROBEG_HEAVY = 32768  # kb_join.cu: a grouped join whose output passes it spreads its heavy probe tiles over the grid (a 2nd launch)


def heavy_pair(heavy, n_heavy=40, n_probe=3000, n_build=140, seed=3):
    """a third of the probe rows and `n_heavy` build rows share the key `heavy`. With n_heavy = 40 the output (over 40 000 rows) passes
    PROBEG_HEAVY and the heavy tiles take the second launch; with n_heavy = 1 it stays below (the control)"""
    g = np.random.default_rng(seed)
    lo = min(heavy, 0xFFFFFFFE - 3000)
    others = np.unique(lo + g.integers(0, 3000, 2 * n_build)).astype(np.uint64)
    others = others[others != heavy][: n_build - n_heavy]
    bk = np.concatenate([np.full(n_heavy, heavy, np.uint64), others]).astype(np.uint32)
    lk = others[g.integers(0, len(others), n_probe)].astype(np.uint32)
    lk[: n_probe // 3] = heavy
    left = ([0, 1], [g.permutation(lk).astype(np.uint32), g.integers(0, 1000, n_probe).astype(np.uint32)])
    right = ([0, 2], [g.permutation(bk), g.integers(0, 1000, len(bk)).astype(np.uint32)])
    return left, right


def star_over_subjects(subj, preds=(101, 102, 103), seed=0):
    """every subject has one object per predicate: a 3-pattern star with single-valued build sides"""
    g = np.random.default_rng(seed)
    n = len(subj)
    rows = [np.stack([subj, np.full(n, p), 5000 + 1000 * i + g.integers(0, 500, n)], axis=1) for i, p in enumerate(preds)]
    tr = np.concatenate(rows).astype(np.uint32)
    return tr[g.permutation(len(tr))]


def star_pats(preds=(101, 102, 103)):
    return [c.pattern(c.V(0), c.K(p), c.V(i + 1)) for i, p in enumerate(preds)]


# kb_join.cu fused_scan_join (R3, index off): rng <= max(4 * n_triples, 2^16) and <= 2^31
R3_MIN = 1 << 16
# kb_store.cu slice_table_update: a persistent table when range <= max(4 * n + 65536, 2^16) and <= 2^28 (n: the slice's rows)
def slice_table_max(n):
    return max(4 * n + 65536, 1 << 16)


# kb_join.cu index_join_built (R2): rng <= max(8 * n_k, 2^16) and <= 2^31
def r2_max(n):
    return max(8 * n, 1 << 16)


def star_threshold(kind, hi, past, seed=0):
    """a 3-predicate star store whose subjects span exactly the threshold range of `kind` (or one id more), ending at `hi`.
    kind: 'r3' (2 000 subjects, index off: fused scan build or not), 'slice' (2 000 subjects, index on: persistent tables and the
    one-kernel index join, or neither), 'r2' (20 000 subjects: too sparse for a persistent table; the index join building its tables
    from the slices, or not). Returns (triples, route taken at the threshold: True on it, False one past it)."""
    n = 20000 if kind == "r2" else 2000
    lim = {"r3": R3_MIN, "slice": slice_table_max(n), "r2": r2_max(n)}[kind]
    if kind == "r3":
        assert 4 * 3 * n < R3_MIN  # the 2^16 side of the max binds
    if kind == "r2":
        assert slice_table_max(n) < lim  # no persistent table at this range
    rng_ = lim + (1 if past else 0)
    subj = spread(np.random.default_rng(seed), hi - rng_ + 1, hi, n)
    return star_over_subjects(subj, seed=seed), not past


DIRECTORY_MIN = 1 << 20  # kb_store.cu index-lookup directories: range <= max(8 * n, 2^20) and <= 2^28


def directory_store(hi, past, seed=0, n=3000):
    """predicate 120 multi-valued in both columns (no persistent table); subject ids span 2^20 (a directory) or 2^20 + 1 (a scan)"""
    g = np.random.default_rng(seed)
    rng_ = DIRECTORY_MIN + (1 if past else 0)
    subj = spread(g, hi - rng_ + 1, hi, 400)
    s = np.concatenate([subj, subj[g.integers(0, len(subj), n - len(subj))]])
    o = 7000 + g.integers(0, 50, n)
    tr = np.unique(np.stack([s, np.full(n, 120), o], axis=1).astype(np.uint32), axis=0)
    return tr, int(subj[0]), int(subj[-1])


RED_MAX_BITS = 1 << 28  # kb_bgp.cu: a reduce bitmap covers [lo, lo + 2^28); ids at or past lo + 2^28 pass unreduced


def bitmap_store(lo, seed=0):
    """a chain BGP ?a P130 ?x . ?x P131 ?b . ?b P132 ?c whose ?x takes lo, lo + 2^28 - 1 and lo + 2^28 in both of its positions,
    with some ?x values of each side lacking a partner on the other. Every subject and object of the store is at least lo, so the
    reduction's bitmap of ?x starts at lo exactly (its lo is the largest of its columns' store-wide minima) and spans 2^28 ids (32 MB)"""
    g = np.random.default_rng(seed)
    xs = np.array([lo, lo + RED_MAX_BITS - 1, lo + RED_MAX_BITS, lo + 5, lo + 77], dtype=np.uint64)
    a = np.stack([lo + 100 + np.arange(8), np.full(8, 130), xs[[0, 1, 2, 3, 0, 1, 2, 2]]], axis=1)
    b = np.stack([xs[[0, 1, 2, 4, 2]], np.full(5, 131), lo + 9000 + np.arange(5)], axis=1)
    d = np.stack([lo + 9000 + np.arange(5), np.full(5, 132), lo + 9500 + g.integers(0, 3, 5)], axis=1)
    tr = np.concatenate([a, b, d]).astype(np.uint32)
    pats = [c.pattern(c.V(0), c.K(130), c.V(1)), c.pattern(c.V(1), c.K(131), c.V(2)), c.pattern(c.V(2), c.K(132), c.V(3))]
    return tr, pats
