"""Seeded sequences of every store mutation, for the maintained store index (tests/test_gpu_store_sequences.py).

A pure-Python model of the store's contents (a bag of tagged segments) is driven by a seeded generator of mutations: the slides
(kb_store_append / _device / _file, kb_store_evict), the set-semantic writes (kb_store_insert / _remove / _remove_template),
kb_store_delete, kb_store_build_index, kb_set_use_index, kb_dict_numeric_load and the Datalog calls (kb_datalog_fixpoint, then
kb_datalog_maintain). The generator reads the model only, so a sequence is fixed by its seed and mode; `apply_device` runs one op on a
context and checks what the call itself returns, and `replay` re-runs a logged sequence on a fresh context to debug one failure.

Data shape, chosen to reach the index's maintenance branches:
  F  functional, one numeric object per subject       -> a typed chunk, a subject table and its rank column
  C  at most 200 distinct objects                     -> one-byte subject codes after a build
  M  1-4 objects per subject (other live subjects)    -> directories, chained or CSR joins
  I  inverse-functional (s + IOFF, I, s)              -> an object table
  N  a name per subject, (s, N, s + NOFF)
  ten filler predicates on some segments              -> more than 8 predicates: the batched indexing path
Subjects come from a dense block that slides upward; now and then a slide brings a subject below the lowest live one, one past the
table headroom, a sparse outlier, or a second F object for a live subject. Every id the data uses — codes, numeric values, subjects,
I subjects and N objects — lies in one dense range, so that the store's key range over any column stays within the bounds of the
direct-table star joins (the fused scan build and the batched join) while no outlier is live: without the index, those are the joins
that read and write the single- and multi-valued hints of kb_ctx. The numeric table has fewer than 65 535 distinct values (exact 16-bit
ranks) or more (coarse buckets), and reloads place new values between the existing ones.
"""
import hashlib
import os
import tempfile

import numpy as np

from kolibrie_b200 import capi as c
from tests.update_reference import batch_insert, batch_remove

F, C, M, I, N, G = 1, 2, 3, 4, 5, 6      # G: the rule's head, (?x F ?v) . (?x C ?c) -> (?x G ?c)
FILLERS = list(range(10, 20))
CODE0, N_CODES = 100, 200                # C objects
VAL0 = 1000                              # numeric value ids VAL0 .. VAL0 + n_values
FAMILIES = {"rank16": 3000, "coarse": 70000}  # initial distinct values: exact 16-bit ranks, or more than 65 535
S_BASE = 48 * 2048                       # subjects, above every value id; a multiple of 2048 so that the shard blocks line up
S_START = S_BASE + 30 * 2048             # the dense block starts here, leaving room below it
IOFF, NOFF = 2048, 4096                  # I subjects and N objects, beside the dense block (multiples of 2048: an I subject is in its
                                         # subject's shard)
N_STRINGS = S_BASE + 400_000             # device dictionary strings "t<id>" for ids below this (kb_store_remove_template)
SPARSE0 = 0x6000_0000
HEADROOM_JUMP = 200_001
RARE_FROM = 8                            # slides before this step bring no rare subject: the first index lives a while
INSERT_TAGS = (500, 501)
ABSENT_TAG = 77_777
INFERRED = c.KB_TAG_INFERRED
SHARD_RANK, SHARD_WORLD = 1, 2
MODES = ("maintained", "never_built", "use_off", "sharded")
SEEDS = (1, 2, 3, 4, 5)
STEPS = 40
EVENTS = ("dup_f_subject", "below_lowest", "past_headroom", "sparse", "over_8_predicates", "multi_segment_evict", "evict_insert_tag",
          "evict_absent", "noop_insert", "remove_absent", "numeric_reload", "rebuild_after_mutation", "maintain_slide", "family_rank16",
          "family_coarse", "filter_present", "filter_between", "filter_below", "filter_above", "dup_f_in_direct_range", "sharded_refusal")


def rules():
    """(?x F ?v) . (?x C ?c) -> (?x G ?c)"""
    return [{"premise": [c.pattern(c.V(0), c.K(F), c.V(1)), c.pattern(c.V(0), c.K(C), c.V(2))],
             "conclusion": [c.pattern(c.V(0), c.K(G), c.V(2))], "filters": []}]


def tmpl():
    """the DELETE template of kb_store_remove_template, over a relation with slots 0, 1, 2 = x, y, v"""
    return [c.pattern(c.V(0), c.K(M), c.V(1)), c.pattern(c.V(0), c.K(F), c.V(2))]


def strings():
    return ["t%d" % i for i in range(N_STRINGS)]


def u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32).reshape(-1, 3)


def keys(rows):
    """one 12-byte key per (s, p, o) row: np.isin / np.unique work on them"""
    return u32(rows).view(np.dtype((np.void, 12))).ravel()


def distinct(rows):
    return np.unique(keys(rows)).view(np.uint32).reshape(-1, 3) if len(rows) else np.empty((0, 3), np.uint32)


def as_set(rows):
    return set(map(tuple, u32(rows).tolist()))


def shard_of(x):
    return (int(x) >> 10) % SHARD_WORLD


def closure(base):
    """closure(B) \\ B under the rule, B = the distinct base rows"""
    b = distinct(base)
    fs = np.unique(b[b[:, 1] == F, 0])
    cr = b[(b[:, 1] == C) & np.isin(b[:, 0], fs)]
    head = np.stack([cr[:, 0], np.full(len(cr), G, np.uint32), cr[:, 2]], axis=1).astype(np.uint32)
    return distinct(head[~np.isin(keys(head), keys(b))]) if len(head) else np.empty((0, 3), np.uint32)


class Model:
    """the store as a list of [tag, rows] segments, as the device keeps them (bag semantics), and the numeric table"""

    def __init__(self, family):
        self.family = family
        nv = FAMILIES[family]
        self.num = np.zeros(VAL0 + nv, np.float64)
        self.isn = np.zeros(VAL0 + nv, np.uint8)
        self.num[VAL0:] = 4.0 * np.arange(nv)
        self.isn[VAL0:] = 1
        self.segs = []
        self.closed = False          # what the device's "closed" token says, conservatively: void after any other op
        self.versioned = 0           # ops that certainly moved the store, index or numeric version (a prepared plan goes stale)
        self.built = False           # kb_store_build_index has run
        self.since_build = 0         # mutations since it did
        self.use_index = True
        self.events = {"family_" + family}

    # ---- reads
    def rows(self):
        return np.concatenate([r for _, r in self.segs]) if self.segs else np.empty((0, 3), np.uint32)

    def tags(self):
        return [t for t, _ in self.segs]

    def base(self):
        parts = [r for t, r in self.segs if t != INFERRED]
        return np.concatenate(parts) if parts else np.empty((0, 3), np.uint32)

    def n_values(self):
        return len(self.num) - VAL0

    # ---- writes, each as its device call documents it
    def _moved(self):
        self.versioned += 1
        self.since_build += 1
        self.closed = False

    def append(self, tag, rows):
        rows = u32(rows)
        live = self.rows()
        lf = live[live[:, 1] == F, 0]
        nf = rows[rows[:, 1] == F, 0]
        if len(lf) and len(nf):
            if np.isin(nf, lf).any():
                self.events.add("dup_f_subject")
            if nf.min() < lf.min():
                self.events.add("below_lowest")
            if int(nf.max()) > int(lf.max()) + HEADROOM_JUMP - 1:
                self.events.add("past_headroom")
            allf = np.concatenate([lf, nf])
            if int(allf.max()) - int(allf.min()) + 1 > 4 * len(allf) + 65536:
                self.events.add("sparse")
        if len(np.unique(rows[:, 1])) > 8:
            self.events.add("over_8_predicates")
        self.segs.append([tag, rows])
        self._moved()

    def evict(self, tag):
        """kb_store_evict: every segment of the tag goes; an absent tag is KB_E_NOT_FOUND and the store stays (at a new version)"""
        hit = [s for s in self.segs if s[0] == tag]
        if not hit:
            self.events.add("evict_absent")
        if len(hit) > 1:
            self.events.add("multi_segment_evict")
        if tag in INSERT_TAGS and hit:
            self.events.add("evict_insert_tag")
        self.segs = [s for s in self.segs if s[0] != tag]
        self._moved()
        return bool(hit)

    def delete(self, rows):
        """kb_store_delete: set-difference by value; every segment stays, emptied or not"""
        gone = keys(rows)
        for s in self.segs:
            s[1] = s[1][~np.isin(keys(s[1]), gone)] if len(s[1]) else s[1]
        self._moved()

    def insert(self, tag, rows):
        """kb_store_insert: BTreeSet::insert in batch order; the new triples go into a segment of the tag"""
        rows = u32(rows)
        flags = batch_insert(as_set(self.rows()), list(map(tuple, rows.tolist())))
        new = rows[np.array(flags, bool)] if len(rows) else rows
        if len(new):
            self.segs.append([tag, new])
            self._moved()
        else:
            self.events.add("noop_insert")
        return flags

    def remove(self, rows):
        """kb_store_remove: BTreeSet::remove in batch order; every stored copy goes, a segment left empty by it leaves the store"""
        rows = u32(rows)
        flags = batch_remove(as_set(self.rows()), list(map(tuple, rows.tolist())))
        if not all(flags):
            self.events.add("remove_absent")
        gone = keys(rows[np.array(flags, bool)]) if len(rows) else keys(rows)
        if len(gone):
            kept = []
            for t, r in self.segs:
                hit = np.isin(keys(r), gone) if len(r) else np.zeros(0, bool)
                if hit.any():
                    r = r[~hit]
                    if not len(r):
                        continue
                kept.append([t, r])
            self.segs = kept
            self._moved()
        return flags

    def template_rows(self, rel):
        """the kb_store_remove batch a DELETE template fills from the relation (x, y, v): pattern by pattern, row by row"""
        rel = np.asarray(rel, np.uint32).reshape(-1, 3)
        out = []
        for r in rel.tolist():
            out.append((r[0], M, r[1]))
            out.append((r[0], F, r[2]))
        return np.array(out, np.uint32).reshape(-1, 3)

    def remove_template(self, rel):
        return sum(self.remove(self.template_rows(rel)))

    def build_index(self):
        if self.built and self.since_build:
            self.events.add("rebuild_after_mutation")
        self.built = True
        self.since_build = 0
        self.versioned += 1
        self.closed = False

    def set_use_index(self, on):
        self.use_index = bool(on)

    def numeric_load(self, values):
        """kb_dict_numeric_load of the table extended by new ids with these values"""
        if len(self.rows()):
            self.events.add("numeric_reload")
        self.num = np.concatenate([self.num, np.asarray(values, np.float64)])
        self.isn = np.concatenate([self.isn, np.ones(len(values), np.uint8)])
        assert len(self.num) <= S_BASE, "value ids reach the subjects"
        self.versioned += 1
        self.closed = False

    def fixpoint(self):
        """kb_datalog_fixpoint on a store without inferred segments (any are evicted first); its facts become one inferred segment"""
        had = INFERRED in self.tags()
        self.segs = [s for s in self.segs if s[0] != INFERRED]
        inf = closure(self.base())
        if len(inf):
            self.segs.append([INFERRED, inf])
        self._moved()
        self.closed = True
        return had, inf

    def maintain(self, evict_tags, add_tag, add):
        """kb_datalog_maintain: the evicted segments go, `add` is one segment, the inferred segments become closure(B') \\ B'"""
        old = as_set(np.concatenate([r for t, r in self.segs if t == INFERRED]) if INFERRED in self.tags() else np.empty((0, 3)))
        if evict_tags and len(add):
            self.events.add("maintain_slide")
        self.segs = [s for s in self.segs if s[0] not in set(evict_tags) and s[0] != INFERRED]
        if len(add):
            self.segs.append([add_tag, u32(add)])
        inf = closure(self.base())
        if len(inf):
            self.segs.append([INFERRED, inf])
        self._moved()
        self.closed = True
        new = as_set(inf)
        return old - new, new - old


# ---- the generator
class Gen:
    def __init__(self, seed, mode):
        self.rng = np.random.default_rng(1000 * seed + MODES.index(mode))
        self.mode = mode
        self.sharded = mode == "sharded"
        self.cursor = 0                 # the dense block's next subject, as a counter
        self.next_tag = 1
        self.family = ("rank16", "coarse")[(seed + MODES.index(mode)) % 2]

    def subj(self, k, foreign=False):
        """the k-th subject of the dense block: in a sharded context, of shard SHARD_RANK's blocks (or another shard's, foreign)"""
        if not self.sharded:
            return S_START + k
        want = (SHARD_RANK + (1 if foreign else 0)) % SHARD_WORLD
        return S_START + ((((k >> 10) * SHARD_WORLD + want) << 10) | (k & 1023))

    def fix_shard(self, x):
        return x ^ 1024 if self.sharded and shard_of(x) != SHARD_RANK else x

    def star(self, model, subjects, fillers=False):
        """the rows of a slide over these subjects: F, C (90 %), M (1-4 other subjects of the slide), I, N"""
        rng = self.rng
        s = np.asarray(subjects, np.uint32)
        n = len(s)
        vals = (VAL0 + rng.integers(0, model.n_values(), n)).astype(np.uint32)
        parts = [np.stack([s, np.full(n, F), vals], 1)]
        hc = rng.random(n) < 0.9
        parts.append(np.stack([s[hc], np.full(hc.sum(), C), CODE0 + rng.integers(0, N_CODES, hc.sum())], 1))
        for j in range(4):
            sel = rng.random(n) < (1.0 if j == 0 else 0.5)
            parts.append(np.stack([s[sel], np.full(sel.sum(), M), s[rng.integers(0, n, sel.sum())]], 1))
        parts.append(np.stack([s + IOFF, np.full(n, I), s], 1))
        parts.append(np.stack([s, np.full(n, N), s + NOFF], 1))
        if fillers:
            for p in FILLERS:
                parts.append(np.stack([s[:50], np.full(min(n, 50), p), s[:50] + NOFF], 1))
        rows = distinct(np.concatenate(parts).astype(np.uint32))  # (an M pair drawn twice is one triple)
        return rows[rng.permutation(len(rows))]

    def live_f(self, model):
        r = model.rows()
        return r[r[:, 1] == F]

    def slide_rows(self, model, step):
        rng = self.rng
        w = int(rng.integers(800, 1600))
        subs = [self.subj(k) for k in range(self.cursor, self.cursor + w)]
        self.cursor += w
        lf = self.live_f(model)
        if len(lf) and step >= RARE_FROM:
            lo, hi = int(lf[:, 0].min()), int(lf[:, 0].max())
            x = rng.random()
            if x < 0.06:
                subs.append(self.fix_shard(lo - int(rng.integers(1500, 3000))))           # below the lowest live subject
            elif x < 0.10:
                subs.append(self.fix_shard(hi + HEADROOM_JUMP + 1100 + int(rng.integers(0, 500))))  # past the table headroom
            elif x < 0.14:
                subs.append(self.fix_shard(SPARSE0 + int(rng.integers(0, 1 << 20))))      # sparse: no table over the range
        if self.sharded and rng.random() < 0.3:
            subs += [self.subj(int(rng.integers(0, self.cursor + 1)), foreign=True) for _ in range(3)]
        rows = self.star(model, sorted(set(subs)), fillers=rng.random() < 0.3)
        if len(lf) and (step >= RARE_FROM or self.mode != "maintained") and rng.random() < 0.2:
            # a live subject gets a second F object and a second C object, and nothing else: F and C become multi-valued (no triple
            # is stored twice)
            x = int(lf[rng.integers(0, len(lf)), 0])
            live = model.rows()
            have = {int(o) for o in live[(live[:, 0] == x) & ((live[:, 1] == F) | (live[:, 1] == C)), 2]}
            v = next(VAL0 + k for k in rng.permutation(model.n_values()) if VAL0 + k not in have)
            cc = next(CODE0 + k for k in rng.permutation(N_CODES) if CODE0 + k not in have)
            rows = np.concatenate([rows, np.array([[x, F, v], [x, C, cc]], np.uint32)])
        live = model.rows()
        live = live[live[:, 1] == M]  # (only M triples are stored twice: a second copy of an F, C, N or I triple would end its table)
        if len(live) and rng.random() < 0.4:  # some triples stored twice: a second copy in this slide
            rows = np.concatenate([rows, live[rng.integers(0, len(live), 40)]])
        return u32(rows)

    def pick_live(self, model, k):
        r = model.rows()
        return r[self.rng.integers(0, len(r), k)] if len(r) else np.empty((0, 3), np.uint32)

    def absent(self, k):
        return np.stack([np.full(k, S_BASE - 5), np.full(k, F), VAL0 + np.arange(k)], 1).astype(np.uint32)

    def op(self, model, step, force=None):
        rng = self.rng
        base_tags = sorted({t for t in model.tags() if t != INFERRED})
        choices = {"append": 22, "evict": 12, "delete": 6, "insert": 10, "remove": 8, "template": 5, "build_index": 6, "use_index": 4,
                   "numeric": 5, "datalog": 8}
        if self.mode == "never_built":
            choices.pop("build_index")
        if self.mode in ("use_off", "maintained"):  # (the maintained mode reads the index it keeps)
            choices.pop("use_index")
        if self.sharded:
            choices["union"] = 4  # kb_store_union into a sharded context: refused, the store stays
        if len(model.rows()) < 20_000:
            choices["append"] += 20
        if len(model.rows()) > 50_000:
            choices["evict"] += 20
        name = force or rng.choice(sorted(choices), p=np.array([choices[k] for k in sorted(choices)]) / sum(choices.values()))
        if name == "append":
            kind = ("host", "device", "file")[int(rng.integers(0, 3))]
            if base_tags and rng.random() < 0.3:
                tag = int(rng.choice(base_tags))
            else:
                tag, self.next_tag = self.next_tag, self.next_tag + 1
            return ("append", {"kind": kind, "tag": tag, "rows": self.slide_rows(model, step)})
        if name == "evict":
            x = rng.random()
            multi = [t for t in base_tags if model.tags().count(t) > 1]
            ins = [t for t in base_tags if t in INSERT_TAGS]
            if x < 0.1 or not base_tags:
                tag = ABSENT_TAG
            elif x < 0.35 and multi:
                tag = int(rng.choice(multi))
            elif x < 0.55 and ins:
                tag = int(rng.choice(ins))
            else:
                tag = int(base_tags[0]) if rng.random() < 0.7 else int(rng.choice(base_tags))  # mostly the oldest: a window slide
            return ("evict", {"tag": tag})
        if name == "delete":
            r = model.rows()
            if len(r):
                _, inv, cnt = np.unique(keys(r), return_inverse=True, return_counts=True)
                dup = r[cnt[inv.ravel()] > 1]
            else:
                dup = r
            parts = [self.pick_live(model, int(rng.integers(50, 300))), self.absent(5)]
            if len(dup):
                parts.append(dup[rng.integers(0, len(dup), 20)])
            return ("delete", {"rows": u32(np.concatenate(parts))})
        if name == "insert":
            tag = int(rng.choice(INSERT_TAGS))
            if rng.random() < 0.15:
                rows = self.pick_live(model, 30)  # every triple already there: nothing changes
            else:
                w = int(rng.integers(20, 200))
                new = self.star(model, [self.subj(k) for k in range(self.cursor, self.cursor + w)])
                self.cursor += w
                rows = np.concatenate([new, self.pick_live(model, 20), new[rng.integers(0, len(new), 10)]])
                rows = rows[rng.permutation(len(rows))]
            return ("insert", {"tag": tag, "rows": u32(rows)})
        if name == "remove":
            rows = np.concatenate([self.pick_live(model, int(rng.integers(20, 300))), self.absent(3)])
            return ("remove", {"rows": u32(np.concatenate([rows, rows[:5]]))})
        if name == "template":
            r = model.rows()
            m = r[(r[:, 1] == M) & (r[:, 0] < N_STRINGS) & (r[:, 2] < N_STRINGS)]
            f = {int(x): int(v) for x, v in self.live_f(model)[:, [0, 2]].tolist()}
            rel = [(x, y, f.get(x, VAL0)) for x, y in m[rng.integers(0, len(m), 8)][:, [0, 2]].tolist()] if len(m) else []
            rel.append((S_BASE - 5, S_BASE - 4, VAL0))  # absent
            return ("template", {"rel": np.array(rel, np.uint32)})
        if name == "build_index":
            return ("build_index", {})
        if name == "union":
            return ("union", {})
        if name == "use_index":
            return ("use_index", {"on": not model.use_index})
        if name == "numeric":
            nv = model.n_values()
            k = np.sort(rng.choice(FAMILIES[self.family], int(rng.integers(200, 2000)), replace=False))
            vals = np.concatenate([4.0 * k + 2.0, [-2.0 - 4 * nv, 4.0 * nv + 1e6 + step]])  # between existing values, below, above
            return ("numeric", {"values": vals})
        if name == "datalog":
            if model.closed:
                evict = [int(rng.choice(base_tags))] if base_tags and rng.random() < 0.8 else []
                add = self.slide_rows(model, step) if rng.random() < 0.8 else np.empty((0, 3), np.uint32)
                tag, self.next_tag = self.next_tag, self.next_tag + 1
                return ("maintain", {"evict": evict, "tag": tag, "rows": u32(add)})
            return ("fixpoint", {})
        raise AssertionError(name)


def apply_model(model, op):
    """the op on the model; returns what the device call must return (flags, counts, found) or None"""
    name, a = op
    if name in ("setup", "union"):  # (a sharded context refuses kb_store_union: nothing changes)
        return None
    if name == "append":
        model.append(a["tag"], a["rows"])
    elif name == "evict":
        return model.evict(a["tag"])
    elif name == "delete":
        model.delete(a["rows"])
    elif name == "insert":
        return model.insert(a["tag"], a["rows"])
    elif name == "remove":
        return model.remove(a["rows"])
    elif name == "template":
        return model.remove_template(a["rel"])
    elif name == "build_index":
        model.build_index()
    elif name == "use_index":
        model.set_use_index(a["on"])
    elif name == "numeric":
        model.numeric_load(a["values"])
    elif name == "fixpoint":
        return model.fixpoint()
    elif name == "maintain":
        return model.maintain(a["evict"], a["tag"], a["rows"])
    else:
        raise AssertionError(name)
    return None


def generate(seed, mode, steps=STEPS):
    """(log, model): the setup entry and `steps` ops, and the model after all of them"""
    g = Gen(seed, mode)
    model = Model(g.family)
    log = [("setup", {"mode": mode, "family": g.family})]
    force = None
    for step in range(steps):
        op = g.op(model, step, force=("append" if step < 3 else force))
        apply_model(model, op)
        # a fixpoint is mostly followed by a maintain, while the store is still closed, and now and then by a second one
        force = "datalog" if g.rng.random() < {"fixpoint": 0.8, "maintain": 0.2}.get(op[0], 0.0) else None
        if op[0] == "append" and step == 2 and mode != "never_built":
            log.append(op)
            op = ("build_index", {})
            apply_model(model, op)
        log.append(op)
    return log, model


def events(seed, mode):
    """the events a sequence reaches, from the model alone: the FILTER constant classes, a multi-valued F while a subject-keyed star
    without the index builds direct tables, and the refused op of a sharded context included"""
    log, _ = generate(seed, mode)
    model = None
    seen = set()
    for op in log:
        if op[0] == "setup":
            model = Model(op[1]["family"])
            continue
        apply_model(model, op)
        seen |= {"filter_" + k for k, _ in filter_constants(model)}
        if op[0] == "union":
            seen.add("sharded_refusal")
        if mode in ("never_built", "use_off") and direct_range(model) and f_multi_valued(model):
            seen.add("dup_f_in_direct_range")
    return seen | model.events


def direct_range(model):
    """whether the store's subject range fits the fused scan build's bound, max(4 n_triples, 2^16): a subject-keyed star without the
    index then builds direct tables, which trust or learn the single-valued hints"""
    r = model.rows()
    return len(r) > 0 and int(r[:, 0].max()) - int(r[:, 0].min()) + 1 <= max(4 * len(r), 1 << 16)


def f_multi_valued(model):
    r = model.rows()
    f = r[r[:, 1] == F, 0]
    return len(np.unique(f)) < len(f)


def filter_constants(model):
    """FILTER constants on ?v from the live F values: one present, one between two values, one below the minimum, one above the maximum"""
    r = model.rows()
    v = np.unique(model.num[r[r[:, 1] == F, 2]])
    if len(v) < 2:
        return []
    i = len(v) // 2
    return [("present", float(v[i])), ("between", float((v[i - 1] + v[i]) / 2)), ("below", float(v[0] - 3)), ("above", float(v[-1] + 3))]


def digest(log):
    h = hashlib.sha256()
    for name, a in log:
        h.update(name.encode())
        for k in sorted(a):
            x = a[k]
            h.update(k.encode())
            h.update(np.ascontiguousarray(x).tobytes() if isinstance(x, np.ndarray) else repr(x).encode())
    return h.hexdigest()


def describe(op):
    name, a = op
    parts = [name]
    for k in sorted(a):
        x = a[k]
        parts.append(f"{k}={len(x)} rows" if isinstance(x, np.ndarray) and x.ndim == 2 else f"{k}=<{len(x)}>" if isinstance(x, np.ndarray) else f"{k}={x}")
    return " ".join(parts)


def report(seed, mode, step, reader, log):
    lines = [f"seed {seed}, mode {mode}, step {step}, reader {reader}; ops up to this step:"]
    lines += [f"  {i:3d} {describe(op)}" for i, op in enumerate(log)]
    return "\n".join(lines)


# ---- the device side
def setup_device(ctx, mode, model, dict_strings=None):
    ctx.store_clear()
    if mode == "sharded":
        ctx.set_sharding(SHARD_RANK, SHARD_WORLD)
    else:
        ctx.set_sharding(0, 1)
    ctx.set_use_index(mode != "use_off")
    ctx.dict_strings_load(dict_strings if dict_strings is not None else strings())
    ctx.dict_numeric_load(model.num, model.isn)


def apply_device(ctx, op, model, want, tmpdir, keep):
    """the op on the context (the model has moved on already: its numeric table is the new one); asserts what the call returns against
    `want`, what apply_model returned"""
    name, a = op
    if name == "append":
        r = a["rows"]
        if a["kind"] == "host":
            ctx.store_append(r[:, 0], r[:, 1], r[:, 2], a["tag"])
        elif a["kind"] == "device":
            import torch

            cols = [torch.from_numpy(np.ascontiguousarray(r[:, j]).view(np.int32)).cuda() for j in range(3)]
            keep.append(cols)
            ctx.store_append_device(cols[0].data_ptr(), cols[1].data_ptr(), cols[2].data_ptr(), len(r), a["tag"])
        else:
            path = os.path.join(tmpdir, "slide.kbs")
            c.segment_write(path, r[:, 0], r[:, 1], r[:, 2], tag=a["tag"])
            ctx.store_append_file(path, a["tag"])
    elif name == "evict":
        try:
            ctx.store_evict(a["tag"])
            found = True
        except c.KolibrieError as e:
            assert e.status == c.KB_E_NOT_FOUND, e
            found = False
        assert found == want, f"evict of tag {a['tag']}: found {found}, the model says {want}"
    elif name == "delete":
        r = a["rows"]
        ctx.store_delete(r[:, 0], r[:, 1], r[:, 2])
    elif name == "insert":
        r = a["rows"]
        got = ctx.store_insert(r[:, 0], r[:, 1], r[:, 2], tag=a["tag"])
        assert got.tolist() == list(want), "insert flags"
    elif name == "remove":
        r = a["rows"]
        got = ctx.store_remove(r[:, 0], r[:, 1], r[:, 2])
        assert got.tolist() == list(want), "remove flags"
    elif name == "template":
        rel = ctx.rel_from_host([0, 1, 2], [a["rel"][:, j] for j in range(3)])
        assert ctx.store_remove_template(rel, tmpl()) == want, "remove_template count"
        rel.free()
    elif name == "union":
        a, b = c.Context(ctx.device), c.Context(ctx.device)
        try:
            ctx.store_union(a, b)
            raise AssertionError("kb_store_union into a sharded context was accepted")
        except c.KolibrieError as e:
            assert e.status == c.KB_E_UNSUPPORTED and "sharded" in e.message, e
        finally:
            a.close()
            b.close()
    elif name == "build_index":
        ctx.build_index()
    elif name == "use_index":
        ctx.set_use_index(a["on"])
    elif name == "numeric":
        ctx.dict_numeric_load(model.num, model.isn)
    elif name == "fixpoint":
        had, inf = want
        if had:
            ctx.store_evict(INFERRED)
        rel, _ = ctx.datalog_fixpoint(rules())
        got = rel.to_numpy([0, 1, 2]) if rel.n_rows else np.empty((0, 3), np.uint32)
        rel.free()
        assert as_set(got) == as_set(inf), "fixpoint facts"
    elif name == "maintain":
        gone, new = want
        add = a["rows"] if len(a["rows"]) else None
        r_gone, r_new, _ = ctx.datalog_maintain(rules(), a["evict"], add, a["tag"])
        for rel, w, what in ((r_gone, gone, "removed"), (r_new, new, "added")):
            got = rel.to_numpy([0, 1, 2]) if rel.n_rows else np.empty((0, 3), np.uint32)
            rel.free()
            assert as_set(got) == w, f"maintain: inferred facts {what}"
    else:
        raise AssertionError(name)


def replay(log, ctx):
    """re-run a logged sequence on a fresh context (debugging one failure); returns the model after it"""
    model = None
    keep = []
    with tempfile.TemporaryDirectory() as tmp:
        for op in log:
            if op[0] == "setup":
                model = Model(op[1]["family"])
                setup_device(ctx, op[1]["mode"], model)
                continue
            want = apply_model(model, op)
            apply_device(ctx, op, model, want, tmp, keep)
    return model
