"""TEST INFRASTRUCTURE: the contract of kb_datalog_maintain restated with full closures on the CPU oracle, behind the method names of
kolibrie_b200.capi.Context, so that the host logic of kolibrie_b200.engine.SimpleR2R (segment and tag bookkeeping, the
fixpoint-then-maintain switch, the fallback after a rule change) runs in the CPU suite. The product never imports this.

    B  = distinct triples of the segments not tagged KB_TAG_INFERRED, I = triples of the KB_TAG_INFERRED segments
    I' = closure(B') \\ B' after the evicted segments left and `add` arrived; removed = I \\ I', added = I' \\ I"""
import numpy as np

from kolibrie_b200 import capi as c
from tests.oracle_ctx import OracleCtx
from tests.sharded_cases import closure_of, rule_predicates


def rows_set(a):
    return set(map(tuple, np.asarray(a, np.uint32).reshape(-1, 3).tolist()))


def as_rows(s):
    return np.array(sorted(s), np.uint32).reshape(-1, 3)


def rules_key(rules):
    """the rules by value (what the device's token compares byte for byte)"""
    t = lambda x: (int(x.is_var), int(x.value))
    pat = lambda p: (t(p.s), t(p.p), t(p.o))
    return repr([([pat(p) for p in r["premise"]], [pat(p) for p in r["conclusion"]],
                  [(f.lhs_slot, f.cmp, f.rhs_is_var, f.rhs_slot, f.rhs_value) for f in r.get("filters", [])]) for r in rules])


def rules_read_numbers(rules):
    """a rule filter takes the numeric branch (a constant right-hand side, or a variable no premise binds): only then does the closure
    depend on the numeric table, and only then does loading it void the token"""
    for r in rules:
        bound = {int(t.value) for p in r["premise"] for t in (p.s, p.p, p.o) if t.is_var}
        for f in r.get("filters", []):
            if f.cmp and (not f.rhs_is_var or int(f.rhs_slot) not in bound):
                return True
    return False


class MaintainStats:
    def __init__(self, **kw):
        for k in ("base_removed", "base_added", "overdeleted", "rederived", "inferred_removed", "inferred_added", "derivations",
                  "overdelete_rounds", "insert_rounds"):
            setattr(self, k, kw.get(k, 0))
        self.device_ms = 0.0


class WindowOracleCtx(OracleCtx):
    """a tagged segment store with the oracle's closure; store_evict, datalog_fixpoint and datalog_maintain keep the closed token the
    way the library does (any other store change voids it; a numeric-table load voids it when a rule filter compares numbers)"""

    def __init__(self):
        super().__init__()
        self.segs = []  # [(tag, rows[n,3])]
        self.version = 0
        self.num_version = 0
        self.token = None
        self.calls = []  # ("fixpoint" | "maintain", args) for the tests

    def _rebuild(self):
        rows = np.concatenate([r for _, r in self.segs], axis=0) if self.segs else np.empty((0, 3), np.uint32)
        self._spo = (rows[:, 0].copy(), rows[:, 1].copy(), rows[:, 2].copy())
        self._make()
        self.version += 1

    def store_load(self, s, p, o):
        self.segs = [(0, np.stack([np.asarray(x, np.uint32) for x in (s, p, o)], axis=1))]
        self._rebuild()

    def store_append(self, s, p, o, tag):
        self.segs.append((int(tag), np.stack([np.asarray(x, np.uint32) for x in (s, p, o)], axis=1).reshape(-1, 3)))
        self._rebuild()

    def store_evict(self, tag):
        if not any(t == tag for t, _ in self.segs):
            raise c.KolibrieError(c.KB_E_NOT_FOUND, f"no segment with tag {tag}")
        self.segs = [(t, r) for t, r in self.segs if t != tag]
        self._rebuild()

    def dict_numeric_load(self, num, isn):
        super().dict_numeric_load(num, isn)
        self.num_version += 1

    def _token(self, rules):
        return (self.version, rules_key(rules), self.num_version if rules_read_numbers(rules) else None)

    def store_download(self):
        rows = np.concatenate([r for _, r in self.segs], axis=0) if self.segs else np.empty((0, 3), np.uint32)
        return rows[:, 0].copy(), rows[:, 1].copy(), rows[:, 2].copy()

    def base(self):
        return set().union(*[rows_set(r) for t, r in self.segs if t != c.KB_TAG_INFERRED])

    def inferred(self):
        return set().union(*[rows_set(r) for t, r in self.segs if t == c.KB_TAG_INFERRED])

    def _closure(self, base_rows):
        st, facts = closure_of(as_rows(base_rows), self._rules, self._num)
        if st != 0:
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, "the oracle declines this rule set")
        return rows_set(facts) - base_rows

    def datalog_fixpoint(self, rules, strategy=0):
        self.calls.append(("fixpoint", None))
        had_inferred = any(t == c.KB_TAG_INFERRED for t, _ in self.segs)
        self._rules = rules
        inf = self._closure(self.base()) - self.inferred()
        if inf:
            self.segs.append((c.KB_TAG_INFERRED, as_rows(inf)))
            self._rebuild()
        self.token = self._token(rules) if not had_inferred and strategy != c.SEMI_NAIVE_PARALLEL else None
        rows = as_rows(inf)
        return self.rel_from_host([0, 1, 2], [rows[:, k].copy() for k in range(3)]), OracleCtx._Stats()

    def datalog_maintain(self, rules, evict_tags=(), add=None, add_tag=0, strategy=0):
        if strategy == c.SEMI_NAIVE_PARALLEL:
            raise c.KolibrieError(c.KB_E_UNSUPPORTED, "KB_SEMI_NAIVE_PARALLEL")
        if c.KB_TAG_INFERRED in evict_tags or (add is not None and add_tag == c.KB_TAG_INFERRED):
            raise c.KolibrieError(c.KB_E_INVALID, "KB_TAG_INFERRED")
        if self.token != self._token(rules):
            raise c.KolibrieError(c.KB_E_INVALID, "store not closed under these rules: run kb_datalog_fixpoint")
        for t in evict_tags:
            if not any(t2 == t for t2, _ in self.segs):
                raise c.KolibrieError(c.KB_E_NOT_FOUND, f"no segment with tag {t}")
        self.calls.append(("maintain", (list(evict_tags), None if add is None else len(add), add_tag)))
        self._rules = rules
        b, i = self.base(), self.inferred()
        if not evict_tags and add is None:
            e = np.empty(0, np.uint32)
            return self.rel_from_host([0, 1, 2], [e] * 3), self.rel_from_host([0, 1, 2], [e] * 3), MaintainStats()
        add_rows = np.asarray(add, np.uint32).reshape(-1, 3) if add is not None else None
        self.segs = [(t, r) for t, r in self.segs if t not in set(evict_tags) and t != c.KB_TAG_INFERRED]
        if add_rows is not None:
            self.segs.append((int(add_tag), add_rows))
        b2 = self.base()
        i2 = self._closure(b2)
        if i2:
            self.segs.append((c.KB_TAG_INFERRED, as_rows(i2)))
        self._rebuild()
        self.token = self._token(rules)
        rem, new = as_rows(i - i2), as_rows(i2 - i)
        preds = rule_predicates(rules)  # (the base counts cover the predicates the rules mention, as the header states)
        in_rules = lambda facts: {t for t in facts if t[1] in preds}
        st = MaintainStats(base_removed=len(in_rules(b - b2)), base_added=len(in_rules(b2 - b)), inferred_removed=len(rem), inferred_added=len(new))
        return (self.rel_from_host([0, 1, 2], [rem[:, k].copy() for k in range(3)]), self.rel_from_host([0, 1, 2], [new[:, k].copy() for k in range(3)]), st)
