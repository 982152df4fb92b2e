"""CPU: the FILTER restatement (tests/filter_reference.py) pinned by cases worked out by hand from the Rust source, then cross-checked
against the C++ oracle's evaluator on random well-typed programs over edge values, unbound cells and quoted ids."""
import numpy as np

from kolibrie_b200 import capi as c
from tests import filter_cases as FC
from tests import filter_reference as R
from tests import oracle_api as O

NONE = R.KB_ID_NONE
CMPS = [c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE]


class Table:
    """ids 0.. carry the given numbers; then one non-numeric literal; ids from `past` on are outside the numeric table"""

    def __init__(self, *values):
        self.values = list(values)
        self.plain = len(values)
        self.past = len(values) + 1
        num = np.array(self.values + [0.0], dtype=np.float64)
        isn = np.array([1] * len(values) + [0], dtype=np.uint8)
        self.terms = R.Terms(num, isn)

    def id(self, v):
        for i, x in enumerate(self.values):
            if np.array_equal(np.float64(x).view(np.uint64), np.float64(v).view(np.uint64)):
                return i
        raise KeyError(v)

    def run(self, prog, **cells):
        """one row: slot k -> the id in cells[f"x{k}"]"""
        cols = {int(k[1:]): np.array([v], dtype=np.uint32) for k, v in cells.items()}
        return bool(R.eval_program(prog, cols, self.terms)[0])


def cmp(slot, op, v):
    return c.fop(c.F_CMP_NUM, slot=slot, cmp=op, value=v)


def NOT():
    return c.fop(c.F_NOT)


def var(slot):
    return c.fop(c.F_PUSH_VAR, slot=slot)


def const(v):
    return c.fop(c.F_PUSH_CONST, value=v)


def op(code):
    return c.fop(code)


def test_nan_fails_every_ordering_and_its_not_passes():
    t = Table(np.nan, np.copysign(np.nan, -1.0), 0.0)
    for x in (t.id(np.nan), 1):
        for k in CMPS:
            for cv in (0.0, np.nan, np.inf, -np.inf):
                assert not t.run([cmp(0, k, cv)], x0=x)
                assert t.run([cmp(0, k, cv), NOT()], x0=x)  # NOT(?x > c) is not ?x <= c
    # a NaN constant: every stored value fails, and NOT passes
    for k in CMPS:
        assert not t.run([cmp(0, k, np.nan)], x0=t.id(0.0)) and t.run([cmp(0, k, np.nan), NOT()], x0=t.id(0.0))


def test_signed_zeros_are_equal_on_both_sides():
    t = Table(0.0, -0.0)
    for x in (0.0, -0.0):
        for cv in (0.0, -0.0):
            got = [t.run([cmp(0, k, cv)], x0=t.id(x)) for k in CMPS]
            assert got == [False, True, False, True], (x, cv)


def test_arithmetic_edges():
    t = Table(np.inf, 1.0, 1e308, 1.0 + 2.0 ** -30, 1.0 - 2.0 ** -30, 0.0)
    truthy = op(c.F_TRUTHY)
    inf, one = t.id(np.inf), t.id(1.0)
    assert t.run([var(0), var(1), op(c.F_SUB), truthy], x0=inf, x1=inf)  # inf - inf = NaN, and NaN != 0.0
    assert not t.run([var(0), const(-0.0), op(c.F_DIV), truthy], x0=one)  # a divisor of -0.0 is a division by zero
    assert t.run([var(0), const(-0.0), op(c.F_DIV), truthy, NOT()], x0=one)
    assert not t.run([var(0), const(0.0), op(c.F_DIV), truthy], x0=one)
    assert t.run([var(0), const(10.0), op(c.F_MUL), truthy], x0=t.id(1e308))  # overflows to inf: valid and truthy
    assert not t.run([var(0), var(0), op(c.F_SUB), truthy], x0=one)
    assert t.run([var(0), var(1), op(c.F_DIV), truthy], x0=t.id(0.0), x1=inf) is False  # 0 / inf = 0.0
    # ?x * ?y - 1: the product rounds to exactly 1.0, so the difference is 0.0 and false; a fused multiply-add would leave -2^-60
    x, y = 1.0 + 2.0 ** -30, 1.0 - 2.0 ** -30
    assert x * y - 1.0 == 0.0
    assert not t.run([var(0), var(1), op(c.F_MUL), const(1.0), op(c.F_SUB), truthy], x0=t.id(x), x1=t.id(y))


def test_non_numeric_and_past_the_table():
    t = Table(5.0)
    for x in (t.plain, t.past, t.past + 1000, 0x80000005):  # non-numeric literal, ids past the table, a quoted-triple id
        assert t.run([cmp(0, c.CMP_GT, -1.0)], x0=x)  # parse().unwrap_or(0.0) = 0.0 > -1
        assert not t.run([cmp(0, c.CMP_GT, 0.0)], x0=x)
        assert not t.run([var(0), op(c.F_TRUTHY)], x0=x)  # not a number: the arithmetic is invalid
        assert not t.run([var(0), const(1.0), op(c.F_ADD), op(c.F_TRUTHY)], x0=x)
    assert t.run([c.fop(c.F_IS_TRIPLE, slot=0)], x0=0x80000005)
    assert not t.run([c.fop(c.F_IS_TRIPLE, slot=0)], x0=t.past)


def test_unbound_operand_in_every_opcode():
    t = Table(5.0, np.nan)
    five = t.id(5.0)
    for k in CMPS:
        for cv in (-1.0, 0.0, 10.0, np.inf, -np.inf, np.nan):
            assert not t.run([cmp(0, k, cv)], x0=NONE)
            assert t.run([cmp(0, k, cv), NOT()], x0=NONE)
    for tid in (five, NONE, t.plain):
        assert not t.run([c.fop(c.F_EQ_ID, slot=0, id=tid)], x0=NONE)
        assert not t.run([c.fop(c.F_NE_ID, slot=0, id=tid)], x0=NONE)  # != is false too (types.rs:143-145)
        assert t.run([c.fop(c.F_NE_ID, slot=0, id=tid), NOT()], x0=NONE)
    assert t.run([c.fop(c.F_NE_ID, slot=0, id=NONE)], x0=five)  # a literal not in the dictionary differs from every bound term
    assert not t.run([c.fop(c.F_EQ_ID, slot=0, id=NONE)], x0=five)
    assert not t.run([c.fop(c.F_IS_TRIPLE, slot=0)], x0=NONE)
    assert t.run([c.fop(c.F_IS_TRIPLE, slot=0), NOT()], x0=NONE)
    for code in (c.F_ADD, c.F_SUB, c.F_MUL, c.F_DIV):
        assert not t.run([var(0), const(1.0), op(code), op(c.F_TRUTHY)], x0=NONE)
        assert not t.run([const(1.0), var(0), op(code), op(c.F_TRUTHY)], x0=NONE)
        assert t.run([var(0), const(1.0), op(code), op(c.F_TRUTHY), NOT()], x0=NONE)
        assert t.run([var(0), const(1.0), op(code), op(c.F_TRUTHY)], x0=five)
    # AND / OR / NOT over a bound and an unbound variable
    assert not t.run([cmp(0, c.CMP_GT, 0.0), cmp(1, c.CMP_GT, 0.0), op(c.F_AND)], x0=five, x1=NONE)
    assert t.run([cmp(0, c.CMP_GT, 0.0), cmp(1, c.CMP_GT, 0.0), op(c.F_OR)], x0=five, x1=NONE)
    assert t.run([cmp(0, c.CMP_GT, 0.0), cmp(1, c.CMP_GT, 0.0), op(c.F_AND), NOT()], x0=five, x1=NONE)


def rule(cmp_, value):
    return c.KbRuleFilter(0, cmp_, 0, 0, value)


def rule_pass(t, f, x):
    return bool(R.rule_filter_pass(f, np.array([x], dtype=np.uint32), None, t.terms)[0])


def test_rule_filters_take_epsilon_literally():
    t = Table(1.0, 1.0 + 2.0 ** -52, 1.0 + 2.0 ** -51, np.nan, np.inf, 0.0, -0.0)
    a = t.id(1.0 + 2.0 ** -52)
    assert rule_pass(t, rule(c.CMP_EQ, 1.0), a) and not rule_pass(t, rule(c.CMP_NE, 1.0), a)  # |a - c| = EPSILON, not > EPSILON
    b = t.id(1.0 + 2.0 ** -51)
    assert not rule_pass(t, rule(c.CMP_EQ, 1.0), b) and rule_pass(t, rule(c.CMP_NE, 1.0), b)
    for k in (c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE, c.CMP_EQ, c.CMP_NE):  # a NaN side makes no rejecting test true: it passes all six
        assert rule_pass(t, rule(k, 1.0), t.id(np.nan)), k
        assert rule_pass(t, rule(k, np.nan), t.id(1.0)), k
    assert rule_pass(t, rule(c.CMP_EQ, np.inf), t.id(np.inf))  # inf - inf = NaN
    assert rule_pass(t, rule(c.CMP_NE, np.inf), t.id(np.inf))
    assert not rule_pass(t, rule(c.CMP_EQ, 1.0), t.id(np.inf))
    assert [rule_pass(t, rule(k, 1.0), t.id(1.0)) for k in (c.CMP_GT, c.CMP_GE, c.CMP_LT, c.CMP_LE)] == [False, True, False, True]
    assert rule_pass(t, rule(c.CMP_EQ, 0.0), t.id(-0.0)) and not rule_pass(t, rule(c.CMP_GT, 0.0), t.id(-0.0))
    assert rule_pass(t, rule(c.CMP_EQ, 0.0), t.plain)  # not a number: 0.0
    assert rule_pass(t, rule(c.CMP_GT, 100.0), NONE)  # unbound: the filter is skipped (rules.rs:139)
    f = c.KbRuleFilter(0, c.CMP_NE, 1, 1, 0.0)
    assert list(R.rule_filter_pass(f, np.array([3, 3], np.uint32), np.array([3, 4], np.uint32), t.terms)) == [False, True]


def test_stack_shape():
    assert R.stack_shape([cmp(0, c.CMP_GT, 1.0), cmp(0, c.CMP_GT, 1.0), op(c.F_AND), NOT()]) == (4, 2)


# ---- random programs against the C++ oracle
LIT0 = 10
N_PLAIN = 8


def edge_table():
    return FC.numeric_table(LIT0 + len(FC.VALUES) + N_PLAIN, LIT0)


def edge_cells(rng, n, n_ids):
    return FC.edge_cells(rng, n, LIT0, N_PLAIN, n_ids)


def random_program(rng, n_slots, consts, ids, max_ops=32, max_depth=10):
    """a well-typed postfix program of at most max_ops ops and max_depth stack slots"""

    def boolean(budget):
        r = rng.random()
        if budget < 4 or r < 0.3:
            k = rng.integers(0, 4)
            s = int(rng.integers(0, n_slots))
            if k == 0:
                return [cmp(s, int(rng.choice(CMPS)), float(rng.choice(consts)))]
            if k == 1:
                return [c.fop(c.F_EQ_ID, slot=s, id=int(rng.choice(ids)))]
            if k == 2:
                return [c.fop(c.F_NE_ID, slot=s, id=int(rng.choice(ids)))]
            return [c.fop(c.F_IS_TRIPLE, slot=s)]
        if r < 0.45:
            return boolean(budget - 1) + [NOT()]
        if r < 0.6:
            return number(budget - 1) + [op(c.F_TRUTHY)]
        a = boolean(budget // 2)
        return a + boolean(budget - len(a) - 1) + [op(c.F_AND if rng.random() < 0.5 else c.F_OR)]

    def number(budget):
        if budget < 3 or rng.random() < 0.4:
            return [var(int(rng.integers(0, n_slots)))] if rng.random() < 0.7 else [const(float(rng.choice(consts)))]
        a = number(budget // 2)
        return a + number(budget - len(a) - 1) + [op(int(rng.choice([c.F_ADD, c.F_SUB, c.F_MUL, c.F_DIV])))]

    while True:
        p = boolean(int(rng.integers(1, max_ops + 1)))
        n, d = R.stack_shape(p)
        if n <= max_ops and d <= max_depth:
            return p


def test_random_programs_vs_oracle():
    rng = np.random.default_rng(20261016)
    num, isn = edge_table()
    terms = R.Terms(num, isn)
    n_rows = 4000
    cols = [edge_cells(rng, n_rows, len(num)) for _ in range(3)]
    rows = np.stack(cols, axis=1)
    consts = FC.boundary_consts(FC.VALUES)
    ids = np.concatenate([np.unique(rows), [NONE, len(num) + 5000]]).astype(np.uint32)
    db = O.Db(np.array([1], np.uint32), np.array([2], np.uint32), np.array([3], np.uint32), num, isn)
    rel = O.rel_from_host([0, 1, 2], cols)
    longest = deepest = 0
    for k in range(400):
        prog = random_program(rng, 3, consts, ids)
        n, d = R.stack_shape(prog)
        longest, deepest = max(longest, n), max(deepest, d)
        want = R.filter_rows(rows, [0, 1, 2], prog, terms)
        got = db.filter(rel, prog).to_numpy([0, 1, 2])
        assert np.array_equal(got, want), (k, [(o.op, o.slot, o.cmp, o.id, o.value) for o in prog])
    assert longest >= 25 and deepest >= 5


def test_single_comparisons_at_every_boundary_vs_oracle():
    num, isn = edge_table()
    terms = R.Terms(num, isn)
    rng = np.random.default_rng(5)
    cells = edge_cells(rng, 3000, len(num))
    db = O.Db(np.array([1], np.uint32), np.array([2], np.uint32), np.array([3], np.uint32), num, isn)
    rel = O.rel_from_host([0], [cells])
    for k in CMPS:
        for cv in FC.boundary_consts(FC.VALUES):
            for prog in ([cmp(0, k, cv)], [cmp(0, k, cv), NOT()]):
                want = R.filter_rows(cells[:, None], [0], prog, terms)
                got = db.filter(rel, prog).to_numpy([0])
                assert np.array_equal(got, want), (k, cv, len(prog))


def test_boundary_consts_hold_every_value_and_its_neighbours():
    cs = FC.boundary_consts(FC.VALUES).view(np.uint64)
    with np.errstate(over="ignore"):
        for v in FC.VALUES:
            for x in (v, np.nextafter(v, np.inf), np.nextafter(v, -np.inf)):
                assert np.float64(x).view(np.uint64) in cs
