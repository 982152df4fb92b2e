"""Exact restatement of FILTER for the tests, written from the Rust source and independent of the C++ oracle.

A `kb_filter_op` postfix program is evaluated over rows of dictionary ids, vectorised with numpy. It restates:
  - `Condition::evaluate_filter_with_ids` (kolibrie/src/streamertail_optimizer/types.rs:119-185), which the Filter operator runs on each
    row (kolibrie/src/streamertail_optimizer/execution/engine.rs:73-85);
  - `ArithmeticExpression::evaluate` (shared/src/query.rs:35-56), the arithmetic inside it;
  - the Datalog rule filters, `evaluate_filters` (datalog/src/reasoning/rules.rs:133-165), separately: their six operators are not the
    ones of a query FILTER.

Operand values. A row's cell is an id; KB_ID_NONE is a variable the row leaves unbound (`result.get(var)` is None). A term's number is
`num_or0[id]` and `is_num[id]` tells whether `decode(id).parse::<f64>()` succeeded; an id at or past the table (a quoted-triple id
included) decodes to nothing numeric, so it counts as 0.0 (`unwrap_or(0.0)`) and as not numeric (`.ok()` is None).

KB_F_CMP_LEGACY is not restated here (tests/test_legacy_path.py has its own restatement).
"""
import numpy as np

from kolibrie_b200 import capi as c

KB_ID_NONE = 0xFFFFFFFF
QUOTED_BIT = 0x80000000
F64_EPSILON = 2.220446049250313e-16  # std::f64::EPSILON = 2^-52
ORDERING = {c.CMP_GT: np.greater, c.CMP_GE: np.greater_equal, c.CMP_LT: np.less, c.CMP_LE: np.less_equal}


def _fields(op):
    """(op, slot, cmp, id, value) of a KbFilterOp or of a tuple in that order"""
    if isinstance(op, c.KbFilterOp):
        return op.op, op.slot, op.cmp, op.id, op.value
    return tuple(op)


class Terms:
    """the numeric side table: num_or0[id] and is_num[id] for ids below its length"""

    def __init__(self, num_or0, is_num):
        self.num = np.ascontiguousarray(num_or0, dtype=np.float64)
        self.isn = np.ascontiguousarray(is_num).astype(bool)

    def number(self, ids):
        """(bound, value, numeric) per cell: value is `parse::<f64>().unwrap_or(0.0)`, numeric is `parse::<f64>().ok().is_some()`"""
        ids = np.asarray(ids, dtype=np.uint32)
        bound = ids != KB_ID_NONE
        inside = ids < len(self.num)
        idx = np.where(inside, ids, 0).astype(np.int64)
        value = np.where(inside, self.num[idx] if len(self.num) else 0.0, 0.0)
        numeric = inside & (self.isn[idx] if len(self.isn) else False)
        return bound, value, numeric & bound


def eval_program(ops, cols, terms: Terms):
    """the rows that pass `ops`: a bool array over the rows of `cols` ({slot: uint32 array}). The program must be well typed: each
    comparison, NOT, AND, OR and TRUTHY yields a boolean, each PUSH and arithmetic op a number (an AST of FilterExpression /
    ArithmeticExpression written in postfix)."""
    ops = [_fields(o) for o in ops]
    n = len(next(iter(cols.values()))) if cols else 0
    if not ops:
        return np.ones(n, dtype=bool)
    st = []  # ("b", bool array) or ("n", valid array, value array)
    with np.errstate(all="ignore"):
        for code, slot, cmp, tid, value in ops:
            if code in (c.F_CMP_NUM, c.F_EQ_ID, c.F_NE_ID, c.F_IS_TRIPLE, c.F_PUSH_VAR):
                ids = np.asarray(cols[slot], dtype=np.uint32)
                bound, num, numeric = terms.number(ids)
            if code == c.F_CMP_NUM:  # types.rs:133-140: parse both sides (unwrap_or(0.0)) and compare; unbound: false (:143-145)
                fn = ORDERING.get(cmp)
                st.append(("b", bound & fn(num, np.float64(value)) if fn is not None else np.zeros(n, dtype=bool)))  # :141 other ops: false
            elif code == c.F_EQ_ID:  # types.rs:131: the decoded string equals the literal <=> the same id; KB_ID_NONE: not in the dictionary
                st.append(("b", bound & (ids == tid) if tid != KB_ID_NONE else np.zeros(n, dtype=bool)))
            elif code == c.F_NE_ID:  # types.rs:132, and false when unbound (:143-145)
                st.append(("b", bound & (ids != tid) if tid != KB_ID_NONE else bound.copy()))
            elif code == c.F_IS_TRIPLE:  # types.rs:167-176: bound and a quoted-triple id
                st.append(("b", bound & ((ids & np.uint32(QUOTED_BIT)) != 0)))
            elif code in (c.F_AND, c.F_OR):  # types.rs:147-154
                (kb, b), (ka, a) = st.pop(), st.pop()
                assert ka == kb == "b", "AND / OR over a number"
                st.append(("b", (a & b) if code == c.F_AND else (a | b)))
            elif code == c.F_NOT:  # types.rs:155-157
                k, a = st.pop()
                assert k == "b", "NOT over a number"
                st.append(("b", ~a))
            elif code == c.F_PUSH_VAR:  # types.rs:159-163: unbound or not a number -> None, and `?` makes the expression invalid
                st.append(("n", numeric, num))
            elif code == c.F_PUSH_CONST:
                st.append(("n", np.ones(n, dtype=bool), np.full(n, value, dtype=np.float64)))
            elif code in (c.F_ADD, c.F_SUB, c.F_MUL, c.F_DIV):  # query.rs:44-54: one IEEE operation, rounded once
                (kb, vb, b), (ka, va, a) = st.pop(), st.pop()
                assert ka == kb == "n", "arithmetic over a boolean"
                valid = va & vb
                if code == c.F_ADD:
                    r = a + b
                elif code == c.F_SUB:
                    r = a - b
                elif code == c.F_MUL:
                    r = a * b
                else:  # query.rs:49: a divisor equal to 0.0 (either sign) is an error
                    valid = valid & (b != 0.0)
                    r = a / b
                st.append(("n", valid, r))
            elif code == c.F_TRUTHY:  # types.rs:164: Ok(v) -> v != 0.0 (so NaN is true), Err -> false
                k, va, a = st.pop()
                assert k == "n", "TRUTHY over a boolean"
                st.append(("b", va & (a != 0.0)))
            else:
                raise NotImplementedError(f"opcode {code}")
    assert len(st) == 1 and st[0][0] == "b", "the program does not leave one boolean"
    return st[0][1]


def filter_rows(rows, slots, ops, terms: Terms):
    """rows (n x k uint32) over `slots` -> the rows that pass"""
    rows = np.asarray(rows, dtype=np.uint32).reshape(-1, len(slots))
    return rows[eval_program(ops, {s: rows[:, j] for j, s in enumerate(slots)}, terms)]


def stack_shape(ops):
    """(number of ops, deepest stack) of a postfix program"""
    depth = top = 0
    for o in ops:
        code = _fields(o)[0]
        top += {c.F_AND: -1, c.F_OR: -1, c.F_ADD: -1, c.F_SUB: -1, c.F_MUL: -1, c.F_DIV: -1, c.F_NOT: 0, c.F_TRUTHY: 0}.get(code, 1)
        depth = max(depth, top)
    return len(ops), depth


# ---- Datalog rule filters (rules.rs:133-165)
def rule_filter_pass(filt, lhs, rhs, terms: Terms):
    """the rows a KbRuleFilter lets through: lhs / rhs are the id columns of its variables (rhs only read when rhs_is_var). A variable
    the row leaves unbound (KB_ID_NONE) skips the filter (rules.rs:139)."""
    lhs = np.asarray(lhs, dtype=np.uint32)
    n = len(lhs)
    bound = lhs != KB_ID_NONE
    if filt.rhs_is_var:  # rules.rs:141-146: ids of two bound variables; only = and != act
        rhs = np.asarray(rhs, dtype=np.uint32)
        if filt.cmp == c.CMP_NE:
            rej = lhs == rhs
        elif filt.cmp == c.CMP_EQ:
            rej = lhs != rhs
        else:
            rej = np.zeros(n, dtype=bool)
        return ~(bound & rej)
    _, a, _ = terms.number(lhs)  # rules.rs:149-151: decode(..).unwrap_or("").parse().unwrap_or(0.0)
    cv = np.float64(filt.rhs_value)
    with np.errstate(all="ignore"):
        rej = {c.CMP_GT: lambda: a <= cv, c.CMP_LT: lambda: a >= cv, c.CMP_GE: lambda: a < cv, c.CMP_LE: lambda: a > cv,
               # rules.rs:157-158, taken literally: a NaN difference (NaN, inf - inf) rejects nothing, so it passes both = and !=
               c.CMP_EQ: lambda: np.abs(a - cv) > F64_EPSILON, c.CMP_NE: lambda: np.abs(a - cv) <= F64_EPSILON}.get(filt.cmp, lambda: np.zeros(n, dtype=bool))()
    return ~(bound & rej)
