"""ORDER BY + LIMIT restated from the Rust source, for the tests of kb_order_by.

apply_order_by (kolibrie/src/execute_query.rs:113-149): for each condition in turn the value of a row is its variable's result string,
or "" when the row lacks the variable; when both values parse with `str::parse::<f64>` they compare by `partial_cmp` with NaN as
Equal, otherwise as `str` (byte order, a proper prefix first); DESC reverses a condition; the first condition that is not Equal
decides. `sort_by` is stable. The LIMIT cut (execute_query.rs:695-699) truncates only when the limit is above 0.

`is_mixed` is the rule under which that comparison is not an order (kb_order_by refuses such a key column): the column holds a number
and a non-empty string that is not a number, or NaN and a number that is not NaN."""
import functools
import math
import re
from typing import Dict, List, Optional, Sequence, Tuple

# Rust's f64 grammar (core::num::dec2flt): optional sign, then inf / infinity / nan in any case, or digits with an optional point and
# an optional exponent; nothing else (no whitespace, no '_', no hex)
_F64 = re.compile(r"[+-]?(?:inf|infinity|nan|(?:[0-9]+\.?[0-9]*|\.[0-9]+)(?:[eE][+-]?[0-9]+)?)", re.IGNORECASE)


def parse_f64(s: str) -> Optional[float]:
    if not s.isascii() or not _F64.fullmatch(s):
        return None
    return float(s)  # Python reads every string the grammar accepts, to the nearest double


def compare(a: str, b: str) -> int:
    x, y = parse_f64(a), parse_f64(b)
    if x is not None and y is not None:
        return -1 if x < y else 1 if x > y else 0  # partial_cmp(..).unwrap_or(Equal): NaN is Equal to everything
    ab, bb = a.encode("utf-8"), b.encode("utf-8")
    return -1 if ab < bb else 1 if ab > bb else 0


def order_rows(rows: Sequence[Dict[str, str]], conditions: Sequence[Tuple[str, bool]], limit: int = 0) -> List[int]:
    """indices of `rows` in the order apply_order_by + LIMIT leave them; conditions = [(variable, descending)]"""

    def cmp(i, j):
        for var, desc in conditions:
            r = compare(rows[i].get(var, ""), rows[j].get(var, ""))
            if desc:
                r = -r
            if r:
                return r
        return 0

    order = sorted(range(len(rows)), key=functools.cmp_to_key(cmp)) if conditions else list(range(len(rows)))
    return order[:limit] if limit > 0 else order


def is_mixed(values: Sequence[str]) -> bool:
    nums = [parse_f64(v) for v in values]
    has_num = any(x is not None and not math.isnan(x) for x in nums)
    has_nan = any(x is not None and math.isnan(x) for x in nums)
    has_str = any(x is None and v != "" for x, v in zip(nums, values))
    return ((has_num or has_nan) and has_str) or (has_nan and has_num)


def render(i: int, strings: Sequence[str], quoted: Dict[int, Tuple[int, int, int]]) -> str:
    """the result string of id i as ExecutionEngine::execute gives it (engine.rs:27-51), "" for an unbound cell (KB_ID_NONE)"""
    if i == 0xFFFFFFFF:
        return ""

    def term(x) -> Optional[str]:  # Dictionary::decode_term (dictionary.rs:60-72)
        if x & 0x80000000:
            comp = quoted.get(x)
            if comp is None:
                return None
            parts = [term(y) for y in comp]
            return None if any(p is None for p in parts) else "<< " + " ".join(parts) + " >>"
        return strings[x] if x < len(strings) else None

    t = term(i)
    return "unknown" if t is None else t
