"""CPU: the ORDER BY restatement (tests/order_reference.py) pinned by hand-worked cases of apply_order_by (execute_query.rs:113-149)."""
import math

from tests import order_reference as R


def order(values, desc=False, limit=0):
    return R.order_rows([{"v": v} for v in values], [("v", desc)], limit)


def test_numbers_compare_as_f64():
    assert R.compare("9", "10") < 0 and R.compare("10", "9") > 0  # not "10" < "9" as strings
    assert R.compare("1e3", "999") > 0
    assert R.compare("-0", "0") == 0 and R.compare("0.0", "-0.0") == 0
    assert R.compare("-inf", "-1e308") < 0 and R.compare("inf", "1e308") > 0 and R.compare("Infinity", "inf") == 0
    assert R.compare("1.0", "1") == 0 and R.compare(".5", "5.") < 0


def test_rust_f64_grammar():
    for ok in ("1", "-1", "+1.5", ".5", "5.", "1e5", "1E-5", "inf", "-Infinity", "NaN", "nan"):
        assert R.parse_f64(ok) is not None, ok
    for bad in ("", " 1", "1 ", "1_0", "0x10", "1e", "e5", "--1", "١", "in f"):
        assert R.parse_f64(bad) is None, bad


def test_strings_compare_by_bytes():
    assert R.compare("", "a") < 0 and R.compare("", "0") < 0  # "" first, also before numbers (it does not parse)
    assert R.compare("ab", "ab\0") < 0 and R.compare("ab\0", "ab\x01") < 0
    assert R.compare("z", "é") < 0  # 0x7a < 0xc3
    base = "http://x/"
    for k in (6, 7, 13, 14):  # first difference at bytes 6, 7, 13 and 14: either side of a 7-byte round
        a = (base * 2)[:k] + "a" + "zzzz"
        b = (base * 2)[:k] + "b"
        assert R.compare(a, b) < 0 and R.compare(b, a) > 0


def test_mixed_columns():
    assert R.is_mixed(["10", "9", "1a"])
    # the cycle that makes it so: 9 < 10 (numbers), 10 < 1a (strings), 1a < 9 (strings)
    assert R.compare("9", "10") < 0 and R.compare("10", "1a") < 0 and R.compare("1a", "9") < 0
    assert R.is_mixed(["NaN", "1", "2"])
    assert not R.is_mixed(["NaN", "nan", ""])  # an all-NaN column (with "") is an order: every NaN ties
    assert not R.is_mixed(["1", "", "2"]) and not R.is_mixed(["a", "", "b"]) and not R.is_mixed([])
    assert R.is_mixed(["1", "unknown"])


def test_stable_sort_and_desc_keeps_ties_in_input_order():
    vals = ["2", "1", "2", "1", "3"]
    assert order(vals) == [1, 3, 0, 2, 4]
    assert order(vals, desc=True) == [4, 0, 2, 1, 3]  # not the ascending order reversed, which would give [4, 2, 0, 3, 1]
    assert order(["-0", "0", "-0.0"], desc=True) == [0, 1, 2]


def test_limit():
    vals = ["c", "a", "b"]
    assert order(vals, limit=0) == [1, 2, 0]  # LIMIT 0 is no limit (execute_query.rs:696)
    assert order(vals, limit=1) == [1]
    assert order(vals, limit=5) == [1, 2, 0]


def test_several_keys_and_missing_variables():
    rows = [{"a": "1", "b": "x"}, {"a": "1"}, {"a": "0", "b": "y"}, {"b": "x"}]
    # "a" DESC, then "b" ASC; a missing variable is "" (execute_query.rs:124-125)
    assert R.order_rows(rows, [("a", True), ("b", False)]) == [1, 0, 2, 3]
    assert R.order_rows(rows, [("zz", False)]) == [0, 1, 2, 3]


def test_render():
    strings = ["a", "", "b"]
    quoted = {0x80000000: (0, 2, 0), 0x80000001: (0, 99, 0), 0x80000002: (0x80000000, 2, 1)}
    assert [R.render(i, strings, quoted) for i in (0, 1, 7, 0xFFFFFFFF)] == ["a", "", "unknown", ""]
    assert R.render(0x80000000, strings, quoted) == "<< a b a >>"
    assert R.render(0x80000001, strings, quoted) == "unknown"
    assert R.render(0x80000002, strings, quoted) == "<< << a b a >> b  >>"
    assert R.render(0x80000009, strings, quoted) == "unknown"
    assert math.isnan(R.parse_f64("-nan"))
