"""The corpus the numeric side table's parse is checked on (tests/test_numparse_cpu.py on the host build, tests/test_gpu_numeric.py on
the device): the fixture's accept and reject lists, printed doubles, long random digit strings, exact halfway points between adjacent
doubles with tails just below and above, the subnormal and overflow edges, saturated exponents, signs and specials, i32 edges, and the
fuzz alphabet of tests/test_cpp_host_cpu.py. Everything is seeded. The reference values come from engine.rust_parse_f64 (CPython's
correctly rounded float() after Rust's grammar) and engine.rust_parse_i32."""
import math
import struct
from fractions import Fraction

import numpy as np

from kolibrie_b200.engine import rust_parse_f64, rust_parse_i32
from tests import helpers as H

FUZZ_ALPHABET = list("0123456789+-.eEinfINFatyN x_\n\t") + ["١", "é"]

EDGES = [
    "2.4703282292062327e-324", "2.4703282292062328e-324", "4.9406564584124654e-324", "2.2250738585072011e-308", "2.2250738585072014e-308",
    "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "1.8e308", "-1.7976931348623159e308",
    "1e99999999999999999999", "-1e99999999999999999999", "0e99999999999999999999", "1e-99999999999999999999", "0e-99999999999999999999",
    "1e65535", "1e65536", "1e-65536", "0.0000000000000000000000000000000000001e37", "1" + "0" * 400 + "e-400", "0." + "0" * 400 + "1e401",
    "-0", "+0", "-0.0", "0.000", "000000000000000000000000000000001", "1.000000000000000000000000000000000", "-.0e-5", "0.", ".0",
    "nan", "-nan", "+nan", "NAN", "-NaN", "inf", "-inf", "+inf", "Infinity", "-INFINITY", "+iNfInItY", "infinit", "infinityy", "nann", "-",
    "9007199254740992", "9007199254740993", "9007199254740993.0000000000000000001", "9007199254740991e22", "9007199254740993e22",
    "123456789012345678901234567890", "1e22", "1e23", "1e37", "9e37", "1e38", "123e35", "4503599627370496.5", "4503599627370497.5",
    "1.00000000000000011102230246251565404236316680908203125", "1.00000000000000011102230246251565404236316680908203124",
    "1.00000000000000011102230246251565404236316680908203126", "0.1", "0.2", "0.3", "3.14159265358979323846264338327950288419716939937510",
    "1e-22", "1e-23", "7e-10", "2147483647", "2147483648", "-2147483648", "-2147483649", "+2147483647", "00000000000000000002147483647",
    "-00000000000000000002147483648", "1" * 40, "+", "+-1", "1e+", "1e-", "1.e5", ".e5", "5e", "e",
]


def _halfway(rng, n):
    """exact midpoints between adjacent doubles of every magnitude (subnormal to max), each printed exactly, 1e-(digits+5) below and
    above it (...4999..9 / ...5000..1 tails), and in positional form"""
    out = []
    for _ in range(n):
        kind = rng.integers(0, 4)
        if kind == 0:
            bits = int(rng.integers(1, 1 << 52))                    # subnormal
        elif kind == 1:
            bits = int(rng.integers(1 << 52, 0x7FEFFFFFFFFFFFFF))  # any finite
        else:
            e = int(rng.integers(1023 - 80, 1023 + 80))            # moderate magnitudes, where the fast paths live
            bits = (e << 52) | int(rng.integers(0, 1 << 52))
        x = Fraction(struct.unpack("<d", struct.pack("<Q", bits))[0])
        y = Fraction(struct.unpack("<d", struct.pack("<Q", bits + 1))[0])
        m = (x + y) / 2
        k = 0
        while (m * 10 ** k).denominator != 1:
            k += 1
        M = int(m * 10 ** k)
        out.append(f"{M}e{-k}")
        out.append(f"{M * 100000 - 1}e{-(k + 5)}")
        out.append(f"{M * 100000 + 1}e{-(k + 5)}")
        s = str(M)
        out.append(f"{s[0]}.{s[1:]}e{len(s) - 1 - k}")
    return out


def _digits(rng, n):
    out = []
    for _ in range(n):
        r = rng.random()
        nd = int(rng.integers(1, 26)) if r < 0.6 else int(rng.integers(26, 101)) if r < 0.9 else int(rng.integers(101, 801))
        d = "".join(map(str, rng.integers(0, 10, nd)))
        cut = int(rng.integers(0, nd + 1))
        body = d[:cut] + "." + d[cut:] if rng.random() < 0.5 and 0 < cut < nd else d
        e = int(rng.integers(-420, 420))
        out.append(body + (f"e{e}" if rng.random() < 0.8 else ""))
    return out


def corpus(seed=2024, scale=1.0):
    """the strings (str) of the corpus; scale < 1 takes a proportional sample of each generated family"""
    rng = np.random.default_rng(seed)
    n = lambda k: max(1, int(k * scale))
    table = H.load("rust_parse_f64.json")
    out = list(table["accept"]) + list(table["reject"]) + EDGES
    bits = rng.integers(0, 1 << 63, n(200_000), dtype=np.uint64) | (rng.integers(0, 2, n(200_000), dtype=np.uint64) << np.uint64(63))
    vals = bits.view(np.float64)
    out += [repr(float(v)) for v in vals]
    logs = (10.0 ** rng.uniform(-30, 30, n(100_000))) * rng.choice([-1.0, 1.0], n(100_000))
    out += [repr(float(v)) for v in logs]
    for fmt in ("%.17e", "%.25e"):
        out += [fmt % float(v) for v in vals[: n(120_000)] if math.isfinite(v)]
        out += [fmt % float(v) for v in logs[: n(30_000)]]
    out += _digits(rng, n(100_000))
    out += _halfway(rng, n(5_000))
    ints = rng.integers(-(1 << 33), 1 << 33, n(80_000))
    out += [("+" if i % 7 == 0 and v >= 0 else "") + ("0" * int(i % 3)) + str(int(v)) for i, v in enumerate(ints)]
    out += ["".join(rng.choice(FUZZ_ALPHABET, size=int(rng.integers(0, 9)))) for _ in range(n(200_000))]
    out += ["http://example.org/employee%d" % i for i in range(n(20_000))] + ["Developer", "ex:salary", "\"lit\"@en", "é", ""]
    return out


def reference(strings):
    """(f64 bits uint64, is_num uint8, i32 int32, is_i32 uint8) of the host mirror's loops"""
    num = np.zeros(len(strings), np.float64)
    isn = np.zeros(len(strings), np.uint8)
    val = np.zeros(len(strings), np.int32)
    isi = np.zeros(len(strings), np.uint8)
    for i, s in enumerate(strings):
        v = rust_parse_f64(s)
        if v is not None:
            num[i] = v
            isn[i] = 1
        w = rust_parse_i32(s)
        if w is not None:
            val[i] = w
            isi[i] = 1
    return num.view(np.uint64), isn, val, isi
