"""CPU: the parse behind kb_dict_numeric_derive (kolibrie_b200/csrc/kb_numparse.cuh), built on the host with g++, against Rust's
`str::parse::<f64>()` as the Python mirror states it (engine.rust_parse_f64: the grammar, then CPython's correctly rounded float()) and
`str::parse::<i32>()` (engine.rust_parse_i32), bit for bit, NaN signs included, on more than 10^6 strings (tests/numparse_corpus.py).
The corpus reaches every route of the parse, the exact slow path included. The 128-bit powers of five are checked against exact
integers."""
import os
import re
import subprocess

import numpy as np

from tests import numparse_corpus as NC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kolibrie_b200", "csrc")
ROUTES = ["reject", "special", "clinger", "clinger_disguised", "lemire_limit", "lemire_subnormal", "lemire", "lemire_many", "slow"]
REC = np.dtype([("route", "<u4"), ("bits", "<u8"), ("is_i32", "<u4"), ("i32", "<i4")])


def run_driver(strings, out_dir):
    """builds tests/cpp/numparse_driver.cpp into out_dir (the repository tree may be read-only) and parses `strings` with it"""
    exe = os.path.join(str(out_dir), "numparse_driver")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", "-I", CSRC, "-o", exe, os.path.join(ROOT, "tests", "cpp", "numparse_driver.cpp")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    enc = [s.encode("utf-8") for s in strings]
    parts = [np.array([len(enc)], np.uint64).tobytes()]
    for b in enc:
        parts.append(np.array([len(b)], np.uint64).tobytes())
        parts.append(b)
    r = subprocess.run([exe], input=b"".join(parts), stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=600)
    assert r.returncode == 0, r.stderr
    out = np.frombuffer(r.stdout, dtype=REC)
    assert len(out) == len(strings)
    return out


def test_host_build_parses_like_rust_bit_for_bit(tmp_path):
    strings = NC.corpus()
    assert len(strings) > 1_000_000
    out = run_driver(strings, tmp_path)
    bits, isn, val, isi = NC.reference(strings)
    route = out["route"]
    got_isn = (route != 0).astype(np.uint8)
    bad = np.nonzero(got_isn != isn)[0]
    assert not len(bad), [(strings[i], int(route[i])) for i in bad[:10]]
    bad = np.nonzero(out["bits"] != bits)[0]
    assert not len(bad), [(strings[i][:80], hex(int(out["bits"][i])), hex(int(bits[i])), ROUTES[int(route[i])]) for i in bad[:10]]
    bad = np.nonzero((out["is_i32"].astype(np.uint8) != isi) | (out["i32"] != val))[0]
    assert not len(bad), [(strings[i], int(out["i32"][i]), int(val[i])) for i in bad[:10]]
    counts = np.bincount(route, minlength=len(ROUTES))
    missing = [ROUTES[k] for k in range(len(ROUTES)) if counts[k] == 0]
    assert not missing, dict(zip(ROUTES, counts.tolist()))


def test_edges_and_signs(tmp_path):
    cases = {"2.4703282292062327e-324": 0, "2.4703282292062328e-324": 1, "1.7976931348623158e308": 0x7FEFFFFFFFFFFFFF,
             "1.7976931348623159e308": 0x7FF0000000000000, "1e99999999999999999999": 0x7FF0000000000000, "0e99999999999999999999": 0,
             "-0": 1 << 63, "-nan": 0xFFF8000000000000, "nan": 0x7FF8000000000000, "-inf": 0xFFF0000000000000}
    out = run_driver(list(cases), tmp_path)
    assert [hex(int(b)) for b in out["bits"]] == [hex(v) for v in cases.values()]
    i32 = {"-2147483648": -2147483648, "2147483648": None, "+": None, "-": None, " 1": None, "+007": 7, "": None, "1.0": None}
    out = run_driver(list(i32), tmp_path)
    assert [int(v) if ok else None for v, ok in zip(out["i32"], out["is_i32"])] == list(i32.values())


def test_power_of_five_table_is_exact():
    """kb_pow5.inc row q: the top 128 bits of 5^q (q >= 0, truncated), or of 2^b / 5^-q rounded up (q < 0) — checked here as the bound
    each row must satisfy, with exact integers"""
    rows = re.findall(r"\{0x([0-9a-f]{16})ull, 0x([0-9a-f]{16})ull\},\s*// 5\^(-?\d+)", open(os.path.join(CSRC, "kb_pow5.inc")).read())
    assert [int(q) for _, _, q in rows] == list(range(-342, 309))
    for hi, lo, q in rows:
        v, q = (int(hi, 16) << 64) | int(lo, 16), int(q)
        assert (1 << 127) <= v < (1 << 128), q
        if q >= 0:
            p = 5 ** q
            sh = p.bit_length() - 128
            exact = p >> sh if sh >= 0 else p << -sh
            assert v == exact, q  # truncation of the normalized 5^q
        else:
            p = 5 ** -q
            # v = floor(2^b / p) + 1 for the b that puts its top bit at 127 (then possibly truncated): 2^b / p < v <= 2^b / p + 1
            b = 127 + p.bit_length() if q >= -27 else None
            if b is not None:
                assert v * p > (1 << b) and (v - 1) * p <= (1 << b), q
            else:
                z = p.bit_length()
                c = (1 << (2 * z + 128)) // p + 1
                sh = c.bit_length() - 128
                assert v == c >> sh, q
