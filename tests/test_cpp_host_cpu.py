"""CPU: the parts of the C++ host mirror that need no device — Rust's str::parse::<f64> acceptance (the numeric side table the FILTER
and rule-filter kernels read is built from it; kolibrie/src/streamertail_optimizer/types.rs:133-148) against the committed table and
against the Python mirror on fuzzed strings, and Dictionary::encode's first-seen ids (shared/src/dictionary.rs:32-48)."""
import math
import os
import subprocess

import numpy as np

from kolibrie_b200.engine import Dictionary, rust_parse_f64
from tests import helpers as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "host_only.cpp")
LIBDIR = os.path.join(ROOT, "kolibrie_b200")


def run(strings, out_dir):
    """builds the host-only program into out_dir (the repository tree may be read-only) and feeds it `strings`"""
    exe = os.path.join(str(out_dir), "host_only")
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-o", exe, SRC, f"-L{LIBDIR}", "-lkolibrie_b200", f"-Wl,-rpath,{LIBDIR}"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    inp = "".join(s.encode("utf-8").hex() + "\n" for s in strings)
    r = subprocess.run([exe], input=inp, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 0, r.stdout
    lines = r.stdout.splitlines()
    progs = [tuple(x.split()[1:]) for x in lines if x.startswith("F ")]
    lines = [x for x in lines if not x.startswith("F ")]
    assert len(lines) == 2 * len(strings) + 1
    parsed = [None if lines[2 * i] == "0" else float.fromhex(lines[2 * i].split()[1]) for i in range(len(strings))]
    ids = [int(lines[2 * i + 1].split()[1]) for i in range(len(strings))]
    n_ids, n_num = (int(x) for x in lines[-1].split()[1:])
    return parsed, ids, n_ids, n_num, progs


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return (math.isnan(a) and math.isnan(b)) or a == b


def test_cpp_mirror_parses_f64_like_rust_and_like_the_python_mirror(tmp_path):
    table = H.load("rust_parse_f64.json")
    rng = np.random.default_rng(12)
    alphabet = list("0123456789+-.eEinfINFatyN x_\n\t") + ["١", "é"]
    fuzz = ["".join(rng.choice(alphabet, size=int(rng.integers(0, 9)))) for _ in range(4000)]
    fuzz = [s for s in fuzz if "\x00" not in s]
    strings = list(table["accept"]) + list(table["reject"]) + fuzz
    parsed, ids, n_ids, n_num, progs = run(strings, tmp_path)
    for s, v in zip(strings[: len(table["accept"])], parsed):
        assert v is not None, f"C++ mirror rejects {s!r}, Rust accepts it"
    for s, v in zip(table["reject"], parsed[len(table["accept"]):]):
        assert v is None, f"C++ mirror accepts {s!r}, Rust rejects it"
    bad = [(s, v, rust_parse_f64(s)) for s, v in zip(strings, parsed) if not same(v, rust_parse_f64(s))]
    assert not bad, bad[:10]
    assert sum(v is not None for v in parsed[len(table["accept"]) + len(table["reject"]):]) > 50, "the fuzz must reach accepted strings too"
    # Dictionary: first-seen ids, and the numeric table marks exactly the ids whose strings parse
    d = Dictionary()
    assert ids == [d.encode(s) for s in strings] and n_ids == len(d.id_to_string)
    assert n_num == sum(rust_parse_f64(s) is not None for s in d.id_to_string)
    # FILTER programs: the expressions tests/cpp/host_only.cpp compiles, through the Python mirror
    from kolibrie_b200.engine import And, Comparison, Condition, Not, Or, SlotMap

    lit = d.id_to_string[0]
    exprs = [
        Comparison("?s", ">", "100000"),
        And(Comparison("?s", ">=", "5."), Comparison("?t", "=", lit)),
        Or(Not(Comparison("?n", "!=", "a literal no triple mentions")), Comparison("?s", "<", "abc")),
        Comparison("?s", "<=", "?t"),
        And(Or(Comparison("t", "=", lit), Comparison("?t", "!=", lit)), Not(Comparison("?s", ">", "-1e3"))),
    ]
    want = []
    for k, e in enumerate(exprs):
        for op in Condition(e).compile(SlotMap(), d):
            want.append((str(k), str(op.op), str(op.slot), str(op.cmp), str(op.id), float(op.value).hex()))
    got = [(a, b, cc, dd, e, float.fromhex(f).hex()) for a, b, cc, dd, e, f in progs]
    assert got == want
