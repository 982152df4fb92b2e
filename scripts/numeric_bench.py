"""kb_dict_numeric_derive on a cfg3-sized dictionary: the employee shape's distinct term strings as scripts/dict_encode_bench.py builds
them (a subject IRI per employee, three predicate IRIs, the titles, the salary literals), 16.8 M ids. Measured:

  full          the f64 table of every id (kb_dict_numeric_derive(F64, 0))
  full + i32    both tables of every id
  append 1M     the f64 table of the last 1 M ids (what a window firing or a load batch that added 1 M strings derives)

Before anything is timed, the derived table is checked against the host loop (Dictionary.numeric_table) on every id. Device time = the
library's CUDA events (kb_stats' `other` family), after a warm-up call, median of --reps calls. Achieved bytes/s = the byte model of
DESIGN.md §3 (8 B of offsets + the bytes read up to the rejecting byte + 9 B written per id, + 5 B with the i32 view) over that time.
The host loop it replaces is timed on a sample of --host-sample ids and scaled. Writes one JSON line per case (card name and power limit
read in the same run) to --out."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.bind_bench import HBM_BYTES_PER_S, card  # noqa: E402


def employee_strings(n_ids: int):
    """distinct strings in first-seen order of the employee shape until n_ids ids: employee{e}, its predicates once, titles, salaries"""
    preds = ["http://xmlns.com/foaf/0.1/name", "http://xmlns.com/foaf/0.1/title", "https://data.cityofchicago.org/resource/xzkq-xp2w/annual_salary"]
    out, seen_sal, e = [], set(), 0
    n_emp = n_ids - 3 - 2 - 120000
    for e in range(n_emp):
        s = f"http://example.org/employee{e}"
        out.append(s)
        if e == 0:
            out += [preds[0], preds[1], "Manager", preds[2]]
        if e == 1:
            out.append("Developer")
        sal = 50000 + e * 7919 % 120000
        if sal not in seen_sal:
            seen_sal.add(sal)
            out.append(str(sal))
    return out[:n_ids]


def bytes_read(strings) -> int:
    """bytes the parse reads: one for a string whose first byte cannot start a number, the whole string otherwise"""
    start = set(b"0123456789+-.iInN")
    return sum(len(s) if s and s.encode()[0] in start else 1 for s in strings)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ids", type=int, default=16_800_000)
    ap.add_argument("--append", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--host-sample", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch

    from kolibrie_b200 import capi as c
    from kolibrie_b200 import engine as E

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    strings = employee_strings(a.ids)
    n = len(strings)
    ctx = c.Context(0)
    ctx.dict_strings_load(strings)
    # correctness first: every id against the host loop
    info = ctx.dict_numeric_derive(c.NUMERIC_F64 | c.NUMERIC_I32, 0)
    d = E.Dictionary()
    d.id_to_string = strings
    sample = E.Dictionary()
    sample.id_to_string = strings[: a.host_sample]
    t0 = time.perf_counter()
    sample.numeric_table()
    host_ms = (time.perf_counter() - t0) * 1e3 * n / min(n, a.host_sample)
    num, isn = ctx.dict_numeric_download(0, n)
    full_num, full_isn = d.numeric_table()
    assert np.array_equal(num.view(np.uint64), full_num.view(np.uint64)) and np.array_equal(isn, full_isn)
    assert info["n_numeric"] == int(full_isn.sum())
    read_all = bytes_read(strings)
    read_tail = bytes_read(strings[n - a.append:])
    cases = {
        "full": (c.NUMERIC_F64, 0, n, 8 * n + read_all + 9 * n),
        "full + i32": (c.NUMERIC_F64 | c.NUMERIC_I32, 0, n, 8 * n + read_all + 14 * n),
        "append 1M": (c.NUMERIC_F64, n - a.append, a.append, 8 * a.append + read_tail + 9 * a.append),
    }
    ctx.set_timing(True)
    lines = []
    for name, (tables, first, ids, alg) in cases.items():
        ctx.dict_numeric_derive(tables, first)  # warm-up
        dev, wall = [], []
        for _ in range(a.reps):
            ctx.synchronize()
            ctx.get_stats(reset=True)
            t0 = time.perf_counter()
            info = ctx.dict_numeric_derive(tables, first)
            wall.append((time.perf_counter() - t0) * 1e3)
            st = ctx.get_stats()
            dev.append(st["other_ms"])
            assert st["h2d_bytes"] == 0
        dms = float(np.median(dev))
        line = {"case": name, "dict_ids": n, "ids_derived": int(info["n_derived"]), "n_numeric": int(info["n_numeric"]), "n_slow": int(info["n_slow"]),
                "device_ms": dms, "call_ms": float(np.median(wall)), "reps": a.reps, "alg_bytes": int(alg), "gb_per_s": alg / (dms * 1e-3) / 1e9,
                "share_of_hbm": alg / (dms * 1e-3) / HBM_BYTES_PER_S,
                "host_loop_ms": host_ms * ids / n, "host_loop_sample_ids": min(n, a.host_sample)}
        lines.append(line)
        print(json.dumps(line), flush=True)
    name, power = card()
    for line in lines:
        line.update(card=name, power_limit=power, workload="numeric_bench: %d distinct employee-shape strings" % n)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
