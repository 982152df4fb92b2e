"""kb_values and a VALUES-based query on cfg2's 10 M-triple store (BASELINE configs[1]: 1 666 667 employees).

Workload: every dictionary id gets a 30-odd-byte IRI string (the employee dataset carries ids only); a VALUES block of 10^6 rows of one
variable ?e, each a subject IRI of the store, about 5 % of them strings the dictionary lacks and about 2 % UNDEF (such a row binds
nothing and is dropped). The query is `VALUES ?e {...}` joined to the cfg2 star (?e title ?t . ?e annual_salary ?s . ?e name ?n), run
as HashJoin(Values, StarJoin) on the device: kb_values, kb_star_join, the row-0 key read and kb_hash_join_keyed.

Reported per step (the dictionary is reloaded between steps, untimed, so that every kb_values call adds the same new strings):
  values_device_ms  CUDA-event time of kb_values' launches (kb_stats `other`), numeric side-table extension included
  values_wall_ms    host clock around the kb_values call, the host-to-device copy of the block included, ending in a synchronise
  bytes_model       least traffic of the operator: every cell byte read once, the 8-byte offsets and 1-byte UNDEF flags read once,
                    a 4-byte id written per defined cell; rate = bytes_model / values_device_ms
  query_wall_ms     host clock around the whole query (values, star join, key read, keyed join), ending in a synchronise
  host_ms           the same work on the host: the Values loop (Dictionary::encode per defined cell, here a Python dict) and a
                    numpy sort-merge join of its ids with the star's rows downloaded once (the download is not counted). A Python
                    restatement, not the reference's Rust: it says what the device replaces, not how fast the reference is.
One JSON line goes to --out with the GPU's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen

CFG2_10M_EMPLOYEES = 1_666_667


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def block(strings, subjects, n_rows, seed=3):
    """the VALUES block as kb_values takes it: undef flags, cell offsets, bytes (one variable)"""
    rng = np.random.default_rng(seed)
    pick = rng.choice(subjects, n_rows)
    u = rng.random(n_rows)
    undef = (u < 0.02).astype(np.uint8)
    new = (u >= 0.02) & (u < 0.07)
    cells = [b"" if undef[k] else (b"<http://example.org/new/%d>" % k if new[k] else strings[int(pick[k])].encode()) for k in range(n_rows)]
    off = np.zeros(n_rows + 1, np.uint64)
    off[1:] = np.cumsum([len(b) for b in cells], dtype=np.uint64)
    return undef, off, np.frombuffer(b"".join(cells), np.uint8).copy(), cells


def run_values(ctx, undef, off, data):
    out, info = C.c_void_p(), c.KbValuesInfo()
    sl = (C.c_uint32 * 1)(0)
    ctx._check(c.lib().kb_values(ctx.h, sl, 1, len(undef), c._ptr(undef), c._ptr(off), c._ptr(data), C.byref(out), C.byref(info)))
    return c.Relation(ctx, out), info.as_dict()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--employees", type=int, default=CFG2_10M_EMPLOYEES)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    name, power = gpu_info()

    d = datagen.employee_dataset(args.employees)
    strings = ["<http://example.org/term/%d>" % i for i in range(d.n_ids)]
    ctx = c.Context(0)
    ctx.store_load(d.s, d.p, d.o)
    ctx.build_index()
    js, pats, _ = datagen.employee_queries(d)["star3"]
    undef, off, data, cells = block(strings, np.unique(d.s), args.rows)

    def reset_dict():
        ctx.dict_strings_load(strings)
        ctx.dict_numeric_derive(c.NUMERIC_F64, 0)
        ctx.synchronize()

    def query():
        rel_v, _ = run_values(ctx, undef, off, data)
        star = ctx.star_join(js, pats)
        v0 = ctx.order_by(rel_v, [], 1)[0].column(0)
        key = [js] if len(v0) and v0[0] != c.KB_ID_NONE else []
        return ctx.hash_join_keyed(rel_v, star, key, c.MERGE_LEFT_FIRST if key else c.MERGE_RIGHT_FIRST)

    ctx.set_timing(True)
    dev_ms, wall_ms, q_ms, info, q_rows = [], [], [], None, 0
    for step in range(args.warmup + args.steps):
        reset_dict()
        ctx.get_stats(reset=True)
        t0 = time.perf_counter()
        rel_v, info = run_values(ctx, undef, off, data)
        ctx.synchronize()
        t1 = time.perf_counter()
        st = ctx.get_stats(reset=True)
        reset_dict()
        ctx.synchronize()
        t2 = time.perf_counter()
        j = query()
        ctx.synchronize()
        t3 = time.perf_counter()
        q_rows = j.n_rows
        if step >= args.warmup:
            dev_ms.append(st["other_ms"])
            wall_ms.append((t1 - t0) * 1e3)
            q_ms.append((t3 - t2) * 1e3)
    n_def = int(len(undef) - undef.sum())
    v_ids = rel_v.column(0)

    # the host: the Values loop and a sort-merge join with the star's rows
    reset_dict()
    star = ctx.star_join(js, pats)
    _, sslots = star.info()
    s_cols = [star.column(i) for i in range(len(sslots))]
    dic = {s: i for i, s in enumerate(strings)}  # the host dictionary before the block
    t0 = time.perf_counter()
    ids = []
    for k, b in enumerate(cells):
        if not undef[k]:
            t = b.decode()
            i = dic.get(t)
            if i is None:
                i = dic[t] = len(dic)
            ids.append(i)
    hv = np.array(ids, np.uint32)
    e = s_cols[sslots.index(js)]
    order = np.argsort(e, kind="stable")
    lo, hi = np.searchsorted(e[order], hv, "left"), np.searchsorted(e[order], hv, "right")
    host_rows = int((hi - lo).sum())
    host_ms = (time.perf_counter() - t0) * 1e3
    assert np.array_equal(hv, v_ids) and host_rows == q_rows

    bytes_model = int(off[-1]) + 8 * (len(undef) + 1) + len(undef) + 4 * n_def
    med = lambda x: float(np.median(x))
    line = {"bench": "values", "gpu": name, "power_limit": power, "store_triples": int(d.n_triples), "block_rows": args.rows,
            "defined_cells": n_def, "cell_bytes": int(off[-1]), "dict_new": info["dict_new"], "rows_dropped": info["rows_dropped"],
            "values_device_ms": med(dev_ms), "values_wall_ms": med(wall_ms), "bytes_model": bytes_model,
            "values_rate_GBps": bytes_model / (med(dev_ms) * 1e-3) / 1e9, "query_rows": int(q_rows), "query_wall_ms": med(q_ms),
            "host_ms": host_ms, "steps": args.steps, "warmup": args.warmup}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
