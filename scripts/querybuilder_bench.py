"""QueryBuilder triple queries on the device (kb_qb_triples / kb_qb_terms) on the 100 M-triple bench store and on cfg2's 10 M-triple
store: per query the device time of each phase (match, selection, sort + dedup, join; the term list's decode as the wall time of its
synchronous call) and the wall time, medians over --reps calls after a warm-up; the match kernel's bytes per its byte model
(DESIGN.md §3) over its phase time; and the numpy restatement of the same query on cfg2, the only baseline (the reference's Rust is
not run). One JSON record per (store, query) to --out, each with the card's name and power limit.
Run: python scripts/querybuilder_bench.py --out profiles/querybuilder.jsonl"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kolibrie_b200 import capi as c  # noqa: E402
from kolibrie_b200 import datagen  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def match_bytes(lens, mode, m):
    """the match kernel's byte model: 8 B of offsets per id, the bytes each mode reads, 1 bit per id written"""
    n = len(lens)
    if mode == c.QB_CONTAINS:
        read = int(lens[lens >= m].sum())
    else:
        read = int(np.minimum(lens, m)[lens >= m].sum())
    return 8 * n + read + (n + 7) // 8


def np_query(d, strings_np, pos, mode, pat):
    """the numpy restatement: the matching ids, the rows whose position holds one, sorted and deduplicated"""
    col = (d.s, d.p, d.o)[pos]
    if mode == c.QB_CONTAINS:
        ok = np.char.find(strings_np, pat) >= 0
    elif mode == c.QB_STARTS:
        ok = np.char.startswith(strings_np, pat)
    else:
        ok = np.char.endswith(strings_np, pat)
    keep = ok[col]
    rows = np.stack([d.s[keep], d.p[keep], d.o[keep]], 1)
    rows = rows[np.lexsort((rows[:, 2], rows[:, 1], rows[:, 0]))]
    first = np.ones(len(rows), bool)
    first[1:] = (rows[1:] != rows[:-1]).any(axis=1)
    return int(first.sum())


def timed(fn, reps):
    fn()  # warm-up
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        out.append((time.perf_counter() - t0, r))
    return out


def run_store(name, d, reps, emit, ctx2=None):
    ctx = c.Context(0)
    strings = datagen.employee_strings(d)
    lens = np.fromiter((len(s.encode()) for s in strings), np.int64, len(strings))
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_strings_load(strings)
    queries = [("with_predicate_ending(annual_salary)", [None, (c.QB_ENDS, "annual_salary"), None], 1),
               ("with_subject_starting(http://example.org/employee1)", [(c.QB_STARTS, "http://example.org/employee1"), None, None], 0),
               ("with_object_like(Developer)", [None, None, (c.QB_CONTAINS, "Developer")], 2),
               ("count()", [None, None, None], None)]
    strings_np = np.array(strings) if name == "cfg2_10m" else None
    for qname, filt, pos in queries:
        count_only = qname == "count()"

        def call():
            rel, info = ctx.qb_triples(filt, count_only=count_only)
            if rel is not None:
                rel.free()
            return info

        runs = timed(call, reps)
        infos = [r for _, r in runs]
        rec = {"store": name, "triples": len(d.s), "query": qname, "rows": infos[0]["n_rows"], "wall_ms": 1e3 * float(np.median([t for t, _ in runs])),
               "phase_ms": {k: float(np.median([i["phase_ms"][j] for i in infos])) for j, k in enumerate(("match", "selection", "sort", "join"))}}
        if pos is not None:
            mode, pat = filt[pos]
            b = match_bytes(lens, mode, len(pat.encode()))
            rec["match_bytes"] = b
            rec["match_gbps"] = b / (rec["phase_ms"]["match"] * 1e-3) / 1e9 if rec["phase_ms"]["match"] > 0 else None
            if strings_np is not None:
                t0 = time.perf_counter()
                np_query(d, strings_np, pos, mode, pat)
                rec["numpy_restatement_ms"] = 1e3 * (time.perf_counter() - t0)
        emit(rec)
    # get_subjects() with distinct(): the whole store's rows, their subjects' distinct strings in byte order
    rel, _ = ctx.qb_triples()

    def terms():  # the synchronous call alone: the strings stay in device memory
        h = c.C.c_void_p()
        ctx._check(c.lib().kb_qb_terms(ctx.h, rel.h, 0, c.QB_TERMS_DISTINCT, c.C.byref(h)))
        n = c.C.c_uint64()
        c.lib().kb_strings_info(h, c.C.byref(n), None)
        c.lib().kb_strings_free(ctx.h, h)
        return n.value

    runs = timed(terms, reps)
    t0 = time.perf_counter()
    ctx.qb_terms(rel, 0, c.QB_TERMS_DISTINCT)
    emit({"store": name, "triples": len(d.s), "query": "get_subjects() distinct", "rows": runs[0][1],
          "decode_wall_ms": 1e3 * float(np.median([t for t, _ in runs])), "with_python_list_ms": 1e3 * (time.perf_counter() - t0)})
    rel.free()
    if ctx2 is not None:  # an OnSubject join against a second context holding a 1 % subject slice
        subj = np.unique(d.s)
        pick = np.isin(d.s, subj[:: 100])
        ctx2.store_load(d.s[pick], d.p[pick], d.o[pick])

        def join():
            rel, info = ctx.qb_triples(join=c.QB_ON_SUBJECT, right=ctx2)
            rel.free()
            return info

        runs = timed(join, reps)
        infos = [r for _, r in runs]
        emit({"store": name, "triples": len(d.s), "query": "join(1% subject slice).join_on_subject()", "right_triples": int(pick.sum()),
              "rows": infos[0]["n_rows"], "wall_ms": 1e3 * float(np.median([t for t, _ in runs])),
              "phase_ms": {k: float(np.median([i["phase_ms"][j] for i in infos])) for j, k in enumerate(("match", "selection", "sort", "join"))}})
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/querybuilder.jsonl")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stores", default="cfg2_10m,bench_100m")
    a = ap.parse_args()
    gpu, power = card()
    f = open(a.out, "w")

    def emit(rec):
        rec.update({"gpu": gpu, "power_limit": power, "reps": a.reps, "statistic": "median"})
        print(json.dumps(rec), flush=True)
        f.write(json.dumps(rec) + "\n")
        f.flush()

    for name in a.stores.split(","):
        n = {"cfg2_10m": 1_666_667, "bench_100m": 16_666_667}[name]
        ctx2 = c.Context(0) if name == "cfg2_10m" else None
        run_store(name, datagen.employee_dataset(n), a.reps, emit, ctx2)
        if ctx2 is not None:
            ctx2.close()
    f.close()


if __name__ == "__main__":
    main()
