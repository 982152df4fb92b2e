"""kb_natural_join on the full-size multi-window emit: cfg2's star split across two windows on ?e (window A = title + salary > 100000,
window B = salary > 100000 + name: 0.69 M rows each, sharing ?e and ?s) plus a static relation with one row per title. One process, arms
in turn after a warm-up of each:

  fast     kb_natural_join(A, B): no unbound shared cell, so one check pass + kb_hash_join
  unbound  kb_natural_join(A, B'), B' = B with 1 % of its ?s cells unbound (KB_ID_NONE): mask pass, partition, two sub-joins
           ((e, s) for the bound group, (e) for the unbound one), coalesce
  emit     a whole emit: A ⋈ B ⋈ static, RSTREAM (kb_r2s_eval), download of every emitted row
  restatement  tests/rsp_join_reference.py's natural_join (the reference's nested loop, restated in Python) on a 2 000 x 2 000 subsample:
           pair checks per second. The Rust nested loop is not run here; no comparison with it is made.

Per arm: median wall ms per call (ending in a device synchronise) and the library's CUDA-event device time (kb_stats: other = check,
mask, partition, coalesce; build + probe = kb_hash_join's launches) against the byte model of DESIGN §3:
  fast:     16·L + 4·c_p·R + 8·R + 4·c_out·R_out (kb_hash_join, build side L) + 4·|S|·(L+R) (check pass)
  unbound:  4·|S|·(L+R) check + 4·|U|·(L+R) mask + 8·c·(L+R) partition (c = |S| + 1 columns moved: shared columns and the row index)
            + each sub-join's kb_hash_join model over its groups (key columns + row index) + 4·c_out·R_out coalesce
Writes one JSON line per arm to --out (default profiles/rsp_multi_window.jsonl) with the card and its power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def hash_join_bytes(build, probe, c_p, c_out, rows):
    return 16 * build + 4 * c_p * probe + 8 * probe + 4 * c_out * rows


def timed(ctx, fn, reps):
    walls, dev = [], []
    for _ in range(reps):
        ctx.get_stats(reset=True)
        t0 = time.perf_counter()
        out = fn()
        ctx.synchronize()
        walls.append((time.perf_counter() - t0) * 1e3)
        st = ctx.get_stats()
        dev.append((st["other_ms"], st["build_ms"] + st["probe_ms"], st["total_ms"], st["other_launches"]))
        if out is not None:
            for r in out:
                r.free()
    dev.sort(key=lambda x: x[2])
    mid = dev[len(dev) // 2]
    return float(np.median(walls)), {"other_ms": mid[0], "join_ms": mid[1], "device_ms": mid[2], "other_launches": mid[3]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--employees", type=int, default=166_667 * 10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "rsp_multi_window.jsonl"))
    a_ = ap.parse_args()
    from kolibrie_b200 import capi as c
    from kolibrie_b200 import datagen
    from tests import rsp_join_reference as J

    gpu, power = card()
    ctx = c.Context(0)
    d = datagen.employee_dataset(a_.employees)
    ctx.store_load(d.s, d.p, d.o)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    ctx.build_index()
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    A = ctx.star_join(js, pats[:2], filt)  # e, t, s
    B = ctx.star_join(js, pats[1:], filt)  # e, s, n
    L, R = A.n_rows, B.n_rows
    Bm = B.to_numpy([0, 2, 3])
    rng = np.random.default_rng(5)
    unb = rng.random(len(Bm)) < 0.01
    Bm[unb, 1] = c.KB_ID_NONE
    Bu = ctx.rel_from_host([0, 2, 3], [np.ascontiguousarray(Bm[:, j]) for j in range(3)])
    titles = np.unique(A.to_numpy([1])[:, 0])
    S = ctx.rel_from_host([1, 9], [titles, titles + 1_000_000])
    ctx.set_timing(True)
    rows_out = ctx.natural_join(A, B).n_rows
    n_unb = int(unb.sum())

    def emit():
        ab = ctx.natural_join(A, B)
        full = ctx.natural_join(ab, S)
        op = ctx.r2s(c.RSTREAM, [0, 1, 2, 3, 9])
        em = op.eval(full)
        cols = [em.column(j) for j in range(5)]
        assert len(cols[0]) == rows_out
        op.free()
        return [ab, full, em]

    arms = {"fast": lambda: [ctx.natural_join(A, B)], "unbound": lambda: [ctx.natural_join(A, Bu)], "emit": emit}
    for f in arms.values():  # warm-up of every shape
        timed(ctx, f, 2)
    n_s, c_out = 2, 4
    model = {
        "fast": hash_join_bytes(L, R, 3, c_out, rows_out) + 4 * n_s * (L + R),
        "unbound": 4 * n_s * (L + R) + 4 * 1 * (L + R) + 8 * (n_s + 1) * (L + R)
        + hash_join_bytes(R - n_unb, L, 3, 4, rows_out - n_unb) + hash_join_bytes(n_unb, L, 2, 3, n_unb) + 4 * c_out * rows_out,
    }
    # the second join (build on the static titles, its check pass over ?t) and the download of the emitted rows
    model["emit"] = model["fast"] + hash_join_bytes(len(titles), rows_out, c_out, 5, rows_out) + 4 * (rows_out + len(titles)) + 4 * 5 * rows_out
    lines = []
    for name, f in arms.items():
        wall, dev = timed(ctx, f, a_.reps)
        rec = {"arm": name, "gpu": gpu, "power_limit": power, "L": L, "R": R, "rows_out": rows_out, "unbound_rows": n_unb if name == "unbound" else 0,
               "wall_ms_median": round(wall, 4), **{k: (round(v, 4) if isinstance(v, float) else v) for k, v in dev.items()},
               "model_bytes": model[name]}
        if dev["device_ms"] > 0:
            rec["model_GBps"] = round(model[name] / (dev["device_ms"] * 1e-3) / 1e9, 1)
            rec["model_share_of_3.35TBps"] = round(model[name] / (dev["device_ms"] * 1e-3) / HBM_BYTES_PER_S, 4)
        lines.append(rec)
    # the restated nested loop on a subsample
    k = 2000
    Ar = [dict(zip((0, 1, 2), map(int, r))) for r in A.to_numpy([0, 1, 2])[:k].tolist()]
    Br = [{kk: v for kk, v in zip((0, 2, 3), map(int, r)) if v != c.KB_ID_NONE} for r in Bm[:k].tolist()]
    t0 = time.perf_counter()
    J.natural_join(Ar, Br)
    dt = time.perf_counter() - t0
    lines.append({"arm": "restatement", "gpu": gpu, "power_limit": power, "left": k, "right": k, "seconds": round(dt, 3),
                  "pairs_per_s": round(k * k / dt), "full_size_pairs": L * R, "full_size_seconds_at_this_rate": round(L * R / (k * k / dt))})
    os.makedirs(os.path.dirname(a_.out), exist_ok=True)
    with open(a_.out, "w") as f:
        for rec in lines:
            line = json.dumps(rec)
            print(line)
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
