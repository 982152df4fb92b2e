"""BIND built-ins on the device (kb_bind) on the workload of scripts/quoted_bench.py: cfg2's 10 M-triple employee store plus one RDF-star
annotation per salary triple (1.67 M quoted triples). Each function runs over a 1.67 M-row relation:

  SUBJECT / OBJECT   BIND(SUBJECT(?t)) over the annotation scan (?t ex:source ?src)
  isTRIPLE           BIND(isTRIPLE(?t)) over the same scan
  TRIPLE existing    BIND(TRIPLE(?e, ds:annual_salary, ?s)) over the salary scan: every triple is quoted already, no new id
  TRIPLE new         BIND(TRIPLE(?s, ds:annual_salary, ?e)): every triple is new (the table is reloaded before each call, so each call
                     also rebuilds the reverse index: its time is included)
  CONCAT             BIND(CONCAT(?e, "/", ?s)) over the salary scan: every concatenation is a new string (the dictionary is reloaded
                     before each call)

Every function's output is checked against the host restatement (ExecutionEngine._bind_host) on the same rows before anything is timed;
the host restatement is timed too. Device time = the library's CUDA events (kb_stats' `other` family, which holds kb_bind's launches);
achieved bytes/s = the algorithmic bytes of DESIGN.md §3 over that time. Writes one JSON line per function (card name and power limit
read in the same run) to --out."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--employees", type=int, default=1_666_667)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch

    from kolibrie_b200 import capi as c
    from kolibrie_b200 import datagen
    from kolibrie_b200 import engine as E

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    data = datagen.annotated_salary_dataset(a.employees)
    R = data.d.n_employees
    strings = ["http://example.org/t%d" % i for i in range(data.n_ids)]
    P = data.d.ids["ds:annual_salary"]
    ctx = c.Context(0)
    ctx.store_load(data.s, data.p, data.o)
    ctx.dict_numeric_load(data.num_or0, data.is_num)

    def fresh_tables():
        ctx.dict_strings_load(strings)
        ctx.quoted_load(data.qt_ids, data.qt_s, data.qt_p, data.qt_o)

    def host_stores():
        d = E.Dictionary()
        for t in strings:
            d.encode(t)
        q = E.QuotedTripleStore()
        q.id_to_components = dict(zip(data.qt_ids.tolist(), zip(data.qt_s.tolist(), data.qt_p.tolist(), data.qt_o.tolist())))
        q.components_to_id = {v: k for k, v in q.id_to_components.items()}
        q.next_qt_id = int(0x80000000 + R)
        return d, q

    fresh_tables()
    ann = ctx.scan([c.pattern(c.V(0), c.K(data.source), c.V(1))])[0]  # t, src
    sal = ctx.scan([c.pattern(c.V(0), c.K(P), c.V(1))])[0]            # e, s
    ann_cols = {"t": ann.column(0), "src": ann.column(1)}
    sal_cols = {"e": sal.column(0), "s": sal.column(1)}
    nxt = int(0x80000000 + R)
    FN_NAME = {c.BIND_SUBJECT: "SUBJECT", c.BIND_OBJECT: "OBJECT", c.BIND_IS_TRIPLE: "isTRIPLE", c.BIND_TRIPLE: "TRIPLE", c.BIND_CONCAT: "CONCAT"}
    str_len = np.array([len(x.encode()) for x in strings], dtype=np.int64)
    # name: (relation, host columns, function, device args, host args, consts, reload tables before each call, algorithmic bytes)
    cases = {
        "SUBJECT": (ann, ann_cols, c.BIND_SUBJECT, [c.V(0)], ["?t"], (), False, 12 * R),
        "OBJECT": (ann, ann_cols, c.BIND_OBJECT, [c.V(0)], ["?t"], (), False, 12 * R),
        "isTRIPLE": (ann, ann_cols, c.BIND_IS_TRIPLE, [c.V(0)], ["?t"], (), False, 12 * R),
        "TRIPLE existing": (sal, sal_cols, c.BIND_TRIPLE, [c.V(0), c.K(P), c.V(1)], ["?e", strings[P], "?s"], (), False, 32 * R),
        "TRIPLE new": (sal, sal_cols, c.BIND_TRIPLE, [c.V(1), c.K(P), c.V(0)], ["?s", strings[P], "?e"], (), True, 60 * R),
        "CONCAT": (sal, sal_cols, c.BIND_CONCAT, [c.V(0), c.K(0), c.V(1)], ["?e", '"/"', "?s"], (b"/",), True, None),
    }
    ctx.set_timing(True)
    lines = []
    for name, (rel, cols, fn, args, hargs, consts, reload, alg) in cases.items():
        next_id = nxt if fn == c.BIND_TRIPLE else 0
        # correctness first: the device's column and tails against the host restatement on the same rows
        fresh_tables()
        d, q = host_stores()
        t0 = time.perf_counter()
        want = E.ExecutionEngine._bind_host(FN_NAME[fn], hargs, cols, R, None, d, q)
        host_ms = (time.perf_counter() - t0) * 1e3
        res, info = ctx.bind(rel, fn, args, 2, next_id, consts)
        got = res.column(res.slots.index(2))
        assert np.array_equal(got, want), name
        new_strings = ctx.dict_strings_download(info["dict_first"], info["dict_new"])
        assert new_strings == d.id_to_string[len(strings):], name
        if info["quoted_new"]:
            qs, qp, qo = ctx.quoted_download(info["quoted_first"], info["quoted_new"])
            assert [q.id_to_components[info["quoted_first"] + k] for k in range(info["quoted_new"])] == list(zip(qs.tolist(), qp.tolist(), qo.tolist()))
        if fn == c.BIND_CONCAT:  # id reads + the strings read + the concatenations written + what the encode reads (hash, probe, compare)
            total = int(sum(str_len[cols[k]].sum() for k in ("e", "s")) + R)
            alg = 8 * R + (total - R) + R + total + 8 * (R + 1) + 3 * total + 4 * R
        res.free()
        # timed reps
        dev, wall = [], []
        for r in range(a.reps):
            if reload:
                fresh_tables()
            ctx.synchronize()
            ctx.get_stats(reset=True)
            t0 = time.perf_counter()
            res, info = ctx.bind(rel, fn, args, 2, next_id, consts)
            ctx.synchronize()
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(ctx.get_stats()["other_ms"])
            res.free()
        dms = float(np.median(dev))
        line = {"function": name, "rows": R, "device_ms": dms, "call_ms": float(np.median(wall)), "host_restatement_ms": host_ms,
                "reps": a.reps, "alg_bytes": int(alg), "gb_per_s": alg / (dms * 1e-3) / 1e9, "share_of_hbm": alg / (dms * 1e-3) / HBM_BYTES_PER_S,
                "n_unbound": int(info["n_unbound"]), "dict_new": int(info["dict_new"]), "quoted_new": int(info["quoted_new"])}
        lines.append(line)
        print(json.dumps(line), flush=True)
    name, power = card()
    for line in lines:
        line.update(card=name, power_limit=power, workload="quoted_bench: %d-triple store + %d annotations" % (len(data.s) - R, R))
    if a.out:
        with open(a.out, "w") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
