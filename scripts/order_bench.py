"""kb_order_by on the headline result: the cfg2 star join over 100 M triples (16 666 667 employees, 6 945 872 result rows, columns e, t, s, n).

Three ways to end `SELECT ... ORDER BY` over that result, each timed over --steps calls after --warmup:
  topk_salary    kb_order_by(DESC ?s, LIMIT 10) on the device, then the 10 rows downloaded
  sort_string    kb_order_by(ASC ?e) on the device, ?e rendered as a 31-byte IRI whose digits do not follow the id order
  host_sort      the alternative without it: download the four columns, then a numpy stable argsort of the ?e strings. It is a LOWER
                 bound on the reference's path, which also decodes every row to a String and sorts BTreeMaps with a comparator that
                 tries f64::parse on both sides of every comparison.
device_ms is the CUDA-event time kb_stats counts in its `other` family (every kb_order_by launch); wall_ms a host clock around the
call, the download included, ending in a synchronise. bytes_model is the least traffic a sort of that result needs: the key column
read once, every column gathered once (4 B per cell read and written); rate = bytes_model / device time. One JSON line per case
goes to --out, with the GPU's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen

E_FULL = 16_666_667


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--employees", type=int, default=E_FULL)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, power = gpu_info()
    d = datagen.employee_dataset(a.employees)
    x = c.Context(0)
    x.dict_numeric_load(d.num_or0, d.is_num)
    x.store_load(d.s, d.p, d.o)
    strings = [(repr(float(d.num_or0[i])) if d.is_num[i] else "http://example.org/e/%010d" % ((i * 2654435761) % (1 << 32))) for i in range(d.n_ids)]
    x.dict_strings_load(strings)
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    rel = x.star_join(js, pats, filt)
    n = rel.n_rows
    sarr = np.array(strings, dtype=object)
    x.set_timing(True)

    def device(keys, limit):
        out, info = x.order_by(rel, keys, limit)
        out.to_numpy([0, 1, 2, 3])
        out.free()
        return info

    def host():
        cols = rel.to_numpy([0, 1, 2, 3])
        order = np.argsort(sarr[cols[:, 0]].astype("S"), kind="stable")
        return cols[order]

    cases = [("topk_salary", lambda: device([(2, True)], 10), 10), ("sort_string", lambda: device([(0, False)], 0), n), ("host_sort", host, n)]
    lines = []
    for label, fn, rows_out in cases:
        for _ in range(a.warmup):
            fn()
        walls, devs, info = [], [], None
        for _ in range(a.steps):
            x.get_stats(reset=True)
            t0 = time.perf_counter()
            info = fn()
            x.synchronize()
            walls.append((time.perf_counter() - t0) * 1e3)
            devs.append(x.get_stats()["other_ms"])
        model = 4 * n + 2 * 4 * 4 * rows_out  # key column read once; four columns gathered (read + write)
        rec = {"case": label, "gpu": name, "power_limit": power, "rows_in": n, "rows_out": rows_out, "steps": a.steps,
               "wall_ms_median": float(np.median(walls)), "wall_ms_min": float(np.min(walls)),
               "device_ms_median": float(np.median(devs)) if label != "host_sort" else None,
               "bytes_model": model, "info": info if isinstance(info, dict) else None}
        if rec["device_ms_median"]:
            rec["model_GBps"] = model / rec["device_ms_median"] / 1e6
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    if a.out:
        with open(a.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    x.close()


if __name__ == "__main__":
    main()
