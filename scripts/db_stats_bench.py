"""kb_store_gather_stats (DatabaseStats::gather_stats_fast on the device) on cfg2's 10 M-triple store (1 666 667 employees) and the
100 M-triple bench store (16 666 667 employees), with max_sample 100 000 (the reference's sampling) and 0 (every triple).

Per store and max_sample, --steps calls after --warmup, each recording:
  phase_ms   device time of the phases (kb_db_stats_info.phase_ms: sort + dedup, gather, counts)
  wall_ms    a host clock around the whole call through capi.Context.store_gather_stats, the download of the maps included
  n_ids      distinct ids in the subject / predicate / object maps
The host baseline is the numpy restatement (tests/stats_reference.gather_stats_numpy) on the same rows, timed once per case. It is
numpy, not the reference's Rust. One JSON line per case goes to --out, with the GPU's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import stats_reference as R

STORES = {"cfg2_10m": 1_666_667, "bench_100m": 16_666_667}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--stores", default=",".join(STORES))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "db_stats.jsonl"))
    args = ap.parse_args()
    name, power = gpu_info()
    ctx = c.Context(0)
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        for store in args.stores.split(","):
            d = datagen.employee_dataset(STORES[store])
            ctx.store_load(d.s, d.p, d.o)
            rows = np.stack([d.s, d.p, d.o], axis=1)
            del d
            for ms in (R.FAST, 0):
                for _ in range(args.warmup):
                    ctx.store_gather_stats(ms)
                phases, walls = [], []
                for _ in range(args.steps):
                    t0 = time.perf_counter()
                    g = ctx.store_gather_stats(ms)
                    walls.append((time.perf_counter() - t0) * 1e3)
                    phases.append(g["phase_ms"])
                t0 = time.perf_counter()
                want = R.gather_stats_numpy(rows, 0, ms)
                host_ms = (time.perf_counter() - t0) * 1e3
                same = all(np.array_equal(g[k][i], want[k][i]) for k in ("subject", "predicate", "object") for i in (0, 1))
                ph = np.median(np.array(phases), axis=0)
                line = {"store": store, "rows": int(len(rows)), "total_triples": g["total_triples"], "max_sample": ms, "take": g["take"],
                        "step": g["step"], "n_ids": g["n_ids"], "steps": args.steps,
                        "phase_ms_median": {"sort_dedup": round(float(ph[0]), 4), "gather": round(float(ph[1]), 4), "counts": round(float(ph[2]), 4)},
                        "wall_ms_median": round(float(np.median(walls)), 3), "wall_ms_min": round(float(np.min(walls)), 3),
                        "host_numpy_ms": round(host_ms, 1), "equal_to_numpy": bool(same), "gpu": name, "power_limit": power}
                print(json.dumps(line), flush=True)
                f.write(json.dumps(line) + "\n")
            ctx.store_clear()
    ctx.close()


if __name__ == "__main__":
    main()
