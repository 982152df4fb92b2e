"""kb_serialize_begin / kb_serialize_next: the device store written as N-Triples-star and Turtle-star text, on cfg2's 10 M-triple store
(1 666 667 employees) and the 100 M-triple bench store (16 666 667 employees).

The dictionary renders entities and predicates as IRIs (http://example.org/e/<10 digits>, bracketed), "F" and the salaries as plain
literals (quoted): every object class of the serializers occurs. Per store and format, --steps full exports after --warmup, each one
kb_serialize_begin and then kb_serialize_next into one reused host buffer of --capacity bytes until the text is complete:
  phase_ms      device time of begin's phases (kb_serialize_info.phase_ms: sort + dedup, render, ranks, unit lengths + scan) and of the
                write kernels of next (kb_stats' `other` family over the next calls)
  wall_ms       a host clock around the whole export, begin and every D2H piece included
  text_bytes    bytes of the text; write_gbps = bytes_model / write device time, where bytes_model = 2 x text bytes (every output byte
                read once, from a rendered term or a literal, and written once into staging) + 21 B per unit (its three u32 term
                indices, its flag byte, its u64 offset); e2e_gbps = text bytes / wall time
The host baseline is the Python restatement of the reference's loops (tests/serialize_reference.py) timed on the first --slice
triples and scaled linearly to the store (its sort is n log n, so the scaled figure is a lower bound). It is Python, not the
reference's Rust. One JSON line per case goes to --out, with the GPU's name and power limit read in the same run."""
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
from tests import serialize_reference as R

STORES = {"cfg2_10m": 1_666_667, "bench_100m": 16_666_667}
FORMATS = {"ntriples": c.SER_NTRIPLES, "turtle": c.SER_TURTLE}
PREFIXES = [("ex", "http://example.org/e/")]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def strings_of(d):
    out = np.array(["http://example.org/e/%010d" % ((i * 2654435761) % (1 << 32)) for i in range(d.n_ids)], dtype=object)
    out[d.ids["F"]] = "F"
    k = np.nonzero(d.is_num)[0]
    out[k] = [str(int(v)) for v in d.num_or0[k]]
    return out.tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stores", default="cfg2_10m,bench_100m")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--capacity", type=int, default=64 << 20)
    ap.add_argument("--slice", type=int, default=200_000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, power = gpu_info()
    x = c.Context(0)
    buf = np.empty(a.capacity, np.uint8)
    import ctypes as C
    L = c.lib()
    lines = []
    for store in a.stores.split(","):
        d = datagen.employee_dataset(STORES[store])
        strings = strings_of(d)
        x.store_load(d.s, d.p, d.o)
        x.dict_strings_load(strings)
        for fmt_name, fmt in FORMATS.items():
            enc = [s.encode() for pr in PREFIXES for s in pr]
            off = np.zeros(len(enc) + 1, np.uint64)
            off[1:] = np.cumsum([len(b) for b in enc])
            data = np.frombuffer(b"".join(enc), np.uint8)
            walls, writes, phases, info = [], [], [], None
            for step in range(a.warmup + a.steps):
                x.set_timing(True)
                x.get_stats(reset=True)
                t0 = time.perf_counter()
                h, inf = C.c_void_p(), c.KbSerializeInfo()
                x._check(L.kb_serialize_begin(x.h, fmt, c._ptr(off), c._ptr(data), len(PREFIXES), C.byref(h), C.byref(inf)))
                x.get_stats(reset=True)  # (begin's own launches are in phase_ms)
                got, total = C.c_uint64(), 0
                while True:
                    x._check(L.kb_serialize_next(x.h, h, c._ptr(buf), a.capacity, C.byref(got)))
                    if got.value == 0:
                        break
                    total += got.value
                wall = (time.perf_counter() - t0) * 1e3
                L.kb_serialize_free(h)
                write_ms = x.get_stats(reset=True)["other_ms"]
                assert total == inf.total_bytes
                if step >= a.warmup:
                    walls.append(wall)
                    writes.append(write_ms)
                    phases.append(list(inf.phase_ms))
                info = inf.as_dict()
            text_bytes = info["total_bytes"]
            model = 2 * text_bytes + 21 * info["n_triples"]
            wmed = float(np.median(writes))
            # host baseline: the Python restatement on a slice, scaled to the store
            n_sl = min(a.slice, d.n_triples)
            trip = list(zip(d.s[:n_sl].tolist(), d.p[:n_sl].tolist(), d.o[:n_sl].tolist()))
            t0 = time.perf_counter()
            if fmt == c.SER_NTRIPLES:
                R.generate_ntriples(trip, strings, {})
            else:
                R.generate_turtle(trip, strings, {}, PREFIXES)
            host_ms = (time.perf_counter() - t0) * 1e3 * d.n_triples / n_sl
            line = {"store": store, "format": fmt_name, "gpu": name, "power_limit": power, "triples": d.n_triples, "steps": a.steps,
                    "capacity": a.capacity, "text_bytes": text_bytes, "info": info,
                    "phase_ms_median": {"sort_dedup": float(np.median([p[0] for p in phases])), "render": float(np.median([p[1] for p in phases])),
                                        "ranks": float(np.median([p[2] for p in phases])), "unit_scan": float(np.median([p[3] for p in phases])),
                                        "write": wmed},
                    "wall_ms_median": float(np.median(walls)), "wall_ms_min": float(np.min(walls)), "bytes_model": model,
                    "write_gbps": model / (wmed * 1e6) if wmed > 0 else None, "e2e_gbps": text_bytes / (float(np.median(walls)) * 1e6),
                    "python_restatement_ms_scaled": host_ms, "python_restatement_slice": n_sl}
            print(json.dumps(line), flush=True)
            lines.append(line)
    x.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
