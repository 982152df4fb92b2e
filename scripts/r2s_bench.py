"""ISTREAM + DSTREAM of a sliding window's result: on the device (kb_r2s_eval) against a download of the whole result and a host set
difference. The window is the cfg5 shape: 10 slides of 1,000,002 triples (employee shape), device-resident slides appended with
kb_store_append_device, query cfg2 through the store index. Per steady-state slide, in one process, the two arms alternate:

  (a) device: star join -> kb_r2s_eval ISTREAM and DSTREAM on the result -> download of the emitted rows only
  (b) host:   star join -> download of every result column -> numpy set difference against the previous firing's rows

Arm (b) is a LOWER BOUND on the reference's host path (Relation2StreamOperator::eval over a HashSet of decoded string rows,
kolibrie/src/rsp/r2s.rs:37-58), not that path itself: it hashes no strings and decodes nothing.

Prints one JSON line per arm (and writes them to --out when given): median ms per slide; for (a) kb_r2s_eval's device time from the
library's CUDA-event timers (kb_stats.other_ms) and its algorithmic bytes over that time against 3.35 TB/s (H100 SXM HBM3);
emitted and total rows; the card and its power limit, read in the same run. Algorithmic bytes of one evaluation over c columns:
4c*R (read the response) + 4c*L (read `last`, DSTREAM only) + 4c*E (write the emitted rows) + 4c*D (write the new state). The hash
table and the flag arrays are counted apart (`table_bytes`: the table initialised, 4 B per slot; `flag_bytes`: the flag / prefix arrays
written once, read by the scan and the write pass)."""
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


def pow2_at_least(x):
    return 1 << max(1, int(x - 1).bit_length())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--per-slide", type=int, default=1_000_002)
    ap.add_argument("--width", type=int, default=10)
    ap.add_argument("--steady", type=int, default=10, help="steady-state slides measured (after the window has filled)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch

    from kolibrie_b200 import capi as c
    from kolibrie_b200 import datagen

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    per_e = a.per_slide // 6
    per = per_e * 6
    n_slides = a.width + a.steady
    d = datagen.employee_dataset(per_e * n_slides)
    ctx = c.Context(0)
    ctx.dict_numeric_load(d.num_or0, d.is_num)
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    slots = [0, 1, 2, 3]  # e, t, s, n
    ds, dp, do = (torch.from_numpy(x).cuda() for x in (d.s, d.p, d.o))
    ist, dst = ctx.r2s(c.ISTREAM, slots), ctx.r2s(c.DSTREAM, slots)
    ctx.set_timing(True)
    prev_v = None
    rec = {"device": [], "host": []}

    def arm_device(t):
        ctx.synchronize()
        t0 = time.perf_counter()
        r = ctx.star_join(js, pats, filt)
        L = ist.info()[0]
        ctx.get_stats(reset=True)
        ei, ed = ist.eval(r), dst.eval(r)
        r2s_ms = ctx.get_stats()["other_ms"]
        rows_i, rows_d = ei.to_numpy(slots), ed.to_numpy(slots)
        ms = (time.perf_counter() - t0) * 1e3
        R, D = r.n_rows, ist.info()[0]
        cc = len(slots)
        alg = 4 * cc * (R + len(rows_i) + D) + 4 * cc * (R + L + len(rows_d) + D)
        flags = 2 * (3 * 4 * R * 3)  # two evaluations x three u32 arrays of R rows, each written, scanned (read + write) and read
        for x in (r, ei, ed):
            x.free()
        return {"ms": ms, "r2s_ms": r2s_ms, "rows": R, "istream_rows": len(rows_i), "dstream_rows": len(rows_d), "alg_bytes": alg,
                "table_bytes": 2 * 4 * pow2_at_least(2 * R), "flag_bytes": flags}

    def arm_host(t):
        nonlocal prev_v
        ctx.synchronize()
        t0 = time.perf_counter()
        r = ctx.star_join(js, pats, filt)
        rows = np.ascontiguousarray(r.to_numpy(slots))
        v = rows.view(np.dtype((np.void, 4 * len(slots)))).ravel()
        if prev_v is None:
            n_i, n_d = len(v), 0
        else:
            n_i = int((~np.isin(v, prev_v)).sum())  # rows not in the previous firing (ISTREAM)
            n_d = int((~np.isin(prev_v, v)).sum())  # previous rows gone (DSTREAM)
        prev_v = v
        ms = (time.perf_counter() - t0) * 1e3
        R = r.n_rows
        r.free()
        return {"ms": ms, "rows": R, "istream_rows": n_i, "dstream_rows": n_d}

    live = []
    for t in range(n_slides):
        if len(live) == a.width:
            ctx.store_evict(live.pop(0))
        lo = t * per
        ctx.store_append_device(ds.data_ptr() + 4 * lo, dp.data_ptr() + 4 * lo, do.data_ptr() + 4 * lo, per, 100 + t)
        live.append(100 + t)
        if t == 0:
            ctx.build_index()
        order = (arm_device, arm_host) if t % 2 == 0 else (arm_host, arm_device)
        for arm in order:
            out = arm(t)
            if t >= a.width:  # steady state: every slide evicts one
                rec["device" if arm is arm_device else "host"].append(out)
    for x, h in zip(rec["device"], rec["host"]):  # both arms saw the same firings
        assert (x["istream_rows"], x["dstream_rows"], x["rows"]) == (h["istream_rows"], h["dstream_rows"], h["rows"]), (x, h)
    name, power = card()
    med = lambda k, arm: float(np.median([x[k] for x in rec[arm]]))
    common = {"card": name, "power_limit": power, "slides_measured": len(rec["device"]), "window_slides": a.width,
              "triples_per_slide": per, "query": "cfg2", "columns": len(slots)}
    r2s_ms = med("r2s_ms", "device")
    alg = med("alg_bytes", "device")
    lines = [
        dict(arm="device", what="star join + kb_r2s_eval ISTREAM + DSTREAM + download of the emitted rows", ms_per_slide=med("ms", "device"),
             r2s_eval_device_ms=r2s_ms, rows=int(med("rows", "device")), istream_rows=int(med("istream_rows", "device")),
             dstream_rows=int(med("dstream_rows", "device")), alg_bytes=int(alg), alg_gb_per_s=alg / (r2s_ms * 1e-3) / 1e9,
             alg_share_of_hbm=alg / (r2s_ms * 1e-3) / HBM_BYTES_PER_S, table_bytes=int(med("table_bytes", "device")),
             flag_bytes=int(med("flag_bytes", "device")), **common),
        dict(arm="host", what="star join + download of every result column + numpy set difference (a lower bound on the reference's "
             "HashSet-of-strings path)", ms_per_slide=med("ms", "host"), rows=int(med("rows", "host")),
             istream_rows=int(med("istream_rows", "host")), dstream_rows=int(med("dstream_rows", "host")), **common),
    ]
    text = "".join(json.dumps(x) + "\n" for x in lines)
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)
    ctx.close()


if __name__ == "__main__":
    main()
