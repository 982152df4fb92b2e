"""Sliding window with rules on the taxonomy stream: one steady-state firing as (a) ONE kb_datalog_maintain (delete-and-rederive from the
slide) against (b) kb_store_evict(KB_TAG_INFERRED) + kb_datalog_fixpoint (what a window re-materialising from scratch pays,
simple_r2r.rs:103-128).

The window: the TBox of datagen.taxonomy_dataset as a segment that never leaves, plus `--slides` ABox rdf:type slides of consecutive
instance ranges (first_instance); rules R1, R2 (datagen.taxonomy_rules). Every firing evicts the oldest slide and adds the next one.
`--scale 1` is the config-4 shape (fanout 10, depth 6, 48.9 M instances in the window: about 50 M live triples); `--scale 0.1` a tenth.
The two arms run one after the other on fresh contexts over the same firings. Per scale: one JSON line with the medians over the timed
firings of each arm's call time (host clock around the synchronous call) and derivations, and whether both arms left the same inferred
set after every timed firing (count + order-independent digest of the whole store, taken outside the timed region: the base segments
are the same in both arms).

    python scripts/window_reasoning_bench.py --scale 0.1 --scale 1 --firings 5 --warmup 2
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kolibrie_b200 import capi as c  # noqa: E402
from kolibrie_b200 import datagen  # noqa: E402

TBOX_TAG = 1 << 40


def slide(k, per, fanout, depth):
    t = datagen.taxonomy_dataset(fanout=fanout, depth=depth, n_instances=per, first_instance=k * per)
    keep = t.p == t.ids["rdf:type"]
    return np.ascontiguousarray(t.s[keep]), np.ascontiguousarray(t.p[keep]), np.ascontiguousarray(t.o[keep])


def store_digest(cx):
    s, p, o = cx.store_download()
    n, ssum, sxor = datagen.row_checksums(np.stack([s, p, o], axis=1))
    return int(n), f"{int(ssum):016x}{int(sxor):016x}"


def run_arm(arm, args, scale, slides_of, tbox, rules):
    cx = c.Context(0)
    try:
        cx.store_append(*tbox, TBOX_TAG)
        for k in range(args.slides):
            cx.store_append(*slides_of(k), k)
        rel, st0 = cx.datalog_fixpoint(rules)
        rel.free()
        times, derivs, digests = [], [], []
        n_fire = args.warmup + args.firings
        for f in range(n_fire):
            old, new = f, args.slides + f
            s, p, o = slides_of(new)
            if arm == "maintain":
                add = cx.rel_from_host([0, 1, 2], [s, p, o])  # (the slide is on the device before the clock starts, as in arm b)
                t0 = time.perf_counter()
                gone, added, st = cx.datalog_maintain(rules, [old], add, new)
                t1 = time.perf_counter()
                gone.free(); added.free(); add.free()
                d = st.derivations
            else:
                cx.store_evict(old)
                cx.store_append(s, p, o, new)
                t0 = time.perf_counter()
                cx.store_evict(c.KB_TAG_INFERRED)
                rel, st = cx.datalog_fixpoint(rules)
                t1 = time.perf_counter()
                rel.free()
                d = st.derivations
            if f >= args.warmup:
                times.append((t1 - t0) * 1e3)
                derivs.append(int(d))
                digests.append(store_digest(cx))
        return {"ms": times, "derivations": derivs, "digests": digests}
    finally:
        cx.close()


def gpu_state():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, action="append")
    ap.add_argument("--slides", type=int, default=10)
    ap.add_argument("--firings", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--fanout", type=int, default=10)
    ap.add_argument("--depth", type=int, default=6)
    args = ap.parse_args()
    fanout, depth = args.fanout, args.depth
    t = datagen.taxonomy_dataset(fanout=fanout, depth=depth, n_instances=1)
    keep = t.p == t.ids["rdfs:subClassOf"]
    tbox = (np.ascontiguousarray(t.s[keep]), np.ascontiguousarray(t.p[keep]), np.ascontiguousarray(t.o[keep]))
    rules = datagen.taxonomy_rules(t)
    for scale in args.scale or [0.1, 1.0]:
        per = int(48_888_890 * scale) // args.slides
        cache = {}

        def slides_of(k):
            if k not in cache:
                cache[k] = slide(k, per, fanout, depth)
            return cache[k]

        before = gpu_state()
        a = run_arm("maintain", args, scale, slides_of, tbox, rules)
        b = run_arm("fixpoint", args, scale, slides_of, tbox, rules)
        med = lambda x: float(np.median(x)) if x else None
        print(json.dumps({
            "bench": "window_reasoning", "scale": scale, "live_triples": int(len(tbox[0]) + per * args.slides), "slide_triples": per,
            "slides_per_window": args.slides, "timed_firings": args.firings, "warmup_firings": args.warmup,
            "maintain_ms_median": med(a["ms"]), "fixpoint_ms_median": med(b["ms"]),
            "maintain_derivations_median": med(a["derivations"]), "fixpoint_derivations_median": med(b["derivations"]),
            "maintain_ms": [round(x, 3) for x in a["ms"]], "fixpoint_ms": [round(x, 3) for x in b["ms"]],
            "same_inferred_every_firing": a["digests"] == b["digests"], "store_rows": [n for n, _ in a["digests"]],
            "gpu_before": before, "gpu_after": gpu_state(),
        }), flush=True)


if __name__ == "__main__":
    main()
