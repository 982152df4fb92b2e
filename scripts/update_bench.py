"""Latency of set-semantic writes to an indexed device store (kb_store_insert / kb_store_remove) next to
the same change made by reloading the store and rebuilding its index (kb_store_load + kb_store_build_index, which is what a front end
that keeps the store on the host does after any change; the host-side walk of its set is not included). Stores: the employee dataset
(6 predicates) at 10 M and 100 M triples. Writes one JSON line per measurement to profiles/update.jsonl (or --out), with the card's
name and power limit read in the same run. Device time: CUDA events around the call on the library's stream (kb_set_timing); wall:
host clock around the call, which returns after its stream synchronises."""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return name, power


def timed(ctx, fn, reps):
    walls, devs = [], []
    for _ in range(reps):
        ctx.get_stats(reset=True)
        t0 = time.perf_counter()
        fn()
        walls.append((time.perf_counter() - t0) * 1e3)
        devs.append(ctx.get_stats()["total_ms"])
    return float(np.median(walls)), float(np.median(devs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000000,100000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "update.jsonl"))
    a = ap.parse_args()
    name, power = card()
    ctx = c.Context(0)
    ctx.set_timing(True)
    out = []

    def rec(size, what, wall, dev, **kw):
        r = dict(store_triples=size, what=what, wall_ms=round(wall, 3), device_ms=None if dev is None else round(dev, 3), gpu=name,
                 power_limit=power, **kw)
        print(json.dumps(r), flush=True)
        out.append(r)

    for size in (int(x) for x in a.sizes.split(",")):
        d = datagen.employee_dataset(size // 6)
        n = len(d.s)
        ctx.store_load(d.s, d.p, d.o)
        ctx.dict_numeric_load(d.num_or0, d.is_num)
        ctx.build_index()
        big = int(max(d.s.max(), d.o.max())) + 1
        one = (np.array([big], np.uint32), np.array([d.p[0]], np.uint32), np.array([big], np.uint32))
        ctx.store_insert(*one)  # warm-up of every shape
        ctx.store_remove(*one)
        ins, rem = [], []
        for _ in range(a.reps):
            ins.append(timed(ctx, lambda: ctx.store_insert(*one), 1))
            rem.append(timed(ctx, lambda: ctx.store_remove(*one), 1))
        rec(n, "one-triple insert (new triple, a segment of its own)", *np.median(np.array(ins), axis=0).tolist())
        rec(n, "one-triple remove of the triple just inserted (its small segment is compacted)", *np.median(np.array(rem), axis=0).tolist())
        # a loaded triple: its segment is the whole loaded store, which the remove compacts and re-indexes
        rng = np.random.default_rng(5)
        walls, devs = [], []
        for j in rng.choice(n, a.reps, replace=False):
            w, dv = timed(ctx, lambda: ctx.store_remove(d.s[j:j + 1], d.p[j:j + 1], d.o[j:j + 1]), 1)
            walls.append(w)
            devs.append(dv)
        rec(n, "one-triple remove of a loaded triple (the loaded segment is compacted and re-indexed)", float(np.median(walls)), float(np.median(devs)))
        m = 1_000_000
        bs = np.arange(big, big + m, dtype=np.uint32)
        bp = np.full(m, d.p[0], np.uint32)
        w, dv = timed(ctx, lambda: ctx.store_insert(bs, bp, bs, tag=1), 1)
        rec(n, "1e6-triple batch insert", w, dv)
        ctx.store_remove(bs, bp, bs)
        # reload + index rebuild: the same change made by uploading the whole store again
        w, _ = timed(ctx, lambda: (ctx.store_load(d.s, d.p, d.o), ctx.build_index()), 2)
        rec(n, "baseline: store_load + build_index", w, None, note="device time not recorded: the 12 B/triple host-to-device copy is not a timed kernel")
        # DELETE { ?s P ?o } WHERE { ?s P ?o } for a predicate the cfg2 star below does not read (it then shows that the index path
        # is still taken after the writes)
        js, pats, filt = datagen.employee_queries(d)["cfg2"]
        P = int(sorted(set(np.unique(d.p).tolist()) - {pt.p.value for pt in pats})[0])
        rel = ctx.scan([c.pattern(c.V(0), c.K(P), c.V(1))])[0]
        rows = rel.to_numpy([0, 1])
        rel.free()
        # the WHERE's rows as one kb_store_remove batch (kb_store_remove_template fills the same batch on the device, but needs the
        # dictionary strings this generated store has none of)
        bp = np.full(len(rows), P, np.uint32)
        ctx.get_stats(reset=True)
        t0 = time.perf_counter()
        removed = int(ctx.store_remove(rows[:, 0], bp, rows[:, 1]).sum())
        wall = (time.perf_counter() - t0) * 1e3
        dev = ctx.get_stats()["total_ms"]
        n0 = ctx.get_stats()["index_joins"]
        ctx.star_join(js, pats, filt).free()
        rec(n, "DELETE of one predicate", wall, dev, api="kb_store_remove of the WHERE's rows (downloaded before the timed call)", removed=removed,
            left=ctx.store_size()[0], star_join_on_index_after=ctx.get_stats()["index_joins"] > n0)
        ctx.store_clear()
    with open(a.out, "a") as f:
        for r in out:
            f.write(json.dumps(r) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
