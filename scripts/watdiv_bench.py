"""The 20 WatDiv-shaped queries (tests/golden/watdiv/queries.json) through kb_bgp_execute on a datagen.watdiv store with the store
index built, as the reference's harness runs them (n_triple_10M.rs:572-589): per query 3 warm-up runs, then the median of 20.
Per query it records the device time (kb_stats with timing on), the wall time of the call, the rows, the route, the reduction's
rounds, modelled bytes and bandwidth (kb_bgp_last_plan), and — with --parent DIR, a build of another checkout — the same call
through that checkout's library, alternating with this one run by run; a query the other library refuses is listed with its status.
The card's name and power limit are read in the same run and written with the results.

The store is WatDiv-SHAPED (datagen.watdiv), not WatDiv: these times are not comparable with the reference's WatDiv latencies.

  python scripts/watdiv_bench.py --triples 10000000 --out profiles/watdiv_10m.jsonl [--parent DIR]"""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kolibrie_b200 import capi as c  # noqa: E402
from kolibrie_b200 import datagen  # noqa: E402
from tests import watdiv_cases as W  # noqa: E402


def load_capi(tree):
    """the capi module of another checkout, bound to that checkout's library"""
    spec = importlib.util.spec_from_file_location("capi_other", os.path.join(tree, "kolibrie_b200", "capi.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def compile_for(api, d, q):
    """the query's patterns in `api`'s own structure types (?vN is slot N)"""
    term = lambda t: api.V(int(t[2:])) if t.startswith("?") else api.K(d.ids[t])
    return [api.pattern(*(term(t) for t in p)) for p in q["patterns"]], [int(v[2:]) for v in q["select"]]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().split("\n")[0]


def one(api, ctx, pats, project):
    """(wall ms, device ms, rows) of one call, or the status it returned"""
    ctx.get_stats(reset=True)
    t0 = time.perf_counter()
    try:
        r = ctx.bgp_execute(pats, None, project)
    except api.KolibrieError as e:
        return e.status
    ctx.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    st = ctx.get_stats()
    n = r.n_rows
    r.free()
    return wall, st["total_ms"], n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--triples", type=int, default=10_000_000)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--parent", default="", help="another checkout whose built library runs the same calls, alternating")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "watdiv_10m.jsonl"))
    args = ap.parse_args()
    d = datagen.watdiv(args.triples)
    arms = [("branch", c)] + ([("parent", load_capi(args.parent))] if args.parent else [])
    ctxs = {}
    for name, api in arms:
        ctx = api.Context(0)
        ctx.store_load(d.s, d.p, d.o)
        ctx.build_index()
        ctx.set_timing(True)
        ctxs[name] = ctx
    gpu = card()
    lines = [{"workload": f"datagen.watdiv({args.triples}): {len(d.s)} triples, WatDiv-shaped (not WatDiv data), store index built",
              "gpu": gpu, "warmup": args.warmup, "iters": args.iters}]
    for q in W.QUERIES:
        per_arm = {name: compile_for(api, d, q) for name, api in arms}
        pats, project = per_arm["branch"]
        rec = {"query": q["name"], "patterns": len(pats)}
        runs = {name: [] for name, _ in arms}
        for it in range(args.warmup + args.iters):
            for name, api in (arms if it % 2 == 0 else arms[::-1]):
                got = one(api, ctxs[name], *per_arm[name])
                if isinstance(got, int):
                    runs[name] = got
                elif isinstance(runs[name], list) and it >= args.warmup:
                    runs[name].append(got)
        for name, _ in arms:
            if isinstance(runs[name], int):
                rec[name] = {"status": runs[name]}
                continue
            rec[name] = {"wall_ms": statistics.median(x[0] for x in runs[name]), "device_ms": statistics.median(x[1] for x in runs[name]),
                         "rows": runs[name][0][2]}
        plan = ctxs["branch"].bgp_last_plan()
        rec["route"] = {c.BGP_STAR: "star", c.BGP_COMPONENTS: "components"}[plan["route"]]
        if plan["route"] == c.BGP_COMPONENTS:
            rec["reduce_rounds"] = plan["reduce_rounds"]
            rec["reduce_bytes"] = plan["reduce_bytes"]
            rec["reduce_bit_ops"] = plan["reduce_bit_ops"]
            rec["max_intermediate"] = plan["max_intermediate"]
            rec["rows_scanned"], rec["rows_reduced"] = plan["rows_scanned"], plan["rows_reduced"]
            f = ctxs["branch"]
            f.get_stats(reset=True)
            r = f.bgp_execute(pats, None, project)
            r.free()
            st = f.get_stats()
            if st["filter_ms"] > 0:  # the reduction's kernels are the `filter` family of this call
                rec["reduce_ms"] = st["filter_ms"]
                rec["reduce_GBps"] = plan["reduce_bytes"] / st["filter_ms"] / 1e6
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")
    for ctx in ctxs.values():
        ctx.close()


if __name__ == "__main__":
    main()
