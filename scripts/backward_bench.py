"""Backward-chaining queries (kb_datalog_query) on the config-4 shape (datagen.taxonomy_dataset: a 10-ary class tree of depth 6 and
48.9 M `x rdf:type C` facts, rules R1/R2), next to the forward route a user has without it: evict the inferred facts, run
kb_datalog_fixpoint and scan the answer. Queries: (x_j type ?C), (?x type C_k), and a ground (x_j type C) that holds. Also the Python
SLD restatement (tests/bc_reference.py, Python, not the reference's Rust) on a small store. Writes one JSON line per measurement to
profiles/backward.jsonl (or --out), with the card's name and power limit read in the same run. Device time: kb_bc_stats.device_ms
(CUDA events around the whole call); wall: host clock around the call, which returns after its stream synchronises."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=48_888_890)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "backward.jsonl"))
    a = ap.parse_args()
    name, power = card()
    t = datagen.taxonomy_dataset(n_instances=a.instances)
    rules = datagen.taxonomy_rules(t)
    ty = t.ids["rdf:type"]
    x0 = 2 + t.n_classes
    j = a.instances // 2
    ctx = c.Context(0)
    ctx.store_load(t.s, t.p, t.o)
    leaf = 2 + t.n_classes - 1
    queries = {
        "(x_j type ?C)": c.pattern(c.K(x0 + j), c.K(ty), c.V(9)),
        "(?x type C_k)": c.pattern(c.V(9), c.K(ty), c.K(2)),  # the root class: every instance
        "(?x type leaf)": c.pattern(c.V(9), c.K(ty), c.K(leaf)),
        "ground (x_j type root)": c.pattern(c.K(x0 + j), c.K(ty), c.K(2)),
    }
    out = []
    base = {"card": name, "power_limit": power, "triples": int(len(t.s)), "instances": a.instances}
    for label, q in queries.items():
        ctx.datalog_query(rules, q)  # warm-up
        walls, devs = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rel, st = ctx.datalog_query(rules, q)
            walls.append((time.perf_counter() - t0) * 1e3)
            devs.append(st.device_ms)
        out.append(dict(base, route="kb_datalog_query", query=label, wall_ms=float(np.median(walls)), device_ms=float(np.median(devs)),
                        rounds=st.rounds, stopped_early=st.stopped_early, base_facts=st.base_facts, derived=st.derived,
                        derivations=st.derivations, answers=st.answers))
        rel.free()
    # forward route: inferred facts evicted, closure, scan of the query (one closure answers every query; timed per query as a user pays it)
    for label, q in queries.items():
        walls = []
        for _ in range(a.reps):
            ctx.store_load(t.s, t.p, t.o)
            t0 = time.perf_counter()
            _, st = ctx.datalog_fixpoint(rules)
            r = ctx.scan([q])[0]
            n = r.n_rows
            walls.append((time.perf_counter() - t0) * 1e3)
        out.append(dict(base, route="kb_datalog_fixpoint + kb_scan", query=label, wall_ms=float(np.median(walls)),
                        device_ms=float(st.device_ms), rounds=st.rounds, derived=int(st.inferred), answers=int(n)))
    ctx.close()
    # the Python SLD restatement on a small store (a 3-ary tree of depth 3, 200 instances)
    from kolibrie_b200.engine import Constant, Variable
    import tests.bc_reference as B
    s = datagen.taxonomy_dataset(fanout=3, depth=3, n_instances=200)
    facts = list(zip(s.s.tolist(), s.p.tolist(), s.o.tolist()))
    A, Bv, Cv, X = Variable("a"), Variable("b"), Variable("c"), Variable("x")
    sc, tyc = Constant(0), Constant(1)
    prules = [([(A, sc, Bv), (Bv, sc, Cv)], [(A, sc, Cv)]), ([(X, tyc, A), (A, sc, Bv)], [(X, tyc, Bv)])]
    q = (Constant(2 + s.n_classes), tyc, Variable("C"))
    t0 = time.perf_counter()
    try:
        got = B.project_sld(B.sld(facts, prules, q, B.MAX_DEPTH, budget=200_000), q)
        status = "ok"
    except B.BudgetExceeded:
        got, status = set(), "budget of 2e5 calls exceeded"
    out.append({"route": "Python SLD restatement (tests/bc_reference.py), host CPU", "query": "(x_0 type ?C), depth 10", "triples": len(facts),
                "wall_ms": (time.perf_counter() - t0) * 1e3, "answers": len(got), "status": status})
    with open(a.out, "w") as f:
        for line in out:
            f.write(json.dumps(line) + "\n")
            print(json.dumps(line))


if __name__ == "__main__":
    main()
