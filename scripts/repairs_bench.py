"""Inconsistency-tolerant queries (kb_datalog_query_repairs) on the config-4 shape: datagen.taxonomy_dataset (a 10-ary class tree of
depth 6, 48.9 M `x rdf:type C` facts) plus a seeded second leaf type for 1 % of the instances (datagen.taxonomy_conflicts), closed by
kb_datalog_fixpoint, plus `disjointWith` between every ordered pair of the ten level-1 classes.
Runs: (i) the constraint (?x type ?a), (?x type ?b), (?a disjointWith ?b): every conflict has three facts, so no subset probe runs;
(ii) the same plus the constraint (?x type C_k) for one level-1 class: conflicts of one and three facts, so the probe runs at scale.
Queries: (x_j type ?C) for a conflicted and for a free x_j, and (?x type C_k).
The only baseline is the Python transcription of compute_repairs + query_with_repairs (tests/repairs_reference.py, Python, not the
reference's Rust) on the largest small store it finishes within a budget; no speed-up is claimed. Writes one JSON line per measurement
to profiles/repairs.jsonl (or --out), with the card's name and power limit read in the same run. Device times: kb_repair_stats (CUDA
events around the whole call and its three phases); wall: host clock around the call, which returns after its stream synchronises."""
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


def transcription_baseline(budget_s):
    """the Python transcription (a) on stores of 4, 6, 8, ... facts with one two-fact conflict, until one takes longer than budget_s"""
    import tests.repairs_reference as R
    out = []
    for n in range(4, 40, 2):
        facts = [(1, 10, k) for k in range(n)]
        cons = [[(1, 10, 0), (1, 10, 1)]]
        t0 = time.perf_counter()
        got, kept = R.transcribe(facts, cons, ("?S", 10, "?O"), facts)
        ms = (time.perf_counter() - t0) * 1e3
        out.append({"route": "Python transcription of compute_repairs (tests/repairs_reference.py), host CPU", "facts": n,
                    "wall_ms": ms, "kept_sets": len(kept), "answers": len(got)})
        if ms > budget_s * 1e3:
            break
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=48_888_890)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--baseline-budget-s", type=float, default=5.0)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "repairs.jsonl"))
    a = ap.parse_args()
    name, power = card()
    t = datagen.taxonomy_dataset(n_instances=a.instances)
    extra, dw, lv1 = datagen.taxonomy_conflicts(t)
    ty = t.ids["rdf:type"]
    x0 = 2 + t.n_classes
    k = int(lv1[3])
    ctx = c.Context(0)
    ctx.store_load(np.concatenate([t.s, extra[0]]), np.concatenate([t.p, extra[1]]), np.concatenate([t.o, extra[2]]))
    ctx.datalog_fixpoint(datagen.taxonomy_rules(t))
    ctx.build_index()
    body = {"premise": [c.pattern(c.V(0), c.K(ty), c.V(1)), c.pattern(c.V(0), c.K(ty), c.V(2)), c.pattern(c.V(1), c.K(dw), c.V(2))]}
    only_k = {"premise": [c.pattern(c.V(0), c.K(ty), c.K(k))]}
    second = extra[0][extra[1] == ty]
    conflicted = int(second[0])  # (not every instance with a second leaf is conflicted: both leaves can share a level-1 class)
    free = x0 + a.instances // 2
    while free in set(second.tolist()):
        free += 1
    queries = {"(x_conflicted type ?C)": c.pattern(c.K(conflicted), c.K(ty), c.V(9)),
               "(x_free type ?C)": c.pattern(c.K(free), c.K(ty), c.V(9)),
               "(?x type C_k)": c.pattern(c.V(9), c.K(ty), c.K(k))}
    out = []
    base = {"card": name, "power_limit": power, "store_triples": int(ctx.store_size()[0]), "instances": a.instances}
    for run, cons in (("(i) disjointness", [body]), ("(ii) disjointness + (?x type C_k)", [body, only_k])):
        for label, q in queries.items():
            ctx.datalog_query_repairs(cons, q)[0].free()  # warm-up
            walls, sts = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                rel, st = ctx.datalog_query_repairs(cons, q)
                walls.append((time.perf_counter() - t0) * 1e3)
                sts.append(st.as_dict())
                rel.free()
            med = {n: float(np.median([s[n] for s in sts])) for n in ("device_ms", "match_ms", "conflict_ms", "answer_ms")}
            last = sts[-1]
            out.append(dict(base, route="kb_datalog_query_repairs", run=run, query=label, wall_ms=float(np.median(walls)), **med,
                            **{n: int(last[n]) for n in ("constraints", "subsets_probed", "matches", "conflicts", "minimal_conflicts",
                                                         "conflicted_facts", "answers")}))
            print(json.dumps(out[-1]), flush=True)
    ctx.close()
    out += transcription_baseline(a.baseline_budget_s)
    with open(a.out, "w") as f:
        for line in out:
            f.write(json.dumps(line) + "\n")
    for line in out[-3:]:
        print(json.dumps(line))


if __name__ == "__main__":
    main()
