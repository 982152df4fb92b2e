"""SparqlDatabase::union and par_join on the device (kb_store_union / kb_store_par_join) at full size: the union of two cfg2 stores
(employee_dataset(1_666_667) with seeds 42 and 45: the same subjects, other titles and salaries; 10 M triples and 1.79 M terms each) and
the par_join of the cfg4 store (taxonomy_dataset(), 50 M triples) with itself on rdfs:subClassOf. Per workload the device time of each
phase and the wall time of the call, medians over --reps repetitions that alternate with the baseline arm: a numpy host restatement of
the same result (not the reference's Rust, which is not run here). Algorithmic bytes come from the shapes (the model is in
union_bytes / par_join_bytes). One JSON record per workload to --out, each with the card's name and power limit read in the same run.
Run: python scripts/union_bench.py --out profiles/union.jsonl"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kolibrie_b200 import capi as c  # noqa: E402
from kolibrie_b200 import datagen  # noqa: E402

UNION_PHASES = ("sets", "terms", "dictionary", "remap", "union")
PAR_JOIN_PHASES = ("selection", "pairs", "joins", "sort")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return name, power


def np_set(t):
    """the distinct rows of an (n, 3) uint32 array in (s, p, o) order (packed into one u64 key when the ids' bits fit)"""
    t = np.asarray(t, dtype=np.uint64).reshape(-1, 3)
    if not len(t):
        return t.astype(np.uint32)
    bits = [max(int(t[:, k].max()).bit_length(), 1) for k in range(3)]
    if sum(bits) <= 64:
        key = (t[:, 0] << np.uint64(bits[1] + bits[2])) | (t[:, 1] << np.uint64(bits[2])) | t[:, 2]
        u = np.sort(key)
        u = u[np.concatenate(([True], u[1:] != u[:-1]))]
        m1, m2 = np.uint64((1 << bits[1]) - 1), np.uint64((1 << bits[2]) - 1)
        return np.stack([u >> np.uint64(bits[1] + bits[2]), (u >> np.uint64(bits[2])) & m1, u & m2], 1).astype(np.uint32)
    t = t[np.lexsort((t[:, 2], t[:, 1], t[:, 0]))]
    keep = np.ones(len(t), bool)
    keep[1:] = (t[1:] != t[:-1]).any(axis=1)
    return t[keep].astype(np.uint32)


def np_union(a_rows, sa, a_index, b_rows, sb):
    """the host restatement of union: b's set, its terms in first-seen order, their ids in a's dictionary or the next ones, the set union"""
    bset = np_set(b_rows)
    seq = bset.reshape(-1)
    order = np.argsort(seq, kind="stable")
    ss = seq[order]
    terms = seq[np.sort(order[np.concatenate(([True], ss[1:] != ss[:-1]))])]  # distinct ids by first position
    new_id = np.empty(len(terms), np.uint32)
    nxt = len(sa)
    for k, t in enumerate(terms.tolist()):
        i = a_index.get(sb[t])
        if i is None:
            i, nxt = nxt, nxt + 1
        new_id[k] = i
    remap = np.zeros(len(sb), np.uint32)
    remap[terms] = new_id
    return np_set(np.concatenate([np_set(a_rows), remap[bset]]))


def np_par_join(rows, pid):
    """the host restatement of par_join(x, x, p): the join a.o = b.s and the rows of A whose object is an object of A, as a set"""
    A = np_set(rows[rows[:, 1] == pid])
    order = np.argsort(A[:, 0], kind="stable")
    bs, bo = A[order, 0], A[order, 2]
    lo, hi = np.searchsorted(bs, A[:, 2], "left"), np.searchsorted(bs, A[:, 2], "right")
    cnt = hi - lo
    li = np.repeat(np.arange(len(A)), cnt)
    ri = np.concatenate([np.arange(l, h) for l, h in zip(lo[cnt > 0], hi[cnt > 0])]) if cnt.any() else np.empty(0, np.int64)
    joined = np.stack([A[li, 0], np.full(len(li), pid, np.uint32), bo[ri]], 1)
    semi = A[np.isin(A[:, 2], A[:, 2])]
    return np_set(np.concatenate([joined, semi]))


def union_bytes(na_raw, nb_raw, na, nb, d, b_ids, a_ids, a_bytes, term_bytes, n_rows):
    """per phase, the bytes the phase must move at least: rows are 12 B (4 B per id), offsets 8 B, strings their bytes"""
    return {"sets": 12 * (na_raw + nb_raw) + 12 * (na + nb),
            "terms": 2 * 12 * nb + 4 * b_ids + 4 * d,
            "dictionary": 4 * d + 2 * term_bytes + 8 * (a_ids + 1) + a_bytes,
            "remap": 4 * d + 12 * nb + 12 * nb,
            "union": 12 * (na + nb) + 12 * n_rows}


def par_join_bytes(na_raw, nb_raw, n_sel_a, n_sel_b, n_join, n_semi, n_rows):
    return {"selection": 12 * (na_raw + nb_raw) + 8 * (n_sel_a + n_sel_b),
            "pairs": 8 * (n_sel_a + 2 * n_sel_b) + 8 * (n_sel_a + 2 * n_sel_b),
            "joins": 8 * (n_sel_a + n_sel_b) + 8 * (n_join + n_semi),
            "sort": 12 * (n_join + n_semi) + 12 * n_rows}


def medians(infos, walls, names):
    return {"phase_ms": {k: float(np.median([i["phase_ms"][j] for i in infos])) for j, k in enumerate(names)},
            "wall_ms": 1e3 * float(np.median(walls))}


def run_union(reps, emit, name, power):
    da, db_ = datagen.employee_dataset(1_666_667, seed=42), datagen.employee_dataset(1_666_667, seed=45)
    sa, sb = datagen.employee_strings(da), datagen.employee_strings(db_)
    a, b, dst = c.Context(0), c.Context(0), c.Context(0)
    a.store_load(da.s, da.p, da.o)
    a.dict_strings_load(sa)
    b.store_load(db_.s, db_.p, db_.o)
    b.dict_strings_load(sb)
    a_rows, b_rows = np.stack([da.s, da.p, da.o], 1), np.stack([db_.s, db_.p, db_.o], 1)
    t0 = time.perf_counter()
    a_index = {s: i for i, s in enumerate(sa)}
    index_s = time.perf_counter() - t0
    dst.store_union(a, b)  # warm-up
    infos, walls, host = [], [], []
    for _ in range(reps):  # the two arms alternate
        t0 = time.perf_counter()
        infos.append(dst.store_union(a, b))
        walls.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        want = np_union(a_rows, sa, a_index, b_rows, sb)
        host.append(time.perf_counter() - t0)
    got = np.stack(dst.store_download(), 1)
    assert len(got) == len(want) and np.array_equal(got, want), "device union differs from the host restatement"
    inf = infos[-1]
    enc = lambda xs: sum(len(x.encode()) for x in xs)
    n_dev, _ = dst.dict_strings_info()
    term_bytes = enc(sb)  # every string of b is one of its terms here
    model = union_bytes(len(da.s), len(db_.s), inf["n_a"], inf["n_b"], inf["n_terms"], len(sb), len(sa), enc(sa), term_bytes, inf["n_rows"])
    rec = {"workload": "union(cfg2 seed 42, cfg2 seed 45)", "card": name, "power_limit": power, "reps": reps,
           "a_triples": len(da.s), "b_triples": len(db_.s), "a_terms": len(sa), "b_terms": inf["n_terms"], "rows": inf["n_rows"],
           "dict_new": inf["dict_new"], "dict_after": n_dev, **medians(infos, walls, UNION_PHASES),
           "algorithmic_bytes": model, "host_restatement": {"what": "numpy restatement (not the reference's Rust)", "median_ms": 1e3 * float(np.median(host)),
                                                            "dictionary_index_ms": 1e3 * index_s}}
    rec["gbps"] = {k: (model[k] / (rec["phase_ms"][k] * 1e-3) / 1e9 if rec["phase_ms"][k] > 0 else None) for k in UNION_PHASES}
    emit(rec)
    for x in (a, b, dst):
        x.close()


def run_par_join(reps, emit, name, power):
    t = datagen.taxonomy_dataset()
    sc = t.ids["rdfs:subClassOf"]
    a, dst = c.Context(0), c.Context(0)
    a.store_load(t.s, t.p, t.o)
    a.dict_strings_load(["rdfs:subClassOf", "rdf:type"])
    rows = np.stack([t.s, t.p, t.o], 1)
    dst.store_par_join(a, a, sc)  # warm-up
    infos, walls, host = [], [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        infos.append(dst.store_par_join(a, a, sc))
        walls.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        want = np_par_join(rows, sc)
        host.append(time.perf_counter() - t0)
    got = np.stack(dst.store_download(), 1)
    assert len(got) == len(want) and np.array_equal(got, want), "device par_join differs from the host restatement"
    inf = infos[-1]
    model = par_join_bytes(len(t.s), len(t.s), inf["n_a"], inf["n_b"], inf["n_join"], inf["n_semi"], inf["n_rows"])
    rec = {"workload": "par_join(cfg4, cfg4, rdfs:subClassOf)", "card": name, "power_limit": power, "reps": reps, "triples": len(t.s),
           "predicate_rows": inf["n_a"], "join_rows": inf["n_join"], "semi_rows": inf["n_semi"], "rows": inf["n_rows"],
           **medians(infos, walls, PAR_JOIN_PHASES), "algorithmic_bytes": model,
           "host_restatement": {"what": "numpy restatement (not the reference's Rust)", "median_ms": 1e3 * float(np.median(host))}}
    rec["gbps"] = {k: (model[k] / (rec["phase_ms"][k] * 1e-3) / 1e9 if rec["phase_ms"][k] > 0 else None) for k in PAR_JOIN_PHASES}
    emit(rec)
    for x in (a, dst):
        x.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/union.jsonl")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    with open(args.out, "w") as f:
        def emit(rec):
            line = json.dumps(rec)
            print(line, flush=True)
            f.write(line + "\n")

        run_union(args.reps, emit, name, power)
        run_par_join(args.reps, emit, name, power)


if __name__ == "__main__":
    main()
