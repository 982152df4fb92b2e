"""RDF-star quoted-triple scan: the device path (kb_scan_quoted) against the path it replaces, on the same seeded data.

Workload: the cfg2 employee store (1,666,667 employees = 10,000,002 triples) plus one annotation per salary triple,
`<< e ds:annual_salary s >> ex:source src_k` (datagen.annotated_salary_dataset: 1,666,667 quoted triples and as many annotation
triples), and the query

    << ?e ds:annual_salary ?s >> ex:source ?src  FILTER(?s > 100000)

Two arms, alternated in one process, each with the store index on and off:

  (a) device: kb_scan_quoted (one match pass over the quoted-triple table + the bind join), kb_filter, kb_rel_decode of the three
      result columns and their download
  (b) host:   what ran before kb_scan_quoted existed — ExecutionEngine._scan_quoted's Python loop over every table entry, the matches
      uploaded with kb_rel_from_host, kb_scan of the outer pattern, kb_hash_join, kb_filter, then the result columns downloaded and
      decoded on the host

Before anything is timed, both arms must return the same bag (row count and order-independent digest), equal to the closed form.
Prints one JSON line per (arm, index) and writes them to --out when given: median wall ms per query (host clock around work that ends
in a download), and for (a) the match kernel's device time (kb_stats.scan_ms over a scan_quoted call with the index on counts the match
launch alone; with the index off it includes the store scan of the bind join) with its algorithmic bytes 12*Q (the table) + 4*(1+v)*M
(entry id + v inner variables per match) over that time, against 3.35 TB/s (H100 SXM HBM3). The card name and power limit are read in
the same run."""
import argparse
import json
import os
import subprocess
import sys
import time
import types

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--employees", type=int, default=1_666_667)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch

    from kolibrie_b200 import capi as c
    from kolibrie_b200 import datagen
    from kolibrie_b200 import engine as E

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    data = datagen.annotated_salary_dataset(a.employees)
    want = datagen.row_checksums(datagen.annotated_salary_answer(data))
    strings = ["http://example.org/t%d" % i for i in range(data.n_ids)]
    ctx = c.Context(0)
    ctx.store_load(data.s, data.p, data.o)
    ctx.dict_numeric_load(data.num_or0, data.is_num)
    ctx.dict_strings_load(strings)
    ctx.quoted_load(data.qt_ids, data.qt_s, data.qt_p, data.qt_o)
    qts = E.QuotedTripleStore()  # the host mirror arm (b) walks
    qts.id_to_components = dict(zip(data.qt_ids.tolist(), zip(data.qt_s.tolist(), data.qt_p.tolist(), data.qt_o.tolist())))
    host_db = types.SimpleNamespace(ctx=ctx, quoted_triple_store=qts)
    pattern = (E.QuotedTriple(E.Variable("?e"), E.Constant(data.d.ids["ds:annual_salary"]), E.Variable("?s")), E.Constant(data.source),
               E.Variable("?src"))
    ctx.set_timing(True)

    def query(arm):
        slots = E.SlotMap()
        ctx.synchronize()
        ctx.get_stats(reset=True)
        t0 = time.perf_counter()
        if arm == "device":
            rel = ctx.scan_quoted(slots.quoted_pattern(pattern))
        else:
            rel = E.ExecutionEngine._scan_quoted(pattern, host_db, slots)
        st = ctx.get_stats()
        f = ctx.filter(rel, [c.fop(c.F_CMP_NUM, slot=slots.of("s"), cmp=c.CMP_GT, value=100000.0)])
        n, rs = f.info()
        if arm == "device":
            cols = [f.decode_strings(i) for i in range(len(rs))]
        else:
            cols = [[strings[x] if x < len(strings) else "unknown" for x in f.column(i).tolist()] for i in range(len(rs))]
        ms = (time.perf_counter() - t0) * 1e3
        order = [slots.of(v) for v in ("e", "s", "src")]
        return ms, st, rel.n_rows, n, f, order, len(cols[0]) if cols else 0

    lines = []
    for use_index in (True, False):
        ctx.set_use_index(use_index)
        if use_index:
            ctx.build_index()
        for arm in ("device", "host"):  # both arms return the closed-form bag before anything is timed
            _, _, _, n, f, order, _ = query(arm)
            got = datagen.row_checksums(f.to_numpy(order))
            assert got == want, (arm, use_index, got, want)
        rec = {"device": [], "host": []}
        for r in range(a.reps):
            for arm in (("device", "host") if r % 2 == 0 else ("host", "device")):
                ms, st, matched, n, f, order, nd = query(arm)
                assert n == want[0] and nd == n
                rec[arm].append((ms, st["scan_ms"], matched))
        Q, M, v = len(data.qt_ids), len(data.qt_ids), 2
        alg = 12 * Q + 4 * (1 + v) * M
        for arm in ("device", "host"):
            ms = float(np.median([x[0] for x in rec[arm]]))
            line = {"arm": arm, "index": use_index, "ms_per_query": ms, "reps": a.reps, "rows_matched": int(rec[arm][0][2]),
                    "rows_out": int(want[0]), "digest": [int(x) for x in want[1:]], "quoted_triples": Q,
                    "store_triples": int(len(data.s))}
            if arm == "device":
                scan_ms = float(np.median([x[1] for x in rec[arm]]))
                line.update(scan_family_device_ms=scan_ms, match_alg_bytes=alg)
                if use_index:  # the scan family holds the match launch alone
                    line.update(match_gb_per_s=alg / (scan_ms * 1e-3) / 1e9, match_share_of_hbm=alg / (scan_ms * 1e-3) / HBM_BYTES_PER_S)
            lines.append(line)
    name, power = card()
    for line in lines:
        line.update(card=name, power_limit=power,
                    what="<< ?e ds:annual_salary ?s >> ex:source ?src FILTER(?s > 100000): " +
                         ("kb_scan_quoted + kb_filter + kb_rel_decode" if line["arm"] == "device" else
                          "host _scan_quoted + kb_rel_from_host + kb_scan + kb_hash_join + kb_filter + host decode"))
        print(json.dumps(line))
    if a.out:
        with open(a.out, "w") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
