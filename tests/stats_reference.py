"""DatabaseStats::gather_stats_fast (kolibrie/src/streamertail_optimizer/stats/database_stats.rs:43-105), restated for the tests.

`gather_stats_fast` is the reference's loop transcribed line by line, with the sample size 100 000 made a parameter `max_sample`
(0: every triple). `gather_stats_numpy` computes the same thing with array operations, for stores too large for the loop. Both take
the triples as a set (or any iterable, repeats collapse as in the BTreeSet) and the quoted-triple store's length.
"""
import numpy as np

FAST = 100_000  # database_stats.rs:50


class Stats:
    def __init__(self, total_triples, quoted_triple_count, take, step, subject, predicate, obj):
        self.total_triples = total_triples
        self.quoted_triple_count = quoted_triple_count
        self.take = take
        self.step = step
        self.subject = subject      # {id: count}
        self.predicate = predicate
        self.object = obj

    def maps(self):
        return self.subject, self.predicate, self.object


def gather_stats_fast(triples, quoted_count=0, max_sample=FAST):
    triples_vec = sorted(set((int(s), int(p), int(o)) for s, p, o in triples))  # database.triples.iter(): BTreeSet order
    total_triples = len(triples_vec)
    sample_size = min(total_triples, max_sample) if max_sample else total_triples
    step = total_triples // sample_size if total_triples > sample_size else 1
    sampled = triples_vec[::step][:sample_size]  # .iter().step_by(step).take(sample_size)
    pred, subj, obj = {}, {}, {}
    for s, p, o in sampled:
        pred[p] = pred.get(p, 0) + 1
        subj[s] = subj.get(s, 0) + 1
        obj[o] = obj.get(o, 0) + 1
    scale = step if step > 1 else 1
    for m in (pred, subj, obj):
        for k in m:
            m[k] *= scale
    return Stats(total_triples, quoted_count, sample_size, step, subj, pred, obj)


def sample_plan(total, max_sample=FAST):
    """(take, step) for T = total"""
    take = min(total, max_sample) if max_sample else total
    return take, (total // take if total > take else 1)


def distinct_sorted(rows):
    """the distinct rows of an (n, 3) array in ascending (s, p, o) order: the BTreeSet's iteration"""
    rows = np.asarray(rows, dtype=np.uint32).reshape(-1, 3)
    sp = rows[:, 0].astype(np.uint64) << np.uint64(32) | rows[:, 1].astype(np.uint64)
    srt = rows[np.lexsort((rows[:, 2], sp))]
    if len(srt):
        keep = np.ones(len(srt), bool)
        keep[1:] = np.any(srt[1:] != srt[:-1], axis=1)
        srt = srt[keep]
    return srt


def gather_stats_numpy(rows, quoted_count=0, max_sample=FAST):
    """the same statistics from an (n, 3) array of (s, p, o) rows, repeats allowed; the maps as (ids ascending, counts) array pairs"""
    srt = distinct_sorted(rows)
    total = len(srt)
    take, step = sample_plan(total, max_sample)
    smp = srt[: take * step: step]
    out = []
    for j in range(3):
        ids, counts = np.unique(smp[:, j], return_counts=True)
        out.append((ids.astype(np.uint32), counts.astype(np.uint64) * np.uint64(step)))
    return {"total_triples": total, "quoted_triple_count": quoted_count, "take": take, "step": step,
            "subject": out[0], "predicate": out[1], "object": out[2]}


def as_arrays(m):
    """{id: count} -> (ids ascending uint32, counts uint64)"""
    ks = sorted(m)
    return np.array(ks, dtype=np.uint32), np.array([m[k] for k in ks], dtype=np.uint64)
