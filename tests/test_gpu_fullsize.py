"""GPU (-m gpu): the BASELINE.json sizes themselves. Results this large are judged through size-independent properties
(SURVEY.md §8d "parity check at scale"): closed-form row counts and CONTENT digests computed from the generator, agreement of the
three product paths (index, scan, one-shot host call), idempotence, additivity over a partition of the subjects, and a full
row-by-row comparison with the oracle on a 1 % subject slice."""
import numpy as np
import pytest

from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from tests import helpers as H
from tests import oracle_api as O

pytestmark = pytest.mark.gpu

E_FULL = 16_666_667  # 100 000 002 triples (BASELINE configs 2/3)
M64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def full():
    d = datagen.employee_dataset(E_FULL)
    cx = c.Context(0)
    cx.dict_numeric_load(d.num_or0, d.is_num)
    cx.store_load(d.s, d.p, d.o)
    yield d, cx
    cx.close()


def digest(rel, order):
    return datagen.row_checksums(rel.to_numpy(order))


def test_cfg2_full_size_properties(full):
    d, cx = full
    js, pats, filt = datagen.employee_queries(d)["cfg2"]  # slots: e, t, s, n
    ids = d.ids
    subj = d.s[d.p == ids["foaf:name"]]
    title = d.o[d.p == ids["foaf:title"]]
    sal = d.o[d.p == ids["ds:annual_salary"]]
    assert len(subj) == len(title) == len(sal) == E_FULL
    keep = d.salary_of_employee > 100000
    # the answer in closed form, straight from the generator: (e, t, s, n = e) for every employee whose salary passes the FILTER
    expect = np.stack([subj[keep], title[keep], sal[keep], subj[keep]], axis=1)
    want = datagen.row_checksums(expect)
    assert want[0] == int(keep.sum()) == 6_945_872

    cx.set_use_index(False)
    r_scan = cx.star_join(js, pats, filt)
    order = sorted(r_scan.slots)
    assert order == [0, 1, 2, 3]
    assert digest(r_scan, order) == want, "scan path"
    cx.set_use_index(True)
    assert cx.build_index()[0] == 6
    before = cx.get_stats()["index_joins"]
    r_idx = cx.star_join(js, pats, filt)
    assert cx.get_stats()["index_joins"] == before + 1
    assert digest(r_idx, order) == want, "index path"
    assert digest(cx.star_join(js, pats, filt), order) == want, "idempotence"

    # the one-shot host call (kb_star_join_host) on the same host columns
    rows, slots = cx.star_join_host(d.s, d.p, d.o, js, pats, filt)
    assert datagen.row_checksums(rows[:, [slots.index(k) for k in order]]) == want, "host one-shot call"

    # row-by-row against the oracle on a 1 % slice of the subjects (a star join on the subject is local to the subject)
    lo, hi = 7_000_000, 7_000_000 + E_FULL // 100
    sub = slice(6 * lo, 6 * hi)
    odb = O.Db(d.s[sub], d.p[sub], d.o[sub], d.num_or0, d.is_num)
    owant = odb.bgp(pats, filt).to_numpy(order)
    got = r_idx.to_numpy(order)
    s_lo, s_hi = subj[lo], subj[hi - 1]
    assert (np.diff(subj[lo:hi].astype(np.int64)) > 0).all()
    H.assert_same_bag(got[(got[:, 0] >= s_lo) & (got[:, 0] <= s_hi)], owant, "1 % slice vs oracle")


def test_cfg2_additive_over_a_partition_of_the_subjects(full):
    """result(store) = result(first half of the employees) + result(second half): counts add, digests add mod 2^64 and xor"""
    d, cx = full
    js, pats, filt = datagen.employee_queries(d)["cfg2"]
    cx.set_use_index(True)
    cx.store_load(d.s, d.p, d.o)
    whole = digest(cx.star_join(js, pats, filt), [0, 1, 2, 3])
    cut = 6 * (E_FULL // 2)
    parts = []
    for sl in (slice(0, cut), slice(cut, None)):
        cx.store_load(d.s[sl], d.p[sl], d.o[sl])
        cx.build_index()
        parts.append(digest(cx.star_join(js, pats, filt), [0, 1, 2, 3]))
    assert whole[0] == parts[0][0] + parts[1][0]
    assert whole[1] == (parts[0][1] + parts[1][1]) & M64
    assert whole[2] == parts[0][2] ^ parts[1][2]
    cx.store_load(d.s, d.p, d.o)  # leave the module's store whole


def test_cfg3_group_by_full_size(full):
    d, cx = full
    js, pats, _ = datagen.employee_queries(d)["cfg3"]
    cx.store_load(d.s, d.p, d.o)
    cx.build_index()
    r = cx.star_join(js, pats)
    assert r.n_rows == E_FULL
    g = cx.group_aggregate(r, [1], [(c.AGG_COUNT, 0), (c.AGG_AVG, 2)])
    title_ids = np.array([d.ids[t] for t in ("Manager", "Developer", "Salesperson")], dtype=np.uint32)
    by_title = {int(k): (int(n), float(v)) for k, n, v in zip(g["keys"][0], g["counts"], g["values"][1])}
    assert sorted(by_title) == sorted(title_ids.tolist())
    for ti, tid in enumerate(title_ids.tolist()):
        m = d.title_of_employee == ti
        assert by_title[tid][0] == int(m.sum())
        # integer salaries: the sum is exact in f64 in any order (< 2^53), so AVG is the correctly rounded quotient, bit for bit
        assert by_title[tid][1] == int(d.salary_of_employee[m].astype(np.int64).sum()) / int(m.sum())


def test_cfg4_closure_full_size():
    """50 M triples -> 293 M inferred facts: closed-form counts per predicate, the reference's round structure, idempotence"""
    fan, depth, n_inst = 10, 6, 48_888_890
    t = datagen.taxonomy_dataset(fan, depth, n_inst, seed=43)
    rules = datagen.taxonomy_rules(t)
    cx = c.Context(0)
    try:
        cx.store_load(t.s, t.p, t.o)
        rel, st = cx.datalog_fixpoint(rules)
        lvl = np.zeros(t.n_classes, dtype=np.int64)
        start = 0
        for k in range(depth + 1):
            lvl[start:start + fan ** k] = k
            start += fan ** k
        cls = t.o[t.p == t.ids["rdf:type"]].astype(np.int64) - 2
        want_type = int(lvl[cls].sum())                                      # an instance of a depth-k class gains k types
        want_sc = sum(fan ** k * (k - 1) for k in range(2, depth + 1))      # a depth-k class gains k-1 proper ancestors
        assert st.inferred == want_type + want_sc == rel.n_rows
        pcol = rel.column(1)
        assert int((pcol == t.ids["rdf:type"]).sum()) == want_type and int((pcol == t.ids["rdfs:subClassOf"]).sum()) == want_sc
        assert st.rounds == 3 and sum(st.round_new[i] for i in range(st.rounds)) == st.inferred
        rel.free()
        rel2, st2 = cx.datalog_fixpoint(rules)  # the store now holds the closure: nothing new
        assert st2.inferred == 0 and st2.rounds == 0
    finally:
        cx.close()


def test_cfg2_permuted_dictionary_and_shuffled_store():
    """cfg2 on a store whose dictionary ids are a random permutation and whose triples come in random order (>= 10 M triples): the
    direct tables still apply (ids dense, predicates functional) and the answer — judged through the closed-form content digest of the
    generator, relabelled — must not depend on either order; scan path, index path (table-mode probe) and the slice-streaming probe agree"""
    E = 2_000_000  # 12 M triples
    d = datagen.employee_dataset(E)
    s, p, o, num, isn, pi = datagen.permuted_dataset(d)
    js, pats0, filt = datagen.employee_queries(d)["cfg2"]
    pats = [c.pattern(c.V(0), c.K(int(pi[pt.p.value])), c.V(v)) for pt, v in zip(pats0, (1, 2, 3))]
    ids = d.ids
    subj = d.s[0::6]
    keep = d.salary_of_employee > 100000
    expect = np.stack([pi[subj[keep]], pi[d.o[1::6][keep]], pi[d.o[5::6][keep]], pi[subj[keep]]], axis=1)
    want = datagen.row_checksums(expect)
    cx = c.Context(0)
    try:
        cx.dict_numeric_load(num, isn)
        cx.store_load(s, p, o)
        got = cx.star_join(js, pats, filt)
        assert datagen.row_checksums(got.to_numpy([0, 1, 2, 3])) == want, "scan path"
        assert cx.build_index()[0] == 6
        n0 = cx.get_stats()["index_joins"]
        got = cx.star_join(js, pats, filt)
        assert cx.get_stats()["index_joins"] == n0 + 1
        rows = got.to_numpy([0, 1, 2, 3])
        assert datagen.row_checksums(rows) == want, "index path"
        assert (np.diff(rows[:, 0].astype(np.int64)) != 0).all()
        g, n_rows = cx.star_join_aggregate(js, pats, filt, [1], [(c.AGG_AVG, 2)])
        assert n_rows == want[0] and len(g["counts"]) == 3
        for ti in range(3):
            m = keep & (d.title_of_employee == ti)
            k = int(pi[d.title_id_by_value[ti]])
            at = g["keys"][0].tolist().index(k)
            assert g["counts"][at] == int(m.sum()) and g["values"][0][at] == int(d.salary_of_employee[m].astype(np.int64).sum()) / int(m.sum())
    finally:
        cx.close()
    # the slice-streaming probe (table mode off) gives the same bag
    import os
    os.environ["KOLIBRIE_PROBE_TABLE"] = "0"
    try:
        cx2 = c.Context(0)
        cx2.dict_numeric_load(num, isn)
        cx2.store_load(s, p, o)
        cx2.build_index()
        assert datagen.row_checksums(cx2.star_join(js, pats, filt).to_numpy([0, 1, 2, 3])) == want, "slice-streaming probe"
        cx2.close()
    finally:
        del os.environ["KOLIBRIE_PROBE_TABLE"]


def test_star_join_with_a_multi_valued_predicate_at_scale():
    """3 objects per subject for one predicate (>= 10 M triples): the star join is 1:N on that pattern — the direct-table paths must
    step aside (duplicate keys) and the answer must still be the relational one: closed-form count and digest, with and without index,
    plus the bound-object lookup through the key-grouped directory"""
    n = 2_200_000  # 3 + 1 + 1 triples per subject = 11 M triples
    s, p, o, num, isn, meta = datagen.multivalued_dataset(n)
    X, T, S, N = 0, 1, 2, 3
    pats = [c.pattern(c.V(X), c.K(1), c.V(T)), c.pattern(c.V(X), c.K(2), c.V(S)), c.pattern(c.V(X), c.K(3), c.V(N))]
    filt = [c.fop(c.F_CMP_NUM, slot=S, cmp=c.CMP_GE, value=500.0)]
    keep = meta["score"] >= 500
    subj, lit = meta["subj"][keep], (meta["score"][keep] + np.uint32(meta["lit0"]))
    expect = np.concatenate([np.stack([subj, tg[keep], lit, subj], axis=1) for tg in meta["tags"]])
    want = datagen.row_checksums(expect)
    assert want[0] == 3 * int(keep.sum())
    rng = np.random.default_rng(3)
    order = rng.permutation(len(s))
    cx = c.Context(0)
    try:
        cx.dict_numeric_load(num, isn)
        cx.store_load(s[order], p[order], o[order])
        for indexed in (False, True):
            if indexed:
                cx.build_index()
            got = cx.star_join(X, pats, filt)
            assert datagen.row_checksums(got.to_numpy([X, T, S, N])) == want, f"indexed={indexed}"
            got.free()
        # (?x tag c): the object is shared by ~1/50 of the subjects x 3 -> a run of the object directory, no scan kernel
        tag = int(meta["tags"][0][123])
        scans0 = cx.get_stats()["scan_launches"]
        r = cx.scan([c.pattern(c.V(X), c.K(1), c.K(tag))])[0]
        assert cx.get_stats()["scan_launches"] == scans0
        assert r.n_rows == sum(int((tg == tag).sum()) for tg in meta["tags"])
    finally:
        cx.close()
