// kb_oracle.cpp — CPU ORACLE. TEST INFRASTRUCTURE ONLY.
//
// A from-scratch C++ restatement of the algorithms on Kolibrie's hot path, used ONLY as the checker in tests/,
// in __graft_entry__.smoke() and as bench.py's CPU baseline. Nothing under kolibrie_b200/ may import, link or
// call it; the product path has no CPU fallback.
//
// Parity status: PINNED for the Datalog fixpoint (14 fc_* known-answer fixtures of
// datalog/tests/reasoning_tests.rs:28-404, replayed in tests/test_oracle_golden.py) and for
// scan/filter (kolibrie/tests/integration_test.rs:19-76,131-299 fixture counts; 4-employee dataset of
// kolibrie/examples/sparql_syntax/simple_select/simple_select_synth_data.rs:16-52).
// Round 2 added, through the host mirror driven by this oracle (tests/test_rdf_star_rsp_golden.py, tests/golden/*.json, generator
// tests/golden/make_fixtures.py): the RDF-star scans, SUBJECT(?t) / isTRIPLE and DELETE WHERE of kolibrie/tests/rdf_star_test.rs
// (:107-145, :281-329, :384-405), the per-firing window contents and ISTREAM / RSTREAM emissions of kolibrie/tests/rsp_engine_test.rs
// (:24-112, :935-1027, :1103-1200), the unit tests of shared/src/quoted_triple_store.rs:82-157, the 4-row answer of
// benches/my_benchmark.rs:29-41, and Rust's str::parse::<f64> acceptance table (tests/golden/rust_parse_f64.json).
// Multi-pattern BGP joins: pinned only by the two joins whose answers kolibrie/tests/integration_test.rs asserts (:286-299 a
// 2-pattern join, :302-342 a 3-pattern join + numeric FILTER; tests/test_oracle_golden.py, both oracle modes). No reference test
// asserts the rows of larger joins through the executor (SURVEY.md §4 "Gap that matters"): beyond those two, parity is UNPINNED and
// the authority is the relational semantics of the cited lines, cross-checked faithful-vs-columnar-vs-brute-force.
// The reference is a Rust workspace and cannot be built in this image (no cargo/rustc), so there is no oracle/_ref
// for the CPU path; oracle/_ref holds only the reference's own CUDA stub (see oracle/Makefile).
//
// Each function cites the reference lines it follows (paths relative to the root of the Kolibrie checkout).
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <limits>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "../include/kolibrie_b200.h"

#define KO_API extern "C" __attribute__((visibility("default")))

namespace {

using u32 = uint32_t;
using u64 = uint64_t;

struct Triple {
    u32 s, p, o;
    bool operator==(const Triple& t) const { return s == t.s && p == t.p && o == t.o; }
    bool operator<(const Triple& t) const {  // shared/src/triple.rs:13-18 derive(Ord): lexicographic s,p,o
        if (s != t.s) return s < t.s;
        if (p != t.p) return p < t.p;
        return o < t.o;
    }
};
struct TripleHash {
    size_t operator()(const Triple& t) const {
        u64 h = (u64)t.s * 0x9E3779B97F4A7C15ull;
        h ^= ((u64)t.p + 0x7F4A7C15ull) * 0xC2B2AE3D27D4EB4Full;
        h = (h ^ (h >> 29)) * 0x165667B19E3779F9ull;
        h ^= (u64)t.o * 0xD6E8FEB86659FD93ull;
        return (size_t)(h ^ (h >> 32));
    }
};

// ---------------------------------------------------------------------------------------------------------------
// Rust `str::parse::<f64>` acceptance (core::num::dec2flt): optional sign; then "inf"/"infinity"/"nan" (ASCII
// case-insensitive) or decimal digits with optional '.', at least one digit overall, optional exponent e[+-]digits.
// No whitespace, no hex, no '_' (SURVEY §7 "FILTER parity").
bool rust_parse_f64(const char* str, size_t len, double* out) {
    size_t i = 0;
    if (len == 0) return false;
    bool neg = false;
    if (str[0] == '+' || str[0] == '-') { neg = str[0] == '-'; i = 1; }
    if (i >= len) return false;
    auto ieq = [&](const char* w) {
        size_t wl = strlen(w);
        if (len - i != wl) return false;
        for (size_t k = 0; k < wl; k++) {
            char c = str[i + k];
            if (c >= 'A' && c <= 'Z') c = (char)(c - 'A' + 'a');
            if (c != w[k]) return false;
        }
        return true;
    };
    if (ieq("inf") || ieq("infinity")) { *out = neg ? -INFINITY : INFINITY; return true; }
    if (ieq("nan")) { *out = NAN; return true; }
    size_t j = i, nd = 0;
    while (j < len && str[j] >= '0' && str[j] <= '9') { j++; nd++; }
    if (j < len && str[j] == '.') { j++; while (j < len && str[j] >= '0' && str[j] <= '9') { j++; nd++; } }
    if (nd == 0) return false;
    if (j < len && (str[j] == 'e' || str[j] == 'E')) {
        j++;
        if (j < len && (str[j] == '+' || str[j] == '-')) j++;
        size_t ne = 0;
        while (j < len && str[j] >= '0' && str[j] <= '9') { j++; ne++; }
        if (ne == 0) return false;
    }
    if (j != len) return false;
    std::string tmp(str, len);  // strtod on a validated decimal string is correctly rounded, like Rust
    *out = strtod(tmp.c_str(), nullptr);
    return true;
}

// ---------------------------------------------------------------------------------------------------------------
// FILTER evaluation: Condition::evaluate_with_ids (kolibrie/src/streamertail_optimizer/types.rs:110-186) on the
// postfix encoding of include/kolibrie_b200.h. `val(slot)` returns the row's id for the variable slot.
struct NumTable {
    const double* num_or0 = nullptr;
    const uint8_t* is_num = nullptr;
    u32 n_ids = 0;
    double num(u32 id) const { return id < n_ids ? num_or0[id] : 0.0; }
    bool isnum(u32 id) const { return id < n_ids ? is_num[id] != 0 : false; }
};

template <class F>
bool eval_filter(const kb_filter_op* ops, u32 n_ops, const NumTable& nt, F&& val) {
    if (n_ops == 0) return true;
    double st[KB_MAX_FILTER_OPS + 1];
    bool ok[KB_MAX_FILTER_OPS + 1];
    int sp = 0;
    for (u32 i = 0; i < n_ops; i++) {
        const kb_filter_op& op = ops[i];
        switch (op.op) {
            case KB_F_CMP_NUM: {
                const u32 id = val(op.slot);
                double a = nt.num(id), b = op.value;
                bool r = false;
                switch (op.cmp) {  // types.rs:133-148
                    case KB_CMP_GT: r = a > b; break;
                    case KB_CMP_GE: r = a >= b; break;
                    case KB_CMP_LT: r = a < b; break;
                    case KB_CMP_LE: r = a <= b; break;
                    default: r = false;
                }
                st[sp] = r && id != KB_ID_NONE; ok[sp++] = true;  // an unbound variable fails every comparison (types.rs:143-145)
            } break;
            case KB_F_EQ_ID: st[sp] = (op.id != KB_ID_NONE && val(op.slot) == op.id); ok[sp++] = true; break;  // types.rs:131
            case KB_F_NE_ID: st[sp] = val(op.slot) != KB_ID_NONE && (op.id == KB_ID_NONE || val(op.slot) != op.id); ok[sp++] = true; break;  // types.rs:132, :143-145
            case KB_F_AND: sp--; st[sp - 1] = (st[sp - 1] != 0.0 && st[sp] != 0.0); break;
            case KB_F_OR: sp--; st[sp - 1] = (st[sp - 1] != 0.0 || st[sp] != 0.0); break;
            case KB_F_NOT: st[sp - 1] = (st[sp - 1] == 0.0); break;
            case KB_F_PUSH_VAR: { u32 id = val(op.slot); st[sp] = nt.num(id); ok[sp++] = id != KB_ID_NONE && nt.isnum(id); } break;  // types.rs:159-163
            case KB_F_PUSH_CONST: st[sp] = op.value; ok[sp++] = true; break;
            case KB_F_ADD: sp--; st[sp - 1] = st[sp - 1] + st[sp]; ok[sp - 1] = ok[sp - 1] && ok[sp]; break;
            case KB_F_SUB: sp--; st[sp - 1] = st[sp - 1] - st[sp]; ok[sp - 1] = ok[sp - 1] && ok[sp]; break;
            case KB_F_MUL: sp--; st[sp - 1] = st[sp - 1] * st[sp]; ok[sp - 1] = ok[sp - 1] && ok[sp]; break;
            case KB_F_DIV: {  // shared/src/query.rs:47-53
                sp--;
                bool v = ok[sp - 1] && ok[sp] && st[sp] != 0.0;
                st[sp - 1] = v ? st[sp - 1] / st[sp] : 0.0;
                ok[sp - 1] = v;
            } break;
            case KB_F_TRUTHY: st[sp - 1] = (ok[sp - 1] && st[sp - 1] != 0.0); ok[sp - 1] = true; break;  // types.rs:168
            case KB_F_IS_TRIPLE: st[sp] = val(op.slot) != KB_ID_NONE && (val(op.slot) & 0x80000000u) != 0; ok[sp++] = true; break;  // types.rs:167-176
            default: return false;
        }
    }
    return sp == 1 && st[0] != 0.0;
}

// ---------------------------------------------------------------------------------------------------------------
// Columnar relation
struct Rel {
    std::vector<u32> slots;
    std::vector<std::vector<u32>> cols;
    u64 n = 0;
    int col_of(u32 slot) const {
        for (size_t i = 0; i < slots.size(); i++) if (slots[i] == slot) return (int)i;
        return -1;
    }
};

inline bool term_match(const kb_term& t, u32 v) { return t.is_var || t.value == v; }

// execute_table_scan_with_ids (engine.rs:510-584): constants must match, variables bind. A variable repeated inside one
// pattern must bind consistently (quirk Q4: enforced here and on the device; the reference's index scans overwrite).
inline bool pattern_match(const kb_pattern& pt, u32 s, u32 p, u32 o) {
    if (!term_match(pt.s, s) || !term_match(pt.p, p) || !term_match(pt.o, o)) return false;
    if (pt.s.is_var && pt.p.is_var && pt.s.value == pt.p.value && s != p) return false;
    if (pt.s.is_var && pt.o.is_var && pt.s.value == pt.o.value && s != o) return false;
    if (pt.p.is_var && pt.o.is_var && pt.p.value == pt.o.value && p != o) return false;
    return true;
}

void pattern_slots(const kb_pattern& pt, std::vector<u32>& slots, std::vector<int>& src) {
    const kb_term* ts[3] = {&pt.s, &pt.p, &pt.o};
    for (int i = 0; i < 3; i++) {
        if (!ts[i]->is_var) continue;
        bool seen = false;
        for (u32 s : slots) if (s == ts[i]->value) seen = true;
        if (!seen) { slots.push_back(ts[i]->value); src.push_back(i); }
    }
}

Rel scan_columnar(const u32* S, const u32* P, const u32* O, u64 n, const kb_pattern& pt) {
    Rel r;
    std::vector<int> src;
    pattern_slots(pt, r.slots, src);
    r.cols.resize(r.slots.size());
    int nt = 1;
#ifdef _OPENMP
    nt = omp_get_max_threads();
#endif
    std::vector<std::vector<u64>> idx(nt);
#pragma omp parallel num_threads(nt)
    {
        int t = 0;
#ifdef _OPENMP
        t = omp_get_thread_num();
#endif
        u64 lo = n * t / nt, hi = n * (t + 1) / nt;
        auto& v = idx[t];
        for (u64 i = lo; i < hi; i++) if (pattern_match(pt, S[i], P[i], O[i])) v.push_back(i);
    }
    std::vector<u64> off(nt + 1, 0);
    for (int t = 0; t < nt; t++) off[t + 1] = off[t] + idx[t].size();
    r.n = off[nt];
    for (auto& c : r.cols) c.resize(r.n);
#pragma omp parallel for num_threads(nt) schedule(static, 1)
    for (int t = 0; t < nt; t++) {
        u64 b = off[t];
        for (size_t k = 0; k < idx[t].size(); k++) {
            u64 i = idx[t][k];
            const u32 vals[3] = {S[i], P[i], O[i]};
            for (size_t c = 0; c < src.size(); c++) r.cols[c][b + k] = vals[src[c]];
        }
    }
    return r;
}

Rel filter_rel(const Rel& in, const kb_filter_op* ops, u32 n_ops, const NumTable& nt) {
    if (n_ops == 0) return in;
    Rel out;
    out.slots = in.slots;
    out.cols.resize(in.cols.size());
    std::vector<uint8_t> keep(in.n);
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < (long long)in.n; i++) {
        keep[i] = eval_filter(ops, n_ops, nt, [&](u32 slot) -> u32 {
            int c = in.col_of(slot);
            return c < 0 ? KB_ID_NONE : in.cols[c][i];
        });
    }
    for (u64 i = 0; i < in.n; i++) if (keep[i]) { for (size_t c = 0; c < in.cols.size(); c++) out.cols[c].push_back(in.cols[c][i]); out.n++; }
    return out;
}

inline u64 mix64(u64 x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

// Natural join on the common variables (execute_optimized_hash_join_with_ids, engine.rs:710-763; execute_hash_join_with_ids
// :766-811; merge variant :970-1039): build a table on the smaller side keyed by the common-variable values, probe with the
// other; output row = union of both rows. No common variable -> cartesian product (:1054-1071). Bag semantics.
Rel hash_join(const Rel& L, const Rel& R) {
    Rel out;
    std::vector<int> lk, rk;
    for (size_t i = 0; i < L.slots.size(); i++) { int c = R.col_of(L.slots[i]); if (c >= 0) { lk.push_back((int)i); rk.push_back(c); } }
    out.slots = L.slots;
    std::vector<int> r_extra;
    for (size_t i = 0; i < R.slots.size(); i++) if (L.col_of(R.slots[i]) < 0) { out.slots.push_back(R.slots[i]); r_extra.push_back((int)i); }
    out.cols.resize(out.slots.size());
    if (L.n == 0 || R.n == 0) return out;  // engine.rs:714-716
    if (lk.empty()) {
        for (u64 i = 0; i < L.n; i++) for (u64 j = 0; j < R.n; j++) {
            for (size_t c = 0; c < L.cols.size(); c++) out.cols[c].push_back(L.cols[c][i]);
            for (size_t c = 0; c < r_extra.size(); c++) out.cols[L.cols.size() + c].push_back(R.cols[r_extra[c]][j]);
            out.n++;
        }
        return out;
    }
    const bool build_left = L.n <= R.n;  // engine.rs:729-733
    const Rel& B = build_left ? L : R;
    const Rel& Pr = build_left ? R : L;
    const std::vector<int>& bk = build_left ? lk : rk;
    const std::vector<int>& pk = build_left ? rk : lk;
    auto keyhash = [&](const Rel& X, const std::vector<int>& kc, u64 i) {
        u64 h = 0x243F6A8885A308D3ull;
        for (int c : kc) h = mix64(h ^ X.cols[c][i]);
        return h;
    };
    u64 cap = 16;
    while (cap < B.n * 2) cap <<= 1;
    std::vector<int64_t> head(cap, -1), next(B.n, -1);
    for (u64 i = 0; i < B.n; i++) {
        u64 h = keyhash(B, bk, i) & (cap - 1);
        next[i] = head[h];
        head[h] = (int64_t)i;
    }
    int nt = 1;
#ifdef _OPENMP
    nt = omp_get_max_threads();
#endif
    std::vector<std::vector<std::pair<u64, u64>>> pairs(nt);  // (left row, right row)
#pragma omp parallel num_threads(nt)
    {
        int t = 0;
#ifdef _OPENMP
        t = omp_get_thread_num();
#endif
        u64 lo = Pr.n * t / nt, hi = Pr.n * (t + 1) / nt;
        auto& v = pairs[t];
        for (u64 i = lo; i < hi; i++) {
            u64 h = keyhash(Pr, pk, i) & (cap - 1);
            for (int64_t j = head[h]; j >= 0; j = next[j]) {
                bool eq = true;
                for (size_t k = 0; k < bk.size(); k++) if (B.cols[bk[k]][j] != Pr.cols[pk[k]][i]) { eq = false; break; }
                if (eq) v.push_back(build_left ? std::make_pair((u64)j, i) : std::make_pair(i, (u64)j));
            }
        }
    }
    std::vector<u64> off(nt + 1, 0);
    for (int t = 0; t < nt; t++) off[t + 1] = off[t] + pairs[t].size();
    out.n = off[nt];
    for (auto& c : out.cols) c.resize(out.n);
#pragma omp parallel for num_threads(nt) schedule(static, 1)
    for (int t = 0; t < nt; t++) {
        u64 b = off[t];
        for (size_t k = 0; k < pairs[t].size(); k++) {
            u64 li = pairs[t][k].first, ri = pairs[t][k].second;
            for (size_t c = 0; c < L.cols.size(); c++) out.cols[c][b + k] = L.cols[c][li];
            for (size_t c = 0; c < r_extra.size(); c++) out.cols[L.cols.size() + c][b + k] = R.cols[r_extra[c]][ri];
        }
    }
    return out;
}

Rel project_rel(const Rel& in, const u32* slots, u32 n) {
    Rel out;
    out.n = in.n;
    for (u32 i = 0; i < n; i++) {
        int c = in.col_of(slots[i]);
        if (c < 0) continue;  // engine.rs:96-103: retain() keeps only the variables that exist
        out.slots.push_back(slots[i]);
        out.cols.push_back(in.cols[c]);
    }
    return out;
}

// ---------------------------------------------------------------------------------------------------------------
// FAITHFUL mode: row-of-maps execution with the UnifiedIndex, as the reference's executor does it.
// Row = small vector of (slot, id) pairs standing in for HashMap<String,u32> (strictly cheaper than the reference's rows).
struct Row {
    u32 n = 0;
    u32 k[KB_MAX_COLS];
    u32 v[KB_MAX_COLS];
    bool get(u32 slot, u32* out) const {
        for (u32 i = 0; i < n; i++) if (k[i] == slot) { *out = v[i]; return true; }
        return false;
    }
    void or_insert(u32 slot, u32 val) {  // HashMap::entry().or_insert (engine.rs:640-642)
        for (u32 i = 0; i < n; i++) if (k[i] == slot) return;
        if (n < KB_MAX_COLS) { k[n] = slot; v[n] = val; n++; }
    }
    void insert(u32 slot, u32 val) {  // HashMap::insert: overwrite
        for (u32 i = 0; i < n; i++) if (k[i] == slot) { v[i] = val; return; }
        if (n < KB_MAX_COLS) { k[n] = slot; v[n] = val; n++; }
    }
};

// UnifiedIndex (shared/src/index_manager.rs:18-26): nested hash maps; only the permutations the scans use.
struct Index {
    std::unordered_map<u32, std::unordered_map<u32, std::vector<u32>>> spo, pos, osp, sop;
    void build(const u32* S, const u32* P, const u32* O, u64 n) {
        for (u64 i = 0; i < n; i++) {
            spo[S[i]][P[i]].push_back(O[i]);
            pos[P[i]][O[i]].push_back(S[i]);
            osp[O[i]][S[i]].push_back(P[i]);
            sop[S[i]][O[i]].push_back(P[i]);
        }
    }
};

struct Db {
    std::vector<u32> S, P, O;
    Index idx;
    bool indexed = false;
    NumTable nt;
    std::vector<double> num;
    std::vector<uint8_t> isnum;
};

// execute_index_scan_with_ids (engine.rs:1192-1245) + scan_*_index_with_ids (:1248-1407)
void index_scan(const Db& db, const kb_pattern& pt, std::vector<Row>& out) {
    const bool bs = !pt.s.is_var, bp = !pt.p.is_var, bo = !pt.o.is_var;
    auto emit2 = [&](u32 k1, u32 v1, u32 k2, u32 v2) { Row r; r.insert(k1, v1); r.insert(k2, v2); out.push_back(r); };
    auto emit1 = [&](u32 k1, u32 v1) { Row r; r.insert(k1, v1); out.push_back(r); };
    if (bs && bp && bo) {
        auto a = db.idx.spo.find(pt.s.value);
        if (a == db.idx.spo.end()) return;
        auto b = a->second.find(pt.p.value);
        if (b == a->second.end()) return;
        for (u32 o : b->second) if (o == pt.o.value) { out.push_back(Row()); return; }
    } else if (bs && bp) {
        auto a = db.idx.spo.find(pt.s.value);
        if (a == db.idx.spo.end()) return;
        auto b = a->second.find(pt.p.value);
        if (b == a->second.end()) return;
        for (u32 o : b->second) emit1(pt.o.value, o);
    } else if (bs && bo) {
        auto a = db.idx.sop.find(pt.s.value);
        if (a == db.idx.sop.end()) return;
        auto b = a->second.find(pt.o.value);
        if (b == a->second.end()) return;
        for (u32 p : b->second) emit1(pt.p.value, p);
    } else if (bp && bo) {
        auto a = db.idx.pos.find(pt.p.value);
        if (a == db.idx.pos.end()) return;
        auto b = a->second.find(pt.o.value);
        if (b == a->second.end()) return;
        for (u32 s : b->second) emit1(pt.s.value, s);
    } else if (bs) {
        auto a = db.idx.spo.find(pt.s.value);
        if (a == db.idx.spo.end()) return;
        for (auto& po : a->second) for (u32 o : po.second) if (pattern_match(pt, pt.s.value, po.first, o)) emit2(pt.p.value, po.first, pt.o.value, o);
    } else if (bp) {
        auto a = db.idx.pos.find(pt.p.value);
        if (a == db.idx.pos.end()) return;
        for (auto& os : a->second) for (u32 s : os.second) if (pattern_match(pt, s, pt.p.value, os.first)) emit2(pt.s.value, s, pt.o.value, os.first);
    } else if (bo) {
        auto a = db.idx.osp.find(pt.o.value);
        if (a == db.idx.osp.end()) return;
        for (auto& sp : a->second) for (u32 p : sp.second) if (pattern_match(pt, sp.first, p, pt.o.value)) emit2(pt.s.value, sp.first, pt.p.value, p);
    } else {  // fully unbound -> table scan (engine.rs:1236-1239)
        for (size_t i = 0; i < db.S.size(); i++) if (pattern_match(pt, db.S[i], db.P[i], db.O[i])) {
            Row r; r.insert(pt.s.value, db.S[i]); r.insert(pt.p.value, db.P[i]); r.insert(pt.o.value, db.O[i]); out.push_back(r);
        }
    }
}

// bind_pattern (engine.rs:888-923)
kb_pattern bind_pattern(const kb_pattern& pt, const Row& b) {
    kb_pattern q = pt;
    kb_term* ts[3] = {&q.s, &q.p, &q.o};
    for (auto* t : ts) { u32 v; if (t->is_var && b.get(t->value, &v)) { t->is_var = 0; t->value = v; } }
    return q;
}

int bound_count(const kb_pattern& pt) { return (!pt.s.is_var) + (!pt.p.is_var) + (!pt.o.is_var); }

// execute_star_join_with_ids (engine.rs:587-691) with the result caps of quirk Q1 OFF (uncapped relational semantics).
std::vector<Row> star_join_faithful(const Db& db, u32 join_slot, const kb_pattern* pats, u32 n) {
    std::vector<Row> results;
    if (n == 0) return results;
    std::vector<std::pair<u32, u64>> est(n);
    for (u32 i = 0; i < n; i++) {
        static const u64 card[4] = {1000000, 10000, 100, 1};  // estimate_pattern_cardinality (engine.rs:694-707)
        est[i] = {i, card[bound_count(pats[i])]};
    }
    std::stable_sort(est.begin(), est.end(), [](auto& a, auto& b) { return a.second < b.second; });  // engine.rs:608
    index_scan(db, pats[est[0].first], results);
    if (results.empty()) return results;
    const bool sequential = results.size() > 10000 || est[0].second > 50000;  // engine.rs:621
    for (u32 k = 1; k < n; k++) {
        const kb_pattern& pt = pats[est[k].first];
        std::vector<Row> next;
        auto one = [&](const Row& binding, std::vector<Row>& dst) {
            u32 jv;
            if (!binding.get(join_slot, &jv)) return;
            Row only; only.insert(join_slot, jv);  // engine.rs:633-636: bound on the join variable ONLY (quirk Q3)
            kb_pattern bp = bind_pattern(pt, only);
            std::vector<Row> matches;
            index_scan(db, bp, matches);
            for (auto& m : matches) { Row merged = binding; for (u32 i = 0; i < m.n; i++) merged.or_insert(m.k[i], m.v[i]); dst.push_back(merged); }
        };
        if (sequential) {
            for (auto& b : results) one(b, next);
        } else {
            int nt = 1;
#ifdef _OPENMP
            nt = omp_get_max_threads();
#endif
            std::vector<std::vector<Row>> part(nt);
#pragma omp parallel for num_threads(nt) schedule(static)
            for (long long i = 0; i < (long long)results.size(); i++) {
                int t = 0;
#ifdef _OPENMP
                t = omp_get_thread_num();
#endif
                one(results[i], part[t]);
            }
            for (auto& p : part) next.insert(next.end(), p.begin(), p.end());
        }
        results.swap(next);
        if (results.empty()) return results;
    }
    return results;
}

// execute_bind_join_with_ids (engine.rs:840-885), caps off: rayon par_chunks -> OpenMP over left rows.
std::vector<Row> bind_join_faithful(const Db& db, const std::vector<Row>& left, const kb_pattern& right) {
    int nt = 1;
#ifdef _OPENMP
    nt = omp_get_max_threads();
#endif
    std::vector<std::vector<Row>> part(nt);
#pragma omp parallel for num_threads(nt) schedule(static)
    for (long long i = 0; i < (long long)left.size(); i++) {
        int t = 0;
#ifdef _OPENMP
        t = omp_get_thread_num();
#endif
        kb_pattern bp = bind_pattern(right, left[i]);
        std::vector<Row> matches;
        index_scan(db, bp, matches);
        for (auto& m : matches) { Row r = left[i]; for (u32 j = 0; j < m.n; j++) r.or_insert(m.k[j], m.v[j]); part[t].push_back(r); }
    }
    std::vector<Row> out;
    for (auto& p : part) out.insert(out.end(), p.begin(), p.end());
    return out;
}

Rel rows_to_rel(const std::vector<Row>& rows, const std::vector<u32>& slots) {
    Rel r;
    r.slots = slots;
    r.cols.resize(slots.size());
    r.n = rows.size();
    for (auto& c : r.cols) c.resize(r.n);
    for (u64 i = 0; i < r.n; i++) for (size_t c = 0; c < slots.size(); c++) { u32 v = KB_ID_NONE; rows[i].get(slots[c], &v); r.cols[c][i] = v; }
    return r;
}

std::vector<u32> bgp_slots(const kb_pattern* pats, u32 n) {
    std::vector<u32> slots;
    std::vector<int> src;
    for (u32 i = 0; i < n; i++) pattern_slots(pats[i], slots, src);
    return slots;
}

// Is this BGP a star on one variable shared by all patterns (optimizer.rs:84-152)? returns slot or -1.
int star_var(const kb_pattern* pats, u32 n) {
    if (n == 0) return -1;
    std::vector<u32> s0; std::vector<int> src;
    pattern_slots(pats[0], s0, src);
    for (u32 cand : s0) {
        bool all = true;
        for (u32 i = 1; i < n && all; i++) {
            std::vector<u32> si; std::vector<int> sr;
            pattern_slots(pats[i], si, sr);
            if (std::find(si.begin(), si.end(), cand) == si.end()) all = false;
        }
        if (all) return (int)cand;
    }
    return -1;
}

// Whole-BGP evaluation.
// mode 0 = columnar (relational restatement: scan each pattern, left-deep natural joins in textual order
//          (build_logical_plan, utils.rs:101-191), FILTER, projection);
// mode 1 = faithful (plans as the reference's optimizer picks them: >=3 patterns sharing a variable -> StarJoin
//          (optimizer.rs:84-152); 2 patterns -> bind join (cost/estimator.rs:99-105); otherwise hash-join chain),
//          rows of maps + UnifiedIndex, quirk-Q1 caps off.
Rel bgp_execute(Db& db, int mode, const kb_pattern* pats, u32 n, const kb_filter_op* f, u32 nf, const u32* proj, u32 nproj) {
    Rel cur;
    const u64 N = db.S.size();
    if (mode == 1) {
        if (!db.indexed) { db.idx.build(db.S.data(), db.P.data(), db.O.data(), N); db.indexed = true; }
        std::vector<u32> slots = bgp_slots(pats, n);
        int sv = star_var(pats, n);
        std::vector<Row> rows;
        if (n >= 3 && sv >= 0) {
            rows = star_join_faithful(db, (u32)sv, pats, n);
        } else {
            index_scan(db, pats[0], rows);
            for (u32 i = 1; i < n; i++) rows = bind_join_faithful(db, rows, pats[i]);
        }
        cur = rows_to_rel(rows, slots);
    } else {
        for (u32 i = 0; i < n; i++) {
            Rel r = scan_columnar(db.S.data(), db.P.data(), db.O.data(), N, pats[i]);
            cur = (i == 0) ? std::move(r) : hash_join(cur, r);
        }
    }
    cur = filter_rel(cur, f, nf, db.nt);
    if (proj) cur = project_rel(cur, proj, nproj);
    return cur;
}

// ---------------------------------------------------------------------------------------------------------------
// GROUP BY + aggregates (group_and_aggregate_results, execute_query.rs:1150-1227); COUNT = rows per group.
struct Groups {
    u32 n_group = 0, n_aggs = 0;
    std::vector<std::vector<u32>> keys;
    std::vector<std::vector<double>> vals;
    std::vector<u64> counts;
};

Groups group_aggregate(const Rel& in, const NumTable& nt, const u32* gslots, u32 ng, const kb_agg* aggs, u32 na) {
    Groups g;
    g.n_group = ng; g.n_aggs = na;
    g.keys.resize(ng); g.vals.resize(na);
    std::vector<int> gc(ng), ac(na);
    for (u32 i = 0; i < ng; i++) gc[i] = in.col_of(gslots[i]);
    for (u32 i = 0; i < na; i++) ac[i] = aggs[i].kind == KB_AGG_COUNT ? -1 : in.col_of(aggs[i].slot);
    std::unordered_map<std::string, u64> idx;
    for (u64 r = 0; r < in.n; r++) {
        std::string key((size_t)ng * 4, '\0');
        for (u32 i = 0; i < ng; i++) { u32 v = gc[i] >= 0 ? in.cols[gc[i]][r] : KB_ID_NONE; memcpy(&key[(size_t)i * 4], &v, 4); }
        auto it = idx.find(key);
        u64 gi;
        bool fresh = false;
        if (it == idx.end()) {
            gi = g.counts.size();
            idx.emplace(key, gi);
            for (u32 i = 0; i < ng; i++) g.keys[i].push_back(gc[i] >= 0 ? in.cols[gc[i]][r] : KB_ID_NONE);
            for (u32 i = 0; i < na; i++) g.vals[i].push_back(0.0);
            g.counts.push_back(0);
            fresh = true;
        } else gi = it->second;
        g.counts[gi]++;
        for (u32 i = 0; i < na; i++) {
            double v = ac[i] >= 0 ? nt.num(in.cols[ac[i]][r]) : 0.0;  // execute_query.rs:1171-1175,1184: unwrap_or(0.0)
            double& acc = g.vals[i][gi];
            if (fresh) { acc = v; continue; }                          // :1198-1201 first row initialises
            switch (aggs[i].kind) {
                case KB_AGG_SUM: case KB_AGG_AVG: acc += v; break;
                case KB_AGG_MIN: acc = std::fmin(acc, v); break;       // f64::min: a NaN operand is ignored
                case KB_AGG_MAX: acc = std::fmax(acc, v); break;       // f64::max
                default: break;
            }
        }
    }
    for (u32 i = 0; i < na; i++) for (size_t gi = 0; gi < g.counts.size(); gi++) {
        if (aggs[i].kind == KB_AGG_AVG) g.vals[i][gi] /= (double)g.counts[gi];   // :1216
        if (aggs[i].kind == KB_AGG_COUNT) g.vals[i][gi] = (double)g.counts[gi];
    }
    return g;
}

// ---------------------------------------------------------------------------------------------------------------
// Datalog. Bindings are fixed-width rows of ids over the rule's variable slots (UNBOUND = KB_ID_NONE); the reference carries
// the same information as BTreeMap<String,String> and re-encodes through the dictionary on every probe.
constexpr u32 UNB = KB_ID_NONE;
constexpr u32 MAXV = 32;
struct Bind { u32 v[MAXV]; };

struct RulePlan {
    u32 n_vars = 0;  // real + synthetic (quirk Q6) variable slots
    struct Prem { int s_var, o_var; bool pred_const; u32 pred; bool s_is_const, o_is_const; u32 s_const, o_const; } prem[KB_MAX_PREMISES];
    u32 n_prem = 0;
};

// extract_join_parameters (shared/src/join_algorithm.rs:466-496): a Constant in subject/object position becomes the synthetic
// variable "__const_subj_{c}" / "__const_obj_{c}" (so it is NOT enforced, and equal constants in the same position of two
// premises join with each other); a Variable predicate becomes "__var_pred_{v}", which is never in the dictionary -> no match
// (:515-521).
RulePlan plan_rule(const kb_rule& r, u32 max_real_slot_plus1) {
    RulePlan pl;
    pl.n_prem = r.n_premise;
    u32 next = max_real_slot_plus1;
    std::unordered_map<u64, u32> synth;
    auto syn = [&](u32 pos, u32 c) {
        u64 k = ((u64)pos << 32) | c;
        auto it = synth.find(k);
        if (it != synth.end()) return it->second;
        u32 s = next++;
        synth.emplace(k, s);
        return s;
    };
    for (u32 i = 0; i < r.n_premise; i++) {
        const kb_pattern& p = r.premise[i];
        pl.prem[i].s_var = (int)(p.s.is_var ? p.s.value : syn(0, p.s.value));
        pl.prem[i].o_var = (int)(p.o.is_var ? p.o.value : syn(2, p.o.value));
        pl.prem[i].pred_const = !p.p.is_var;
        pl.prem[i].pred = p.p.value;
        pl.prem[i].s_is_const = !p.s.is_var; pl.prem[i].s_const = p.s.value;
        pl.prem[i].o_is_const = !p.o.is_var; pl.prem[i].o_const = p.o.value;
    }
    pl.n_vars = next;
    return pl;
}

struct PairHash { size_t operator()(const std::pair<u32, u32>& p) const { return (size_t)mix64(((u64)p.first << 32) | p.second); } };

// perform_hash_join_for_rules (join_algorithm.rs:499-570) + build_simple_hash_table (:582-622) + process_triple_fast (:625-677)
std::vector<Bind> join_premise(const RulePlan::Prem& pr, const Triple* facts, u64 n_facts, const std::vector<Bind>& cur, bool strict = false) {
    std::vector<Bind> out;
    if (cur.empty()) return out;        // :510-512
    if (!pr.pred_const) return out;     // :515-521 variable predicate never matches
    std::vector<const Triple*> filt;    // :528-534 predicate pre-filter
    for (u64 i = 0; i < n_facts; i++) {
        if (facts[i].p != pr.pred) continue;
        // strict = matches_rule_pattern (rules.rs:9-72): constants in subject / object position must equal the fact's
        if (strict && ((pr.s_is_const && facts[i].s != pr.s_const) || (pr.o_is_const && facts[i].o != pr.o_const))) continue;
        filt.push_back(&facts[i]);
    }
    if (filt.empty()) return out;
    std::unordered_map<std::pair<u32, u32>, std::vector<u32>, PairHash> both;
    std::unordered_map<u32, std::vector<u32>> sb, ob;
    std::vector<u32> neither;
    for (u32 i = 0; i < cur.size(); i++) {
        u32 s = cur[i].v[pr.s_var], o = cur[i].v[pr.o_var];
        if (s != UNB && o != UNB) both[{s, o}].push_back(i);
        else if (s != UNB) sb[s].push_back(i);
        else if (o != UNB) ob[o].push_back(i);
        else neither.push_back(i);
    }
    for (const Triple* t : filt) {
        auto b = both.find({t->s, t->o});
        if (b != both.end()) { for (u32 i : b->second) out.push_back(cur[i]); continue; }  // :637-642 early return
        auto s = sb.find(t->s);
        if (s != sb.end()) for (u32 i : s->second) { Bind r = cur[i]; r.v[pr.o_var] = t->o; out.push_back(r); }
        auto o = ob.find(t->o);
        if (o != ob.end()) for (u32 i : o->second) { Bind r = cur[i]; r.v[pr.s_var] = t->s; out.push_back(r); }
        for (u32 i : neither) { Bind r = cur[i]; r.v[pr.s_var] = t->s; r.v[pr.o_var] = t->o; out.push_back(r); }  // insert s then o (:668-675)
    }
    return out;
}

// evaluate_filters (datalog/src/reasoning/rules.rs:133-165)
bool rule_filters_pass(const kb_rule& r, const Bind& b, const NumTable& nt) {
    for (u32 i = 0; i < r.n_filters; i++) {
        const kb_rule_filter& f = r.filters[i];
        u32 lhs = b.v[f.lhs_slot];
        if (lhs == UNB) continue;  // :139 `if let Some(..)`
        if (f.rhs_is_var && b.v[f.rhs_slot] != UNB) {
            u32 rhs = b.v[f.rhs_slot];
            if (f.cmp == KB_CMP_NE && lhs == rhs) return false;
            if (f.cmp == KB_CMP_EQ && lhs != rhs) return false;
        } else {
            double a = nt.num(lhs), c = f.rhs_value;
            switch (f.cmp) {
                case KB_CMP_GT: if (a <= c) return false; break;
                case KB_CMP_LT: if (a >= c) return false; break;
                case KB_CMP_GE: if (a < c) return false; break;
                case KB_CMP_LE: if (a > c) return false; break;
                case KB_CMP_EQ: if (std::fabs(a - c) > std::numeric_limits<double>::epsilon()) return false; break;
                case KB_CMP_NE: if (std::fabs(a - c) <= std::numeric_limits<double>::epsilon()) return false; break;
                default: break;
            }
        }
    }
    return true;
}

struct FixpointOut {
    std::vector<Triple> inferred;
    std::vector<u64> round_new;
    u64 derivations = 0;
    int status = 0;
};

// Reasoner::infer_with_strategy (infer_generic.rs:27-53) with SemiNaiveStrategy (semi_naive.rs:17-85) or NaiveStrategy
// (my_naive.rs:18-69).
FixpointOut fixpoint(const std::vector<Triple>& base, const kb_rule* rules, u32 n_rules, u32 strategy, const NumTable& nt) {
    FixpointOut fo;
    std::vector<Triple> all = base;
    std::unordered_set<Triple, TripleHash> known(all.begin(), all.end());
    const size_t idx_before = all.size();
    std::vector<RulePlan> plans;
    for (u32 r = 0; r < n_rules; r++) {
        u32 mx = 0;
        auto upd = [&](const kb_term& t) { if (t.is_var) mx = std::max(mx, t.value + 1); };
        for (u32 i = 0; i < rules[r].n_premise; i++) { upd(rules[r].premise[i].s); upd(rules[r].premise[i].p); upd(rules[r].premise[i].o); }
        for (u32 i = 0; i < rules[r].n_conclusion; i++) { upd(rules[r].conclusion[i].s); upd(rules[r].conclusion[i].p); upd(rules[r].conclusion[i].o); }
        for (u32 i = 0; i < rules[r].n_filters; i++) { mx = std::max(mx, rules[r].filters[i].lhs_slot + 1); if (rules[r].filters[i].rhs_is_var) mx = std::max(mx, rules[r].filters[i].rhs_slot + 1); }
        plans.push_back(plan_rule(rules[r], mx));
        if (plans.back().n_vars > MAXV) { fo.status = KB_E_LIMIT; return fo; }
    }
    size_t delta_start = 0;
    for (;;) {
        std::unordered_set<Triple, TripleHash> round;
        const size_t end = all.size();
        const Triple* delta = all.data() + delta_start;
        const u64 n_delta = end - delta_start;
        delta_start = end;
        for (u32 r = 0; r < n_rules; r++) {
            const kb_rule& rule = rules[r];
            const RulePlan& pl = plans[r];
            std::vector<Bind> sols;
            Bind empty;
            for (u32 k = 0; k < MAXV; k++) empty.v[k] = UNB;
            const bool strict = strategy == KB_SEMI_NAIVE_PARALLEL;
            if (strict && rule.n_premise != 1 && rule.n_premise != 2) continue;  // semi_naive_parallel.rs:149 `_ => {}`
            if (strategy == KB_NAIVE) {
                if (rule.n_premise > 0) {
                    std::vector<Bind> cur{empty};
                    for (u32 j = 0; j < rule.n_premise; j++) { cur = join_premise(pl.prem[j], all.data(), end, cur); if (cur.empty()) break; }
                    sols = std::move(cur);
                }
            } else {
                for (u32 i = 0; i < rule.n_premise; i++) {  // semi_naive.rs:22-44
                    std::vector<Bind> cur{empty};
                    cur = join_premise(pl.prem[i], delta, n_delta, cur, strict);
                    for (u32 j = 0; j < rule.n_premise; j++) {
                        if (j == i) continue;
                        cur = join_premise(pl.prem[j], all.data(), end, cur, strict);
                        if (cur.empty()) break;
                    }
                    sols.insert(sols.end(), cur.begin(), cur.end());
                }
            }
            for (const Bind& b : sols) {
                if (!strict && !rule_filters_pass(rule, b, nt)) continue;  // the parallel variant never evaluates rule.filters
                for (u32 c = 0; c < rule.n_conclusion; c++) {
                    const kb_pattern& h = rule.conclusion[c];
                    auto term = [&](const kb_term& t, bool* ok) -> u32 {
                        if (!t.is_var) return t.value;
                        if (b.v[t.value] == UNB) { *ok = false; return 0; }  // quirk Q8 (materialisation.rs:13-27, :40-49): unsafe head
                        return b.v[t.value];
                    };
                    bool ok = true;
                    Triple f{term(h.s, &ok), term(h.p, &ok), term(h.o, &ok)};
                    if (!ok) { fo.status = KB_E_UNSUPPORTED; return fo; }
                    fo.derivations++;
                    if (!known.count(f)) round.insert(f);  // semi_naive.rs:76-78
                }
            }
        }
        if (round.empty()) break;  // infer_generic.rs:38-40
        u64 added = 0;
        for (const Triple& f : round) if (!known.count(f)) { known.insert(f); all.push_back(f); added++; }
        fo.round_new.push_back(added);
    }
    fo.inferred.assign(all.begin() + idx_before, all.end());
    std::sort(fo.inferred.begin(), fo.inferred.end());
    return fo;
}

}  // namespace

// =================================================================================================================
// C API (ctypes) — handles are opaque pointers
struct ko_db { Db db; };
struct ko_rel { Rel r; };
struct ko_groups { Groups g; };
struct ko_fix { FixpointOut f; };

KO_API ko_db* ko_db_create(const u32* s, const u32* p, const u32* o, u64 n) {
    ko_db* d = new ko_db;
    d->db.S.assign(s, s + n); d->db.P.assign(p, p + n); d->db.O.assign(o, o + n);
    return d;
}
KO_API void ko_db_numeric(ko_db* d, const double* num_or0, const uint8_t* is_num, u32 n_ids) {
    d->db.num.assign(num_or0, num_or0 + n_ids);
    d->db.isnum.assign(is_num, is_num + n_ids);
    d->db.nt.num_or0 = d->db.num.data(); d->db.nt.is_num = d->db.isnum.data(); d->db.nt.n_ids = n_ids;
}
KO_API void ko_db_build_index(ko_db* d) {
    if (!d->db.indexed) { d->db.idx.build(d->db.S.data(), d->db.P.data(), d->db.O.data(), d->db.S.size()); d->db.indexed = true; }
}
KO_API void ko_db_free(ko_db* d) { delete d; }

KO_API ko_rel* ko_bgp_execute(ko_db* d, int mode, const kb_pattern* pats, u32 n, const kb_filter_op* f, u32 nf, const u32* proj, u32 nproj) {
    ko_rel* r = new ko_rel;
    r->r = bgp_execute(d->db, mode, pats, n, f, nf, proj, nproj);
    return r;
}
KO_API ko_rel* ko_scan(ko_db* d, const kb_pattern* pat, const kb_filter_op* f, u32 nf) {
    ko_rel* r = new ko_rel;
    r->r = filter_rel(scan_columnar(d->db.S.data(), d->db.P.data(), d->db.O.data(), d->db.S.size(), *pat), f, nf, d->db.nt);
    return r;
}
KO_API ko_rel* ko_rel_from_host(const u32* slots, u32 n_cols, const u32* const* cols, u64 n_rows) {
    ko_rel* r = new ko_rel;
    r->r.n = n_rows;
    for (u32 c = 0; c < n_cols; c++) { r->r.slots.push_back(slots[c]); r->r.cols.emplace_back(cols[c], cols[c] + n_rows); }
    return r;
}
KO_API ko_rel* ko_hash_join(const ko_rel* a, const ko_rel* b) { ko_rel* r = new ko_rel; r->r = hash_join(a->r, b->r); return r; }
KO_API ko_rel* ko_filter(ko_db* d, const ko_rel* a, const kb_filter_op* f, u32 nf) { ko_rel* r = new ko_rel; r->r = filter_rel(a->r, f, nf, d->db.nt); return r; }
KO_API ko_rel* ko_project(const ko_rel* a, const u32* slots, u32 n) { ko_rel* r = new ko_rel; r->r = project_rel(a->r, slots, n); return r; }
KO_API u64 ko_rel_rows(const ko_rel* r) { return r->r.n; }
KO_API u32 ko_rel_cols(const ko_rel* r) { return (u32)r->r.slots.size(); }
KO_API u32 ko_rel_slot(const ko_rel* r, u32 c) { return r->r.slots[c]; }
KO_API const u32* ko_rel_col(const ko_rel* r, u32 c) { return r->r.cols[c].data(); }
KO_API void ko_rel_free(ko_rel* r) { delete r; }

KO_API ko_groups* ko_group_aggregate(ko_db* d, const ko_rel* in, const u32* gslots, u32 ng, const kb_agg* aggs, u32 na) {
    ko_groups* g = new ko_groups;
    g->g = group_aggregate(in->r, d->db.nt, gslots, ng, aggs, na);
    return g;
}
KO_API u64 ko_groups_n(const ko_groups* g) { return g->g.counts.size(); }
KO_API const u32* ko_groups_keys(const ko_groups* g, u32 c) { return g->g.keys[c].data(); }
KO_API const double* ko_groups_values(const ko_groups* g, u32 a) { return g->g.vals[a].data(); }
KO_API const u64* ko_groups_counts(const ko_groups* g) { return g->g.counts.data(); }
KO_API void ko_groups_free(ko_groups* g) { delete g; }

KO_API ko_fix* ko_datalog_fixpoint(ko_db* d, const kb_rule* rules, u32 n_rules, u32 strategy) {
    std::vector<Triple> base(d->db.S.size());
    for (size_t i = 0; i < base.size(); i++) base[i] = Triple{d->db.S[i], d->db.P[i], d->db.O[i]};
    // index_manager.query(None,None,None) dumps the spo index: set semantics (index_manager.rs:41-57 dedups on insert)
    std::sort(base.begin(), base.end());
    base.erase(std::unique(base.begin(), base.end()), base.end());
    ko_fix* f = new ko_fix;
    f->f = fixpoint(base, rules, n_rules, strategy, d->db.nt);
    return f;
}
KO_API int ko_fix_status(const ko_fix* f) { return f->f.status; }
KO_API u64 ko_fix_n(const ko_fix* f) { return f->f.inferred.size(); }
KO_API void ko_fix_copy(const ko_fix* f, u32* s, u32* p, u32* o) {
    for (size_t i = 0; i < f->f.inferred.size(); i++) { s[i] = f->f.inferred[i].s; p[i] = f->f.inferred[i].p; o[i] = f->f.inferred[i].o; }
}
KO_API u32 ko_fix_rounds(const ko_fix* f) { return (u32)f->f.round_new.size(); }
KO_API u64 ko_fix_round_new(const ko_fix* f, u32 r) { return f->f.round_new[r]; }
KO_API u64 ko_fix_derivations(const ko_fix* f) { return f->f.derivations; }
KO_API void ko_fix_free(ko_fix* f) { delete f; }

// legacy FFI semantics as repaired (SURVEY A.4): ascending indices of triples with p == predicate (and o == *literal)
KO_API u32 ko_legacy_select(const u32* p, const u32* o, u32 n, u32 pred, const u32* literal, u32* out_idx) {
    u32 c = 0;
    for (u32 i = 0; i < n; i++) if (p[i] == pred && (!literal || o[i] == *literal)) out_idx[c++] = i;
    return c;
}

KO_API int ko_rust_parse_f64(const char* s, u64 len, double* out) { return rust_parse_f64(s, (size_t)len, out) ? 1 : 0; }
KO_API int ko_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
KO_API void ko_set_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}
