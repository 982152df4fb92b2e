// kb_backward.cu — what kb_datalog_query adds to the Datalog driver (kb_datalog.cu): the demand patterns of a query (host), the demand
// selection of a predicate relation, and the answer pass that projects the facts matching the query onto its variables, each distinct
// binding once.
//
// Reasoner::backward_chaining (datalog/src/reasoning/backward_chaining.rs:165-259) answers a pattern by SLD resolution down to
// MAX_DEPTH = 10. Its distinct bindings of the query's variables are those of the query's instances in T^depth, the facts with a proof of
// height <= depth (premise constants enforced, rule filters ignored): semi-naive rounds stopped after `depth` rounds. Every subgoal of
// that search is an instance of a demand pattern (below), so facts that match none of their predicate's demand patterns take no part in
// any proof of an answer and are left out of the rounds.
#include <algorithm>
#include <deque>

#include "kb_internal.hpp"

namespace kb {

namespace {
constexpr u32 ANY = KB_ID_NONE;
bool subsumes(uint2 a, uint2 b) { return (a.x == ANY || a.x == b.x) && (a.y == ANY || a.y == b.y); }
}  // namespace

void bc_demand_compile(const kb_rule* rules, u32 n_rules, const kb_pattern& q, BcDemand* d) {
    d->relevant.assign(n_rules, false);
    d->pats.clear();
    std::deque<std::pair<u32, uint2>> work;
    auto add = [&](u32 p, uint2 x) {
        auto& v = d->pats[p];
        for (const uint2& e : v) if (subsumes(e, x)) return;
        v.erase(std::remove_if(v.begin(), v.end(), [&](const uint2& e) { return subsumes(x, e); }), v.end());
        if (v.size() >= BC_MAX_DEMAND) {  // too many patterns for one predicate: all of its facts are demanded (sound, and bounds the work)
            x = make_uint2(ANY, ANY);
            v.clear();
        }
        v.push_back(x);
        work.push_back({p, x});
    };
    // the query: a constant that a variable of the query repeats is not known here, so a repeated variable demands any value
    auto qv = [&](const kb_term& t) { return t.is_var ? ANY : t.value; };
    const uint2 q0 = make_uint2(qv(q.s), qv(q.o));
    if (!q.p.is_var) add(q.p.value, q0);
    else
        for (u32 r = 0; r < n_rules; r++)
            for (u32 c = 0; c < rules[r].n_conclusion; c++) add(rules[r].conclusion[c].p.value, q0);
    while (!work.empty()) {
        const auto [p, x] = work.front();
        work.pop_front();
        for (u32 r = 0; r < n_rules; r++) {
            const kb_rule& rule = rules[r];
            for (u32 c = 0; c < rule.n_conclusion; c++) {
                const kb_pattern& h = rule.conclusion[c];
                if (h.p.value != p) continue;
                // unify the head with the demand: a head constant must equal a demanded constant, a head variable takes it
                std::map<u32, u32> bind;
                bool ok = true;
                auto unify = [&](const kb_term& t, u32 v) {
                    if (v == ANY) return;
                    if (!t.is_var) { ok = ok && t.value == v; return; }
                    auto it = bind.find(t.value);
                    if (it == bind.end()) bind[t.value] = v;
                    else ok = ok && it->second == v;
                };
                unify(h.s, x.x);
                unify(h.o, x.y);
                if (!ok) continue;
                d->relevant[r] = true;
                auto term = [&](const kb_term& t) {
                    if (!t.is_var) return t.value;
                    auto it = bind.find(t.value);
                    return it == bind.end() ? ANY : it->second;
                };
                for (u32 i = 0; i < rule.n_premise; i++) add(rule.premise[i].p.value, make_uint2(term(rule.premise[i].s), term(rule.premise[i].o)));
            }
        }
    }
    d->n_patterns = 0;
    for (auto& kv : d->pats) d->n_patterns += (u32)kv.second.size();
}

kb_status bc_demand_upload(kb_ctx* ctx, const BcDemand& d, const std::vector<u32>& preds, BcDemandDev* out) {
    // a predicate nothing demands gets an empty pattern list (none of its facts is needed); one with (any, any) is not restricted. When
    // the patterns exceed the device table, the predicates with the most patterns are left unrestricted until the rest fit.
    std::vector<std::pair<u32, std::vector<uint2>>> lists;
    for (u32 p : preds) {
        auto it = d.pats.find(p);
        if (it == d.pats.end()) { lists.push_back({p, {}}); continue; }
        if (it->second.size() == 1 && it->second[0].x == ANY && it->second[0].y == ANY) continue;
        lists.push_back({p, it->second});
    }
    std::stable_sort(lists.begin(), lists.end(), [](const auto& a, const auto& b) { return a.second.size() < b.second.size(); });
    std::vector<uint2> tab;
    std::vector<std::pair<u32, std::pair<u32, u32>>> at;  // predicate -> (first, count)
    for (auto& l : lists) {
        if (tab.size() + l.second.size() > BC_MAX_DEMAND) break;
        at.push_back({l.first, {(u32)tab.size(), (u32)l.second.size()}});
        tab.insert(tab.end(), l.second.begin(), l.second.end());
    }
    out->of.clear();
    if (at.empty()) return KB_OK;
    KB_TRY(alloc_buf(ctx, BC_MAX_DEMAND * sizeof(uint2), &out->tab));
    // (from pageable memory: the call returns once `tab` has been staged, so the vector may go out of scope before the copy runs)
    if (!tab.empty()) KB_CUDA(ctx, cudaMemcpyAsync(out->tab->p, tab.data(), tab.size() * sizeof(uint2), cudaMemcpyHostToDevice, ctx->st));
    const uint2* base = static_cast<const uint2*>(out->tab->p);
    for (auto& a : at) out->of[a.first] = {base + a.second.first, a.second.second};
    return KB_OK;
}

// ---- kernels and their launch formats (private to this file)
// out = the rows (s,o) that match one of the n_dem demand patterns, in no particular order; *out_count = their number (zeroed)
static __global__ void __launch_bounds__(256) bc_demand_select_kernel(const u32* __restrict__ s, const u32* __restrict__ o, u32 n, const uint2* dem,
                                                                      u32 n_dem, u32* out_s, u32* out_o, u32* out_count) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        u32 a = 0, b = 0;
        bool take = false;
        if (i < n) {
            a = s[i];
            b = o[i];
            take = bc_demanded(dem, n_dem, a, b);
        }
        emit_pair(take, a, b, out_s, out_o, out_count);
    }
}
static void launch_bc_demand_select(const u32* s, const u32* o, u32 n, const uint2* dem, u32 n_dem, u32* out_s, u32* out_o, u32* out_count,
                                    int n_sms, cudaStream_t st) {
    if (n == 0) return;
    bc_demand_select_kernel<<<grid_1d(n, n_sms), 256, 0, st>>>(s, o, n, dem, n_dem, out_s, out_o, out_count);
}

// The answer pass of kb_datalog_query over n rows of (s, p, o) (in[k] null: every row holds cval[k] there): a row matches the query when
// every constant position holds q_val and every repeated variable holds the value of its first position; the projection onto the
// query's n_vars distinct variables (out column j = the value at position var_pos[j]) enters a key set (64-bit keys up to 2 variables,
// 96-bit keys for 3) and is appended to out[] when it was new.
struct BcAnswerParams {
    const u32* in[3];
    u32 cval[3];
    u32 n;
    u32 q_is_var[3], q_val[3];  // per position: a variable (q_val = the position of its first appearance) or the constant q_val
    u32 n_vars, var_pos[3];
    u64* set64;                 // n_vars <= 2
    uint4* set96;               // n_vars == 3
    u32 set_slots;              // power of two
    u32* out[3];
    u32 out_cap;
    u32* out_count;
    u32* overflow;              // set or output full
    // kb_datalog_query_repairs (null for kb_datalog_query): a row whose fact (s, p, o) is in the fact set `excl` at a slot whose byte
    // excl_flag[slot] is non-zero is dropped
    const uint4* excl;
    u32 excl_slots;
    const u8* excl_flag;
};
static __global__ void __launch_bounds__(256) bc_answer_kernel(const __grid_constant__ BcAnswerParams P) {
    const int lane = threadIdx.x & 31;
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (P.n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        u32 v[3] = {0, 0, 0}, key[3] = {0, 0, 0};
        bool fresh = false;
        if (i < P.n) {
            bool ok = true;
#pragma unroll
            for (int k = 0; k < 3; k++) v[k] = P.in[k] ? P.in[k][i] : P.cval[k];
#pragma unroll
            for (int k = 0; k < 3; k++) ok = ok && (P.q_is_var[k] ? v[k] == v[P.q_val[k]] : v[k] == P.q_val[k]);
            if (ok && P.excl) {
                const u32 slot = set_find(P.excl, P.excl_slots, v[0], v[1], v[2]);
                ok = slot == EMPTY32 || P.excl_flag[slot] == 0;
            }
            if (ok) {
#pragma unroll
                for (int j = 0; j < 3; j++) key[j] = j < (int)P.n_vars ? v[P.var_pos[j]] : 0u;
                const u32 r = P.n_vars == 3 ? set_insert(P.set96, P.set_slots, key[0], key[1], key[2])
                                            : set64_insert(P.set64, P.set_slots, key[0], key[1]);
                if (r == 2u) *P.overflow = 1u;
                fresh = r == 1u;
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, fresh);
        if (!m) continue;
        u32 base = 0;
        if (lane == __ffs(m) - 1) base = atomicAdd(P.out_count, (u32)__popc(m));
        base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
        if (fresh) {
            const u32 r = base + (u32)__popc(m & ((1u << lane) - 1u));
            if (r < P.out_cap) {
                for (u32 j = 0; j < P.n_vars; j++) P.out[j][r] = key[j];
            } else *P.overflow = 1u;
        }
    }
}
static void launch_bc_answer(const BcAnswerParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    bc_answer_kernel<<<grid_1d(p.n, n_sms), 256, 0, st>>>(p);
}

// ---- host side of the two passes
kb_status bc_demand_select(kb_ctx* ctx, const uint2* dem, u32 n_dem, const Col& s, const Col& o, u64 n, Col* out_s, Col* out_o, u32 count_word) {
    KB_TRY(alloc_col(ctx, n, out_s));
    KB_TRY(alloc_col(ctx, n, out_o));
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + count_word, 0, sizeof(u32), ctx->st));
    timer_begin(ctx, F_FILTER);
    launch_bc_demand_select(s.ptr, o.ptr, (u32)n, dem, n_dem, out_s->ptr, out_o->ptr, ctx->ctrl + count_word, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

kb_status bc_answer(kb_ctx* ctx, const kb_pattern& q, const std::vector<BcSource>& src, std::unique_ptr<kb_rel>* out, const BcExclude* excl) {
    // the query's distinct variables in s, p, o first-appearance order (kb_scan's column order)
    BcAnswerParams P{};
    if (excl) {
        P.excl = excl->set;
        P.excl_slots = excl->slots;
        P.excl_flag = excl->flag;
    }
    const kb_term* qt[3] = {&q.s, &q.p, &q.o};
    std::vector<u32> slots;
    for (u32 k = 0; k < 3; k++) {
        P.q_is_var[k] = qt[k]->is_var;
        if (!qt[k]->is_var) { P.q_val[k] = qt[k]->value; continue; }
        u32 first = k;
        for (u32 j = 0; j < k; j++) if (qt[j]->is_var && qt[j]->value == qt[k]->value) { first = j; break; }
        P.q_val[k] = first;
        if (first == k) { P.var_pos[slots.size()] = k; slots.push_back(qt[k]->value); }
    }
    P.n_vars = (u32)slots.size();
    u64 rows = 0;
    for (auto& sc : src) rows += sc.n;
    if (rows >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "the answer pass reads more than 2^32 - 16 rows");
    u64 slots_n = 1024;
    while (slots_n < 2 * rows) slots_n <<= 1;
    if (slots_n > (1ull << 31)) return fail(ctx, KB_E_LIMIT, "the answer set would need more than 2^31 slots");
    Buf set;
    const size_t slot_bytes = P.n_vars == 3 ? sizeof(uint4) : sizeof(u64);
    KB_TRY(alloc_buf(ctx, slots_n * slot_bytes, &set));
    // 64-bit keys: all ones is the empty slot; 96-bit slots: state word 0 is free
    KB_CUDA(ctx, cudaMemsetAsync(set->p, P.n_vars == 3 ? 0x00 : 0xFF, slots_n * slot_bytes, ctx->st));
    if (P.n_vars == 3) P.set96 = static_cast<uint4*>(set->p);
    else P.set64 = static_cast<u64*>(set->p);
    P.set_slots = (u32)slots_n;
    auto res = std::make_unique<kb_rel>();
    res->slots = slots;
    for (u32 j = 0; j < P.n_vars; j++) {
        Col c;
        KB_TRY(alloc_col(ctx, std::max<u64>(rows, 1), &c));
        res->cols.push_back(c);
        P.out[j] = c.ptr;
    }
    P.out_cap = (u32)std::max<u64>(rows, 1);
    const u32 off = ctrl_alloc(ctx, 2);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 2 * sizeof(u32), ctx->st));
    P.out_count = ctx->ctrl + off;
    P.overflow = ctx->ctrl + off + 1;
    timer_begin(ctx, F_BUILD, (int)std::max<size_t>(src.size(), 1));
    for (auto& sc : src) {
        for (int k = 0; k < 3; k++) { P.in[k] = sc.in[k]; P.cval[k] = sc.cval[k]; }
        P.n = (u32)sc.n;
        launch_bc_answer(P, ctx->n_sms, ctx->st);
    }
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    if (ctx->h_ctrl[off + 1]) return fail(ctx, KB_E_LIMIT, "answer set overflow");
    res->n = ctx->h_ctrl[off];
    *out = std::move(res);
    return KB_OK;
}

}  // namespace kb
