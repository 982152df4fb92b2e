// kb_repairs.cu — kb_datalog_query_repairs: Reasoner::query_with_repairs (datalog/src/reasoning/repairs.rs:10-43) under IAR semantics.
//
// The constraints are denial constraints: a fact set violates one iff its premises match inside the set, which is monotone in the set.
// So the minimal inconsistent subsets of the store are the minimal ones among the fact sets of single matches, and a fact lies in every
// maximal repair iff it lies in none of them. The call computes that set of facts and answers the query over the rest:
//   matches       each constraint's premises through kb_bgp_execute (bgp_execute_impl)
//   K1 conflict   per match row: instantiate the premises, enter each fact into the fact set F (96-bit keys, 16-byte slots; a fact's id
//                 is its slot), sort the d <= 6 distinct ids in registers, enter (ids, d) into the conflict set C (32-byte slots), and
//                 keep the smallest and largest d
//   K2 minimal    per slot of C: with dmin < dmax, probe each proper subset of at least dmin ids in C (at most 62); a conflict without
//                 a sub-conflict is minimal (with dmin == dmax every conflict is, and no probe runs) and flags its facts in a byte
//                 array over F's slots
//   answer        the query's matches (scan_store, one pattern) through bc_answer, which drops a match whose fact has its flag set
// Byte model. K1 per match row: 4 B per variable column read; per premise one 16-byte slot of F probed (and written once per distinct
// fact); one 32-byte slot of C. K2 per slot of C: 32 B read; with the probe up to 62 more 32-byte slots; per minimal conflict d atomic
// byte flags. The answer pass per query match: its columns, one 16-byte slot of F and one flag byte.
#include <algorithm>

#include "kb_internal.hpp"

namespace kb {
namespace {

constexpr u32 NP = KB_MAX_PREMISES;  // conflict ids per key
static_assert(NP == 6, "the conflict key holds 6 ids and a state word in 32 bytes");

struct ConflictParams {
    const u32* col[KB_MAX_COLS];     // the match rows' variable columns
    u32 n;                           // match rows
    u32 np;                          // premises
    u32 tcol[NP][3];                 // per premise and position: the column that holds the term, or EMPTY32 for a constant ...
    u32 tval[NP][3];                 // ... which is this id
    uint4* facts;                    // F: {s, p, o, state}
    u32 fact_slots;
    uint4* conf;                     // C: two uint4 per slot: {id0, id1, id2, id3}, {id4, id5, d, state}
    u32 conf_slots;
    u32* ctrl;                       // [0] distinct conflicts, [1] dmin, [2] dmax, [3] overflow
};
struct MinimalParams {
    const uint4* conf;
    u32 conf_slots;
    u32 probe;                       // 0: every conflict is minimal
    u32 dmin;
    u32* flag_words;                 // the fact flags: byte `slot` of this array
    u32* ctrl;                       // [4] minimal conflicts, [5] conflicted facts
};

__device__ __forceinline__ void cswap(u32& a, u32& b) {
    const u32 lo = min(a, b), hi = max(a, b);
    a = lo;
    b = hi;
}
// ascending, EMPTY32 (free entries) last
__device__ __forceinline__ void sort6(u32 (&v)[NP]) {
#pragma unroll
    for (int i = 0; i < 6; i++)
#pragma unroll
        for (int j = (i & 1); j + 1 < 6; j += 2) cswap(v[j], v[j + 1]);
}
__device__ __forceinline__ u32 conf_hash(const u32 (&v)[NP]) {
    u32 h = 0x2545F491u;
#pragma unroll
    for (int i = 0; i < 6; i++) h = mix32(h ^ (v[i] * 0x9E3779B1u + (u32)i));
    return h;
}
__device__ __forceinline__ bool conf_equal(const uint4 a, const uint4 b, const u32 (&v)[NP]) {
    return a.x == v[0] && a.y == v[1] && a.z == v[2] && a.w == v[3] && b.x == v[4] && b.y == v[5];
}
// 1 inserted now, 0 already there, 2 table full
__device__ __forceinline__ u32 conf_insert(uint4* set, u32 n_slots, const u32 (&v)[NP], u32 d) {
    const u32 mask = n_slots - 1u;
    u32 slot = conf_hash(v) & mask;
    for (u32 probes = 0; probes < n_slots; probes++) {
        u32* st_ptr = reinterpret_cast<u32*>(&set[2 * slot + 1]) + 3;
        u32 st = atomicCAS(st_ptr, 0u, 1u);
        if (st == 0u) {
            set[2 * slot] = make_uint4(v[0], v[1], v[2], v[3]);
            u32* w = reinterpret_cast<u32*>(&set[2 * slot + 1]);
            w[0] = v[4]; w[1] = v[5]; w[2] = d;
            __threadfence();
            atomicExch(st_ptr, 2u);
            return 1u;
        }
        while (st == 1u) st = *reinterpret_cast<volatile u32*>(st_ptr);
        __threadfence();
        const volatile u32* w = reinterpret_cast<const volatile u32*>(&set[2 * slot]);
        const uint4 a = make_uint4(w[0], w[1], w[2], w[3]), b = make_uint4(w[4], w[5], w[6], w[7]);
        if (conf_equal(a, b, v)) return 0u;
        slot = (slot + 1u) & mask;
    }
    return 2u;
}
__device__ __forceinline__ bool conf_find(const uint4* set, u32 n_slots, const u32 (&v)[NP]) {
    const u32 mask = n_slots - 1u;
    u32 slot = conf_hash(v) & mask;
    for (u32 probes = 0; probes < n_slots; probes++) {
        const uint4 b = set[2 * slot + 1];
        if (b.w == 0u) return false;
        if (conf_equal(set[2 * slot], b, v)) return true;
        slot = (slot + 1u) & mask;
    }
    return false;
}

__global__ void __launch_bounds__(256) rp_conflict_kernel(const __grid_constant__ ConflictParams P) {
    u32 dmin = 0xFFFFFFFFu, dmax = 0, fresh = 0;
    bool overflow = false;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        u32 id[NP];
#pragma unroll
        for (int k = 0; k < (int)NP; k++) {
            id[k] = EMPTY32;
            if (k >= (int)P.np) continue;
            u32 t[3];
#pragma unroll
            for (int j = 0; j < 3; j++) t[j] = P.tcol[k][j] == EMPTY32 ? P.tval[k][j] : __ldg(P.col[P.tcol[k][j]] + i);
            u32 at = EMPTY32;
            if (set_insert_at(P.facts, P.fact_slots, t[0], t[1], t[2], &at) == 2u) overflow = true;
            id[k] = at;
        }
        if (overflow) continue;
        // the distinct ids: sort, blank each repeat (compared with its unblanked left neighbour), sort the blanks to the end
        sort6(id);
#pragma unroll
        for (int k = 5; k > 0; k--) if (id[k] == id[k - 1]) id[k] = EMPTY32;
        sort6(id);
        u32 d = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) d += id[k] != EMPTY32 ? 1u : 0u;
        const u32 r = conf_insert(P.conf, P.conf_slots, id, d);
        if (r == 2u) overflow = true;
        fresh += r == 1u ? 1u : 0u;
        dmin = min(dmin, d);
        dmax = max(dmax, d);
    }
    // one atomic per warp for each statistic
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        fresh += __shfl_xor_sync(0xffffffffu, fresh, s);
        dmin = min(dmin, __shfl_xor_sync(0xffffffffu, dmin, s));
        dmax = max(dmax, __shfl_xor_sync(0xffffffffu, dmax, s));
    }
    if (__any_sync(0xffffffffu, overflow) && (threadIdx.x & 31) == 0) P.ctrl[3] = 1u;
    if ((threadIdx.x & 31) == 0 && dmax) {
        atomicAdd(P.ctrl + 0, fresh);
        atomicMin(P.ctrl + 1, dmin);
        atomicMax(P.ctrl + 2, dmax);
    }
}

__global__ void __launch_bounds__(256) rp_minimal_kernel(const __grid_constant__ MinimalParams P) {
    for (u32 c = blockIdx.x * blockDim.x + threadIdx.x; c < P.conf_slots; c += gridDim.x * blockDim.x) {
        const uint4 b = P.conf[2 * c + 1];
        if (b.w == 0u) continue;
        const uint4 a = P.conf[2 * c];
        const u32 id[NP] = {a.x, a.y, a.z, a.w, b.x, b.y};
        const u32 d = b.z;
        bool minimal = true;
        if (P.probe) {
            // proper subsets of at least dmin ids; a subset of sorted ids, compacted by the sort, is a key in canonical form
            for (u32 m = 1; minimal && m + 1 < (1u << d); m++) {
                if ((u32)__popc(m) < P.dmin) continue;
                u32 sub[NP];
#pragma unroll
                for (int k = 0; k < 6; k++) sub[k] = (m >> k) & 1u ? id[k] : EMPTY32;
                sort6(sub);
                if (conf_find(P.conf, P.conf_slots, sub)) minimal = false;
            }
        }
        if (!minimal) continue;
        atomicAdd(P.ctrl + 4, 1u);
        u32 newly = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) {
            if ((u32)k >= d) break;
            const u32 bit = 1u << ((id[k] & 3u) * 8u);
            newly += (atomicOr(P.flag_words + (id[k] >> 2), bit) & bit) ? 0u : 1u;
        }
        if (newly) atomicAdd(P.ctrl + 5, newly);
    }
}

}  // namespace
}  // namespace kb

using namespace kb;

// Reasoner::query_with_repairs under IAR semantics (file comment). Reads the store and leaves it, its index and every state kept for the
// forward calls as they were.
extern "C" kb_status kb_datalog_query_repairs(kb_ctx* ctx, const kb_rule* constraints, uint32_t n_constraints, const kb_pattern* query,
                                              kb_rel** out, kb_repair_stats* stats) {
    KB_ENTER(ctx);
    if ((n_constraints && !constraints) || !query || !out) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (ctx->shard_world > 1) return fail(ctx, KB_E_UNSUPPORTED, "a sharded context: constraints are checked against one store");
    auto pattern_ok = [&](const kb_pattern& pt, const char* what, u32 r) -> kb_status {
        for (const kb_term* t : {&pt.s, &pt.p, &pt.o})
            if (t->is_var == KB_TERM_QUOTED) return fail(ctx, KB_E_UNSUPPORTED, "%s %u: a quoted-triple term (it matches no fact)", what, r);
        return check_pattern(ctx, pt);
    };
    KB_TRY(pattern_ok(*query, "query", 0));
    for (u32 r = 0; r < n_constraints; r++) {
        const kb_rule& c = constraints[r];
        if (c.n_premise > KB_MAX_PREMISES) return fail(ctx, KB_E_LIMIT, "constraint %u: %u premises (at most %d)", r, c.n_premise, KB_MAX_PREMISES);
        if (c.n_premise && !c.premise) return fail(ctx, KB_E_INVALID, "constraint %u: NULL premise array", r);
        std::vector<u32> slots, src;
        for (u32 i = 0; i < c.n_premise; i++) {
            KB_TRY(pattern_ok(c.premise[i], "constraint", r));
            pattern_vars(c.premise[i], &slots, &src);
        }
        if (slots.size() > KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "constraint %u: more than %d variables", r, KB_MAX_COLS);
    }
    ScopedEvent ev0, ev1, ev2, ev3;
    cudaEventRecord(ev0, ctx->st);
    kb_repair_stats rs{};

    // ---- matches of every constraint body (all of them first: the sets are sized once from their rows)
    std::vector<std::pair<const kb_rule*, std::unique_ptr<kb_rel>>> bodies;
    u64 fact_refs = 0;
    for (u32 r = 0; r < n_constraints; r++) {
        const kb_rule& c = constraints[r];
        if (c.n_premise == 0) continue;  // never fires
        rs.constraints++;
        std::unique_ptr<kb_rel> m;
        KB_TRY(bgp_execute_impl(ctx, c.premise, c.n_premise, nullptr, 0, nullptr, 0, &m));
        if (m->n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "constraint %u has more than 2^32 - 16 matches", r);
        rs.matches += m->n;
        fact_refs += (u64)c.n_premise * m->n;
        if (m->n) bodies.push_back({&c, std::move(m)});
    }
    cudaEventRecord(ev1, ctx->st);

    // ---- conflicts and the flags of the facts in minimal ones
    BcExclude excl;
    Buf facts, conf, flags;
    if (!bodies.empty()) {
        u64 fact_slots = 1024, conf_slots = 1024;
        while (fact_slots < 2 * fact_refs) fact_slots <<= 1;
        while (conf_slots < 2 * rs.matches) conf_slots <<= 1;
        if (fact_slots > (1ull << 31)) return fail(ctx, KB_E_LIMIT, "the fact set would need more than 2^31 slots");
        if (conf_slots > (1ull << 31)) return fail(ctx, KB_E_LIMIT, "the conflict set would need more than 2^31 slots");
        KB_TRY(alloc_buf(ctx, fact_slots * sizeof(uint4), &facts));
        KB_TRY(alloc_buf(ctx, conf_slots * 2 * sizeof(uint4), &conf));
        KB_TRY(alloc_buf(ctx, fact_slots, &flags));
        KB_CUDA(ctx, cudaMemsetAsync(facts->p, 0, fact_slots * sizeof(uint4), ctx->st));
        KB_CUDA(ctx, cudaMemsetAsync(conf->p, 0, conf_slots * 2 * sizeof(uint4), ctx->st));
        KB_CUDA(ctx, cudaMemsetAsync(flags->p, 0, fact_slots, ctx->st));
        const u32 off = ctrl_alloc(ctx, 6);
        const u32 init[6] = {0u, 0xFFFFFFFFu, 0u, 0u, 0u, 0u};  // (pageable: staged before the call returns)
        KB_CUDA(ctx, cudaMemcpyAsync(ctx->ctrl + off, init, sizeof init, cudaMemcpyHostToDevice, ctx->st));
        ConflictParams K{};
        K.facts = static_cast<uint4*>(facts->p);
        K.fact_slots = (u32)fact_slots;
        K.conf = static_cast<uint4*>(conf->p);
        K.conf_slots = (u32)conf_slots;
        K.ctrl = ctx->ctrl + off;
        timer_begin(ctx, F_BUILD, (int)bodies.size());
        for (auto& b : bodies) {
            const kb_rule& c = *b.first;
            const kb_rel& m = *b.second;
            for (size_t j = 0; j < m.cols.size(); j++) K.col[j] = m.cols[j].ptr;
            K.n = (u32)m.n;
            K.np = c.n_premise;
            for (u32 k = 0; k < c.n_premise; k++) {
                const kb_term* t[3] = {&c.premise[k].s, &c.premise[k].p, &c.premise[k].o};
                for (int j = 0; j < 3; j++) {
                    K.tcol[k][j] = t[j]->is_var ? (u32)m.col_of(t[j]->value) : EMPTY32;
                    K.tval[k][j] = t[j]->is_var ? 0u : t[j]->value;
                }
            }
            rp_conflict_kernel<<<grid_1d(m.n, ctx->n_sms), 256, 0, ctx->st>>>(K);
        }
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        if (ctx->h_ctrl[off + 3]) return fail(ctx, KB_E_LIMIT, "internal: the fact or conflict set filled up");
        rs.conflicts = ctx->h_ctrl[off];
        const u32 dmin = ctx->h_ctrl[off + 1], dmax = ctx->h_ctrl[off + 2];
        rs.subsets_probed = dmin != dmax ? 1u : 0u;
        MinimalParams M{};
        M.conf = K.conf;
        M.conf_slots = K.conf_slots;
        M.probe = rs.subsets_probed;
        M.dmin = dmin;
        M.flag_words = static_cast<u32*>(flags->p);
        M.ctrl = K.ctrl;
        timer_begin(ctx, F_BUILD);
        rp_minimal_kernel<<<grid_1d(conf_slots, ctx->n_sms), 256, 0, ctx->st>>>(M);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        rs.minimal_conflicts = ctx->h_ctrl[off + 4];
        rs.conflicted_facts = ctx->h_ctrl[off + 5];
        excl.set = K.facts;
        excl.slots = K.fact_slots;
        excl.flag = static_cast<const u8*>(flags->p);
    }
    bodies.clear();
    cudaEventRecord(ev2, ctx->st);

    // ---- answers: the query's matches in the store, minus the facts of minimal conflicts, each distinct binding once
    std::vector<std::unique_ptr<kb_rel>> scanned;
    KB_TRY(scan_store(ctx, query, 1, {}, &scanned));
    const kb_rel& qm = *scanned[0];
    std::vector<BcSource> src(1);
    const kb_term* qt[3] = {&query->s, &query->p, &query->o};
    for (int k = 0; k < 3; k++) {
        if (qt[k]->is_var) src[0].in[k] = qm.cols[qm.col_of(qt[k]->value)].ptr;
        else src[0].cval[k] = qt[k]->value;
    }
    src[0].n = qm.n;
    if (!src[0].n) src.clear();
    std::unique_ptr<kb_rel> res;
    KB_TRY(bc_answer(ctx, *query, src, &res, excl.set ? &excl : nullptr));
    cudaEventRecord(ev3, ctx->st);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    timers_flush(ctx);
    float ms[3] = {0.f, 0.f, 0.f}, all = 0.f;
    cudaEventElapsedTime(&ms[0], ev0, ev1);
    cudaEventElapsedTime(&ms[1], ev1, ev2);
    cudaEventElapsedTime(&ms[2], ev2, ev3);
    cudaEventElapsedTime(&all, ev0, ev3);
    rs.answers = res->n;
    rs.device_ms = all;
    rs.match_ms = ms[0];
    rs.conflict_ms = ms[1];
    rs.answer_ms = ms[2];
    if (stats) *stats = rs;
    ctx->stats.rows_out = res->n;
    *out = res.release();
    return KB_OK;
}
