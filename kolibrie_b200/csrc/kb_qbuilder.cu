// kb_qbuilder.cu — QueryBuilder triple queries (query_builder.rs:355-643) over the device store: what apply_filters, apply_join and the
// get_* result methods compute, without decoding a triple to text.
//
// kb_qb_triples runs four phases, each timed in kb_qb_info.phase_ms:
//   match      one pass over the device dictionary per CONTAINS / STARTS / ENDS filter (qb_match_kernel): bit id of a bitmap over the
//              ids is set when the id's string matches. A text filter is thereby decided once per distinct term instead of once per
//              triple. A warp takes 32 consecutive ids and writes their bitmap word with one ballot. STARTS / ENDS read at most m bytes
//              of each string; CONTAINS is tested by each lane on its own string up to QB_LONG bytes, and by the whole warp, one string
//              at a time, on longer ones (the lanes try 32 start positions at once), so a long literal does not stall its warp's other
//              31 strings behind one thread. The pattern sits in shared memory (at most KB_QB_PATTERN_MAX bytes).
//   selection  one pass over the raw store rows (qb_select_kernel): each position's test (id equality or the bitmap bit; a quoted id
//              or an id past the dictionary fails a text filter) and the survivors compacted, a warp reserving its slots with one
//              atomic. No filter: no pass, the segments go to the sort as they are.
//   sort       store_distinct (kb_serialize.cu) of the survivors: ascending (s, p, o), duplicates dropped (the BTreeSet<Triple>).
//   join       per KB_QB_ON_* condition the distinct (key, carried) pairs of the filtered set and of the whole right store (a sort and
//              a unique of packed u64 pairs each), the exact output size as sum over left pairs of the right pairs with the key
//              (binary searches in the sorted right pairs), then hash_join_impl of the two pair relations. A condition's output is
//              duplicate-free already (per key it is the product of two distinct sets); the union of the conditions and its order
//              come from store_distinct again.
// OFFSET / LIMIT are a slice of the sorted rows; the result columns are split from it (qb_split_kernel).
// kb_qb_terms renders a column as Dictionary::decode(id).unwrap_or("") (decode_ids' Plain mode, kb_dict.cu): every row, the rows that
// decode, or the distinct strings of those in byte order (a sort-unique of the ids, rank_values of kb_order.cu over their texts, the
// ids scattered into rank order and rendered).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>

#include "kb_internal.hpp"

using kb::u32;
using kb::u64;
using kb::u8;

namespace kb {
namespace {

constexpr int QT = 256;     // threads per block of every kernel here
constexpr u32 QB_LONG = 128;  // CONTAINS: strings longer than this are searched by the whole warp

__device__ __forceinline__ bool bytes_at(const u8* __restrict__ s, const u8* __restrict__ pat, u32 m) {
    for (u32 k = 0; k < m; k++)
        if (__ldg(s + k) != pat[k]) return false;
    return true;
}

// bits[w] bit l = string of id 32 w + l matches `mode` against the m pattern bytes (KB_QB_CONTAINS / _STARTS / _ENDS)
__global__ void __launch_bounds__(QT) qb_match_kernel(const unsigned long long* __restrict__ off, const u8* __restrict__ bytes, u32 n_ids,
                                                      const u8* __restrict__ pattern, u32 m, u32 mode, u32* __restrict__ bits) {
    extern __shared__ u8 pat[];
    for (u32 k = threadIdx.x; k < m; k += blockDim.x) pat[k] = pattern[k];
    __syncthreads();
    const u32 lane = threadIdx.x & 31u;
    const u32 n_words = (n_ids + 31u) >> 5;
    const u32 warps = (gridDim.x * blockDim.x) >> 5;
    for (u32 w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_words; w += warps) {
        const u32 id = (w << 5) + lane;
        const bool valid = id < n_ids;
        unsigned long long a = 0;
        u32 len = 0;
        if (valid) {
            a = off[id];
            len = (u32)(off[id + 1] - a);
        }
        const u8* s = bytes + a;
        bool hit = false, longs = false;
        if (valid && len >= m) {
            if (mode == KB_QB_STARTS) hit = bytes_at(s, pat, m);
            else if (mode == KB_QB_ENDS) hit = bytes_at(s + (len - m), pat, m);
            else if (len > QB_LONG) longs = true;
            else
                for (u32 i = 0; i + m <= len && !hit; i++) hit = bytes_at(s + i, pat, m);
        }
        // CONTAINS on long strings: the warp searches each one, 32 start positions a step
        for (u32 todo = __ballot_sync(0xffffffffu, longs); todo; todo &= todo - 1u) {
            const u32 r = (u32)__ffs(todo) - 1u;
            const unsigned long long ra = __shfl_sync(0xffffffffu, a, r);
            const u32 rl = __shfl_sync(0xffffffffu, len, r);
            const u8* rs = bytes + ra;
            bool found = false;
            for (u32 base = 0; base + m <= rl && !found; base += 32u) {
                const u32 i = base + lane;
                found = __any_sync(0xffffffffu, i + m <= rl && bytes_at(rs + i, pat, m));
            }
            if (lane == r) hit = found;
        }
        const u32 word = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) bits[w] = word;
    }
}

struct PosTest {
    u32 mode;  // 0 any, 1 id equality, 2 bitmap bit
    u32 id;
    const u32* bits;
};
struct SelectParams {
    PosTest t[3];
    u32 dict_ids;
    const u32 *s, *p, *o;
    u64 n;
    u32 *os, *op, *oo;  // survivors, at *count and on
    u32* count;
};

__device__ __forceinline__ bool pos_pass(const PosTest& t, u32 id, u32 dict_ids) {
    if (t.mode == 0) return true;
    if (t.mode == 1) return id == t.id;
    return id < dict_ids && ((__ldg(t.bits + (id >> 5)) >> (id & 31u)) & 1u);
}

__global__ void __launch_bounds__(QT) qb_select_kernel(const __grid_constant__ SelectParams P) {
    const u32 lane = threadIdx.x & 31u;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 base = blockIdx.x * (u64)blockDim.x + (threadIdx.x & ~31u); base < P.n; base += stride) {
        const u64 i = base + lane;
        u32 s = 0, p = 0, o = 0;
        bool keep = false;
        if (i < P.n) {
            s = P.s[i];
            p = P.p[i];
            o = P.o[i];
            keep = pos_pass(P.t[0], s, P.dict_ids) && pos_pass(P.t[1], p, P.dict_ids) && pos_pass(P.t[2], o, P.dict_ids);
        }
        const u32 b = __ballot_sync(0xffffffffu, keep);
        if (!b) continue;
        u32 at = 0;
        if (lane == 0) at = atomicAdd(P.count, (u32)__popc(b));
        at = __shfl_sync(0xffffffffu, at, 0);
        if (keep) {
            const u32 r = at + (u32)__popc(b & ((1u << lane) - 1u));
            P.os[r] = s;
            P.op[r] = p;
            P.oo[r] = o;
        }
    }
}

// rows [lo, lo + n) of the sorted (S, PO) as three columns
__global__ void __launch_bounds__(QT) qb_split_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u64 lo, u64 n,
                                                      u32* __restrict__ s, u32* __restrict__ p, u32* __restrict__ o) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const unsigned long long po = PO[lo + i];
        s[i] = S[lo + i];
        p[i] = (u32)(po >> 32);
        o[i] = (u32)po;
    }
}

__global__ void __launch_bounds__(QT) qb_pack_kernel(const u32* __restrict__ key, const u32* __restrict__ car, u64 n, unsigned long long* __restrict__ out) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        out[i] = (unsigned long long)key[i] << 32 | car[i];
}

__global__ void __launch_bounds__(QT) qb_unpack_kernel(const unsigned long long* __restrict__ in, u32 n, u32* __restrict__ key, u32* __restrict__ car) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long x = in[i];
        key[i] = (u32)(x >> 32);
        car[i] = (u32)x;
    }
}

__device__ __forceinline__ u32 lower_bound_u64(const unsigned long long* a, u32 n, unsigned long long x) {
    u32 lo = 0, len = n;
    while (len > 0) {
        const u32 h = len >> 1;
        if (a[lo + h] < x) { lo += h + 1; len -= h + 1; }
        else len = h;
    }
    return lo;
}

// *total += for each left pair, the right pairs with its key (both sorted, packed key << 32 | carried)
__global__ void __launch_bounds__(QT) qb_join_count_kernel(const unsigned long long* __restrict__ L, u32 nl, const unsigned long long* __restrict__ R, u32 nr,
                                                           unsigned long long* total) {
    unsigned long long t = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += gridDim.x * blockDim.x) {
        const unsigned long long k = L[i] & 0xFFFFFFFF00000000ull;
        const u32 a = lower_bound_u64(R, nr, k);
        const u32 b = (k >> 32) == 0xFFFFFFFFull ? nr : lower_bound_u64(R, nr, k + (1ull << 32));
        t += b - a;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(total, t);
}

struct Decodable {
    u32 n;
    __device__ bool operator()(u32 id) const { return id < n; }
};

__global__ void __launch_bounds__(QT) qb_scatter_kernel(const u32* __restrict__ ids, const u32* __restrict__ rank_of, u32 n, u32* __restrict__ out) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[rank_of[i]] = ids[i];
}

auto U = [](const Buf& b) { return static_cast<u32*>(b->p); };
auto U64 = [](const Buf& b) { return static_cast<unsigned long long*>(b->p); };

}  // namespace

// the distinct (key << 32 | carried) pairs of the n rows (key[i], car[i]), sorted: *out, *n_out of them
kb_status distinct_pairs(kb_ctx* ctx, const std::vector<std::pair<const u32*, const u32*>>& cols, const std::vector<u64>& rows, Buf* out, u32* n_out) {
    u64 n = 0;
    for (u64 r : rows) n += r;
    *n_out = 0;
    if (n == 0) return KB_OK;
    Buf raw, sorted;
    KB_TRY(alloc_buf(ctx, n * 8, &raw));
    KB_TRY(alloc_buf(ctx, n * 8, &sorted));
    KB_TRY(alloc_buf(ctx, n * 8, out));
    u64 at = 0;
    timer_begin(ctx, F_OTHER, (int)cols.size() + 2);
    for (size_t k = 0; k < cols.size(); k++) {
        if (rows[k]) qb_pack_kernel<<<grid_1d(rows[k], ctx->n_sms, QT), QT, 0, ctx->st>>>(cols[k].first, cols[k].second, rows[k], U64(raw) + at);
        at += rows[k];
    }
    const u32 c = ctrl_alloc(ctx, 1);
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, U64(raw), U64(sorted), (u32)n, 0, 64, ctx->st); }));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceSelect::Unique(t, b, U64(sorted), U64(*out), ctx->ctrl + c, (u32)n, ctx->st); }));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    *n_out = ctx->h_ctrl[c];
    return KB_OK;
}

// n sorted distinct pairs as a two-column relation over (key slot, carried slot)
kb_status pair_rel(kb_ctx* ctx, const Buf& pairs, u32 n, u32 key_slot, u32 car_slot, std::unique_ptr<kb_rel>* out) {
    auto r = std::make_unique<kb_rel>();
    r->slots = {key_slot, car_slot};
    r->cols.resize(2);
    r->n = n;
    for (Col& c : r->cols) KB_TRY(alloc_col(ctx, n, &c));
    if (n) {
        timer_begin(ctx, F_OTHER, 1);
        qb_unpack_kernel<<<grid_1d(n, ctx->n_sms, QT), QT, 0, ctx->st>>>(U64(pairs), n, r->cols[0].ptr, r->cols[1].ptr);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
    }
    *out = std::move(r);
    return KB_OK;
}

kb_status pair_join_count(kb_ctx* ctx, const Buf& lp, u32 nl, const Buf& rp, u32 nr, u64* cnt) {
    *cnt = 0;
    if (!nl || !nr) return KB_OK;
    const u32 c = ctrl_alloc(ctx, 2);
    timer_begin(ctx, F_OTHER, 1);
    qb_join_count_kernel<<<grid_1d(nl, ctx->n_sms, QT), QT, 0, ctx->st>>>(U64(lp), nl, U64(rp), nr, reinterpret_cast<unsigned long long*>(ctx->ctrl + c));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    unsigned long long v = 0;
    memcpy(&v, ctx->h_ctrl + c, sizeof v);
    *cnt = v;
    return KB_OK;
}

kb_status split_sorted(kb_ctx* ctx, const Buf& S, const Buf& PO, u64 lo, u64 n, u32* s, u32* p, u32* o) {
    if (!n) return KB_OK;
    timer_begin(ctx, F_OTHER, 1);
    qb_split_kernel<<<grid_1d(n, ctx->n_sms, QT), QT, 0, ctx->st>>>(U(S), U64(PO), lo, n, s, p, o);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

namespace {

struct JoinCond {
    u32 bit;
    int lkey, lcar;  // left position (0 s, 1 p, 2 o) of the key and of the carried id
    int rkey, rcar;  // right position
    int out[3];      // output s, p, o: 0 key, 1 left carried, 2 right carried
};
constexpr JoinCond JOINS[3] = {
    {KB_QB_ON_SUBJECT, 0, 1, 0, 2, {0, 1, 2}},    // (l.s, l.p, r.o) for l.s == r.s
    {KB_QB_ON_PREDICATE, 1, 0, 1, 2, {1, 0, 2}},  // (l.s, l.p, r.o) for l.p == r.p
    {KB_QB_ON_OBJECT, 2, 0, 2, 1, {1, 2, 0}},     // (l.s, r.p, r.o) for l.o == r.o
};

kb_status qb_triples(kb_ctx* ctx, const kb_qb_spec& spec, const kb_ctx* right, const u32* slots, kb_rel** out, kb_qb_info* info) {
    bool text = false;
    for (int k = 0; k < 3; k++) {
        const kb_qb_filter& f = spec.pos[k];
        if (f.mode > KB_QB_ENDS) return fail(ctx, KB_E_INVALID, "unknown filter mode %u at position %d", f.mode, k);
        if (f.mode >= KB_QB_CONTAINS) {
            if (f.len && !f.pattern) return fail(ctx, KB_E_INVALID, "NULL pattern at position %d", k);
            if (f.len > KB_QB_PATTERN_MAX) return fail(ctx, KB_E_LIMIT, "a pattern of %llu bytes at position %d (limit KB_QB_PATTERN_MAX = %u)",
                                                        (unsigned long long)f.len, k, KB_QB_PATTERN_MAX);
            text = true;
        }
    }
    if (spec.join & ~7u) return fail(ctx, KB_E_INVALID, "unknown join bits 0x%x", spec.join);
    const bool join = right && spec.join;
    if (right && right->device != ctx->device) return fail(ctx, KB_E_INVALID, "the right context is on device %d, this one on device %d", right->device, ctx->device);
    if (ctx->shard_world > 1 || (join && right->shard_world > 1)) return fail(ctx, KB_E_UNSUPPORTED, "a sharded context: the query reads one whole store");
    if (text && !ctx->dict_ids) return fail(ctx, KB_E_UNSUPPORTED, "text filters need the device dictionary's strings (kb_dict_strings_load)");
    u64 n_raw = 0, n_right = 0;
    std::vector<ColSpan> spans = store_spans(ctx, &n_raw), rspans;
    if (n_raw >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "a store of %llu triples (QueryBuilder: limit 2^32 - 16)", (unsigned long long)n_raw);
    if (join) {
        rspans = store_spans(right, &n_right);
        if (n_right >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "a right store of %llu triples (limit 2^32 - 16)", (unsigned long long)n_right);
    }
    info->n_raw = n_raw;
    PhaseTimer<5> pt;
    pt.mark(ctx->st);

    // ---- match: a bitmap over the ids per text filter
    SelectParams P{};
    P.dict_ids = ctx->dict_ids;
    bool none = false;  // an EXACT id with bit 31: nothing matches
    Buf bits[3];
    const u32 n_words = (ctx->dict_ids + 31u) / 32u;
    const DictTab dict = dicttab(ctx);
    for (int k = 0; k < 3; k++) {
        const kb_qb_filter& f = spec.pos[k];
        P.t[k].mode = f.mode == KB_QB_ANY ? 0u : f.mode == KB_QB_EXACT ? 1u : 2u;
        P.t[k].id = f.id;
        if (f.mode == KB_QB_EXACT && (f.id & 0x80000000u)) none = true;
        if (f.mode < KB_QB_CONTAINS || n_raw == 0) continue;
        Buf pat;
        const u32 m = (u32)f.len;
        KB_TRY(alloc_buf(ctx, (size_t)n_words * 4 + 16, &bits[k]));
        KB_TRY(alloc_buf(ctx, m + 16, &pat));
        if (m) KB_CUDA(ctx, cudaMemcpyAsync(pat->p, f.pattern, m, cudaMemcpyHostToDevice, ctx->st));
        ctx->stats.h2d_bytes += m;
        timer_begin(ctx, F_OTHER, 1);
        qb_match_kernel<<<grid_1d((u64)n_words * 32, ctx->n_sms, QT), QT, m, ctx->st>>>(dict.off, dict.bytes, dict.ids, static_cast<const u8*>(pat->p), m,
                                                                                       f.mode, U(bits[k]));
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        P.t[k].bits = U(bits[k]);
    }
    pt.mark(ctx->st);

    // ---- selection: the rows that pass, compacted
    Buf sel;
    u64 n_sel_raw = n_raw;
    const bool filtered = P.t[0].mode || P.t[1].mode || P.t[2].mode;
    if (none || n_raw == 0) {
        spans.clear();
        n_sel_raw = 0;
    } else if (filtered) {
        KB_TRY(alloc_buf(ctx, n_raw * 12, &sel));
        const u32 c = ctrl_alloc(ctx, 1);
        P.os = U(sel);
        P.op = U(sel) + n_raw;
        P.oo = U(sel) + 2 * n_raw;
        P.count = ctx->ctrl + c;
        for (const ColSpan& sp : spans) {
            if (sp.ready) KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, sp.ready, 0));
            P.s = sp.s; P.p = sp.p; P.o = sp.o; P.n = sp.n;
            timer_begin(ctx, F_OTHER, 1);
            qb_select_kernel<<<grid_1d(sp.n, ctx->n_sms, QT), QT, 0, ctx->st>>>(P);
            timer_end(ctx);
        }
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        n_sel_raw = ctx->h_ctrl[c];
        spans.assign(1, ColSpan{P.os, P.op, P.oo, n_sel_raw, nullptr});
    }
    for (Buf& b : bits) b.reset();
    pt.mark(ctx->st);

    // ---- sort + dedup: the filtered set
    Buf S, PO;
    u32 n = 0;
    if (n_sel_raw) KB_TRY(store_distinct(ctx, spans, &S, &PO, &n));
    sel.reset();
    info->n_selected = n;
    pt.mark(ctx->st);

    // ---- join with the right store
    if (join) {
        Col lc[3];
        for (Col& c : lc) KB_TRY(alloc_col(ctx, n, &c));
        KB_TRY(split_sorted(ctx, S, PO, 0, n, lc[0].ptr, lc[1].ptr, lc[2].ptr));
        S.reset(); PO.reset();
        if (n_right) KB_CUDA(ctx, cudaStreamSynchronize(right->st));  // the right store's last writes are done
        std::vector<std::unique_ptr<kb_rel>> parts;
        std::vector<ColSpan> out_spans;
        u64 total = 0;
        for (const JoinCond& jc : JOINS) {
            if (!(spec.join & jc.bit)) continue;
            Buf lp, rp;
            u32 nl = 0, nr = 0;
            KB_TRY(distinct_pairs(ctx, {{lc[jc.lkey].ptr, lc[jc.lcar].ptr}}, {n}, &lp, &nl));
            std::vector<std::pair<const u32*, const u32*>> rc;
            std::vector<u64> rrows;
            for (const ColSpan& sp : rspans) {
                if (sp.ready) KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, sp.ready, 0));
                const u32* col[3] = {sp.s, sp.p, sp.o};
                rc.push_back({col[jc.rkey], col[jc.rcar]});
                rrows.push_back(sp.n);
            }
            KB_TRY(distinct_pairs(ctx, rc, rrows, &rp, &nr));
            if (!nl || !nr) continue;
            u64 cnt = 0;
            KB_TRY(pair_join_count(ctx, lp, nl, rp, nr, &cnt));
            total += cnt;
            if (total >= 0xFFFFFFF0ull)
                return fail(ctx, KB_E_LIMIT, "the join gives %llu rows or more before the union (limit 2^32 - 16)", (unsigned long long)total);
            if (!cnt) continue;
            std::unique_ptr<kb_rel> L, R, J;
            KB_TRY(pair_rel(ctx, lp, nl, 0, 1, &L));
            KB_TRY(pair_rel(ctx, rp, nr, 0, 2, &R));
            lp.reset(); rp.reset();
            KB_TRY(hash_join_impl(ctx, *L, *R, nullptr, &J));
            if (J->n != cnt) return fail(ctx, KB_E_CUDA, "the join gave %llu rows, %llu counted", (unsigned long long)J->n, cnt);
            const u32* jcol[3] = {J->cols[J->col_of(0)].ptr, J->cols[J->col_of(1)].ptr, J->cols[J->col_of(2)].ptr};
            out_spans.push_back({jcol[jc.out[0]], jcol[jc.out[1]], jcol[jc.out[2]], J->n, nullptr});
            parts.push_back(std::move(J));
        }
        n = 0;
        if (total) KB_TRY(store_distinct(ctx, out_spans, &S, &PO, &n));
    }
    info->n_joined = n;
    pt.mark(ctx->st);

    // ---- OFFSET / LIMIT
    const u64 lo = spec.offset;
    if (lo > n) return fail(ctx, KB_E_INVALID, "offset %llu past the %u rows (the reference panics)", (unsigned long long)lo, n);
    const u64 hi = spec.limit >= (u64)n - lo ? (u64)n : lo + spec.limit;  // offset + limit saturates
    info->n_rows = hi - lo;
    if (out) {
        auto r = std::make_unique<kb_rel>();
        r->slots.assign(slots, slots + 3);
        r->n = hi - lo;
        KB_TRY(alloc_strided_cols(ctx, r->n, 3, &r->cols));
        KB_TRY(split_sorted(ctx, S, PO, lo, r->n, r->cols[0].ptr, r->cols[1].ptr, r->cols[2].ptr));
        *out = r.release();
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    for (int k = 0; k < 4; k++) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, pt.e[k], pt.e[k + 1]);
        info->phase_ms[k] = ms;
    }
    timers_flush(ctx);
    return KB_OK;
}

kb_status qb_terms(kb_ctx* ctx, const kb_rel& rows, u32 col, u32 mode, kb_strings** out) {
    auto res = std::make_unique<kb_strings>();
    const u32 n = (u32)rows.n;
    const u32* ids = rows.cols[col].ptr;
    Buf kept, sorted, uniq, ordered;
    u32 m = n;
    if (mode != KB_QB_TERMS_EMPTY && n) {  // the rows whose id decodes
        KB_TRY(alloc_buf(ctx, (size_t)n * 4, &kept));
        const u32 c = ctrl_alloc(ctx, 1);
        timer_begin(ctx, F_OTHER, 1);
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceSelect::If(t, b, ids, U(kept), ctx->ctrl + c, n, Decodable{ctx->dict_ids}, ctx->st); }));
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        m = ctx->h_ctrl[c];
        ids = U(kept);
    }
    if (mode == KB_QB_TERMS_DISTINCT && m) {  // sort-unique of the ids, their texts ranked by bytes, the ids in rank order
        KB_TRY(alloc_buf(ctx, (size_t)m * 4, &sorted));
        KB_TRY(alloc_buf(ctx, (size_t)m * 4, &uniq));
        const u32 c = ctrl_alloc(ctx, 1);
        timer_begin(ctx, F_OTHER, 2);
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, ids, U(sorted), m, 0, 32, ctx->st); }));
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceSelect::Unique(t, b, U(sorted), U(uniq), ctx->ctrl + c, m, ctx->st); }));
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        const u32 d = ctx->h_ctrl[c];
        Buf toff, tbytes, rank_of;
        KB_TRY(decode_ids(ctx, U(uniq), d, 0, Decode::Plain, "the column", &toff, &tbytes, nullptr));
        KB_TRY(alloc_buf(ctx, (size_t)d * 4, &rank_of));
        u32 n_values = 0, rounds = 0;
        KB_TRY(rank_values(ctx, d, nullptr, U(toff), static_cast<const u8*>(tbytes->p), U(rank_of), &n_values, &rounds));
        if (n_values != d) return fail(ctx, KB_E_CUDA, "%u distinct ids gave %u distinct strings", d, n_values);
        KB_TRY(alloc_buf(ctx, (size_t)d * 4, &ordered));
        timer_begin(ctx, F_OTHER, 1);
        qb_scatter_kernel<<<grid_1d(d, ctx->n_sms, QT), QT, 0, ctx->st>>>(U(uniq), U(rank_of), d, U(ordered));
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        ids = U(ordered);
        m = d;
    }
    res->n = m;
    KB_TRY(decode_ids(ctx, ids, m, 0, Decode::Plain, "the column", &res->off, &res->bytes, &res->total));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    timers_flush(ctx);
    *out = res.release();
    return KB_OK;
}

}  // namespace
}  // namespace kb

extern "C" {

kb_status kb_qb_triples(kb_ctx* ctx, const kb_qb_spec* spec, const kb_ctx* right, const uint32_t* slots, kb_rel** out, kb_qb_info* info) {
    KB_ENTER(ctx);
    kb_qb_info local{};
    if (!info) info = &local;
    *info = kb_qb_info{};
    if (out) *out = nullptr;
    if (!spec || !slots) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    return kb::qb_triples(ctx, *spec, right, slots, out, info);
}

kb_status kb_qb_terms(kb_ctx* ctx, const kb_rel* rows, uint32_t col, uint32_t mode, kb_strings** out) {
    KB_ENTER(ctx);
    if (!rows || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (col >= rows->cols.size() || rows->pair) return kb::fail(ctx, KB_E_INVALID, "column %u out of range", col);
    if (mode > KB_QB_TERMS_DISTINCT) return kb::fail(ctx, KB_E_INVALID, "unknown term-list mode %u", mode);
    if (rows->n >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "relation too large");
    if (rows->n && !ctx->dict_ids) return kb::fail(ctx, KB_E_UNSUPPORTED, "term lists need the device dictionary's strings (kb_dict_strings_load)");
    return kb::qb_terms(ctx, *rows, col, mode, out);
}

}  // extern "C"
