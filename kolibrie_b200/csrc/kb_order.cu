// kb_order.cu — ORDER BY and LIMIT over a device relation (kb_order_by): apply_order_by and the LIMIT cut that end the optimizer path
// (execute_query.rs:113-149, 693-699), so that an `ORDER BY ... LIMIT k` query downloads and decodes k rows instead of its whole result.
//
// Every key column becomes one u32 per row: the dense rank of the row's value among the column's distinct values.
//   distinct   sort-unique of the column's ids (CUB); K1 order_classify_kernel sorts every distinct id into "" / number / NaN / string,
//              counts them (a mixed column is refused) and writes a number's order key (kb_numrank.cuh's order_key_total).
//   rank       the D distinct values are ranked by refinement rounds over a global order `ord` and group starts `grp`: each round sorts
//              the positions of the unresolved groups by (group, key) with two stable radix sorts, splits the groups where the key
//              changes, and keeps only the groups that are still tied and whose strings go on. A numeric key is one round on its order
//              key; a string key has one round per 7 bytes on (next 7 bytes, big-endian | number of valid bytes), the strings rendered
//              by the decode kernels of kb_rel_decode.
//   rows       K rowrank: a lower bound over the distinct ids gives each row its rank; DESC is R - 1 - rank.
// Then either a stable LSD radix sort of row indices over the ranks, last key first (full sort), or, for a small LIMIT over at most
// two keys, a radix select of the k-th smallest packed key and an order-preserving compaction (top-k). Every column of `in` is
// gathered in the new order. Launches and device time count in kb_stats' `other` family.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>

#include "kb_internal.hpp"
#include "kb_numrank.cuh"

namespace kb {
namespace {

constexpr int OT = 256;  // threads per block of every kernel here
// top-k is taken for limit * ORDER_TOPK_RATIO <= rows: its select reads the packed keys once per 8-bit digit and its compaction twice,
// about what two passes of a radix sort cost, and it sorts only the rows below T; with a larger share of the rows kept, that sort
// approaches the full sort it was meant to avoid
constexpr u64 ORDER_TOPK_RATIO = 16;

enum : u32 { OC_EMPTY = 0, OC_NUM = 1, OC_NAN = 2, OC_STR = 3 };

struct ClassifyParams {
    const u32* ids; u32 d;                                     // the column's distinct ids, ascending (KB_ID_NONE last)
    const double* num; const u8* isnum; u32 n_ids;             // numeric side table
    const unsigned long long* dict_off; u32 dict_ids;          // device dictionary (null: none loaded)
    u32 quoted_slots;
    unsigned long long* key;                                   // order key of a number, 0 for ""
    u32* ctr;                                                  // [0] numbers, [1] NaNs, [2] non-empty strings, [3] quoted ids, no table
};

__global__ void __launch_bounds__(OT) order_classify_kernel(const __grid_constant__ ClassifyParams P) {
    u32 c[4] = {0, 0, 0, 0};
    for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < P.d; j += gridDim.x * blockDim.x) {
        const u32 id = P.ids[j];
        u32 cls = OC_STR;
        unsigned long long k = 0;
        if (id == EMPTY32) cls = OC_EMPTY;
        else if (id & 0x80000000u) c[3] += P.quoted_slots == 0u;   // `<< s p o >>` or "unknown": a string either way
        else if (P.dict_off && id >= P.dict_ids) cls = OC_STR;     // "unknown"
        else if (id < P.n_ids && P.isnum[id]) {
            const double x = P.num[id];
            cls = x != x ? OC_NAN : OC_NUM;
            k = kb_nr::order_key_total(x);
        } else if (P.dict_off && P.dict_off[id + 1] == P.dict_off[id]) cls = OC_EMPTY;
        if (cls == OC_NUM) c[0]++;
        if (cls == OC_NAN) c[1]++;
        if (cls == OC_STR) c[2]++;
        P.key[j] = k;
    }
    for (int w = 0; w < 4; w++) {
        const u32 s = __reduce_add_sync(0xffffffffu, c[w]);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd(P.ctr + w, s);
    }
}

struct RefineParams {
    const u32* act; u32 m;                      // positions of the unresolved groups, ascending
    u32* ord; u32* grp;                         // value index at every position; start position of its group
    const u32* str_off; const u8* bytes;        // string key: rendered values (null: numeric key)
    const unsigned long long* nkey;             // numeric key: order key of every value
    u32 round;
    unsigned long long* key; u32* gkey; u32* s_of; u32* idx;  // per active item j (before the sorts)
};

// (next 7 bytes from byte 7 * round, big-endian, zero-padded) << 8 | how many of them the string has: "ab" sorts before "ab\0"
__device__ __forceinline__ unsigned long long chunk_key(const u32* off, const u8* bytes, u32 s, u32 round) {
    const u32 a = off[s], len = off[s + 1] - a, at = round * 7u;
    const u32 cnt = len > at ? min(7u, len - at) : 0u;
    unsigned long long k = 0;
#pragma unroll
    for (u32 b = 0; b < 7u; b++) k = (k << 8) | (b < cnt ? (unsigned long long)bytes[a + at + b] : 0ull);
    return (k << 8) | cnt;
}

__global__ void __launch_bounds__(OT) refine_prep_kernel(const __grid_constant__ RefineParams P) {
    for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < P.m; j += gridDim.x * blockDim.x) {
        const u32 p = P.act[j], s = P.ord[p];
        P.s_of[j] = s;
        P.gkey[j] = P.grp[p];
        P.key[j] = P.str_off ? chunk_key(P.str_off, P.bytes, s, P.round) : P.nkey[s];
        P.idx[j] = j;
    }
}

__global__ void __launch_bounds__(OT) gather_u32_kernel(const u32* __restrict__ src, const u32* __restrict__ idx, u32 n, u32* __restrict__ dst) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}

// sorted item j (original active index i = idx[j]) takes position act[j]; a head starts a new group
__global__ void __launch_bounds__(OT) refine_assign_kernel(const __grid_constant__ RefineParams P, const u32* __restrict__ idx, u32* __restrict__ head,
                                                          u32* __restrict__ hp) {
    for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < P.m; j += gridDim.x * blockDim.x) {
        const u32 i = idx[j];
        bool h = j == 0u;
        if (!h) {
            const u32 q = idx[j - 1];
            h = P.gkey[q] != P.gkey[i] || P.key[q] != P.key[i];
        }
        P.ord[P.act[j]] = P.s_of[i];
        head[j] = h;
        hp[j] = h ? P.act[j] : 0u;
    }
}

// hp holds its running maximum here: the position of the group's first item. An item stays active while its group has another
// item and its string goes on past this round's 7 bytes.
__global__ void __launch_bounds__(OT) refine_flag_kernel(const __grid_constant__ RefineParams P, const u32* __restrict__ idx, const u32* __restrict__ head,
                                                        const u32* __restrict__ hp, u8* __restrict__ more) {
    for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < P.m; j += gridDim.x * blockDim.x) {
        P.grp[P.act[j]] = hp[j];
        const bool single = head[j] && (j + 1u == P.m || head[j + 1u]);
        more[j] = P.str_off && !single && (P.key[idx[j]] & 0xFFull) == 7ull;
    }
}

__global__ void __launch_bounds__(OT) iota_kernel(u32* __restrict__ a, u32 n) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) a[i] = i;
}

__global__ void __launch_bounds__(OT) group_head_kernel(const u32* __restrict__ grp, u32 d, u32* __restrict__ head) {
    for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < d; p += gridDim.x * blockDim.x) head[p] = p == 0u || grp[p] != grp[p - 1u];
}

// rank_of[value] = (inclusive count of group heads up to its position) - 1
__global__ void __launch_bounds__(OT) value_rank_kernel(const u32* __restrict__ ord, const u32* __restrict__ incl, u32 d, u32* __restrict__ rank_of) {
    for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < d; p += gridDim.x * blockDim.x) rank_of[ord[p]] = incl[p] - 1u;
}

__global__ void __launch_bounds__(OT) row_rank_kernel(const u32* __restrict__ col, u32 n, const u32* __restrict__ ids, u32 d, const u32* __restrict__ rank_of,
                                                     u32 flip, u32* __restrict__ out) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 id = col[i];
        u32 lo = 0, len = d;
        while (len > 0) {
            const u32 h = len >> 1;
            if (ids[lo + h] < id) { lo += h + 1; len -= h + 1; }
            else len = h;
        }
        const u32 r = rank_of[lo];
        out[i] = flip ? flip - r : r;
    }
}

// top-k: the packed key of every row (rank0 * n1 + rank1) and the digit histograms of the radix select
__global__ void __launch_bounds__(OT) pack_key_kernel(const u32* __restrict__ r0, const u32* __restrict__ r1, u64 n1, u32 n, unsigned long long* __restrict__ key) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) key[i] = (u64)r0[i] * n1 + (r1 ? r1[i] : 0u);
}

__global__ void __launch_bounds__(OT) select_hist_kernel(const unsigned long long* __restrict__ key, u32 n, unsigned long long hi_mask, unsigned long long prefix,
                                                        u32 shift, u32* __restrict__ hist) {
    __shared__ u32 h[256];
    for (int b = threadIdx.x; b < 256; b += blockDim.x) h[b] = 0;
    __syncthreads();
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long k = key[i];
        if ((k & hi_mask) == prefix) atomicAdd(&h[(k >> shift) & 0xFFu], 1u);
    }
    __syncthreads();
    for (int b = threadIdx.x; b < 256; b += blockDim.x)
        if (h[b]) atomicAdd(hist + b, h[b]);
}

__global__ void __launch_bounds__(OT) topk_flags_kernel(const unsigned long long* __restrict__ key, u32 n, unsigned long long t, u32* __restrict__ less,
                                                       u32* __restrict__ eq) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long k = key[i];
        less[i] = k < t;
        eq[i] = k == t;
    }
}

// less / eq hold their exclusive prefixes: rows below T go to [0, n_less) and the first `need` rows equal to T to [n_less, k), both in
// input order
__global__ void __launch_bounds__(OT) topk_place_kernel(const unsigned long long* __restrict__ key, u32 n, unsigned long long t, const u32* __restrict__ less,
                                                       const u32* __restrict__ eq, u32 n_less, u32 need, unsigned long long* __restrict__ okey,
                                                       u32* __restrict__ oidx) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long k = key[i];
        if (k < t) { okey[less[i]] = k; oidx[less[i]] = i; }
        else if (k == t && eq[i] < need) oidx[n_less + eq[i]] = i;
    }
}

struct OrderGatherParams {
    const u32* in[KB_MAX_COLS];
    u32* out[KB_MAX_COLS];
    u32 n_cols, n;
    const u32* idx;
};
__global__ void __launch_bounds__(OT) order_gather_kernel(const __grid_constant__ OrderGatherParams P) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        const u32 r = P.idx[i];
        for (u32 c = 0; c < P.n_cols; c++) P.out[c][i] = P.in[c][r];
    }
}


struct MaxOp {
    __device__ __forceinline__ u32 operator()(u32 a, u32 b) const { return a > b ? a : b; }
};

struct KeyRank {
    Buf rank;        // u32 per row (DESC applied)
    u32 n_values = 0;  // distinct ranks R
    u32 kind = KB_ORDER_CONST, distinct = 0, rounds = 0;
};

}  // namespace

// (declared in kb_internal.hpp: kb_serialize.cu ranks rendered terms with it)
kb_status rank_values(kb_ctx* ctx, u32 d, const unsigned long long* nkey, const u32* str_off, const u8* bytes, u32* rank_of, u32* n_values, u32* rounds) {
    Buf ord, grp, act, act2, key, key2, gkey, gs, gs2, s_of, idx, idx2, idx3, head, hp, more;
    const size_t n4 = (size_t)d * sizeof(u32);
    for (Buf* b : {&ord, &grp, &act, &act2, &gkey, &gs, &gs2, &s_of, &idx, &idx2, &idx3, &head, &hp}) KB_TRY(alloc_buf(ctx, n4, b));
    KB_TRY(alloc_buf(ctx, (size_t)d * 8, &key));
    KB_TRY(alloc_buf(ctx, (size_t)d * 8, &key2));
    KB_TRY(alloc_buf(ctx, d, &more));
    const int g = grid_1d(d, ctx->n_sms);
    auto U = [](Buf& b) { return static_cast<u32*>(b->p); };
    timer_begin(ctx, F_OTHER, 2);
    iota_kernel<<<g, OT, 0, ctx->st>>>(U(ord), d);
    iota_kernel<<<g, OT, 0, ctx->st>>>(U(act), d);
    timer_end(ctx);
    KB_CUDA(ctx, cudaMemsetAsync(grp->p, 0, n4, ctx->st));
    const u32 gbits = std::max(1u, bits_of(d - 1));
    u32 m = d, r = 0;
    while (m > 1) {
        RefineParams P{};
        P.act = U(act); P.m = m; P.ord = U(ord); P.grp = U(grp);
        P.str_off = str_off; P.bytes = bytes; P.nkey = nkey; P.round = r;
        P.key = static_cast<unsigned long long*>(key->p); P.gkey = U(gkey); P.s_of = U(s_of); P.idx = U(idx);
        unsigned long long* k2 = static_cast<unsigned long long*>(key2->p);
        const int gm = grid_1d(m, ctx->n_sms);
        timer_begin(ctx, F_OTHER, 4);
        refine_prep_kernel<<<gm, OT, 0, ctx->st>>>(P);
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, P.key, k2, P.idx, U(idx2), m, 0, 64, ctx->st); }));
        gather_u32_kernel<<<gm, OT, 0, ctx->st>>>(P.gkey, U(idx2), m, U(gs));
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, U(gs), U(gs2), U(idx2), U(idx3), m, 0, (int)gbits, ctx->st); }));
        refine_assign_kernel<<<gm, OT, 0, ctx->st>>>(P, U(idx3), U(head), U(hp));
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveScan(t, b, U(hp), U(hp), MaxOp(), m, ctx->st); }));
        refine_flag_kernel<<<gm, OT, 0, ctx->st>>>(P, U(idx3), U(head), U(hp), static_cast<u8*>(more->p));
        const u32 c = ctrl_alloc(ctx, 4);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 4 * sizeof(u32), ctx->st));
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) {
            return cub::DeviceSelect::Flagged(t, b, U(act), static_cast<const u8*>(more->p), U(act2), ctx->ctrl + c, m, ctx->st);
        }));
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        m = ctx->h_ctrl[c];
        std::swap(act, act2);
        r++;
    }
    *rounds = r;
    // dense ranks: one per group, in position order
    timer_begin(ctx, F_OTHER, 2);
    group_head_kernel<<<g, OT, 0, ctx->st>>>(U(grp), d, U(head));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveSum(t, b, U(head), U(hp), d, ctx->st); }));
    value_rank_kernel<<<g, OT, 0, ctx->st>>>(U(ord), U(hp), d, rank_of);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_CUDA(ctx, cudaMemcpyAsync(n_values, U(hp) + d - 1, sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += sizeof(u32);
    return KB_OK;
}

namespace {

// the rank column of one key; refusals (KB_E_UNSUPPORTED) before any output exists
kb_status rank_key(kb_ctx* ctx, const kb_rel& in, u32 col, bool desc, KeyRank* kr) {
    const u32 n = (u32)in.n;
    const u32* ids = in.cols[col].ptr;
    Buf sorted, uniq, nkey, rank_of;
    KB_TRY(alloc_buf(ctx, (size_t)n * 4, &sorted));
    KB_TRY(alloc_buf(ctx, (size_t)n * 4, &uniq));
    u32* d_sorted = static_cast<u32*>(sorted->p);
    u32* d_uniq = static_cast<u32*>(uniq->p);
    const u32 c = ctrl_alloc(ctx, 8);  // [0] distinct ids, [4..7] classify counts
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 8 * sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER, 0);
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, ids, d_sorted, n, 0, 32, ctx->st); }));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceSelect::Unique(t, b, d_sorted, d_uniq, ctx->ctrl + c, n, ctx->st); }));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32 d = ctx->h_ctrl[c];
    kr->distinct = d;
    KB_TRY(alloc_buf(ctx, (size_t)d * 8, &nkey));
    ClassifyParams P{};
    P.ids = d_uniq; P.d = d;
    P.num = ctx->num ? static_cast<const double*>(ctx->num->p) : nullptr;
    P.isnum = ctx->isnum ? static_cast<const u8*>(ctx->isnum->p) : nullptr;
    P.n_ids = P.num ? ctx->n_ids : 0u;
    const DictTab dict = dicttab(ctx);
    P.dict_off = dict.off;
    P.dict_ids = dict.ids;
    P.quoted_slots = ctx->quoted_slots;
    P.key = static_cast<unsigned long long*>(nkey->p);
    P.ctr = ctx->ctrl + c + 4;
    timer_begin(ctx, F_OTHER, 1);
    order_classify_kernel<<<grid_1d(d, ctx->n_sms, OT), OT, 0, ctx->st>>>(P);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32 n_num = ctx->h_ctrl[c + 4], n_nan = ctx->h_ctrl[c + 5], n_str = ctx->h_ctrl[c + 6], n_qt = ctx->h_ctrl[c + 7];
    if ((n_num + n_nan > 0 && n_str > 0) || (n_nan > 0 && n_num > 0))
        return fail(ctx, KB_E_UNSUPPORTED, "ORDER BY column of slot %u mixes %s: the reference's comparison is not an order on it", in.slots[col],
                    n_str ? "numbers and strings that are not numbers" : "NaN and other numbers");
    if (n_qt) return fail(ctx, KB_E_UNSUPPORTED, "the ORDER BY column holds quoted-triple ids (bit 31) and no quoted-triple table is loaded (kb_quoted_load)");
    if (n_str && !ctx->dict_ids) return fail(ctx, KB_E_UNSUPPORTED, "a string ORDER BY key needs the device dictionary's strings (kb_dict_strings_load)");
    KB_TRY(alloc_buf(ctx, (size_t)d * 4, &rank_of));
    if (n_str) {
        // render the distinct values as kb_rel_decode does; KB_ID_NONE (last, when present) is "" and not decoded
        u32 none = 0;
        KB_CUDA(ctx, cudaMemcpyAsync(&none, d_uniq + d - 1, sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        ctx->stats.d2h_bytes += sizeof(u32);
        const u32 dr = none == EMPTY32 ? d - 1 : d;
        Buf off, bytes;
        KB_TRY(decode_ids(ctx, d_uniq, dr, d - dr, Decode::Unknown, "the ORDER BY column", &off, &bytes, nullptr));
        KB_TRY(rank_values(ctx, d, nullptr, static_cast<const u32*>(off->p), static_cast<const u8*>(bytes->p), static_cast<u32*>(rank_of->p), &kr->n_values,
                           &kr->rounds));
        kr->kind = KB_ORDER_STRING;
    } else {
        u32 rounds = 0;
        KB_TRY(rank_values(ctx, d, P.key, nullptr, nullptr, static_cast<u32*>(rank_of->p), &kr->n_values, &rounds));
        kr->kind = KB_ORDER_NUMERIC;
    }
    if (kr->n_values <= 1) kr->kind = KB_ORDER_CONST;
    KB_TRY(alloc_buf(ctx, (size_t)n * 4, &kr->rank));
    timer_begin(ctx, F_OTHER, 1);
    row_rank_kernel<<<grid_1d(n, ctx->n_sms, OT), OT, 0, ctx->st>>>(ids, n, d_uniq, d, static_cast<const u32*>(rank_of->p), desc ? kr->n_values - 1u : 0u,
                                                                 static_cast<u32*>(kr->rank->p));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

}  // namespace

static kb_status order_by_impl(kb_ctx* ctx, const kb_rel& in, const kb_order_key* keys, u32 n_keys, u64 limit, std::unique_ptr<kb_rel>* out, kb_order_info* info) {
    const u32 n = (u32)in.n;
    const u32 n_out = limit > 0 && limit < n ? (u32)limit : n;
    info->n_rows_in = n;
    info->n_rows_out = n_out;
    // the key ranks, first key first; a key whose values all compare equal does not order anything
    std::vector<KeyRank> ranks(n_keys);
    std::vector<u32> sort_keys;
    if (n) {
        bool any_col = false;
        for (u32 k = 0; k < n_keys; k++) any_col = any_col || in.col_of(keys[k].slot) >= 0;
        if (any_col && ctx->n_ids < ctx->dict_ids)  // a stale is_num would sort numbers as strings
            return fail(ctx, KB_E_UNSUPPORTED, "the numeric side table covers %u ids, the device dictionary %u: run kb_dict_numeric_derive",
                        ctx->n_ids, ctx->dict_ids);
        for (u32 k = 0; k < n_keys; k++) {
            const int col = in.col_of(keys[k].slot);
            if (col < 0) continue;  // "" in every row (execute_query.rs:124-125): no effect
            KB_TRY(rank_key(ctx, in, (u32)col, keys[k].descending != 0, &ranks[k]));
            if (ranks[k].kind != KB_ORDER_CONST) sort_keys.push_back(k);
        }
    }
    for (u32 k = 0; k < n_keys; k++) {
        info->key_kind[k] = ranks[k].kind;
        info->n_distinct[k] = ranks[k].distinct;
        info->string_rounds[k] = ranks[k].rounds;
    }
    if (sort_keys.empty()) {  // the input order is the sorted order: a view of the first n_out rows
        info->route = KB_ORDER_VIEW;
        auto r = select_cols(in, in.slots);
        r->n = n_out;
        *out = std::move(r);
        return KB_OK;
    }
    auto U = [](const Buf& b) { return static_cast<u32*>(b->p); };
    Buf order;  // row indices in sorted order, n_out of them
    const u32 nk = (u32)sort_keys.size();
    const int g = grid_1d(n, ctx->n_sms);
    if (limit > 0 && nk <= 2 && (u64)limit * ORDER_TOPK_RATIO <= n) {
        // top-k: T = the k-th smallest packed key; rows below T sorted, then the first rows equal to T in input order
        info->route = KB_ORDER_TOPK;
        const KeyRank& a = ranks[sort_keys[0]];
        const KeyRank* b = nk == 2 ? &ranks[sort_keys[1]] : nullptr;
        const u64 n1 = b ? b->n_values : 1u;
        const u64 kmax = (u64)(a.n_values - 1) * n1 + (n1 - 1);
        Buf key, less, eq, okey, okey2, oidx, oidx2, scratch;
        KB_TRY(alloc_buf(ctx, (size_t)n * 8, &key));
        unsigned long long* d_key = static_cast<unsigned long long*>(key->p);
        timer_begin(ctx, F_OTHER, 1);
        pack_key_kernel<<<g, OT, 0, ctx->st>>>(U(a.rank), b ? U(b->rank) : nullptr, n1, n, d_key);
        timer_end(ctx);
        unsigned long long prefix = 0;
        u32 need = n_out;
        for (int shift = (int)((std::max(1u, bits_of(kmax)) - 1) / 8) * 8; shift >= 0; shift -= 8) {
            const u32 c = ctrl_alloc(ctx, 256);
            KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 256 * sizeof(u32), ctx->st));
            const unsigned long long hi = shift + 8 >= 64 ? 0ull : ~0ull << (shift + 8);
            timer_begin(ctx, F_OTHER, 1);
            select_hist_kernel<<<g, OT, 0, ctx->st>>>(d_key, n, hi, prefix, (u32)shift, ctx->ctrl + c);
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
            KB_TRY(ctrl_read(ctx));
            u32 digit = 0;
            for (; digit < 256; digit++) {
                const u32 h = ctx->h_ctrl[c + digit];
                if (need <= h) break;
                need -= h;
            }
            prefix |= (unsigned long long)digit << shift;
        }
        const u32 n_less = n_out - need;  // rows whose key is below T; `need` rows equal to T complete the k
        for (Buf* x : {&less, &eq, &oidx, &oidx2}) KB_TRY(alloc_buf(ctx, (size_t)n * 4, x));
        KB_TRY(alloc_buf(ctx, (size_t)n_out * 8, &okey));
        KB_TRY(alloc_buf(ctx, (size_t)n_out * 8, &okey2));
        unsigned long long* d_ok = static_cast<unsigned long long*>(okey->p);
        unsigned long long* d_ok2 = static_cast<unsigned long long*>(okey2->p);
        timer_begin(ctx, F_OTHER, 2);
        topk_flags_kernel<<<g, OT, 0, ctx->st>>>(d_key, n, prefix, U(less), U(eq));
        KB_TRY(cub_run(ctx, [&](void* t, size_t& s) { return cub::DeviceScan::ExclusiveSum(t, s, U(less), U(less), n, ctx->st); }));
        KB_TRY(cub_run(ctx, [&](void* t, size_t& s) { return cub::DeviceScan::ExclusiveSum(t, s, U(eq), U(eq), n, ctx->st); }));
        topk_place_kernel<<<g, OT, 0, ctx->st>>>(d_key, n, prefix, U(less), U(eq), n_less, need, d_ok, U(oidx));
        if (n_less > 1) {
            KB_TRY(cub_run(ctx, [&](void* t, size_t& s) {
                return cub::DeviceRadixSort::SortPairs(t, s, d_ok, d_ok2, U(oidx), U(oidx2), n_less, 0, (int)std::max(1u, bits_of(kmax)), ctx->st);
            }));
            KB_CUDA(ctx, cudaMemcpyAsync(U(oidx), U(oidx2), (size_t)n_less * 4, cudaMemcpyDeviceToDevice, ctx->st));
        }
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        order = oidx;
    } else {
        // full sort: stable LSD radix sorts of the row indices, last key first
        info->route = KB_ORDER_SORT;
        Buf idx, idx2, k1, k2;
        for (Buf* x : {&idx, &idx2, &k1, &k2}) KB_TRY(alloc_buf(ctx, (size_t)n * 4, x));
        timer_begin(ctx, F_OTHER, 1);
        iota_kernel<<<g, OT, 0, ctx->st>>>(U(idx), n);
        timer_end(ctx);
        for (int s = (int)nk - 1; s >= 0; s--) {
            const KeyRank& kr = ranks[sort_keys[s]];
            timer_begin(ctx, F_OTHER, 1);
            gather_u32_kernel<<<g, OT, 0, ctx->st>>>(U(kr.rank), U(idx), n, U(k1));
            KB_TRY(cub_run(ctx, [&](void* t, size_t& b) {
                return cub::DeviceRadixSort::SortPairs(t, b, U(k1), U(k2), U(idx), U(idx2), n, 0, (int)std::max(1u, bits_of(kr.n_values - 1)), ctx->st);
            }));
            timer_end(ctx);
            std::swap(idx, idx2);
        }
        KB_CUDA(ctx, cudaGetLastError());
        order = idx;
    }
    // every column of `in`, gathered in the sorted order
    auto r = std::make_unique<kb_rel>();
    r->slots = in.slots;
    r->n = n_out;
    KB_TRY(alloc_strided_cols(ctx, n_out, (u32)in.cols.size(), &r->cols));
    OrderGatherParams G{};
    G.n_cols = (u32)in.cols.size();
    G.n = n_out;
    G.idx = U(order);
    for (u32 c = 0; c < G.n_cols; c++) { G.in[c] = in.cols[c].ptr; G.out[c] = r->cols[c].ptr; }
    if (n_out) {
        timer_begin(ctx, F_OTHER, 1);
        order_gather_kernel<<<grid_1d(n_out, ctx->n_sms, OT), OT, 0, ctx->st>>>(G);
        timer_end(ctx);
    }
    KB_CUDA(ctx, cudaGetLastError());
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    timers_flush(ctx);
    *out = std::move(r);
    return KB_OK;
}

}  // namespace kb

extern "C" {

kb_status kb_order_by(kb_ctx* ctx, const kb_rel* in, const kb_order_key* keys, uint32_t n_keys, uint64_t limit, kb_rel** out, kb_order_info* info) {
    if (!ctx) return KB_E_INVALID;
    kb::DeviceGuard guard(ctx->device);
    KB_TRY(kb::begin_call(ctx));
    kb_order_info local{};
    if (!info) info = &local;
    *info = kb_order_info{};
    if (!in || !out || (n_keys && !keys)) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_keys > KB_MAX_COLS) return kb::fail(ctx, KB_E_INVALID, "at most %d ORDER BY keys (got %u)", KB_MAX_COLS, n_keys);
    if (in->n > 0xFFFFFFFFull) return kb::fail(ctx, KB_E_LIMIT, "a relation of %llu rows (limit 2^32-1)", (unsigned long long)in->n);
    std::unique_ptr<kb_rel> r;
    KB_TRY(kb::order_by_impl(ctx, *in, keys, n_keys, limit, &r, info));
    ctx->stats.rows_out = r->n;
    *out = r.release();
    return KB_OK;
}

}  // extern "C"
