// kb_natjoin.cu — the natural join of SPARQL mappings over relations whose cells may be unbound (KB_ID_NONE): what the RSP engine's
// emit step joins window results and static data with (natural_join, kolibrie/src/rsp_engine.rs:684-718). The semantics are in
// include/kolibrie_b200.h; here:
//   fast route     no shared column holds KB_ID_NONE (one check pass tells): exactly kb_hash_join (hash_join_impl)
//   unbound route  U = the shared slots that hold KB_ID_NONE on some side (|U| <= 4)
//     K1 natjoin_mask_kernel       every row's bound-mask over U (bit j: U[j] is bound) and a histogram per side and mask
//     K2 natjoin_partition_kernel  counting sort of each side by mask: the row index and the shared columns, every mask group starting
//                                  on a 256-byte boundary, so a group is a zero-copy column view
//     sub-joins                    for every pair of non-empty groups (mL, mR): hash_join_impl on the key (S \ U) ∪ (U ∩ mL ∩ mR),
//                                  carrying the two row indices (an empty key is the groups' cartesian product)
//     K3 natjoin_coalesce_kernel   the output rows from the sub-joins' row-index pairs: the right cell if bound, else the left one
// and kb_hash_join_keyed, the hash joins of the Streamertail engine over rows that may leave variables unbound (engine.rs:710-811, 970-1071):
//   check pass                   natjoin_check_kernel over the key columns: a KB_ID_NONE there is refused
//   K4 keyed_index_kernel        every side's row index
//   sub-join                     hash_join_impl of the (key columns, row index) views: the row-index pairs
//   K3                           the output rows, every non-key shared slot coalesced by the call's merge policy
#include <algorithm>

#include "kb_internal.hpp"

namespace kb {
namespace {

constexpr u32 NJ_MAX_U = 4, NJ_MASKS = 1u << NJ_MAX_U;
constexpr u64 NJ_ALIGN = 64;  // rows: a mask group starts on a 256-byte boundary (column views must be 16-byte aligned)

struct NjCheckSide { const u32* col[KB_MAX_COLS]; u32 n; };
struct NjCheckParams { NjCheckSide side[2]; u32 n_cols; u32* flags; /* [2]: bit c = shared column c holds KB_ID_NONE */ };

struct NjMaskSide { const u32* col[NJ_MAX_U]; u32 n; u8* mask; };
struct NjMaskParams { NjMaskSide side[2]; u32 n_u; u32* hist; /* [2][NJ_MASKS] */ };

struct NjPartSide {
    const u32* in[KB_MAX_COLS];
    u32* out[KB_MAX_COLS];
    const u8* mask;
    u32* perm;                // original row index of every sorted row
    u32* cursor;              // [NJ_MASKS] rows placed so far per mask
    u32 start[NJ_MASKS];      // first row of every mask group
    u32 n;
};
struct NjPartParams { NjPartSide side[2]; u32 n_cols; };

struct NjCoalesceParams {
    const u32* li;            // the sub-join's left / right row indices
    const u32* ri;
    u32 n;
    u64 base;                 // first output row of this sub-join
    const u32* l[KB_MAX_COLS];  // source column of output column c on each side (null: the side lacks the slot)
    const u32* r[KB_MAX_COLS];
    u32* out[KB_MAX_COLS];
    u32 n_out;
    u32 right_first;          // a slot both sides hold: the preferred side's cell if bound, else the other side's
};

__global__ void __launch_bounds__(256) natjoin_check_kernel(const __grid_constant__ NjCheckParams P) {
    const NjCheckSide& S = P.side[blockIdx.y];
    u32 f = 0;
    for (u32 c = 0; c < P.n_cols; c++) {
        const u32* col = S.col[c];
        for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < S.n; i += gridDim.x * blockDim.x)
            if (__ldg(col + i) == KB_ID_NONE) f |= 1u << c;
    }
    f = __reduce_or_sync(0xffffffffu, f);
    if ((threadIdx.x & 31) == 0 && f) atomicOr(P.flags + blockIdx.y, f);
}

__global__ void __launch_bounds__(256) natjoin_mask_kernel(const __grid_constant__ NjMaskParams P) {
    __shared__ u32 s_hist[NJ_MASKS];
    const NjMaskSide& S = P.side[blockIdx.y];
    if (threadIdx.x < NJ_MASKS) s_hist[threadIdx.x] = 0;
    __syncthreads();
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < S.n; i += gridDim.x * blockDim.x) {
        u32 m = 0;
        for (u32 j = 0; j < P.n_u; j++) m |= (__ldg(S.col[j] + i) != KB_ID_NONE ? 1u : 0u) << j;
        S.mask[i] = (u8)m;
        atomicAdd(&s_hist[m], 1u);
    }
    __syncthreads();
    if (threadIdx.x < NJ_MASKS && s_hist[threadIdx.x]) atomicAdd(P.hist + blockIdx.y * NJ_MASKS + threadIdx.x, s_hist[threadIdx.x]);
}

// a block places one tile of blockDim.x rows at a time: ranks inside the tile from shared counters, the tile's base per mask from ONE
// global atomic per mask (the order inside a group is unspecified, as the operator's row order is)
__global__ void __launch_bounds__(256) natjoin_partition_kernel(const __grid_constant__ NjPartParams P) {
    __shared__ u32 s_cnt[NJ_MASKS], s_base[NJ_MASKS];
    const NjPartSide& S = P.side[blockIdx.y];
    for (u64 tile = (u64)blockIdx.x * blockDim.x; tile < S.n; tile += (u64)gridDim.x * blockDim.x) {
        if (threadIdx.x < NJ_MASKS) s_cnt[threadIdx.x] = 0;
        __syncthreads();
        const u64 i = tile + threadIdx.x;
        u32 m = 0, local = 0;
        if (i < S.n) {
            m = S.mask[i];
            local = atomicAdd(&s_cnt[m], 1u);
        }
        __syncthreads();
        if (threadIdx.x < NJ_MASKS && s_cnt[threadIdx.x]) s_base[threadIdx.x] = atomicAdd(S.cursor + threadIdx.x, s_cnt[threadIdx.x]);
        __syncthreads();
        if (i < S.n) {
            const u32 pos = S.start[m] + s_base[m] + local;
            S.perm[pos] = (u32)i;
            for (u32 c = 0; c < P.n_cols; c++) S.out[c][pos] = __ldg(S.in[c] + i);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) natjoin_coalesce_kernel(const __grid_constant__ NjCoalesceParams P) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        const u32 li = __ldg(P.li + i), ri = __ldg(P.ri + i);
        for (u32 c = 0; c < P.n_out; c++) {
            const u32 lv = P.l[c] ? __ldg(P.l[c] + li) : KB_ID_NONE, rv = P.r[c] ? __ldg(P.r[c] + ri) : KB_ID_NONE;
            P.out[c][P.base + i] = P.right_first ? (rv != KB_ID_NONE ? rv : lv) : (lv != KB_ID_NONE ? lv : rv);
        }
    }
}

__global__ void __launch_bounds__(256) keyed_index_kernel(u32* idx, u32 n) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) idx[i] = i;
}


// a view of rows [start, start + n) of the sorted side: the key columns of `key` (positions into the shared slots) plus the row index
std::unique_ptr<kb_rel> group_view(const std::vector<u32>& shared, const std::vector<u32>& key, const std::vector<Buf>& keycols, const Buf& perm, u32 idx_slot,
                                   u64 start, u64 n) {
    auto v = std::make_unique<kb_rel>();
    v->n = n;
    for (u32 k : key) {
        v->slots.push_back(shared[k]);
        v->cols.push_back(Col{keycols[k], static_cast<u32*>(keycols[k]->p) + start});
    }
    v->slots.push_back(idx_slot);
    v->cols.push_back(Col{perm, static_cast<u32*>(perm->p) + start});
    return v;
}

// the two slots that name no variable of either side and carry the row indices through a sub-join
void index_slots(const kb_rel& L, const kb_rel& R, u32 idx_slot[2]) {
    u32 cand = 0xFFFFFFFEu;
    for (int k = 0; k < 2; k++) {
        while (L.col_of(cand) >= 0 || R.col_of(cand) >= 0) cand--;
        idx_slot[k] = cand--;
    }
}

kb_status natural_join_impl(kb_ctx* ctx, const kb_rel& L, const kb_rel& R, std::unique_ptr<kb_rel>* out) {
    std::vector<u32> shared, out_slots = L.slots;
    for (u32 s : R.slots) {
        if (L.col_of(s) >= 0) shared.push_back(s);
        else out_slots.push_back(s);
    }
    if (out_slots.size() > KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "join result has more than %d columns", KB_MAX_COLS);
    // empty sides (rsp_engine.rs:688-690) and no shared slot (the cartesian product): nothing can be unbound in a key
    if (shared.empty() || L.n == 0 || R.n == 0) return hash_join_impl(ctx, L, R, nullptr, out);
    if (L.n >= 0xFFFFFFF0ull || R.n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "relation too large");
    const kb_rel* side[2] = {&L, &R};
    const u32 nS = (u32)shared.size();

    // route check: which shared columns hold KB_ID_NONE on either side
    NjCheckParams C{};
    C.n_cols = nS;
    for (int s = 0; s < 2; s++) {
        C.side[s].n = (u32)side[s]->n;
        for (u32 c = 0; c < nS; c++) C.side[s].col[c] = side[s]->cols[side[s]->col_of(shared[c])].ptr;
    }
    const u32 cw = ctrl_alloc(ctx, 2 + 2 * NJ_MASKS + 2 * NJ_MASKS);  // flags, histograms, cursors
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + cw, 0, (2 + 4 * NJ_MASKS) * sizeof(u32), ctx->st));
    C.flags = ctx->ctrl + cw;
    timer_begin(ctx, F_OTHER);
    natjoin_check_kernel<<<dim3(grid_1d(std::max(L.n, R.n), ctx->n_sms), 2), 256, 0, ctx->st>>>(C);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32 none_cols = ctx->h_ctrl[cw] | ctx->h_ctrl[cw + 1];
    if (!none_cols) return hash_join_impl(ctx, L, R, nullptr, out);  // fast route

    // unbound route
    std::vector<u32> U, fixed;  // positions into `shared`
    for (u32 c = 0; c < nS; c++) (none_cols >> c & 1u ? U : fixed).push_back(c);
    if (U.size() > NJ_MAX_U)
        return fail(ctx, KB_E_LIMIT, "%zu shared variables are unbound on some side (limit %u: at most %u mask pairs)", U.size(), NJ_MAX_U,
                    NJ_MASKS * NJ_MASKS);
    NjMaskParams M{};
    M.n_u = (u32)U.size();
    M.hist = ctx->ctrl + cw + 2;
    Buf masks[2];
    for (int s = 0; s < 2; s++) {
        KB_TRY(alloc_buf(ctx, side[s]->n, &masks[s]));
        M.side[s].n = (u32)side[s]->n;
        M.side[s].mask = static_cast<u8*>(masks[s]->p);
        for (u32 j = 0; j < M.n_u; j++) M.side[s].col[j] = C.side[s].col[U[j]];
    }
    timer_begin(ctx, F_OTHER);
    natjoin_mask_kernel<<<dim3(grid_1d(std::max(L.n, R.n), ctx->n_sms), 2), 256, 0, ctx->st>>>(M);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    u32 hist[2][NJ_MASKS];
    memcpy(hist, ctx->h_ctrl + cw + 2, sizeof hist);

    // counting sort by mask
    NjPartParams Pp{};
    Pp.n_cols = nS;
    std::vector<Buf> keycols[2];
    Buf perm[2];
    for (int s = 0; s < 2; s++) {
        NjPartSide& S = Pp.side[s];
        u64 rows = 0;
        for (u32 m = 0; m < NJ_MASKS; m++) {
            S.start[m] = (u32)rows;
            rows += (hist[s][m] + NJ_ALIGN - 1) / NJ_ALIGN * NJ_ALIGN;
        }
        if (rows >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "relation too large");
        KB_TRY(alloc_buf(ctx, rows * sizeof(u32), &perm[s]));
        keycols[s].resize(nS);
        for (u32 c = 0; c < nS; c++) {
            KB_TRY(alloc_buf(ctx, rows * sizeof(u32), &keycols[s][c]));
            S.in[c] = C.side[s].col[c];
            S.out[c] = static_cast<u32*>(keycols[s][c]->p);
        }
        S.mask = M.side[s].mask;
        S.perm = static_cast<u32*>(perm[s]->p);
        S.cursor = ctx->ctrl + cw + 2 + 2 * NJ_MASKS + s * NJ_MASKS;
        S.n = (u32)side[s]->n;
    }
    timer_begin(ctx, F_OTHER);
    natjoin_partition_kernel<<<dim3(grid_1d(std::max(L.n, R.n), ctx->n_sms), 2), 256, 0, ctx->st>>>(Pp);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());

    u32 idx_slot[2];
    index_slots(L, R, idx_slot);
    struct Sub { std::unique_ptr<kb_rel> rel; u64 base; };
    std::vector<Sub> subs;
    u64 total = 0;
    for (u32 ml = 0; ml < NJ_MASKS; ml++) {
        if (!hist[0][ml]) continue;
        for (u32 mr = 0; mr < NJ_MASKS; mr++) {
            if (!hist[1][mr]) continue;
            std::vector<u32> key = fixed;
            for (u32 j = 0; j < U.size(); j++)
                if ((ml & mr) >> j & 1u) key.push_back(U[j]);
            std::sort(key.begin(), key.end());
            auto lv = group_view(shared, key, keycols[0], perm[0], idx_slot[0], Pp.side[0].start[ml], hist[0][ml]);
            auto rv = group_view(shared, key, keycols[1], perm[1], idx_slot[1], Pp.side[1].start[mr], hist[1][mr]);
            std::unique_ptr<kb_rel> j;
            KB_TRY(hash_join_impl(ctx, *lv, *rv, nullptr, &j));
            if (!j->n) continue;
            subs.push_back(Sub{std::move(j), total});
            total += subs.back().rel->n;
            if (total >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "join result of more than 2^32 rows");
        }
    }

    auto rel = std::make_unique<kb_rel>();
    rel->slots = out_slots;
    rel->n = total;
    NjCoalesceParams Q{};
    Q.n_out = (u32)out_slots.size();
    Q.right_first = 1;  // merged.insert: the right value overwrites (rsp_engine.rs:708-711)
    for (u32 c = 0; c < Q.n_out; c++) {
        Col col;
        KB_TRY(alloc_col(ctx, total, &col));
        rel->cols.push_back(col);
        Q.out[c] = col.ptr;
        const int lc = L.col_of(out_slots[c]), rc = R.col_of(out_slots[c]);
        Q.l[c] = lc >= 0 ? L.cols[lc].ptr : nullptr;
        Q.r[c] = rc >= 0 ? R.cols[rc].ptr : nullptr;
    }
    if (!subs.empty()) {
        timer_begin(ctx, F_OTHER, (int)subs.size());
        for (auto& s : subs) {
            Q.li = s.rel->cols[s.rel->col_of(idx_slot[0])].ptr;
            Q.ri = s.rel->cols[s.rel->col_of(idx_slot[1])].ptr;
            Q.n = (u32)s.rel->n;
            Q.base = s.base;
            natjoin_coalesce_kernel<<<grid_1d(s.rel->n, ctx->n_sms), 256, 0, ctx->st>>>(Q);
        }
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
    }
    *out = std::move(rel);
    return KB_OK;
}

kb_status keyed_join_impl(kb_ctx* ctx, const kb_rel& L, const kb_rel& R, const u32* key, u32 n_key, u32 merge, std::unique_ptr<kb_rel>* out) {
    std::vector<u32> out_slots = L.slots;
    for (u32 s : R.slots)
        if (L.col_of(s) < 0) out_slots.push_back(s);
    if (out_slots.size() > KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "join result has more than %d columns", KB_MAX_COLS);
    if (L.n >= 0xFFFFFFF0ull || R.n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "relation too large");
    const kb_rel* side[2] = {&L, &R};
    // a key cell without a value: the reference's hash joins panic on `tuple[var]`, its merge join compares keys of another shape
    if (n_key && L.n && R.n) {
        NjCheckParams C{};
        C.n_cols = n_key;
        for (int s = 0; s < 2; s++) {
            C.side[s].n = (u32)side[s]->n;
            for (u32 k = 0; k < n_key; k++) C.side[s].col[k] = side[s]->cols[side[s]->col_of(key[k])].ptr;
        }
        const u32 cw = ctrl_alloc(ctx, 2);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + cw, 0, 2 * sizeof(u32), ctx->st));
        C.flags = ctx->ctrl + cw;
        timer_begin(ctx, F_OTHER);
        natjoin_check_kernel<<<dim3(grid_1d(std::max(L.n, R.n), ctx->n_sms), 2), 256, 0, ctx->st>>>(C);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        const u32 f = ctx->h_ctrl[cw] | ctx->h_ctrl[cw + 1];
        if (f) {
            u32 k = 0;
            while (!(f >> k & 1u)) k++;
            return fail(ctx, KB_E_UNSUPPORTED, "kb_hash_join_keyed: key slot %u is unbound in a %s row (the reference panics there)", key[k],
                        ctx->h_ctrl[cw] >> k & 1u ? "left" : "right");
        }
    }
    u32 idx_slot[2];
    index_slots(L, R, idx_slot);
    Buf idx[2];
    std::unique_ptr<kb_rel> view[2];
    for (int s = 0; s < 2; s++) {
        KB_TRY(alloc_buf(ctx, std::max<u64>(side[s]->n, 1) * sizeof(u32), &idx[s]));
        if (side[s]->n) {
            timer_begin(ctx, F_OTHER);
            keyed_index_kernel<<<grid_1d(side[s]->n, ctx->n_sms), 256, 0, ctx->st>>>(static_cast<u32*>(idx[s]->p), (u32)side[s]->n);
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
        }
        view[s] = std::make_unique<kb_rel>();
        view[s]->n = side[s]->n;
        for (u32 k = 0; k < n_key; k++) {
            view[s]->slots.push_back(key[k]);
            view[s]->cols.push_back(side[s]->cols[side[s]->col_of(key[k])]);
        }
        view[s]->slots.push_back(idx_slot[s]);
        view[s]->cols.push_back(Col{idx[s], static_cast<u32*>(idx[s]->p)});
    }
    std::unique_ptr<kb_rel> j;
    KB_TRY(hash_join_impl(ctx, *view[0], *view[1], nullptr, &j));
    if (j->n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "join result of more than 2^32 rows");

    auto rel = std::make_unique<kb_rel>();
    rel->slots = out_slots;
    rel->n = j->n;
    NjCoalesceParams Q{};
    Q.n_out = (u32)out_slots.size();
    Q.right_first = merge == KB_MERGE_RIGHT_FIRST;
    for (u32 c = 0; c < Q.n_out; c++) {
        Col col;
        KB_TRY(alloc_col(ctx, j->n, &col));
        rel->cols.push_back(col);
        Q.out[c] = col.ptr;
        const int lc = L.col_of(out_slots[c]), rc = R.col_of(out_slots[c]);
        Q.l[c] = lc >= 0 ? L.cols[lc].ptr : nullptr;
        Q.r[c] = rc >= 0 ? R.cols[rc].ptr : nullptr;
    }
    if (j->n) {
        Q.li = j->cols[j->col_of(idx_slot[0])].ptr;
        Q.ri = j->cols[j->col_of(idx_slot[1])].ptr;
        Q.n = (u32)j->n;
        timer_begin(ctx, F_OTHER);
        natjoin_coalesce_kernel<<<grid_1d(j->n, ctx->n_sms), 256, 0, ctx->st>>>(Q);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
    }
    *out = std::move(rel);
    return KB_OK;
}

}  // namespace
}  // namespace kb

extern "C" {

kb_status kb_natural_join(kb_ctx* ctx, const kb_rel* left, const kb_rel* right, kb_rel** out) {
    if (!ctx) return KB_E_INVALID;
    kb::DeviceGuard guard(ctx->device);
    KB_TRY(kb::begin_call(ctx));
    if (!left || !right || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (left->pair || right->pair) return kb::fail(ctx, KB_E_INVALID, "internal pair relation");
    std::unique_ptr<kb_rel> r;
    KB_TRY(kb::natural_join_impl(ctx, *left, *right, &r));
    ctx->stats.rows_out = r->n;
    *out = r.release();
    return KB_OK;
}

}  // extern "C"

extern "C" {

kb_status kb_hash_join_keyed(kb_ctx* ctx, const kb_rel* left, const kb_rel* right, const uint32_t* key_slots, uint32_t n_key, uint32_t merge,
                             kb_rel** out) {
    KB_ENTER(ctx);
    if (!left || !right || !out || (n_key && !key_slots)) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (left->pair || right->pair) return kb::fail(ctx, KB_E_INVALID, "internal pair relation");
    if (merge != KB_MERGE_LEFT_FIRST && merge != KB_MERGE_RIGHT_FIRST) return kb::fail(ctx, KB_E_INVALID, "kb_hash_join_keyed: unknown merge policy %u", merge);
    if (n_key > 4) return kb::fail(ctx, KB_E_LIMIT, "kb_hash_join_keyed: %u key slots (a hash join key holds at most 4)", n_key);
    for (uint32_t k = 0; k < n_key; k++) {
        if (left->col_of(key_slots[k]) < 0 || right->col_of(key_slots[k]) < 0)
            return kb::fail(ctx, KB_E_INVALID, "kb_hash_join_keyed: key slot %u is not a column of both sides", key_slots[k]);
        for (uint32_t m = 0; m < k; m++)
            if (key_slots[m] == key_slots[k]) return kb::fail(ctx, KB_E_INVALID, "kb_hash_join_keyed: key slot %u repeated", key_slots[k]);
    }
    std::unique_ptr<kb_rel> r;
    KB_TRY(kb::keyed_join_impl(ctx, *left, *right, key_slots, n_key, merge, &r));
    ctx->stats.rows_out = r->n;
    *out = r.release();
    return KB_OK;
}

}  // extern "C"
