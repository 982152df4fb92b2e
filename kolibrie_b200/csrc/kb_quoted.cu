// kb_quoted.cu — the quoted-triple table (QuotedTripleStore, quoted_triple_store.rs:28-55) on the device: kb_quoted_load, its growth and
// its reverse index, TRIPLE's batch encode (quoted_encode, called by kb_bind), the match pass of kb_scan_quoted and kb_quoted_download.
// Every quoted_* field of kb_ctx is written here.
#include <algorithm>

#include "kb_internal.hpp"
#include "kb_tagtab.cuh"

namespace kb {

// =================================================================================================================
// Quoted-triple match (kb_scan_quoted; match_term over QuotedTripleStore entries, engine.rs:1088-1107): ONE streaming pass over the
// table's three columns, QM_TILE-entry tiles TMA-staged into shared memory (two stages), matches compacted with warp ballots (row order
// unspecified). The inner pattern(s) are compiled into at most 6 checks on the entry's components.
constexpr int QM_TILE = 1024, QM_THREADS = 256;
enum QmCheck : u32 { QM_NONE = 0, QM_CONST = 1 /* comp == arg */, QM_EQ = 2 /* comp == component arg */, QM_QUOTED = 3 /* comp has bit 31 */ };
struct QuotedMatchParams {
    QuotedTab t;
    u32 n_tiles;
    u32 n_chk;
    u32 chk_kind[6], chk_comp[6], chk_arg[6];  // check k: kind, component (0 s, 1 p, 2 o), argument
    u32 n_out;                                 // 1 + inner variables
    u32 out_comp[7];                           // component of output column c >= 1 (column 0 = entry id)
    u32* out[7];                               // [t.n] each
    u32* count;                                // zeroed: rows written
    u32* ticket;                               // zeroed: tile counter
};
// The table's s, p, o columns stream through two shared stages of QM_TILE entries each; an entry that passes every check is one output row
// (entry id, inner variables), appended with a warp ballot and one atomic per warp.
__device__ __forceinline__ u32 qm_comp(u32 k, u32 s, u32 p, u32 o) { return k == 0u ? s : k == 1u ? p : o; }

__global__ void __launch_bounds__(QM_THREADS) quoted_match_kernel(const __grid_constant__ QuotedMatchParams P) {
    __shared__ __align__(128) u32 sbuf[2][3][QM_TILE];
    __shared__ __align__(8) u64 bars[2];
    __shared__ u32 s_tile[2];
    const int tid = threadIdx.x, lane = tid & 31;
    auto issue = [&](u32 stage) {  // one thread: take the next tile and start its three column copies into `stage`
        const u32 t = atomicAdd(P.ticket, 1u);
        s_tile[stage] = t;
        if (t < P.n_tiles) {
            const u32 b = t * (u32)QM_TILE;
            const u32 c = min((u32)QM_TILE, P.t.n - b);
            const u32 bytes = (c * 4u + 15u) & ~15u;  // columns are padded to 256 B: the rounded-up read stays in bounds
            mbar_arrive_expect_tx(&bars[stage], bytes * 3u);
            tma_load_1d(sbuf[stage][0], P.t.s + b, bytes, &bars[stage]);
            tma_load_1d(sbuf[stage][1], P.t.p + b, bytes, &bars[stage]);
            tma_load_1d(sbuf[stage][2], P.t.o + b, bytes, &bars[stage]);
        }
    };
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_mbar_init();
        issue(0);
        issue(1);
    }
    __syncthreads();
    // a CTA's tickets grow with its iterations: once a stage draws a ticket past the end, no copy is in flight in the other one
    for (u32 it = 0;; it++) {
        const u32 stage = it & 1u;
        const u32 tile = s_tile[stage];
        if (tile >= P.n_tiles) break;
        mbar_wait(&bars[stage], (it >> 1) & 1u);
        const u32 base = tile * (u32)QM_TILE;
        const u32 cnt = min((u32)QM_TILE, P.t.n - base);
        for (u32 j = (u32)tid; j < (u32)QM_TILE; j += QM_THREADS) {  // the same trip count in every lane: the ballot sees the whole warp
            u32 s = 0, p = EMPTY32, o = 0;
            if (j < cnt) { s = sbuf[stage][0][j]; p = sbuf[stage][1][j]; o = sbuf[stage][2][j]; }
            bool ok = p != EMPTY32;  // (empty slots and the tail of the last tile)
#pragma unroll
            for (int k = 0; k < 6; k++) {
                if ((u32)k >= P.n_chk) break;
                const u32 v = qm_comp(P.chk_comp[k], s, p, o), a = P.chk_arg[k];
                const u32 kind = P.chk_kind[k];
                ok = ok && (kind == QM_CONST ? v == a : kind == QM_EQ ? v == qm_comp(a, s, p, o) : kind == QM_QUOTED ? (v & 0x80000000u) != 0u : true);
            }
            const unsigned b = __ballot_sync(0xffffffffu, ok);
            if (!b) continue;
            u32 at = 0;
            if (lane == __ffs(b) - 1) at = atomicAdd(P.count, (u32)__popc(b));
            at = __shfl_sync(0xffffffffu, at, __ffs(b) - 1);
            if (ok) {
                const u32 r = at + (u32)__popc(b & ((1u << lane) - 1u));
                P.out[0][r] = 0x80000000u | (base + j);
#pragma unroll
                for (int c = 1; c < 7; c++)
                    if ((u32)c < P.n_out) P.out[c][r] = qm_comp(P.out_comp[c], s, p, o);
            }
        }
        __syncthreads();  // every thread is done with the stage: it takes the tile after next
        if (tid == 0) issue(stage);
    }
}
static void launch_quoted_match(const QuotedMatchParams& p, int n_sms, cudaStream_t st) {
    if (p.n_tiles == 0) return;
    const int grid = grid_for((const void*)quoted_match_kernel, QM_THREADS, 0, n_sms, p.n_tiles);
    quoted_match_kernel<<<grid, QM_THREADS, 0, st>>>(p);
}


// =================================================================================================================
// TRIPLE: QuotedTripleStore::encode of a batch, kb_dict_encode's scheme (kb_tagtab.cuh) on a 96-bit key. The reverse index
// (s, p, o) -> table index holds table indices, compared against the forward table on a tag match; the batch table keeps the smallest row
// of every new triple.
struct BindTripleParams {
    const u32* col[3];        // argument columns (null: the constant cval[k])
    u32 cval[3];
    u32 n;
    QuotedTab qt;             // forward table: lookups compare against it
    const u64* rev;           // reverse index (null: empty table)
    u64 rev_mask;
    u64* batch;               // all ~0 beforehand
    u64 batch_mask;
    u32* hit;                 // [n] id the table holds, else EMPTY32
    u32* slot_of;             // [n] batch slot of a new triple's row, EMPTY32 for a hit or an unbound row
    u32* first;               // [n + 1] 1 on the first row of every new triple; then its exclusive prefix (the rank)
    u32* overflow;
    u32 next_qt_id;           // the assign pass: ids next_qt_id + rank, entries written into ws / wp / wo at (next_qt_id & 0x7FFFFFFF) + rank
    u32 *ws, *wp, *wo;
    const u32* old;
    u32* out;
    unsigned long long* n_unbound;
};
__device__ __forceinline__ u64 triple_hash(u32 s, u32 p, u32 o) {
    u64 h = ((u64)s << 32 | p) * 0x9E3779B97F4A7C15ull;
    h ^= (u64)o * 0xC2B2AE3D27D4EB4Full;
    h ^= h >> 31;  // murmur3 64-bit finaliser
    h *= 0xff51afd7ed558ccdull;
    h ^= h >> 33;
    h *= 0xc4ceb9fe1a85ec53ull;
    h ^= h >> 33;
    return h;
}
__device__ __forceinline__ void bind_triple_row(const BindTripleParams& P, u32 i, u32* s, u32* p, u32* o) {
    *s = P.col[0] ? P.col[0][i] : P.cval[0];
    *p = P.col[1] ? P.col[1][i] : P.cval[1];
    *o = P.col[2] ? P.col[2][i] : P.cval[2];
}

__global__ void __launch_bounds__(256) bind_triple_resolve_kernel(const __grid_constant__ BindTripleParams P) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        u32 s, p, o;
        bind_triple_row(P, i, &s, &p, &o);
        u32 hit = EMPTY32, slot_of = EMPTY32;
        if (s != EMPTY32 && p != EMPTY32 && o != EMPTY32) {
            const u64 h = triple_hash(s, p, o);
            if (P.rev) {
                const u32 x = tag_find(P.rev, P.rev_mask, h, [&](u32 x) { return __ldg(P.qt.s + x) == s && __ldg(P.qt.p + x) == p && __ldg(P.qt.o + x) == o; });
                if (x != EMPTY32) hit = 0x80000000u | x;
            }
            // a row holding the slot's triple (the slot's row may be lowered concurrently: always the same triple)
            if (hit == EMPTY32 && !tag_claim_min(P.batch, P.batch_mask, h, i, [&](u32 r) {
                    u32 rs, rp, ro;
                    bind_triple_row(P, r, &rs, &rp, &ro);
                    return rs == s && rp == p && ro == o;
                }, &slot_of))
                *P.overflow = 1u;
        }
        P.hit[i] = hit;
        P.slot_of[i] = slot_of;
    }
}
__global__ void __launch_bounds__(256) bind_triple_mark_kernel(const __grid_constant__ BindTripleParams P) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        const u32 so = P.slot_of[i];
        P.first[i] = so != EMPTY32 && (u32)P.batch[so] == i ? 1u : 0u;
    }
}
__global__ void __launch_bounds__(256) bind_triple_assign_kernel(const __grid_constant__ BindTripleParams P) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 end = (P.n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
        u32 v = EMPTY32;
        if (i < P.n) {
            const u32 so = P.slot_of[i];
            if (so != EMPTY32) {
                const u32 fp = (u32)P.batch[so];
                const u32 r = P.first[fp];
                v = P.next_qt_id + r;
                if (fp == i) {
                    u32 s, p, o;
                    bind_triple_row(P, i, &s, &p, &o);
                    const u32 x = (P.next_qt_id & 0x7FFFFFFFu) + r;
                    P.ws[x] = s;
                    P.wp[x] = p;
                    P.wo[x] = o;
                }
            } else {
                v = P.hit[i];
                if (v == EMPTY32 && P.old) v = P.old[i];
            }
            P.out[i] = v;
        }
        bind_count_unbound(i < P.n && v == EMPTY32, P.n_unbound);
    }
}
__global__ void __launch_bounds__(256) quoted_rev_insert_kernel(const QuotedTab qt, u32 first, u32 n, u64* __restrict__ rev, u64 mask, u32* overflow) {
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const u32 x = first + k;
        const u32 s = qt.s[x], p = qt.p[x], o = qt.o[x];
        if (p == EMPTY32) continue;  // a hole
        u32 slot;  // the same triple twice in the table: the smaller index answers
        if (!tag_claim_min(rev, mask, triple_hash(s, p, o), x, [&](u32 y) { return qt.s[y] == s && qt.p[y] == p && qt.o[y] == o; }, &slot)) *overflow = 1u;
    }
}

}  // namespace kb

using namespace kb;

namespace {

// no table, no reverse index
void quoted_reset(kb_ctx* ctx) {
    ctx->quoted_s.reset(); ctx->quoted_p.reset(); ctx->quoted_o.reset();
    ctx->quoted_slots = ctx->quoted_cap = 0;
    ctx->quoted_rev = TagIndex{};
}

// the reverse index holds every entry of the table and stays below load 1/2 with `extra` more entries
kb_status quoted_rev_ensure(kb_ctx* ctx, u64 extra) {
    const QuotedTab qt = quotedtab(ctx);
    return tag_index_ensure(ctx, &ctx->quoted_rev, ctx->quoted_slots, extra, "quoted-triple reverse index", [&](u32 first, u32 n, u64* tab, u64 mask, u32* overflow) {
        quoted_rev_insert_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(qt, first, n, tab, mask, overflow);
    });
}

// the table's buffers hold at least `slots` entries; new slots are EMPTY32. The buffers keep alloc_buf's padding past their capacity,
// which the match kernel's rounded-up TMA reads of the last tile rely on.
kb_status quoted_grow(kb_ctx* ctx, u32 slots) {
    if (slots <= ctx->quoted_cap) return KB_OK;
    const u32 cap = (u32)std::min<u64>(KB_QUOTED_MAX_SLOTS, std::max<u64>((u64)slots + slots / 2, 1024));
    Buf* cols[3] = {&ctx->quoted_s, &ctx->quoted_p, &ctx->quoted_o};
    Buf nb[3];
    for (int k = 0; k < 3; k++) {
        KB_TRY(alloc_buf(ctx, (size_t)cap * sizeof(u32), &nb[k]));
        launch_fill_u32(static_cast<u32*>(nb[k]->p), EMPTY32, cap, ctx->st);
        if (ctx->quoted_slots)
            KB_CUDA(ctx, cudaMemcpyAsync(nb[k]->p, (*cols[k])->p, (size_t)ctx->quoted_slots * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    }
    ctx->stats.kernel_launches += 3;
    KB_CUDA(ctx, cudaGetLastError());
    for (int k = 0; k < 3; k++) *cols[k] = nb[k];
    ctx->quoted_cap = cap;
    return KB_OK;
}

}  // namespace

QuotedTab kb::quotedtab(const kb_ctx* ctx) {
    QuotedTab t{};
    if (ctx->quoted_slots) {
        t.s = static_cast<const u32*>(ctx->quoted_s->p);
        t.p = static_cast<const u32*>(ctx->quoted_p->p);
        t.o = static_cast<const u32*>(ctx->quoted_o->p);
        t.n = ctx->quoted_slots;
    }
    return t;
}

kb_status kb::quoted_encode(kb_ctx* ctx, const u32* const* col, const u32* cval, u32 n, u32 next_qt_id, const u32* old, u32* out,
                            unsigned long long* n_unbound, kb_bind_info* info) {
    KB_TRY(quoted_rev_ensure(ctx, n));
    u64 bslots = 0;
    Buf batch, hit, slot_of, first, scratch;
    KB_TRY(tag_batch_table(ctx, n, &batch, &bslots));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &hit));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &slot_of));
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &first));
    KB_TRY(alloc_buf(ctx, (((size_t)n + 1) / 2048 + 4) * sizeof(u32), &scratch));
    KB_CUDA(ctx, cudaMemsetAsync(static_cast<u32*>(first->p) + n, 0, sizeof(u32), ctx->st));
    BindTripleParams P{};
    for (int k = 0; k < 3; k++) { P.col[k] = col[k]; P.cval[k] = cval[k]; }
    P.n = n;
    P.qt = quotedtab(ctx);
    P.rev = static_cast<const u64*>(ctx->quoted_rev.tab->p);
    P.rev_mask = ctx->quoted_rev.slots - 1;
    P.batch = static_cast<u64*>(batch->p);
    P.batch_mask = bslots - 1;
    P.hit = static_cast<u32*>(hit->p);
    P.slot_of = static_cast<u32*>(slot_of->p);
    P.first = static_cast<u32*>(first->p);
    const u32 c = ctrl_alloc(ctx, 2);  // [0] overflow, [1] new triples (first[n] after the scan)
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 2 * sizeof(u32), ctx->st));
    P.overflow = ctx->ctrl + c;
    const int grid = grid_1d(n, ctx->n_sms);
    timer_begin(ctx, F_OTHER, 5);
    bind_triple_resolve_kernel<<<grid, 256, 0, ctx->st>>>(P);
    bind_triple_mark_kernel<<<grid, 256, 0, ctx->st>>>(P);
    launch_exclusive_scan_u32(P.first, n + 1, static_cast<u32*>(scratch->p), ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->ctrl + c + 1, P.first + n, sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    if (ctx->h_ctrl[c]) return fail(ctx, KB_E_LIMIT, "TRIPLE batch table overflow");
    const u32 n_new = ctx->h_ctrl[c + 1];
    const u32 base = next_qt_id & 0x7FFFFFFFu;
    if (n_new && (u64)base + n_new > KB_QUOTED_MAX_SLOTS)
        return fail(ctx, KB_E_LIMIT, "TRIPLE: %u new quoted triples from id 0x%08x would pass the table's %u slots", n_new, next_qt_id, KB_QUOTED_MAX_SLOTS);
    // nothing has changed so far (the reverse index is a cache of the table); from here on the table grows
    if (n_new) KB_TRY(quoted_grow(ctx, base + n_new));
    P.next_qt_id = next_qt_id;
    P.ws = n_new ? static_cast<u32*>(ctx->quoted_s->p) : nullptr;
    P.wp = n_new ? static_cast<u32*>(ctx->quoted_p->p) : nullptr;
    P.wo = n_new ? static_cast<u32*>(ctx->quoted_o->p) : nullptr;
    P.old = old;
    P.out = out;
    P.n_unbound = n_unbound;
    timer_begin(ctx, F_OTHER);
    bind_triple_assign_kernel<<<grid, 256, 0, ctx->st>>>(P);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    if (n_new) {
        ctx->quoted_slots = base + n_new;
        KB_TRY(quoted_rev_ensure(ctx, 0));  // the new entries enter the reverse index
    }
    info->quoted_first = n_new ? next_qt_id : 0;
    info->quoted_new = n_new;
    return KB_OK;
}

kb_status kb::quoted_copy(kb_ctx* dst, const kb_ctx* src) {
    const u32 slots = src->quoted_slots;
    if (!slots) {
        quoted_reset(dst);
        return KB_OK;
    }
    const Buf* from[3] = {&src->quoted_s, &src->quoted_p, &src->quoted_o};
    Buf nb[3];  // the copy is complete before it replaces dst's table
    for (int k = 0; k < 3; k++) {
        KB_TRY(alloc_buf(dst, (size_t)slots * sizeof(u32), &nb[k]));
        KB_CUDA(dst, cudaMemcpyAsync(nb[k]->p, (*from[k])->p, (size_t)slots * sizeof(u32), cudaMemcpyDeviceToDevice, dst->st));
    }
    quoted_reset(dst);
    dst->quoted_s = nb[0]; dst->quoted_p = nb[1]; dst->quoted_o = nb[2];
    dst->quoted_slots = dst->quoted_cap = slots;
    return KB_OK;
}

extern "C" {

kb_status kb_quoted_load(kb_ctx* ctx, const uint32_t* ids, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n) {
    KB_ENTER(ctx);
    if (n == 0) {
        quoted_reset(ctx);
        return KB_OK;
    }
    if (!ids || !s || !p || !o) return fail(ctx, KB_E_INVALID, "NULL argument");
    u32 slots = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (!(ids[i] & 0x80000000u) || ids[i] == KB_ID_NONE)
            return fail(ctx, KB_E_INVALID, "entry %llu: id 0x%08x is not a quoted-triple id (bit 31, not KB_ID_NONE)", (unsigned long long)i, ids[i]);
        if (s[i] == KB_ID_NONE || p[i] == KB_ID_NONE || o[i] == KB_ID_NONE)
            return fail(ctx, KB_E_INVALID, "entry %llu: component KB_ID_NONE (reserved)", (unsigned long long)i);
        const u32 x = ids[i] & 0x7FFFFFFFu;
        if (x >= KB_QUOTED_MAX_SLOTS) return fail(ctx, KB_E_LIMIT, "quoted-triple id 0x%08x: index beyond the table's %u slots", ids[i], KB_QUOTED_MAX_SLOTS);
        slots = std::max(slots, x + 1u);
    }
    std::vector<u32> h((size_t)slots * 3, EMPTY32);  // s | p | o
    for (uint64_t i = 0; i < n; i++) {
        const u32 x = ids[i] & 0x7FFFFFFFu;
        if (h[(size_t)slots + x] != EMPTY32) return fail(ctx, KB_E_INVALID, "quoted-triple id 0x%08x given twice", ids[i]);
        h[x] = s[i];
        h[(size_t)slots + x] = p[i];
        h[2 * (size_t)slots + x] = o[i];
    }
    Buf bs, bp, bo;  // the new table is complete before it replaces the old one
    KB_TRY(alloc_buf(ctx, (size_t)slots * sizeof(u32), &bs));
    KB_TRY(alloc_buf(ctx, (size_t)slots * sizeof(u32), &bp));
    KB_TRY(alloc_buf(ctx, (size_t)slots * sizeof(u32), &bo));
    KB_CUDA(ctx, cudaMemcpyAsync(bs->p, h.data(), (size_t)slots * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(bp->p, h.data() + slots, (size_t)slots * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(bo->p, h.data() + 2 * (size_t)slots, (size_t)slots * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.h2d_bytes += (u64)slots * 12u;
    quoted_reset(ctx);  // (TRIPLE rebuilds the reverse index on its next call)
    ctx->quoted_s = bs; ctx->quoted_p = bp; ctx->quoted_o = bo;
    ctx->quoted_slots = ctx->quoted_cap = slots;
    return KB_OK;
}

// resolve_quoted_triple_scan (engine.rs:1111-1188): the match kernel gives one row (entry id in a fresh slot F, inner variables) per
// accepted entry; the outer pattern with F in the quoted position(s) is bind-joined to those rows, which merges the bindings and drops
// the rows whose shared variables conflict; F is projected away.
kb_status kb_scan_quoted(kb_ctx* ctx, const kb_quoted_pattern* qp, kb_rel** out) {
    KB_ENTER(ctx);
    if (!qp || !out) return fail(ctx, KB_E_INVALID, "NULL argument");
    const kb_pattern& op = qp->outer;
    if (op.p.is_var == KB_TERM_QUOTED) return fail(ctx, KB_E_UNSUPPORTED, "quoted triple in predicate position");
    const bool qs = op.s.is_var == KB_TERM_QUOTED, qo = op.o.is_var == KB_TERM_QUOTED;
    if (!qs && !qo) return fail(ctx, KB_E_INVALID, "kb_scan_quoted: neither subject nor object is quoted (use kb_scan)");
    // the terms in reading order: s, p, o with each quoted term inlined as its own s, p, o; inner terms carry their component
    struct T { const kb_term* t; int comp; };  // comp -1: a term of the outer pattern
    std::vector<T> terms;
    auto inline_pos = [&](const kb_term& t, const kb_pattern& in) {
        if (t.is_var == KB_TERM_QUOTED) { terms.push_back({&in.s, 0}); terms.push_back({&in.p, 1}); terms.push_back({&in.o, 2}); }
        else terms.push_back({&t, -1});
    };
    inline_pos(op.s, qp->inner_s);
    terms.push_back({&op.p, -1});
    inline_pos(op.o, qp->inner_o);
    std::vector<u32> used, order;  // every variable; the result's columns
    for (const T& x : terms) {
        if (x.t->is_var > KB_TERM_QUOTED || (x.comp < 0 && x.t->is_var == KB_TERM_QUOTED))
            return fail(ctx, KB_E_INVALID, "kb_term.is_var must be 0 or 1 (or KB_TERM_QUOTED in a quoted position / inside an inner pattern)");
        if (x.t->is_var == 0 && x.t->value == KB_ID_NONE) return fail(ctx, KB_E_INVALID, "constant id 0xFFFFFFFF is reserved (KB_ID_NONE)");
        if (x.t->is_var == 1) {
            if (x.t->value >= 4096) return fail(ctx, KB_E_LIMIT, "variable slot %u too large (max 4095)", x.t->value);
            if (std::find(order.begin(), order.end(), x.t->value) == order.end()) order.push_back(x.t->value);
        }
    }
    u32 F = 0;  // a slot no variable of the pattern uses
    while (std::find(order.begin(), order.end(), F) != order.end()) F++;
    // the match: checks on the entry's components, output columns (entry id, inner variables in order of first appearance)
    QuotedMatchParams P{};
    P.t = quotedtab(ctx);
    std::vector<u32> mslots{F};
    std::vector<std::pair<u32, u32>> first;  // inner variable -> component of its first occurrence
    for (const T& x : terms) {
        if (x.comp < 0) continue;
        if (x.t->is_var != 1u) {
            P.chk_kind[P.n_chk] = x.t->is_var == KB_TERM_QUOTED ? QM_QUOTED : QM_CONST;
            P.chk_comp[P.n_chk] = (u32)x.comp;
            P.chk_arg[P.n_chk++] = x.t->value;
        } else {
            auto it = std::find_if(first.begin(), first.end(), [&](const std::pair<u32, u32>& f) { return f.first == x.t->value; });
            if (it == first.end()) {
                first.push_back({x.t->value, (u32)x.comp});
                P.out_comp[mslots.size()] = (u32)x.comp;
                mslots.push_back(x.t->value);
            } else if (it->second != (u32)x.comp) {  // a repeated variable: equal components (the same entry fills both quoted positions)
                P.chk_kind[P.n_chk] = QM_EQ;
                P.chk_comp[P.n_chk] = (u32)x.comp;
                P.chk_arg[P.n_chk++] = it->second;
            }
        }
    }
    P.n_out = (u32)mslots.size();
    std::unique_ptr<kb_rel> res;
    if (P.t.n == 0) {
        KB_TRY(empty_rel(ctx, order, &res));
        ctx->stats.rows_out = 0;
        *out = res.release();
        return KB_OK;
    }
    auto m = std::make_unique<kb_rel>();
    m->slots = mslots;
    KB_TRY(alloc_strided_cols(ctx, P.t.n, P.n_out, &m->cols));
    for (u32 c = 0; c < P.n_out; c++) P.out[c] = m->cols[c].ptr;
    const u32 off = ctrl_alloc(ctx, 4);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 4 * sizeof(u32), ctx->st));
    P.count = ctx->ctrl + off;
    P.ticket = ctx->ctrl + off + 1;
    P.n_tiles = (P.t.n + QM_TILE - 1) / QM_TILE;
    timer_begin(ctx, F_SCAN);
    launch_quoted_match(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    m->n = ctx->h_ctrl[off];
    ctx->stats.rows_scanned += P.t.n;
    if (m->n == 0) {
        KB_TRY(empty_rel(ctx, order, &res));
    } else {
        kb_pattern po = op;
        if (qs) po.s = kb_term{1, F};
        if (qo) po.o = kb_term{1, F};
        std::unique_ptr<kb_rel> j;
        KB_TRY(bind_join_impl(ctx, *m, po, &j));
        res = select_cols(*j, order);
    }
    ctx->stats.rows_out = res->n;
    *out = res.release();
    return KB_OK;
}

kb_status kb_quoted_download(kb_ctx* ctx, uint32_t first_id, uint32_t n, uint32_t* s, uint32_t* p, uint32_t* o) {
    KB_ENTER(ctx);
    if (n == 0) return KB_OK;
    if (!s || !p || !o) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (!(first_id & 0x80000000u)) return fail(ctx, KB_E_INVALID, "0x%08x is not a quoted-triple id", first_id);
    const u64 x = first_id & 0x7FFFFFFFu;
    if (x + n > 0x7FFFFFFFull) return fail(ctx, KB_E_INVALID, "id range past 0xFFFFFFFE");
    const u64 held = x < ctx->quoted_slots ? std::min<u64>(n, ctx->quoted_slots - x) : 0;
    uint32_t* dst[3] = {s, p, o};
    const Buf* src[3] = {&ctx->quoted_s, &ctx->quoted_p, &ctx->quoted_o};
    for (int k = 0; k < 3; k++) {
        if (held) KB_CUDA(ctx, cudaMemcpyAsync(dst[k], static_cast<const u32*>((*src[k])->p) + x, held * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        std::fill(dst[k] + held, dst[k] + n, KB_ID_NONE);
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += held * 12u;
    return KB_OK;
}

}  // extern "C"
