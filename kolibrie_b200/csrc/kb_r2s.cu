// kb_r2s.cu — Relation-to-Stream operators on the device: Relation2StreamOperator::eval (kolibrie/src/rsp/r2s.rs:37-58) applied to
// a firing's result where the result already lives, so that a stream user downloads the rows that changed instead of the window's
// whole result. The operator keeps `last` (the distinct rows of the previous evaluation, first-occurrence order) and a table over it in
// device memory; one evaluation is: build a table over the response -> mark (representatives; ISTREAM: rows `last` lacks; DSTREAM:
// rows of `last` the response lacks) -> exclusive scans -> write the emitted rows and the new state. The new state is built in fresh
// buffers and replaces `last` only when every step succeeded.
#include <algorithm>

#include "kb_internal.hpp"

using namespace kb;

namespace kb {

// ---------------------------------------------------------------------------------------------------------------
// Relation-to-Stream operators (kb_r2s_eval; Relation2StreamOperator::eval, r2s.rs:37-58). A set of rows is an open-addressing table
// of u32 row indices (EMPTY32 = free slot) keyed by a 64-bit mix of the row's columns in the operator's slot order; a hash hit is
// confirmed by comparing every column.
struct R2sRows {
    const u32* col[KB_MAX_COLS];  // columns in the operator's slot order
    u32 n;
    u32* tab;                     // table over the rows (unused when n == 0)
    u32 mask;                     // table slots - 1
};
struct R2sParams {
    R2sRows cur;      // the response: its table is built, then remapped to the new state's columns
    R2sRows last;     // the previous state (read only)
    u32 n_cols;
    u32 probe_last;   // ISTREAM: flag the response rows whose tuple `last` does not hold
    u32* rep;         // [cur.n] 1 where row i is its tuple's representative (first occurrence); then its exclusive prefix
    u32* slot_of;     // [cur.n] table slot of row i's tuple
    u32* emit;        // ISTREAM: [cur.n] emitted response rows; DSTREAM: [last.n] rows of `last` that are gone (flags, then prefix)
    u32* counts;      // [2] zeroed: representatives, emitted rows
    u32 n_rep, n_emit;  // write passes: the totals of the two flag arrays
    u32* out_state[KB_MAX_COLS];
    u32* out_emit[KB_MAX_COLS];
};

// =================================================================================================================
// Relation-to-Stream operators (kb_r2s_eval). Row indices are 64-bit in the loops: a response may hold up to 2^32-1 rows.
__device__ __forceinline__ u64 r2s_mix64(u64 x) {  // murmur3 64-bit finaliser
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}
// home slot of row i: the columns are mixed in order, so rows that differ only by swapping two columns' values hash apart
__device__ __forceinline__ u32 r2s_home(const u32* const* col, u32 n_cols, u32 i, u32 mask) {
    u64 h = 0x9E3779B97F4A7C15ull;
    for (u32 c = 0; c < n_cols; c++) h = r2s_mix64(h ^ (u64)col[c][i]);
    return (u32)h & mask;
}
__device__ __forceinline__ bool r2s_equal(const u32* const* a, u32 ia, const u32* const* b, u32 ib, u32 n_cols) {
    for (u32 c = 0; c < n_cols; c++)
        if (a[c][ia] != b[c][ib]) return false;
    return true;
}
// does the set T hold the tuple of row i of `col`?
__device__ __forceinline__ bool r2s_contains(const R2sRows& T, const u32* const* col, u32 i, u32 n_cols) {
    if (T.n == 0u) return false;
    u32 slot = r2s_home(col, n_cols, i, T.mask);
    while (true) {
        const u32 held = T.tab[slot];
        if (held == EMPTY32) return false;
        if (r2s_equal(T.col, held, col, i, n_cols)) return true;
        slot = (slot + 1u) & T.mask;
    }
}
// warp-aggregated count of the lanes whose flag is set (every lane of the warp calls it)
__device__ __forceinline__ void r2s_count(bool flag, u32* counter) {
    const u32 b = __ballot_sync(0xffffffffu, flag);
    if ((threadIdx.x & 31u) == 0u && b) atomicAdd(counter, (u32)__popc(b));
}

__global__ void __launch_bounds__(256) r2s_build_kernel(const __grid_constant__ R2sParams P) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < P.cur.n; k += stride) {
        const u32 i = (u32)k;
        u32 slot = r2s_home(P.cur.col, P.n_cols, i, P.cur.mask);
        while (true) {
            u32 held = *(volatile u32*)&P.cur.tab[slot];
            if (held == EMPTY32) {
                held = atomicCAS(&P.cur.tab[slot], EMPTY32, i);
                if (held == EMPTY32) break;
            }
            // a slot only ever moves to a smaller index of the same tuple: the comparison with `held` stays valid
            if (r2s_equal(P.cur.col, held, P.cur.col, i, P.n_cols)) {
                if (held > i) atomicMin(&P.cur.tab[slot], i);
                break;
            }
            slot = (slot + 1u) & P.cur.mask;
        }
    }
}
__global__ void __launch_bounds__(256) r2s_mark_kernel(const __grid_constant__ R2sParams P) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 n_round = ((u64)P.cur.n + 31ull) & ~31ull;
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < n_round; k += stride) {
        bool rep = false, emit = false;
        if (k < P.cur.n) {
            const u32 i = (u32)k;
            u32 slot = r2s_home(P.cur.col, P.n_cols, i, P.cur.mask);
            u32 held;
            while (true) {  // the tuple was inserted: it is found before any free slot
                held = P.cur.tab[slot];
                if (held != EMPTY32 && r2s_equal(P.cur.col, held, P.cur.col, i, P.n_cols)) break;
                slot = (slot + 1u) & P.cur.mask;
            }
            rep = held == i;
            P.rep[i] = rep ? 1u : 0u;
            P.slot_of[i] = slot;
            if (P.probe_last) {
                emit = !r2s_contains(P.last, P.cur.col, i, P.n_cols);
                P.emit[i] = emit ? 1u : 0u;
            }
        }
        r2s_count(rep, &P.counts[0]);
        r2s_count(emit, &P.counts[1]);
    }
}
__global__ void __launch_bounds__(256) r2s_gone_mark_kernel(const __grid_constant__ R2sParams P) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 n_round = ((u64)P.last.n + 31ull) & ~31ull;
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < n_round; k += stride) {
        bool gone = false;
        if (k < P.last.n) {
            gone = !r2s_contains(P.cur, P.last.col, (u32)k, P.n_cols);
            P.emit[k] = gone ? 1u : 0u;
        }
        r2s_count(gone, &P.counts[1]);
    }
}
// a row is taken iff its exclusive prefix differs from the next row's (the last row: from the total)
__device__ __forceinline__ bool r2s_taken(const u32* off, u64 k, u64 n, u32 total, u32* at) {
    *at = off[k];
    return (k + 1ull < n ? off[k + 1] : total) != *at;
}
__global__ void __launch_bounds__(256) r2s_write_kernel(const __grid_constant__ R2sParams P) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < P.cur.n; k += stride) {
        const u32 i = (u32)k;
        u32 at;
        if (r2s_taken(P.rep, k, P.cur.n, P.n_rep, &at)) {
            for (u32 c = 0; c < P.n_cols; c++) P.out_state[c][at] = P.cur.col[c][i];
            P.cur.tab[P.slot_of[i]] = at;  // the table now indexes the new state's columns
        }
        if (P.probe_last && r2s_taken(P.emit, k, P.cur.n, P.n_emit, &at))
            for (u32 c = 0; c < P.n_cols; c++) P.out_emit[c][at] = P.cur.col[c][i];
    }
}
__global__ void __launch_bounds__(256) r2s_gone_write_kernel(const __grid_constant__ R2sParams P) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < P.last.n; k += stride) {
        u32 at;
        if (r2s_taken(P.emit, k, P.last.n, P.n_emit, &at))
            for (u32 c = 0; c < P.n_cols; c++) P.out_emit[c][at] = P.last.col[c][(u32)k];
    }
}
// build: every response row goes into cur's table (atomicCAS on a free slot, atomicMin on a slot holding an equal row: the slot ends
// up holding the tuple's first occurrence, whatever the thread order)
static void launch_r2s_build(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.cur.n) r2s_build_kernel<<<grid_1d(p.cur.n, n_sms), 256, 0, st>>>(p);
}
// mark: rep, slot_of and, with probe_last, emit (+ counts)
static void launch_r2s_mark(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.cur.n) r2s_mark_kernel<<<grid_1d(p.cur.n, n_sms), 256, 0, st>>>(p);
}
// DSTREAM mark: emit[j] = row j of `last` has no equal row in the response (+ counts[1]); runs before the remap
static void launch_r2s_gone_mark(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.last.n) r2s_gone_mark_kernel<<<grid_1d(p.last.n, n_sms), 256, 0, st>>>(p);
}
// write, after the exclusive scans: the representatives into out_state (and cur's table remapped to them), with probe_last the
// emitted rows into out_emit
static void launch_r2s_write(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.cur.n) r2s_write_kernel<<<grid_1d(p.cur.n, n_sms), 256, 0, st>>>(p);
}
// DSTREAM write: the gone rows of `last` into out_emit, in `last` order
static void launch_r2s_gone_write(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.last.n) r2s_gone_write_kernel<<<grid_1d(p.last.n, n_sms), 256, 0, st>>>(p);
}

}  // namespace kb

struct kb_r2s {
    u32 op = KB_RSTREAM;
    std::vector<u32> slots;  // column order of every row the operator compares, stores and emits
    std::vector<Col> cols;   // last: distinct rows, in the order of their first occurrence in the response that set them
    u64 n = 0;
    Buf tab;                 // table over `cols` (null when n == 0)
    u32 mask = 0;
};

namespace {

// the response's columns in the operator's slot order; false when its slot set is not the operator's
bool canonical_cols(const kb_r2s& op, const kb_rel& r, const u32** cols) {
    if (r.pair || r.slots.size() != op.slots.size() || r.cols.size() != op.slots.size()) return false;
    for (size_t c = 0; c < op.slots.size(); c++) {
        const int k = r.col_of(op.slots[c]);
        if (k < 0) return false;
        cols[c] = r.cols[k].ptr;
    }
    return true;
}

kb_status r2s_eval(kb_ctx* ctx, kb_r2s* op, const kb_rel* response, kb_rel** emitted) {
    const u32 nc = (u32)op->slots.size();
    R2sParams P{};
    if (!canonical_cols(*op, *response, P.cur.col))
        return fail(ctx, KB_E_INVALID, "the response's variables are not the %u slots the stream operator was created with", nc);
    if (op->op == KB_RSTREAM)  // r2s.rs:39: the response itself; `last` is not touched
        return kb_project(ctx, response, response->slots.data(), (u32)response->slots.size(), emitted);
    if (response->n > 0xFFFFFFFFull) return fail(ctx, KB_E_LIMIT, "a response of %llu rows (limit 2^32-1)", (unsigned long long)response->n);
    const u64 n = response->n, L = op->n;
    const bool istream = op->op == KB_ISTREAM;
    P.n_cols = nc;
    P.cur.n = (u32)n;
    P.last.n = (u32)L;
    for (u32 c = 0; c < nc; c++) P.last.col[c] = op->cols[c].ptr;
    P.last.tab = op->tab ? static_cast<u32*>(op->tab->p) : nullptr;
    P.last.mask = op->mask;
    P.probe_last = istream ? 1u : 0u;

    // the new table: 2x the response rows, a power of two (capped at 2^32 slots: the row indices are u32, so it never fills)
    const u64 slots = n ? std::min<u64>(1ull << 32, std::max<u64>(2ull, 1ull << (64 - __builtin_clzll(2 * n - 1)))) : 0;
    Buf tab, rep, slot_of, emit, scratch;
    const u64 flags = istream ? n : L;  // rows the emit flags cover
    if (n) {
        KB_TRY(alloc_buf(ctx, slots * sizeof(u32), &tab));
        KB_TRY(alloc_buf(ctx, n * sizeof(u32), &rep));
        KB_TRY(alloc_buf(ctx, n * sizeof(u32), &slot_of));
        KB_CUDA(ctx, cudaMemsetAsync(tab->p, 0xFF, slots * sizeof(u32), ctx->st));
        P.cur.tab = static_cast<u32*>(tab->p);
        P.cur.mask = (u32)(slots - 1);
        P.rep = static_cast<u32*>(rep->p);
        P.slot_of = static_cast<u32*>(slot_of->p);
    }
    if (flags) {
        KB_TRY(alloc_buf(ctx, flags * sizeof(u32), &emit));
        P.emit = static_cast<u32*>(emit->p);
    }
    const u64 scan_n = std::max(n, flags);
    if (scan_n) KB_TRY(alloc_buf(ctx, ((scan_n + 2047) / 2048 + 1) * sizeof(u32), &scratch));
    const u32 cw = ctrl_alloc(ctx, 4);
    P.counts = ctx->ctrl + cw;
    KB_CUDA(ctx, cudaMemsetAsync(P.counts, 0, 4 * sizeof(u32), ctx->st));

    // build, mark, scans (a scan is 3 launches)
    const int k_mark = (n ? 2 + 3 : 0) + (flags ? 3 : 0) + (!istream && L ? 1 : 0);
    if (k_mark) {
        timer_begin(ctx, F_OTHER, k_mark);
        launch_r2s_build(P, ctx->n_sms, ctx->st);
        launch_r2s_mark(P, ctx->n_sms, ctx->st);
        if (!istream) launch_r2s_gone_mark(P, ctx->n_sms, ctx->st);
        if (n) launch_exclusive_scan_u32(P.rep, (u32)n, static_cast<u32*>(scratch->p), ctx->st);
        if (flags) launch_exclusive_scan_u32(P.emit, (u32)flags, static_cast<u32*>(scratch->p), ctx->st);
        timer_end(ctx);
    }
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    P.n_rep = ctx->h_ctrl[cw];
    P.n_emit = ctx->h_ctrl[cw + 1];

    // the emitted rows and the new state, each in buffers of exactly its size
    auto out = std::make_unique<kb_rel>();
    out->slots = op->slots;
    out->n = P.n_emit;
    std::vector<Col> state(nc);
    for (u32 c = 0; c < nc; c++) {
        Col e;
        KB_TRY(alloc_col(ctx, P.n_emit, &e));
        out->cols.push_back(e);
        P.out_emit[c] = e.ptr;
        KB_TRY(alloc_col(ctx, P.n_rep, &state[c]));
        P.out_state[c] = state[c].ptr;
    }
    const int k_write = (n ? 1 : 0) + (!istream && L ? 1 : 0);
    if (k_write) {
        timer_begin(ctx, F_OTHER, k_write);
        launch_r2s_write(P, ctx->n_sms, ctx->st);
        if (!istream) launch_r2s_gone_write(P, ctx->n_sms, ctx->st);
        timer_end(ctx);
    }
    KB_CUDA(ctx, cudaGetLastError());
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    timers_flush(ctx);

    // every step succeeded: the response's distinct rows become `last`
    op->cols = std::move(state);
    op->n = P.n_rep;
    op->tab = tab;
    op->mask = n ? P.cur.mask : 0u;
    ctx->stats.rows_out = out->n;
    *emitted = out.release();
    return KB_OK;
}

}  // namespace

extern "C" {

kb_status kb_r2s_create(kb_ctx* ctx, uint32_t stream_op, const uint32_t* slots, uint32_t n_cols, kb_r2s** out) {
    if (!ctx) return KB_E_INVALID;
    ctx->err.clear();
    if (!slots || !out) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (stream_op > KB_DSTREAM) return fail(ctx, KB_E_INVALID, "unknown stream operator %u", stream_op);
    if (n_cols == 0 || n_cols > KB_MAX_COLS) return fail(ctx, KB_E_INVALID, "a stream operator compares 1..%d columns (got %u)", KB_MAX_COLS, n_cols);
    for (u32 c = 0; c < n_cols; c++)
        for (u32 d = 0; d < c; d++)
            if (slots[c] == slots[d]) return fail(ctx, KB_E_INVALID, "duplicate slot %u", slots[c]);
    auto op = std::make_unique<kb_r2s>();
    op->op = stream_op;
    op->slots.assign(slots, slots + n_cols);
    op->cols.resize(n_cols);
    *out = op.release();
    return KB_OK;
}

kb_status kb_r2s_eval(kb_ctx* ctx, kb_r2s* op, const kb_rel* response, kb_rel** emitted) {
    if (!ctx) return KB_E_INVALID;
    DeviceGuard guard(ctx->device);
    KB_TRY(begin_call(ctx));
    if (!op || !response || !emitted) return fail(ctx, KB_E_INVALID, "NULL argument");
    return r2s_eval(ctx, op, response, emitted);
}

kb_status kb_r2s_info(const kb_r2s* op, uint64_t* last_rows, uint32_t* stream_op) {
    if (!op) return KB_E_INVALID;
    if (last_rows) *last_rows = op->n;
    if (stream_op) *stream_op = op->op;
    return KB_OK;
}

void kb_r2s_free(kb_ctx* ctx, kb_r2s* op) {
    if (!op) return;
    if (ctx) {
        DeviceGuard guard(ctx->device);
        delete op;
    } else delete op;
}

}  // extern "C"
