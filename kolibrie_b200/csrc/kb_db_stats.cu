// kb_db_stats.cu — the optimizer's store statistics: DatabaseStats::gather_stats_fast (database_stats.rs:43-105) over the device store.
//
// kb_store_gather_stats works in three phases, each timed in kb_db_stats_info.phase_ms:
//   sort + dedup  store_distinct (kb_serialize.cu): the live segments' distinct triples in ascending (s, p, o) order, the reference's
//                 BTreeSet<Triple> iteration order
//   gather        the `take` sampled rows (positions 0, step, 2 step, ...) as three u32 columns
//   counts        subjects need no sort: any subsequence of the (s, p, o) order is grouped by s. Predicates and objects take a radix
//                 sort of `take` keys. Each column then gets a run-length encode: head flags, the run starts selected by CUB, and
//                 one pass that writes (id, run length * step). One control-arena read gives the run counts, and the maps come back to
//                 the host.
// The quoted-triple count is a count of the table's entries (a hole has p = EMPTY32) in the same control-arena read.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>

#include "kb_internal.hpp"

using kb::u32;
using kb::u64;
using kb::u8;

struct kb_db_stats {
    std::vector<u32> ids[3];
    std::vector<uint64_t> counts[3];
};

namespace kb {
namespace {

constexpr int DT = 256;  // threads per block of every kernel here

struct Cols3 {
    const u32* c[3];
};

// the sampled rows: row k is distinct triple k * step; cols = s | p | o, `take` entries each
__global__ void __launch_bounds__(DT) dbs_gather_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u64 take, u64 step,
                                                        u32* __restrict__ cols) {
    for (u64 k = blockIdx.x * (u64)blockDim.x + threadIdx.x; k < take; k += (u64)gridDim.x * blockDim.x) {
        const u64 i = k * step;
        const unsigned long long po = PO[i];
        cols[k] = S[i];
        cols[take + k] = (u32)(po >> 32);
        cols[2 * take + k] = (u32)po;
    }
}

// heads[j * m + i] = 1 where row i of sorted column j starts a run
__global__ void __launch_bounds__(DT) dbs_heads_kernel(const __grid_constant__ Cols3 C, u32 m, u8* __restrict__ heads) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x)
#pragma unroll
        for (int j = 0; j < 3; j++) heads[(u64)j * m + i] = i == 0u || C.c[j][i] != C.c[j][i - 1];
}

// run r of column j starts at starts[j * m + r]; runs[j] runs: ids[j * m + r] = its id, counts[j * m + r] = its length * step
__global__ void __launch_bounds__(DT) dbs_counts_kernel(const __grid_constant__ Cols3 C, const u32* __restrict__ starts, const u32* __restrict__ runs,
                                                        u32 m, u64 step, u32* __restrict__ ids, unsigned long long* __restrict__ counts) {
    const u32 nr[3] = {runs[0], runs[1], runs[2]};
    for (u32 r = blockIdx.x * blockDim.x + threadIdx.x; r < m; r += gridDim.x * blockDim.x)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            if (r >= nr[j]) continue;
            const u32* st = starts + (u64)j * m;
            const u32 a = st[r], b = r + 1u < nr[j] ? st[r + 1] : m;
            ids[(u64)j * m + r] = C.c[j][a];
            counts[(u64)j * m + r] = (unsigned long long)(b - a) * step;
        }
}

// entries of the quoted-triple table: slots whose predicate is not EMPTY32
__global__ void __launch_bounds__(DT) dbs_quoted_count_kernel(const u32* __restrict__ qp, u32 n, u32* count) {
    u32 c = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) c += qp[i] != EMPTY32;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

kb_status gather_stats(kb_ctx* ctx, u64 max_sample, kb_db_stats* out, kb_db_stats_info* info) {
    u64 n_raw = 0;
    const std::vector<ColSpan> spans = store_spans(ctx, &n_raw);
    if (n_raw >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "a store of %llu triples (statistics: limit 2^32 - 16)", (unsigned long long)n_raw);
    auto U = [](const Buf& b) { return static_cast<u32*>(b->p); };
    const u32 cq = ctrl_alloc(ctx, 4);  // [0..2] runs per column, [3] quoted-triple entries
    if (ctx->quoted_slots) {
        timer_begin(ctx, F_OTHER, 1);
        dbs_quoted_count_kernel<<<grid_1d(ctx->quoted_slots, ctx->n_sms, DT), DT, 0, ctx->st>>>(quotedtab(ctx).p, ctx->quoted_slots, ctx->ctrl + cq + 3);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
    }
    if (n_raw == 0) {
        if (ctx->quoted_slots) KB_TRY(ctrl_read(ctx));
        info->quoted_triple_count = ctx->quoted_slots ? ctx->h_ctrl[cq + 3] : 0u;
        info->step = 1;
        return KB_OK;
    }
    ScopedEvent ev[4];
    KB_CUDA(ctx, cudaEventRecord(ev[0], ctx->st));
    Buf S, PO;
    u32 T = 0;
    KB_TRY(store_distinct(ctx, spans, &S, &PO, &T));
    KB_CUDA(ctx, cudaEventRecord(ev[1], ctx->st));

    const u64 take = max_sample ? std::min<u64>(T, max_sample) : T;
    const u64 step = max_sample && T > max_sample ? T / take : 1;
    const u32 m = (u32)take;  // T >= 1, so m >= 1
    Buf cols, sorted;
    KB_TRY(alloc_buf(ctx, 3ull * m * 4, &cols));
    timer_begin(ctx, F_OTHER, 1);
    dbs_gather_kernel<<<grid_1d(m, ctx->n_sms, DT), DT, 0, ctx->st>>>(U(S), static_cast<const unsigned long long*>(PO->p), m, step, U(cols));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    S.reset(); PO.reset();
    KB_CUDA(ctx, cudaEventRecord(ev[2], ctx->st));

    KB_TRY(alloc_buf(ctx, 3ull * m * 4, &sorted));
    Cols3 C{{U(cols), U(sorted) + m, U(sorted) + 2ull * m}};  // subjects are grouped already
    timer_begin(ctx, F_OTHER, 2);
    for (int j = 1; j < 3; j++)
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, U(cols) + (u64)j * m, U(sorted) + (u64)j * m, m, 0, 32, ctx->st); }));
    timer_end(ctx);
    Buf heads, starts, ids, counts;
    KB_TRY(alloc_buf(ctx, 3ull * m, &heads));
    KB_TRY(alloc_buf(ctx, 3ull * m * 4, &starts));
    KB_TRY(alloc_buf(ctx, 3ull * m * 4, &ids));
    KB_TRY(alloc_buf(ctx, 3ull * m * 8, &counts));
    const u8* h = static_cast<const u8*>(heads->p);
    timer_begin(ctx, F_OTHER, 5);
    dbs_heads_kernel<<<grid_1d(m, ctx->n_sms, DT), DT, 0, ctx->st>>>(C, m, static_cast<u8*>(heads->p));
    for (int j = 0; j < 3; j++)
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) {
            return cub::DeviceSelect::Flagged(t, b, thrust::counting_iterator<u32>(0), h + (u64)j * m, U(starts) + (u64)j * m, ctx->ctrl + cq + j, m, ctx->st);
        }));
    dbs_counts_kernel<<<grid_1d(m, ctx->n_sms, DT), DT, 0, ctx->st>>>(C, U(starts), ctx->ctrl + cq, m, step, U(ids),
                                                                       static_cast<unsigned long long*>(counts->p));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_CUDA(ctx, cudaEventRecord(ev[3], ctx->st));
    KB_TRY(ctrl_read(ctx));
    for (int j = 0; j < 3; j++) {
        const u32 runs = ctx->h_ctrl[cq + j];
        out->ids[j].resize(runs);
        out->counts[j].resize(runs);
        KB_CUDA(ctx, cudaMemcpyAsync(out->ids[j].data(), U(ids) + (u64)j * m, (size_t)runs * 4, cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(out->counts[j].data(), static_cast<const unsigned long long*>(counts->p) + (u64)j * m, (size_t)runs * 8,
                                     cudaMemcpyDeviceToHost, ctx->st));
        ctx->stats.d2h_bytes += (u64)runs * 12;
        info->n_ids[j] = runs;
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    info->total_triples = T;
    info->quoted_triple_count = ctx->quoted_slots ? ctx->h_ctrl[cq + 3] : 0u;
    info->take = take;
    info->step = step;
    for (int k = 0; k < 3; k++) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev[k], ev[k + 1]);
        info->phase_ms[k] = ms;
    }
    return KB_OK;
}

}  // namespace
}  // namespace kb

extern "C" {

kb_status kb_store_gather_stats(kb_ctx* ctx, uint64_t max_sample, kb_db_stats** out, kb_db_stats_info* info) {
    KB_ENTER(ctx);
    kb_db_stats_info local{};
    if (!info) info = &local;
    *info = kb_db_stats_info{};
    if (!out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    auto st = std::make_unique<kb_db_stats>();
    KB_TRY(kb::gather_stats(ctx, max_sample, st.get(), info));
    *out = st.release();
    return KB_OK;
}

kb_status kb_db_stats_counts(const kb_db_stats* st, uint32_t position, const uint32_t** ids, const uint64_t** counts, uint64_t* n) {
    if (!st || !ids || !counts || !n || position > 2) return KB_E_INVALID;
    *ids = st->ids[position].data();
    *counts = st->counts[position].data();
    *n = st->ids[position].size();
    return KB_OK;
}

void kb_db_stats_free(kb_db_stats* st) { delete st; }

}  // extern "C"
