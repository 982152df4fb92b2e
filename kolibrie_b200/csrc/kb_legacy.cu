// kb_legacy.cu — the FFI symbol Kolibrie already binds (include/cudajoin.h): predicate (+ optional object-literal) select.
// Replaces kolibrie/src/cuda/cuda_join.cu:48-118. Only the columns the select reads are uploaded (the reference uploads
// subjects and objects it never touches, cuda_join.cu:68-70), the kernel is the same fused TMA scan used everywhere else,
// and the indices come back ascending.
#include <cstdlib>
#include <mutex>

#include "../../include/cudajoin.h"
#include "kb_internal.hpp"

using namespace kb;

static std::mutex g_legacy_mutex;
static kb_ctx* g_legacy_ctx = nullptr;

static kb_status legacy_select(kb_ctx* ctx, const u32* h_p, const u32* h_o, u32 n, u32 pred, const u32* literal, u32** out_idx, u32* out_n) {
    KB_TRY(begin_call(ctx));
    ctx->ordered = 1;  // the legacy contract returns ascending indices
    Segment sg;  // scanned on its own: the context's store is not involved
    sg.n = n;
    KB_TRY(alloc_col(ctx, n, &sg.p));
    KB_CUDA(ctx, cudaMemcpyAsync(sg.p.ptr, h_p, (size_t)n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    sg.s = sg.p;  // the select never looks at subjects: alias instead of uploading 4N more bytes
    if (literal) {
        KB_TRY(alloc_col(ctx, n, &sg.o));
        KB_CUDA(ctx, cudaMemcpyAsync(sg.o.ptr, h_o, (size_t)n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    } else {
        sg.o = sg.p;
    }
    ctx->stats.h2d_bytes += (literal ? 2ull : 1ull) * n * sizeof(u32);
    kb_pattern pt;
    pt.s = kb_term{1, 0};
    pt.p = kb_term{0, pred};
    pt.o = literal ? kb_term{0, *literal} : kb_term{1, 1};
    std::vector<std::unique_ptr<kb_rel>> rels;
    std::vector<FilterProg> none;
    KB_TRY(scan_segments(ctx, {sg}, &pt, 1, none, ScanOut::RowIndex, &rels));
    const u64 m = rels[0]->n;
    u32* idx = static_cast<u32*>(malloc(std::max<size_t>(m * sizeof(u32), 4)));
    if (!idx) return fail(ctx, KB_E_OOM, "malloc failed");
    if (m) {
        KB_CUDA(ctx, cudaMemcpyAsync(idx, rels[0]->cols[0].ptr, m * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        ctx->stats.d2h_bytes += m * sizeof(u32);
    }
    *out_idx = idx;
    *out_n = (u32)m;
    return KB_OK;
}

extern "C" void perform_hash_join_cuda(const uint32_t* h_subjects, const uint32_t* h_predicates, const uint32_t* h_objects,
                                       uint32_t num_triples, uint32_t predicate_filter, uint32_t* literal_filter, uint32_t** h_indices,
                                       uint32_t* h_result_count) {
    (void)h_subjects;
    if (!h_indices || !h_result_count) return;
    *h_result_count = 0;
    *h_indices = nullptr;
    std::lock_guard<std::mutex> lock(g_legacy_mutex);
    kb_status rc = KB_OK;
    if (!g_legacy_ctx) rc = kb_ctx_create(0, &g_legacy_ctx);
    if (rc == KB_OK && num_triples > 0 && h_predicates && (!literal_filter || h_objects) && predicate_filter != KB_ID_NONE &&
        (!literal_filter || *literal_filter != KB_ID_NONE)) {
        int prev = -1;
        cudaGetDevice(&prev);
        cudaSetDevice(g_legacy_ctx->device);
        u32* idx = nullptr;
        u32 m = 0;
        rc = legacy_select(g_legacy_ctx, h_predicates, h_objects, num_triples, predicate_filter, literal_filter, &idx, &m);
        if (prev >= 0) cudaSetDevice(prev);
        if (rc == KB_OK) {
            *h_indices = idx;
            *h_result_count = m;
            return;
        }
        fprintf(stderr, "kolibrie_b200: perform_hash_join_cuda failed: %s\n", kb_last_error(g_legacy_ctx));
    } else if (rc != KB_OK) {
        fprintf(stderr, "kolibrie_b200: perform_hash_join_cuda: %s\n", kb_last_error(nullptr));
    }
    // error / empty: count 0 and a non-null malloc'd pointer (Rust's Vec::from_raw_parts needs non-null, cuda_join.rs:55)
    *h_indices = static_cast<uint32_t*>(malloc(4));
    *h_result_count = 0;
}
