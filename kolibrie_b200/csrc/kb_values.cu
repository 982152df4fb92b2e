// kb_values.cu — `PhysicalOperator::Values` (kolibrie/src/streamertail_optimizer/execution/engine.rs:279-308) on the device, so that a
// VALUES block, which the plan builder makes the base of the whole join chain (streamertail_optimizer/utils.rs:110-171), does not send the
// plan to the CPU. The semantics are in include/kolibrie_b200.h; here:
//   K1 values_flag_kernel     thread per row: defined[cell] and keep[row] (the row has a defined cell)
//      two exclusive scans    position of every defined cell in encode order (row-major, UNDEF skipped), output row of every kept row
//   K2 values_compact_kernel  the defined cells' offsets in encode order (an UNDEF cell is empty, so the next defined offset closes it)
//      dict_encode_device     kb_dict_encode's body: the ids of the sequential Dictionary::encode loop, new strings in first-seen order
//   K3 values_scatter_kernel  thread per kept row: per column the id of the row's LAST defined cell of that slot, else KB_ID_NONE
// then kb_dict_numeric_derive's body extends the f64 side table over the new ids.
#include <algorithm>

#include "kb_internal.hpp"
#include "kb_kernels.cuh"

namespace kb {
namespace {

struct ValuesParams {
    const u8* undef;          // [n_rows * n_vars]
    const u64* off;           // [n_cells + 1] cell offsets into the batch bytes
    const u32* var_col;       // [n_vars] output column of header variable v
    u32 n_rows, n_vars, n_cols;
    u32* cell_rank;           // [n_cells + 1] defined flag, then its exclusive prefix
    u32* row_rank;            // [n_rows + 1] keep flag, then its exclusive prefix
    u64* enc_off;             // [n_def + 1] offsets of the defined cells in encode order
    const u32* ids;           // [n_def] ids in encode order
    u32* out[KB_MAX_COLS];
};

__global__ void __launch_bounds__(256) values_flag_kernel(const __grid_constant__ ValuesParams P) {
    for (u32 r = blockIdx.x * blockDim.x + threadIdx.x; r < P.n_rows; r += gridDim.x * blockDim.x) {
        u32 any = 0;
        for (u32 v = 0; v < P.n_vars; v++) {
            const u64 i = (u64)r * P.n_vars + v;
            const u32 d = __ldg(P.undef + i) ? 0u : 1u;
            P.cell_rank[i] = d;
            any |= d;
        }
        P.row_rank[r] = any;  // `if !row.is_empty()` (engine.rs:302)
    }
}

// cells [0, n_cells]: the closing offset of the batch goes behind the last defined cell
__global__ void __launch_bounds__(256) values_compact_kernel(const __grid_constant__ ValuesParams P) {
    const u64 n_cells = (u64)P.n_rows * P.n_vars;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= n_cells; i += (u64)gridDim.x * blockDim.x)
        if (i == n_cells || !__ldg(P.undef + i)) P.enc_off[P.cell_rank[i]] = __ldg(P.off + i);
}

__global__ void __launch_bounds__(256) values_scatter_kernel(const __grid_constant__ ValuesParams P) {
    for (u32 r = blockIdx.x * blockDim.x + threadIdx.x; r < P.n_rows; r += gridDim.x * blockDim.x) {
        const u32 o = P.row_rank[r];
        if (P.row_rank[r + 1] == o) continue;  // dropped row
        for (u32 c = 0; c < P.n_cols; c++) {
            u32 val = KB_ID_NONE;
            for (u32 v = 0; v < P.n_vars; v++) {  // header order: a repeated variable keeps its later defined cell (row.insert overwrites)
                const u64 i = (u64)r * P.n_vars + v;
                if (__ldg(P.var_col + v) == c && !__ldg(P.undef + i)) val = __ldg(P.ids + P.cell_rank[i]);
            }
            P.out[c][o] = val;
        }
    }
}

}  // namespace
}  // namespace kb

using namespace kb;

extern "C" {

kb_status kb_values(kb_ctx* ctx, const uint32_t* slots, uint32_t n_vars, uint64_t n_rows, const uint8_t* undef, const uint64_t* offsets,
                    const uint8_t* bytes, kb_rel** out, kb_values_info* info) {
    KB_ENTER(ctx);
    if (!out || !offsets || (n_vars && !slots)) return fail(ctx, KB_E_INVALID, "NULL argument");
    const u64 n_cells = n_rows * (u64)n_vars;
    if (n_rows >= 0xFFFFFFF0ull || n_cells >= 0xFFFFFFF0ull)
        return fail(ctx, KB_E_LIMIT, "kb_values: %llu rows of %u cells (limit 2^32-16 rows and cells per call)", (unsigned long long)n_rows, n_vars);
    if (n_cells && !undef) return fail(ctx, KB_E_INVALID, "NULL undef mask");
    // the columns: one per distinct slot, in order of first appearance in the header
    std::vector<u32> cols, var_col(n_vars);
    for (u32 v = 0; v < n_vars; v++) {
        u32 c = 0;
        while (c < cols.size() && cols[c] != slots[v]) c++;
        if (c == cols.size()) {
            if (cols.size() == KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "kb_values: more than %d distinct variables", KB_MAX_COLS);
            cols.push_back(slots[v]);
        }
        var_col[v] = c;
    }
    if (offsets[0] != 0) return fail(ctx, KB_E_INVALID, "kb_values: offsets must start at 0");
    for (u64 i = 0; i < n_cells; i++) {
        if (offsets[i + 1] < offsets[i]) return fail(ctx, KB_E_INVALID, "kb_values: offsets decrease at cell %llu", (unsigned long long)i);
        if (undef[i] && offsets[i + 1] != offsets[i]) return fail(ctx, KB_E_INVALID, "kb_values: UNDEF cell %llu is not empty", (unsigned long long)i);
    }
    const u64 total = offsets[n_cells];
    if (total > 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "kb_values: %llu bytes of cells (limit 2^32-16 per call)", (unsigned long long)total);
    if (total && !bytes) return fail(ctx, KB_E_INVALID, "NULL bytes");
    kb_values_info inf{};
    inf.dict_first = ctx->dict_ids;
    std::unique_ptr<kb_rel> r;
    if (n_cells == 0) {
        KB_TRY(empty_rel(ctx, cols, &r));
        inf.rows_dropped = n_rows;
        if (info) *info = inf;
        ctx->stats.rows_out = 0;
        *out = r.release();
        return KB_OK;
    }
    const u32 nr = (u32)n_rows;
    Buf d_undef, d_off, d_bytes, d_varcol, cell_rank, row_rank, scratch;
    KB_TRY(alloc_buf(ctx, (size_t)n_cells, &d_undef));
    KB_TRY(alloc_buf(ctx, ((size_t)n_cells + 1) * sizeof(u64), &d_off));
    KB_TRY(alloc_buf(ctx, (size_t)total + 16, &d_bytes));
    KB_TRY(alloc_buf(ctx, (size_t)n_vars * sizeof(u32), &d_varcol));
    KB_TRY(alloc_buf(ctx, ((size_t)n_cells + 1) * sizeof(u32), &cell_rank));
    KB_TRY(alloc_buf(ctx, ((size_t)nr + 1) * sizeof(u32), &row_rank));
    KB_TRY(alloc_buf(ctx, (((size_t)n_cells + 1) / 2048 + 4) * sizeof(u32), &scratch));
    KB_CUDA(ctx, cudaMemcpyAsync(d_undef->p, undef, (size_t)n_cells, cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(d_off->p, offsets, ((size_t)n_cells + 1) * sizeof(u64), cudaMemcpyHostToDevice, ctx->st));
    if (total) KB_CUDA(ctx, cudaMemcpyAsync(d_bytes->p, bytes, (size_t)total, cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(d_varcol->p, var_col.data(), (size_t)n_vars * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    ctx->stats.h2d_bytes += n_cells + (n_cells + 1) * sizeof(u64) + total + (u64)n_vars * sizeof(u32);
    ValuesParams P{};
    P.undef = static_cast<const u8*>(d_undef->p);
    P.off = static_cast<const u64*>(d_off->p);
    P.var_col = static_cast<const u32*>(d_varcol->p);
    P.n_rows = nr;
    P.n_vars = n_vars;
    P.n_cols = (u32)cols.size();
    P.cell_rank = static_cast<u32*>(cell_rank->p);
    P.row_rank = static_cast<u32*>(row_rank->p);
    KB_CUDA(ctx, cudaMemsetAsync(P.cell_rank + n_cells, 0, sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(P.row_rank + nr, 0, sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER, 3);
    values_flag_kernel<<<grid_1d(nr, ctx->n_sms), 256, 0, ctx->st>>>(P);
    launch_exclusive_scan_u32(P.cell_rank, (u32)n_cells + 1, static_cast<u32*>(scratch->p), ctx->st);
    launch_exclusive_scan_u32(P.row_rank, nr + 1, static_cast<u32*>(scratch->p), ctx->st);
    timer_end(ctx);
    const u32 c = ctrl_alloc(ctx, 2);  // [0] defined cells, [1] kept rows
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->ctrl + c, P.cell_rank + n_cells, sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->ctrl + c + 1, P.row_rank + nr, sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32 n_def = ctx->h_ctrl[c], n_kept = ctx->h_ctrl[c + 1];
    if ((u64)ctx->dict_ids + n_def >= 0x80000000ull) return fail(ctx, KB_E_LIMIT, "kb_values: dictionary ids would reach bit 31");
    // checked: the dictionary changes from here on
    Buf enc_off, ids;
    KB_TRY(alloc_buf(ctx, ((size_t)n_def + 1) * sizeof(u64), &enc_off));
    KB_TRY(alloc_buf(ctx, std::max<size_t>((size_t)n_def, 1) * sizeof(u32), &ids));
    P.enc_off = static_cast<u64*>(enc_off->p);
    P.ids = static_cast<const u32*>(ids->p);
    timer_begin(ctx, F_OTHER);
    values_compact_kernel<<<grid_1d(n_cells + 1, ctx->n_sms), 256, 0, ctx->st>>>(P);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    u32 n_new = 0;
    KB_TRY(dict_encode_device(ctx, P.enc_off, static_cast<const unsigned char*>(d_bytes->p), n_def, total, static_cast<u32*>(ids->p), &n_new, nullptr));
    inf.dict_new = n_new;
    inf.rows_dropped = n_rows - n_kept;
    r = std::make_unique<kb_rel>();
    r->slots = cols;
    r->n = n_kept;
    for (u32 k = 0; k < P.n_cols; k++) {
        Col col;
        KB_TRY(alloc_col(ctx, n_kept, &col));
        r->cols.push_back(col);
        P.out[k] = col.ptr;
    }
    if (n_kept) {
        timer_begin(ctx, F_OTHER);
        values_scatter_kernel<<<grid_1d(nr, ctx->n_sms), 256, 0, ctx->st>>>(P);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
    }
    // the f64 side table learns the new strings, as after kb_bind's CONCAT, when it covers exactly the ids the dictionary held: a
    // shorter table (never derived, or behind) would be parsed from its end, a longer one is another dictionary's; both are left
    // to their owner (kb_dict_numeric_derive)
    if (n_new && ctx->n_ids == inf.dict_first) KB_TRY(numeric_derive(ctx, KB_NUMERIC_F64, KB_NUMERIC_APPEND, nullptr));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));  // the host inputs' device copies are released with the stream order anyway
    ctx->stats.rows_out = r->n;
    if (info) *info = inf;
    *out = r.release();
    return KB_OK;
}

}  // extern "C"
