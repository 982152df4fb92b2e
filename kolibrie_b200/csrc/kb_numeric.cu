// kb_numeric.cu — the numeric side tables derived on the device from the device dictionary (kb_dict_numeric_derive): num_or0 / is_num
// (`str::parse::<f64>()`, read by FILTER comparisons, arithmetic, aggregates and rule filters) and the legacy executor's i32 view
// (`str::parse::<i32>()`). The strings are in HBM already (kb_dict_strings_load, kb_dict_encode, kb_bind's CONCAT / isTRIPLE), so a
// table costs one pass over the ids it adds and no host-to-device copy.
//   K1 numeric_derive_kernel  thread per id: kb_numparse.cuh's parse_f64 / parse_i32 of the id's string. Most terms are IRIs and names,
//                             rejected on their first byte. An id whose value Eisel–Lemire cannot decide is appended to a list.
//   K2 numeric_slow_kernel    thread per listed id: slow_f64, the exact decimal conversion (its 788-byte decimal lives in local memory)
// and, for the store index's rank columns, the value order of the f64 table (ensure_num_order, kb_numrank.cuh).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <climits>

#include "kb_internal.hpp"
#include "kb_numparse.cuh"
#include "kb_numrank.cuh"

namespace kb {

__device__ const kb_np::Tables d_np_tables = {
    {
#include "kb_pow5.inc"
    },
    KB_NP_POW10_INIT,
    KB_NP_IPOW10_INIT,
};

struct NumDeriveParams {
    const unsigned long long* off; const unsigned char* bytes;  // the device dictionary
    u32 lo, n;                                                  // ids [lo, n) are parsed
    double* num; u8* isnum; u32 first_f;                        // f64 table (null: not derived), written for ids >= first_f
    int* i32v; u8* isi32; u32 first_i;                          // i32 table (null: not derived), written for ids >= first_i
    u32* slow;                                                  // ids left to numeric_slow_kernel
    u32* ctr;                                                   // [0] slow ids, [1] numeric ids, [2] i32 ids
};

__global__ void __launch_bounds__(256) numeric_derive_kernel(const __grid_constant__ NumDeriveParams P) {
    u32 n_num = 0, n_i32 = 0;
    for (u32 id = P.lo + blockIdx.x * blockDim.x + threadIdx.x; id < P.n; id += gridDim.x * blockDim.x) {
        const unsigned long long a = __ldg(P.off + id);
        const u64 len = __ldg(P.off + id + 1) - a;
        const u8* s = P.bytes + a;
        if (P.num && id >= P.first_f) {
            u64 bits;
            const u32 route = kb_np::parse_f64(s, len, &d_np_tables, &bits);
            if (route == kb_np::NUM_SLOW) P.slow[atomicAdd(P.ctr, 1u)] = id;  // (num_or0[id] is written by K2)
            else P.num[id] = __longlong_as_double((long long)bits);
            P.isnum[id] = route != kb_np::NUM_REJECT;
            n_num += route != kb_np::NUM_REJECT;
        }
        if (P.i32v && id >= P.first_i) {
            int v;
            const bool ok = kb_np::parse_i32(s, len, &v);
            P.i32v[id] = v;
            P.isi32[id] = ok;
            n_i32 += ok;
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        n_num += __shfl_down_sync(0xffffffffu, n_num, o);
        n_i32 += __shfl_down_sync(0xffffffffu, n_i32, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (n_num) atomicAdd(P.ctr + 1, n_num);
        if (n_i32) atomicAdd(P.ctr + 2, n_i32);
    }
}

__global__ void __launch_bounds__(128) numeric_slow_kernel(const unsigned long long* __restrict__ off, const unsigned char* __restrict__ bytes,
                                                           const u32* __restrict__ slow, u32 n_slow, double* __restrict__ num) {
    kb_np::Decimal dec;
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n_slow; k += gridDim.x * blockDim.x) {
        const u32 id = slow[k];
        const unsigned long long a = off[id];
        num[id] = __longlong_as_double((long long)kb_np::slow_f64(bytes + a, off[id + 1] - a, &dec));
    }
}

// a table of `n` entries of elem_a + elem_b bytes that keeps its first `keep` entries: in place when the buffers hold n, else in new
// buffers with headroom (an append per window firing must not reallocate and copy each time)
static kb_status numeric_grow(kb_ctx* ctx, Buf* a, Buf* b, size_t elem_a, u32 keep, u32 n) {
    if (*a && *b && (*a)->bytes >= (size_t)n * elem_a && (*b)->bytes >= (size_t)n) return KB_OK;
    const size_t cap = (size_t)n + n / 2 + 1024;
    Buf na, nb;
    KB_TRY(alloc_buf(ctx, cap * elem_a, &na));
    KB_TRY(alloc_buf(ctx, cap, &nb));
    if (keep) {
        KB_CUDA(ctx, cudaMemcpyAsync(na->p, (*a)->p, (size_t)keep * elem_a, cudaMemcpyDeviceToDevice, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(nb->p, (*b)->p, (size_t)keep, cudaMemcpyDeviceToDevice, ctx->st));
    }
    *a = na;
    *b = nb;
    return KB_OK;
}

// the value order's keys (kb_numrank.cuh: order_key / order_value); id n is the extra 0.0
__global__ void __launch_bounds__(256) numorder_keys_kernel(const double* __restrict__ num, u32 n, unsigned long long* __restrict__ keys) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (u64)gridDim.x * blockDim.x) keys[i] = kb_nr::order_key(i < n ? num[i] : 0.0);
}
__global__ void __launch_bounds__(256) numorder_values_kernel(const unsigned long long* __restrict__ keys, u32 n, double* __restrict__ out) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = kb_nr::order_value(keys[i]);
}
// the value order of the numeric side table: keys[i] = order-preserving u64 of fold(num_or0[i]) for i < n, of 0.0 for i == n and for NaN
static void launch_numorder_keys(const double* num_or0, u32 n, unsigned long long* keys, int n_sms, cudaStream_t st) {
    const int grid = grid_1d((u64)n + 1, n_sms);
    numorder_keys_kernel<<<grid, 256, 0, st>>>(num_or0, n, keys);
}
// the inverse, over the sorted distinct keys
static void launch_numorder_values(const unsigned long long* keys, u32 n, double* out, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    numorder_values_kernel<<<grid, 256, 0, st>>>(keys, n, out);
}

// The value order V of the f64 table (kb_numrank.cuh): every value as an order-preserving u64 key (NaN as 0.0, -0.0 as +0.0, one extra
// 0.0), a radix sort, the distinct keys, back to doubles; then the host copy that FILTER constants are resolved against. Run by the
// index build for its rank columns, never by a query.
kb_status ensure_num_order(kb_ctx* ctx, bool* ok) {
    *ok = true;
    if (ctx->numv && ctx->numv_version == ctx->num_version) return KB_OK;
    ctx->numv.reset();
    ctx->h_numv.clear();
    const u64 m = (u64)ctx->n_ids + 1;
    if (m > (u64)INT32_MAX) { *ok = false; return KB_OK; }
    Buf a, b, cnt, tmp;
    KB_TRY(alloc_buf(ctx, m * sizeof(unsigned long long), &a));
    KB_TRY(alloc_buf(ctx, m * sizeof(unsigned long long), &b));
    KB_TRY(alloc_buf(ctx, sizeof(int), &cnt));
    unsigned long long* ka = static_cast<unsigned long long*>(a->p);
    unsigned long long* kb_ = static_cast<unsigned long long*>(b->p);
    int* d_cnt = static_cast<int*>(cnt->p);
    size_t t_sort = 0, t_uniq = 0;
    KB_CUDA(ctx, cub::DeviceRadixSort::SortKeys(nullptr, t_sort, ka, kb_, (int)m, 0, 64, ctx->st));
    KB_CUDA(ctx, cub::DeviceSelect::Unique(nullptr, t_uniq, kb_, ka, d_cnt, (int)m, ctx->st));
    KB_TRY(alloc_buf(ctx, std::max<size_t>(std::max(t_sort, t_uniq), 16), &tmp));
    launch_numorder_keys(ctx->num ? static_cast<const double*>(ctx->num->p) : nullptr, ctx->n_ids, ka, ctx->n_sms, ctx->st);
    KB_CUDA(ctx, cub::DeviceRadixSort::SortKeys(tmp->p, t_sort, ka, kb_, (int)m, 0, 64, ctx->st));
    KB_CUDA(ctx, cub::DeviceSelect::Unique(tmp->p, t_uniq, kb_, ka, d_cnt, (int)m, ctx->st));
    int n_v = 0;
    KB_CUDA(ctx, cudaMemcpyAsync(&n_v, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    Buf v;
    KB_TRY(alloc_buf(ctx, (size_t)n_v * sizeof(double), &v));
    launch_numorder_values(ka, (u32)n_v, static_cast<double*>(v->p), ctx->n_sms, ctx->st);
    KB_CUDA(ctx, cudaGetLastError());
    ctx->stats.kernel_launches += 2;
    ctx->h_numv.resize((size_t)n_v);
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->h_numv.data(), v->p, (size_t)n_v * sizeof(double), cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += sizeof(int) + (size_t)n_v * sizeof(double);
    ctx->numv = v;
    ctx->numv_version = ctx->num_version;
    return KB_OK;
}

kb_status numeric_derive(kb_ctx* ctx, uint32_t tables, uint32_t first_id, kb_numeric_info* info) {
    if (info) *info = kb_numeric_info{};
    if (tables == 0 || (tables & ~(KB_NUMERIC_F64 | KB_NUMERIC_I32)))
        return fail(ctx, KB_E_INVALID, "tables must be a non-empty combination of KB_NUMERIC_F64 and KB_NUMERIC_I32 (got 0x%x)", tables);
    const bool F = tables & KB_NUMERIC_F64, I = tables & KB_NUMERIC_I32;
    const u32 n = ctx->dict_ids;
    const u32 first_f = first_id == KB_NUMERIC_APPEND ? ctx->n_ids : first_id;
    const u32 first_i = first_id == KB_NUMERIC_APPEND ? ctx->n_i32 : first_id;
    if (F && first_f > ctx->n_ids) return fail(ctx, KB_E_INVALID, "first_id %u would leave a hole: the f64 table holds %u ids", first_f, ctx->n_ids);
    if (I && first_i > ctx->n_i32) return fail(ctx, KB_E_INVALID, "first_id %u would leave a hole: the i32 table holds %u ids", first_i, ctx->n_i32);
    if ((F && first_f > n) || (I && first_i > n)) return fail(ctx, KB_E_INVALID, "first_id is past the %u ids of the device dictionary", n);
    // checked: nothing changes before this point
    if (F) KB_TRY(numeric_grow(ctx, &ctx->num, &ctx->isnum, sizeof(double), first_f, n));
    if (I) KB_TRY(numeric_grow(ctx, &ctx->i32val, &ctx->isi32, sizeof(int32_t), first_i, n));
    const u32 lo = F && I ? std::min(first_f, first_i) : F ? first_f : first_i;
    u32 n_slow = 0, n_num = 0, n_i32 = 0;
    if (lo < n) {
        Buf slow;
        KB_TRY(alloc_buf(ctx, (size_t)(F ? n - first_f : 1) * sizeof(u32) + 16, &slow));
        const u32 c = ctrl_alloc(ctx, 4);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 4 * sizeof(u32), ctx->st));
        NumDeriveParams P{};
        const DictTab dict = dicttab(ctx);
        P.off = dict.off;
        P.bytes = dict.bytes;
        P.lo = lo;
        P.n = n;
        if (F) { P.num = static_cast<double*>(ctx->num->p); P.isnum = static_cast<u8*>(ctx->isnum->p); P.first_f = first_f; }
        if (I) { P.i32v = static_cast<int*>(ctx->i32val->p); P.isi32 = static_cast<u8*>(ctx->isi32->p); P.first_i = first_i; }
        P.slow = static_cast<u32*>(slow->p);
        P.ctr = ctx->ctrl + c;
        timer_begin(ctx, F_OTHER, 1);
        numeric_derive_kernel<<<grid_1d(n - lo, ctx->n_sms), 256, 0, ctx->st>>>(P);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        n_slow = ctx->h_ctrl[c];
        n_num = ctx->h_ctrl[c + 1];
        n_i32 = ctx->h_ctrl[c + 2];
        if (n_slow) {
            timer_begin(ctx, F_OTHER, 1);
            numeric_slow_kernel<<<grid_1d(n_slow, ctx->n_sms, 128, 4), 128, 0, ctx->st>>>(P.off, P.bytes, P.slow, n_slow, P.num);
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
        }
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));  // (`slow` is released with the stream order anyway; the counts are final here)
        timers_flush(ctx);
    }
    if (F) {
        ctx->n_ids = n;
        ctx->num_version++;  // typed index columns and prepared plans read the table: as after kb_dict_numeric_load
    }
    if (I) ctx->n_i32 = n;
    if (info) {
        info->n_ids = n;
        info->n_derived = n - lo;
        info->n_numeric = n_num;
        info->n_i32 = n_i32;
        info->n_slow = n_slow;
    }
    return KB_OK;
}

}  // namespace kb

using namespace kb;

extern "C" {

kb_status kb_dict_numeric_derive(kb_ctx* ctx, uint32_t tables, uint32_t first_id, kb_numeric_info* info) {
    KB_ENTER(ctx);
    return numeric_derive(ctx, tables, first_id, info);
}

kb_status kb_dict_numeric_download(kb_ctx* ctx, uint32_t first, uint32_t n, double* num_or0, uint8_t* is_num, int32_t* val, uint8_t* is_i32) {
    KB_ENTER(ctx);
    if (n == 0) return KB_OK;
    if ((num_or0 || is_num) && (u64)first + n > ctx->n_ids) return fail(ctx, KB_E_INVALID, "ids [%u, %u + %u) are past the f64 table's %u", first, first, n, ctx->n_ids);
    if ((val || is_i32) && (u64)first + n > ctx->n_i32) return fail(ctx, KB_E_INVALID, "ids [%u, %u + %u) are past the i32 table's %u", first, first, n, ctx->n_i32);
    size_t bytes = 0;
    if (num_or0) { KB_CUDA(ctx, cudaMemcpyAsync(num_or0, static_cast<const double*>(ctx->num->p) + first, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->st)); bytes += (size_t)n * 8; }
    if (is_num) { KB_CUDA(ctx, cudaMemcpyAsync(is_num, static_cast<const u8*>(ctx->isnum->p) + first, n, cudaMemcpyDeviceToHost, ctx->st)); bytes += n; }
    if (val) { KB_CUDA(ctx, cudaMemcpyAsync(val, static_cast<const int32_t*>(ctx->i32val->p) + first, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->st)); bytes += (size_t)n * 4; }
    if (is_i32) { KB_CUDA(ctx, cudaMemcpyAsync(is_i32, static_cast<const u8*>(ctx->isi32->p) + first, n, cudaMemcpyDeviceToHost, ctx->st)); bytes += n; }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += bytes;
    return KB_OK;
}

}  // extern "C"
