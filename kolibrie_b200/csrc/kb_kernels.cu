// kb_kernels.cu — the sm_90a kernels more than one file launches: the direct-table build from a pair relation (the star join's
// tables, kb_join.cu, and the store index's, kb_store.cu, share one layout), a column's min/max, the exclusive scan and the fill.
// Kernels with a single caller live in the file that launches them, with their launch formats.
#include "kb_internal.hpp"

namespace kb {

template <bool TRUSTED>
__global__ void __launch_bounds__(256) build_direct_pairs_kernel(const uint2* __restrict__ kv, u32 key_is_y, u32 n, u32* __restrict__ table,
                                                                 u32 kmin, u32 range, u32 cshift, u32* dup_flag) {
    const u32 stride = gridDim.x * blockDim.x;
    bool dup = false;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint2 e = kv[i];
        const u32 off = compact_key(key_is_y ? e.y : e.x, cshift) - kmin;
        const u32 v = key_is_y ? e.x : e.y;
        if (off < range) {
            if (TRUSTED) table[off] = v;
            else dup = dup || (atomicExch(&table[off], v) != EMPTY32);
        } else dup = true;
    }
    if (__any_sync(0xffffffffu, dup) && (threadIdx.x & 31) == 0) *dup_flag = 1u;
}
void launch_build_direct_pairs(const uint2* kv, u32 key_is_y, u32 n, u32* table, u32 kmin, u32 range, u32 cshift, u32* dup_flag, u32 trusted,
                               int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    if (trusted) build_direct_pairs_kernel<true><<<grid, 256, 0, st>>>(kv, key_is_y, n, table, kmin, range, cshift, dup_flag);
    else build_direct_pairs_kernel<false><<<grid, 256, 0, st>>>(kv, key_is_y, n, table, kmin, range, cshift, dup_flag);
}

__global__ void __launch_bounds__(256) col_minmax_kernel(const u32* __restrict__ col, u32 n, u32* out_min, u32* out_max) {
    u32 mn = EMPTY32, mx = 0u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 v = col[i];
        mn = min(mn, v);
        mx = max(mx, v);
    }
    mn = __reduce_min_sync(0xffffffffu, mn);
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0) { atomicMin(out_min, mn); atomicMax(out_max, mx); }
}
void launch_col_minmax(const u32* col, u32 n, u32* out_min, u32* out_max, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    col_minmax_kernel<<<grid_1d(n, n_sms, 256, 4), 256, 0, st>>>(col, n, out_min, out_max);
}

// exclusive scan in three passes over 2048-element tiles: tile sums, scan of the tile sums by one CTA, local scan + tile base
constexpr u32 SCAN_TILE_ELEMS = 2048;
__device__ __forceinline__ u32 cta_excl_scan_256(u32 v, u32* s_w, u32* total) {  // 256 threads; returns the exclusive prefix of v
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const u32 w = lane < 8 ? s_w[lane] : 0u;
        u32 wi = w;
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            const u32 y = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += y;
        }
        if (lane < 8) s_w[lane] = wi - w;
        if (lane == 7) s_w[8] = wi;
    }
    __syncthreads();
    const u32 ex = s_w[warp] + incl - v;
    *total = s_w[8];
    __syncthreads();
    return ex;
}
__global__ void __launch_bounds__(256) scan_tile_sums_kernel(const u32* __restrict__ a, u32 n, u32* __restrict__ sums) {
    __shared__ u32 s_w[9];
    const u32 base = blockIdx.x * SCAN_TILE_ELEMS;
    u32 v = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const u32 i = base + (u32)j * 256u + threadIdx.x;
        v += i < n ? a[i] : 0u;
    }
    u32 tot;
    cta_excl_scan_256(v, s_w, &tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(256) scan_sums_kernel(u32* sums, u32 n_tiles) {  // one CTA: exclusive scan of the tile sums, total at [n_tiles]
    __shared__ u32 s_w[9];
    u32 run = 0;
    for (u32 b = 0; b < n_tiles; b += 256u) {
        const u32 i = b + threadIdx.x;
        const u32 v = i < n_tiles ? sums[i] : 0u;
        u32 tot;
        const u32 ex = cta_excl_scan_256(v, s_w, &tot);
        if (i < n_tiles) sums[i] = run + ex;
        run += tot;
    }
    if (threadIdx.x == 0) sums[n_tiles] = run;
}
__global__ void __launch_bounds__(256) scan_apply_kernel(u32* __restrict__ a, u32 n, const u32* __restrict__ sums) {
    __shared__ u32 s_w[9];
    const u32 base = blockIdx.x * SCAN_TILE_ELEMS + threadIdx.x * 8u;  // 8 consecutive elements per thread
    u32 v[8];
    u32 t = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) { v[j] = base + (u32)j < n ? a[base + (u32)j] : 0u; t += v[j]; }
    u32 tot;
    u32 ex = cta_excl_scan_256(t, s_w, &tot) + sums[blockIdx.x];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (base + (u32)j < n) a[base + (u32)j] = ex;
        ex += v[j];
    }
}
void launch_exclusive_scan_u32(u32* a, u32 n, u32* scratch, cudaStream_t st) {
    if (n == 0) return;
    const u32 n_tiles = (n + SCAN_TILE_ELEMS - 1) / SCAN_TILE_ELEMS;
    scan_tile_sums_kernel<<<n_tiles, 256, 0, st>>>(a, n, scratch);
    scan_sums_kernel<<<1, 256, 0, st>>>(scratch, n_tiles);
    scan_apply_kernel<<<n_tiles, 256, 0, st>>>(a, n, scratch);
}

__global__ void fill_kernel(u32* p, u32 v, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) p[i] = v;
}
void launch_fill_u32(u32* p, u32 v, u64 n, cudaStream_t st) {
    if (n == 0) return;
    fill_kernel<<<grid_1d(n, (int)H100_SMS), 256, 0, st>>>(p, v, n);
}

}  // namespace kb
