// kb_api.cu — C ABI of libkolibrie_b200.so: context, device triple store, relations and the operator entry points.
// Host code only orchestrates: every data-touching step is an sm_90a kernel. The ones this file launches, the multi-GPU shuffle's
// partition, count and fused scatter, are defined here with their launch format.
#include <cstdarg>
#include <cstdlib>
#include <algorithm>
#include <chrono>
#include <mutex>

#include "kb_internal.hpp"
#include "kb_numrank.cuh"

using namespace kb;

namespace kb {

// fused partition + transfer of the multi-GPU join-key shuffle: a tile of rows is sorted by destination rank d = shard_of(key, n_parts)
// in shared memory, one range per (tile, destination) is reserved with an atomicAdd on *cursor_ptrs[d] — the destination's own cursor
// in peer memory (push mode, base = 0) or a local cursor behind a precomputed base[d] — and the runs are streamed into d's receive
// buffer (peer memory over NVLink) as 128-byte-aligned warp stores
struct ShuffleParams {
    const u32* key;
    u32 n, n_parts, n_cols;
    const u32* in[KB_MAX_COLS];
    u32* const* peer_cols;     // device array [n_parts * n_cols]
    u32* const* cursor_ptrs;   // device array [n_parts]: word the range of destination d is reserved on
    const u32* base;           // device array [n_parts]
    u32 capacity;
    u32* overflow;
    u32* ticket;               // zeroed tile counter
    u32 tile, n_tiles, stride, pow2_mask;  // set by the launcher
};

// partition rows by mix32(key) % n_parts (multi-GPU shuffle): count then scatter

__global__ void __launch_bounds__(256) part_count_kernel(const u32* key, u32 n, u32 n_parts, u32* counts) {
    __shared__ u32 sc[64];
    if (threadIdx.x < 64) sc[threadIdx.x] = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const u32 n_round = (n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += gridDim.x * blockDim.x) {
        const bool valid = i < n;
        const u32 part = valid ? shard_of(key[i], n_parts) : 0xFFFFu;
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (!valid) continue;
        // one shared atomic per (warp, destination) instead of one per row: with a handful of destinations the rows of a warp
        // pile up on a handful of addresses
        const unsigned peers = __match_any_sync(act, part);
        if (lane == __ffs(peers) - 1) atomicAdd(&sc[part], (u32)__popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < n_parts && sc[threadIdx.x]) atomicAdd(&counts[threadIdx.x], sc[threadIdx.x]);
}
static void launch_part_count(const u32* key, u32 n, u32 n_parts, u32* counts, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms, 256, 4);
    part_count_kernel<<<grid, 256, 0, st>>>(key, n, n_parts, counts);
}
struct PartScatterParams {
    const u32* in[KB_MAX_COLS];
    u32* out[KB_MAX_COLS];
    u32 n_cols;
};
__global__ void __launch_bounds__(256) part_scatter_kernel(const u32* key, u32 n, u32 n_parts, u32* cursors, const PartScatterParams P) {
    const int lane = threadIdx.x & 31;
    const u32 n_round = (n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += gridDim.x * blockDim.x) {
        const bool valid = i < n;
        const u32 part = valid ? shard_of(key[i], n_parts) : 0xFFFFu;
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (!valid) continue;
        const unsigned peers = __match_any_sync(act, part);
        const int leader = __ffs(peers) - 1;
        u32 basepos = 0;
        if (lane == leader) basepos = atomicAdd(&cursors[part], (u32)__popc(peers));
        basepos = __shfl_sync(peers, basepos, leader);
        const u32 r = basepos + (u32)__popc(peers & ((1u << lane) - 1u));
        for (u32 c = 0; c < P.n_cols; c++) P.out[c][r] = P.in[c][i];
    }
}
static void launch_part_scatter(const u32* key, u32 n, u32 n_parts, u32* cursors, const u32* const* in_cols, u32* const* out_cols, u32 n_cols,
                                int n_sms, cudaStream_t st) {
    if (n == 0) return;
    PartScatterParams P;
    P.n_cols = n_cols;
    for (u32 c = 0; c < n_cols; c++) { P.in[c] = in_cols[c]; P.out[c] = out_cols[c]; }
    int grid = grid_1d(n, n_sms, 256, 4);
    part_scatter_kernel<<<grid, 256, 0, st>>>(key, n, n_parts, cursors, P);
}

// Join-key shuffle FUSED with its transfer (SURVEY.md 8e). A CTA takes a tile of rows, sorts it by destination rank in shared memory
// (histogram -> offsets -> staged columns), reserves ONE range per (tile, destination) in the destination's receive buffer — an
// atomicAdd on the cursor the destination owns (peer memory: no count pass and no count exchange before the transfer), or on a local
// cursor when the caller fixed the ranges beforehand — and then streams every (destination, column) run out of shared memory with
// warp stores whose 32-lane windows are aligned to 128-byte lines of the REMOTE address: NVLink carries full lines, not the 4-byte
// scatter a row-at-a-time kernel produces.
// Rows per thread and tile are fixed (8): the keys, the rows' values (NC <= 2 columns: kept in registers from ONE round of independent
// loads; more columns: re-read when the row is staged), their destination and their rank inside the tile stay in registers from the
// histogram pass to the staging pass — the first version re-read the inputs and took the ranks with a second round of shared atomics
// (5.6 warp instructions per row, most stalls on the dependent global loads: far above the HBM floor with all eight destinations
// LOCAL, i.e. the SM side alone). DIRECT (8 or more destinations): the rank is the
// return value of a plain shared atomic per row (a warp's 32 rows spread over >= 8 counters: a few passes) instead of match.any +
// leader election + shuffle (52 instructions per row slot and warp). Flush: the staged run of a destination starts at a shared-memory
// offset congruent to its place in the receive buffer modulo 16 bytes, so its body goes out as 16-byte vector stores on 128-byte
// boundaries (512 contiguous bytes per warp instruction: whole NVLink lines), head and tail as one predicated scalar store each.
constexpr u32 SHUF_ITEMS = 8;
template <int NC, int THREADS, bool DIRECT>
__global__ void __launch_bounds__(THREADS) shuffle_scatter_kernel(const __grid_constant__ ShuffleParams P) {
    extern __shared__ __align__(16) u32 sh_stage[];  // [n_cols][stride] columns sorted by destination
    __shared__ u32 s_cnt[64], s_off[64], s_gbase[64];
    __shared__ u32 s_tile;
    constexpr u32 TILE = SHUF_ITEMS * THREADS;
    constexpr int NV = NC > 0 ? NC : 1;
    const u32 STRIDE = P.stride;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 pm = P.pow2_mask;
    for (;;) {
        if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
        if (tid < 64) s_cnt[tid] = 0u;
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= P.n_tiles) break;
        const u32 row0 = tile * TILE;
        const u32 cnt = min(TILE, P.n - row0);
        // ---- 0. every load of the tile in flight at once
        u32 key[SHUF_ITEMS], val[SHUF_ITEMS][NV];
#pragma unroll
        for (u32 j = 0; j < SHUF_ITEMS; j++) {
            const u32 r = j * THREADS + (u32)tid;
            key[j] = r < cnt ? __ldg(P.key + row0 + r) : 0u;
        }
        if (NC > 0) {
#pragma unroll
            for (int c = 0; c < NV; c++) {
                if (P.in[c] == P.key) {
#pragma unroll
                    for (u32 j = 0; j < SHUF_ITEMS; j++) val[j][c] = key[j];
                } else {
#pragma unroll
                    for (u32 j = 0; j < SHUF_ITEMS; j++) {
                        const u32 r = j * THREADS + (u32)tid;
                        val[j][c] = r < cnt ? __ldg(P.in[c] + row0 + r) : 0u;
                    }
                }
            }
        }
        // ---- 1. destinations, histogram, rank of the row among the tile's rows for its destination
        u32 dest[SHUF_ITEMS], rank[SHUF_ITEMS];
#pragma unroll
        for (u32 j = 0; j < SHUF_ITEMS; j++) {
            const u32 r = j * THREADS + (u32)tid;
            const bool valid = r < cnt;
            const u32 blk = key[j] >> SHARD_B;
            dest[j] = pm ? (blk & pm) : (blk % P.n_parts);  // == shard_of(key, n_parts)
            rank[j] = 0u;
            if (DIRECT) {
                if (valid) rank[j] = atomicAdd(&s_cnt[dest[j]], 1u);
            } else {
                const unsigned act = __ballot_sync(0xffffffffu, valid);
                if (valid) {
                    const unsigned peers = __match_any_sync(act, dest[j]);
                    const int leader = __ffs(peers) - 1;
                    u32 b = 0;
                    if (lane == leader) b = atomicAdd(&s_cnt[dest[j]], (u32)__popc(peers));
                    b = __shfl_sync(peers, b, leader);
                    rank[j] = b + (u32)__popc(peers & ((1u << lane) - 1u));
                }
            }
        }
        __syncthreads();
        // ---- 2. one range reservation per destination (remote cursor: the receiver's own word); offsets inside the tile: every
        // destination gets a 16-byte aligned slot of its count + 8 elements and starts in it at (its place in the receive buffer mod 4)
        if (warp == 0) {
            u32 run = 0;
            for (u32 d0 = 0; d0 < P.n_parts; d0 += 32u) {
                const u32 d = d0 + (u32)lane;
                const u32 c = d < P.n_parts ? s_cnt[d] : 0u;
                const u32 padded = d < P.n_parts ? ((c + 3u + 3u + 3u) & ~3u) : 0u;
                u32 incl = padded;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += y;
                }
                if (d < P.n_parts) {
                    u32 g = 0u;
                    if (c) g = P.base[d] + atomicAdd_system(P.cursor_ptrs[d], c);
                    if (c && (u64)g + c > (u64)P.capacity) { *P.overflow = 1u; g = EMPTY32; }
                    s_gbase[d] = g;
                    s_off[d] = run + incl - padded + (g & 3u);
                }
                run += __shfl_sync(0xffffffffu, incl, 31);
            }
        }
        __syncthreads();
        // ---- 3. stage the columns sorted by destination: position = the destination's offset in the tile + the rank of step 1
#pragma unroll
        for (u32 j = 0; j < SHUF_ITEMS; j++) {
            const u32 r = j * THREADS + (u32)tid;
            if (r >= cnt) continue;
            const u32 pos = s_off[dest[j]] + rank[j];
            if (NC > 0) {
#pragma unroll
                for (int c = 0; c < NV; c++) sh_stage[c * STRIDE + pos] = val[j][c];
            } else {
                for (u32 c = 0; c < P.n_cols; c++) sh_stage[c * STRIDE + pos] = __ldg(P.in[c] + row0 + r);
            }
        }
        __syncthreads();
        // ---- 4. flush every (destination, column) run
        const u32 n_runs = P.n_parts * P.n_cols;
        for (u32 q = (u32)warp; q < n_runs; q += THREADS / 32) {
            const u32 d = q / P.n_cols, c = q - d * P.n_cols;
            const u32 m = s_cnt[d];
            const u32 g = s_gbase[d];
            if (m == 0u || g == EMPTY32) continue;
            u32* dst = P.peer_cols[q] + g;
            const u32* src = sh_stage + c * STRIDE + s_off[d];
            const u32 mis = (u32)((reinterpret_cast<uintptr_t>(dst) >> 2) & 31u);  // elements past the previous 128-byte boundary
            if ((reinterpret_cast<uintptr_t>(P.peer_cols[q]) & 15u) == 0u) {
                const u32 head = min(m, (32u - mis) & 31u);
                if ((u32)lane < head) dst[lane] = src[lane];
                const u32 body = (m - head) >> 2;  // 16-byte vectors, the first one on a 128-byte boundary of the receive buffer
                const uint4* s4 = reinterpret_cast<const uint4*>(src + head);
                uint4* d4 = reinterpret_cast<uint4*>(dst + head);
                for (u32 e = (u32)lane; e < body; e += 32u) d4[e] = s4[e];
                const u32 t0 = head + (body << 2);
                if (t0 + (u32)lane < m) dst[t0 + lane] = src[t0 + lane];
            } else {
                for (int e0 = -(int)mis; e0 < (int)m; e0 += 32) {
                    const int e = e0 + lane;
                    if (e >= 0 && e < (int)m) dst[e] = src[e];
                }
            }
        }
        __syncthreads();
    }
    __threadfence_system();  // the stores must be visible to the peers before the barrier that follows the launch
}
template <int NC, int THREADS>
static void launch_shuffle_t(ShuffleParams p, int n_sms, cudaStream_t st) {
    p.tile = SHUF_ITEMS * THREADS;
    p.n_tiles = (p.n + p.tile - 1u) / p.tile;
    p.stride = (p.tile + 12u * p.n_parts + 3u) & ~3u;
    p.pow2_mask = (p.n_parts & (p.n_parts - 1u)) == 0u ? p.n_parts - 1u : 0u;
    if (p.n_parts == 1u) p.pow2_mask = 0u;  // (x % 1 == 0; a zero mask selects the modulo path)
    const size_t smem = (size_t)p.n_cols * p.stride * sizeof(u32);
    static const bool direct_env = !(getenv("KOLIBRIE_SHUFFLE_DIRECT") && getenv("KOLIBRIE_SHUFFLE_DIRECT")[0] == '0');
    if (p.n_parts >= 8u && direct_env) {
        cudaFuncSetAttribute(shuffle_scatter_kernel<NC, THREADS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        const int grid = grid_for((const void*)shuffle_scatter_kernel<NC, THREADS, true>, THREADS, smem, n_sms, p.n_tiles);
        shuffle_scatter_kernel<NC, THREADS, true><<<grid, THREADS, smem, st>>>(p);
    } else {
        cudaFuncSetAttribute(shuffle_scatter_kernel<NC, THREADS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        const int grid = grid_for((const void*)shuffle_scatter_kernel<NC, THREADS, false>, THREADS, smem, n_sms, p.n_tiles);
        shuffle_scatter_kernel<NC, THREADS, false><<<grid, THREADS, smem, st>>>(p);
    }
}
static void launch_shuffle_scatter(const ShuffleParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    static const int threads_env = getenv("KOLIBRIE_SHUFFLE_THREADS") ? atoi(getenv("KOLIBRIE_SHUFFLE_THREADS")) : 0;
    const bool wide = threads_env ? threads_env >= 512 : true;  // 4096-row tiles (512 threads) for the register-resident cases
    if (p.n_cols == 1) { if (wide) launch_shuffle_t<1, 512>(p, n_sms, st); else launch_shuffle_t<1, 256>(p, n_sms, st); }
    else if (p.n_cols == 2) { if (wide) launch_shuffle_t<2, 512>(p, n_sms, st); else launch_shuffle_t<2, 256>(p, n_sms, st); }
    else if (p.n_cols <= 6) launch_shuffle_t<0, 512>(p, n_sms, st);  // <= 6 x (4096 + 768) x 4 B = 114 KB of staging
    else launch_shuffle_t<0, 128>(p, n_sms, st);                    // 16 columns x (1024 + 768) x 4 B = 112 KB
}

static std::string g_create_err;

kb_status fail(kb_ctx* ctx, kb_status code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf; else g_create_err = buf;
    return code;
}

kb_status alloc_buf(kb_ctx* ctx, size_t bytes, Buf* out) {
    auto b = std::make_shared<DevBuf>();
    b->bytes = round256(bytes) + 256;  // every column can be over-read to the next 16-byte boundary by the TMA tile loads
    b->st = ctx->st;
    b->life = ctx->life;
    static const bool cache_on = !(getenv("KOLIBRIE_BUF_CACHE") && getenv("KOLIBRIE_BUF_CACHE")[0] == '0');
    if (!cache_on) ctx->life->cache_off = true;
    if (b->bytes >= Life::MIN_BYTES && cache_on) {  // best fit among the recycled buffers (at most 25 % larger than asked)
        Life& L = *ctx->life;
        int best = -1;
        for (size_t i = 0; i < L.cache.size(); i++)
            if (L.cache[i].bytes >= b->bytes && L.cache[i].bytes <= b->bytes + b->bytes / 4 && (best < 0 || L.cache[i].bytes < L.cache[best].bytes)) best = (int)i;
        if (best >= 0) {
            b->p = L.cache[best].p;
            b->bytes = L.cache[best].bytes;
            L.cached_bytes -= b->bytes;
            L.cache.erase(L.cache.begin() + best);
            *out = b;
            return KB_OK;
        }
    }
    cudaError_t e = cudaMallocAsync(&b->p, b->bytes, ctx->st);
    if (e != cudaSuccess && !ctx->life->cache.empty()) {  // out of memory with buffers parked in the cache: give them back and try once more
        cudaGetLastError();
        for (auto& cb : ctx->life->cache) cudaFreeAsync(cb.p, ctx->st);
        ctx->life->cache.clear();
        ctx->life->cached_bytes = 0;
        cudaStreamSynchronize(ctx->st);
        e = cudaMallocAsync(&b->p, b->bytes, ctx->st);
    }
    if (e != cudaSuccess) {
        b->p = nullptr;
        cudaGetLastError();
        return fail(ctx, KB_E_OOM, "device allocation of %zu bytes failed: %s", b->bytes, cudaGetErrorString(e));
    }
    *out = b;
    return KB_OK;
}

kb_status tag_batch_table(kb_ctx* ctx, u64 n, Buf* tab, u64* slots) {
    u64 s = 1024;
    while (s < 2 * n) s <<= 1;
    KB_TRY(alloc_buf(ctx, s * sizeof(u64), tab));
    KB_CUDA(ctx, cudaMemsetAsync((*tab)->p, 0xFF, s * sizeof(u64), ctx->st));
    *slots = s;
    return KB_OK;
}

kb_status alloc_col(kb_ctx* ctx, u64 rows, Col* out) {
    Buf b;
    KB_TRY(alloc_buf(ctx, (size_t)rows * sizeof(u32), &b));
    out->buf = b;
    out->ptr = static_cast<u32*>(b->p);
    return KB_OK;
}

kb_status begin_call(kb_ctx* ctx) {
    ctx->err.clear();
    ctx->ctrl_used = 0;
    if (ctx->ctrl_dirty) {
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl, 0, kb_ctx::CTRL_WORDS * sizeof(u32), ctx->st));
        ctx->ctrl_dirty = false;
    }
    return KB_OK;
}

u32 ctrl_alloc(kb_ctx* ctx, u32 words) {
    ctx->ctrl_dirty = true;
    u32 off = ctx->ctrl_used;
    ctx->ctrl_used += (words + 3u) & ~3u;
    if (ctx->ctrl_used > kb_ctx::CTRL_WORDS) {  // wrap: callers never keep more than a few hundred words live per call
        off = 0;
        ctx->ctrl_used = (words + 3u) & ~3u;
    }
    return off;
}

kb_status ctrl_read(kb_ctx* ctx) {
    const u32 words = kb_ctx::CTRL_WORDS;  // whole arena: allocations may have wrapped
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->h_ctrl, ctx->ctrl, words * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += words * sizeof(u32);
    timers_flush(ctx);
    return KB_OK;
}

kb_status ensure_tile_state(kb_ctx* ctx, u64 tiles) {
    if (ctx->tile_state && tiles <= ctx->tile_state_tiles) return KB_OK;  // (a scan of a store never loaded asks for 0 tiles: still allocate)
    u64 want = std::max<u64>(tiles, 1024) * 2;
    Buf b, b2;
    KB_TRY(alloc_buf(ctx, want * MAXP * sizeof(u64), &b));
    KB_TRY(alloc_buf(ctx, (want / 32 + 2) * MAXP * sizeof(u64), &b2));
    KB_CUDA(ctx, cudaMemsetAsync(b->p, 0, want * MAXP * sizeof(u64), ctx->st));  // epoch 0 is never used by a launch
    KB_CUDA(ctx, cudaMemsetAsync(b2->p, 0, (want / 32 + 2) * MAXP * sizeof(u64), ctx->st));
    ctx->tile_state = b;
    ctx->block_state = b2;
    ctx->tile_state_tiles = want;
    return KB_OK;
}

NumTab numtab(const kb_ctx* ctx) {
    NumTab nt;
    nt.num_or0 = ctx->num ? static_cast<const double*>(ctx->num->p) : nullptr;
    nt.is_num = ctx->isnum ? static_cast<const u8*>(ctx->isnum->p) : nullptr;
    nt.n_ids = ctx->n_ids;
    nt.i32_val = ctx->i32val ? static_cast<const int*>(ctx->i32val->p) : nullptr;
    nt.is_i32 = ctx->isi32 ? static_cast<const u8*>(ctx->isi32->p) : nullptr;
    nt.n_i32 = ctx->n_i32;
    return nt;
}

static cudaEvent_t get_event(kb_ctx* ctx) {
    if (!ctx->ev_pool.empty()) {
        cudaEvent_t e = ctx->ev_pool.back();
        ctx->ev_pool.pop_back();
        return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
void timer_begin(kb_ctx* ctx, int fam, int n_kernels) {
    ctx->stats.kernel_launches += (u64)n_kernels;
    switch (fam) {
        case F_SCAN: ctx->stats.scan_launches++; break;
        case F_BUILD: ctx->stats.build_launches++; break;
        case F_PROBE: ctx->stats.probe_launches++; break;
        case F_FILTER: ctx->stats.filter_launches++; break;
        case F_GROUP: ctx->stats.group_launches++; break;
        default: ctx->stats.other_launches++; break;
    }
    if (!ctx->timing) return;
    PendingTimer t;
    t.a = get_event(ctx);
    t.b = get_event(ctx);
    t.fam = fam;
    cudaEventRecord(t.a, ctx->st);
    ctx->timers.push_back(t);
}
void timer_end(kb_ctx* ctx) {
    if (!ctx->timing || ctx->timers.empty()) return;
    cudaEventRecord(ctx->timers.back().b, ctx->st);
}
void timers_flush(kb_ctx* ctx) {
    size_t kept = 0;
    for (auto& t : ctx->timers) {
        float ms = 0.f;
        if (cudaEventQuery(t.b) == cudaErrorNotReady) {  // launched by an asynchronous submit that has not finished: next flush
            ctx->timers[kept++] = t;
            continue;
        }
        if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) {
            switch (t.fam) {
                case F_SCAN: ctx->stats.scan_ms += ms; break;
                case F_BUILD: ctx->stats.build_ms += ms; break;
                case F_PROBE: ctx->stats.probe_ms += ms; break;
                case F_FILTER: ctx->stats.filter_ms += ms; break;
                case F_GROUP: ctx->stats.group_ms += ms; break;
                default: ctx->stats.other_ms += ms; break;
            }
            ctx->stats.total_ms += ms;
        } else {
            cudaGetLastError();
        }
        ctx->ev_pool.push_back(t.a);
        ctx->ev_pool.push_back(t.b);
    }
    cudaGetLastError();  // cudaErrorNotReady is sticky in the per-thread last-error slot
    ctx->timers.resize(kept);
}

// ---------------------------------------------------------------------------------------------------------------
// FILTER program helpers
static int op_arity(u32 op) {
    switch (op) {
        case KB_F_CMP_NUM: case KB_F_EQ_ID: case KB_F_NE_ID: case KB_F_PUSH_VAR: case KB_F_PUSH_CONST: case KB_F_IS_TRIPLE: case KB_F_CMP_LEGACY: return 0;
        case KB_F_NOT: case KB_F_TRUTHY: return 1;
        case KB_F_AND: case KB_F_OR: case KB_F_ADD: case KB_F_SUB: case KB_F_MUL: case KB_F_DIV: return 2;
        default: return -1;
    }
}
static bool op_has_slot(u32 op) {
    return op == KB_F_CMP_NUM || op == KB_F_EQ_ID || op == KB_F_NE_ID || op == KB_F_PUSH_VAR || op == KB_F_IS_TRIPLE || op == KB_F_CMP_LEGACY;
}

kb_status validate_filter(kb_ctx* ctx, const kb_filter_op* ops, u32 n) {
    if (n == 0) return KB_OK;
    if (!ops) return fail(ctx, KB_E_INVALID, "filter program is NULL");
    if (n > KB_MAX_FILTER_OPS) return fail(ctx, KB_E_LIMIT, "filter program longer than %d ops", KB_MAX_FILTER_OPS);
    int depth = 0;
    for (u32 i = 0; i < n; i++) {
        int a = op_arity(ops[i].op);
        if (a < 0) return fail(ctx, KB_E_INVALID, "filter op %u: unknown opcode %u", i, ops[i].op);
        if (depth < a) return fail(ctx, KB_E_INVALID, "filter op %u: stack underflow", i);
        depth += 1 - a;
        if (depth > 10) return fail(ctx, KB_E_LIMIT, "filter expression too deep");
    }
    if (depth != 1) return fail(ctx, KB_E_INVALID, "filter program leaves %d values on the stack", depth);
    return KB_OK;
}

static void split_rec(const kb_filter_op* ops, const std::vector<u32>& begin, u32 b, u32 e, std::vector<FilterProg>* out) {
    if (ops[e - 1].op == KB_F_AND) {
        const u32 right_b = begin[e - 2];
        split_rec(ops, begin, b, right_b, out);
        split_rec(ops, begin, right_b, e - 1, out);
        return;
    }
    FilterProg f;
    f.ops.assign(ops + b, ops + e);
    out->push_back(std::move(f));
}

bool split_conjuncts(const kb_filter_op* ops, u32 n, std::vector<FilterProg>* out) {
    out->clear();
    if (n == 0) return true;
    std::vector<u32> begin(n), stack;
    for (u32 i = 0; i < n; i++) {
        int a = op_arity(ops[i].op);
        if (a < 0 || (int)stack.size() < a) return false;
        u32 b = i;
        for (int k = 0; k < a; k++) { b = stack.back(); stack.pop_back(); }
        begin[i] = b;
        stack.push_back(b);
    }
    if (stack.size() != 1) return false;
    split_rec(ops, begin, 0, n, out);
    return true;
}

std::set<u32> filter_slots(const FilterProg& f) {
    std::set<u32> s;
    for (auto& op : f.ops) if (op_has_slot(op.op)) s.insert(op.slot);
    return s;
}

kb_status compile_prog(kb_ctx* ctx, const FilterProg& f, const std::vector<u32>& slots, std::vector<FilterOp>* ops,
                       const std::vector<u32>* pos) {
    ops->clear();
    for (auto& op : f.ops) {
        FilterOp d;
        d.op = op.op; d.slot = op.slot; d.cmp = op.cmp; d.id = op.id; d.value = op.value;
        if (op_has_slot(op.op)) {
            bool bound = false;
            for (size_t i = 0; i < slots.size(); i++) {
                if (slots[i] != op.slot) continue;
                d.slot = pos ? (*pos)[i] : (u32)i;
                bound = true;
            }
            if (!bound) return fail(ctx, KB_E_INVALID, "filter uses a variable that is not bound where it is evaluated");
        }
        ops->push_back(d);
    }
    if (ops->size() > KB_MAX_FILTER_OPS) return fail(ctx, KB_E_LIMIT, "filter too long");
    return KB_OK;
}

void pattern_vars(const kb_pattern& pt, std::vector<u32>* slots, std::vector<u32>* src) {
    const kb_term* ts[3] = {&pt.s, &pt.p, &pt.o};
    for (u32 i = 0; i < 3; i++) {
        if (!ts[i]->is_var) continue;
        if (std::find(slots->begin(), slots->end(), ts[i]->value) == slots->end()) {
            slots->push_back(ts[i]->value);
            src->push_back(i);
        }
    }
}

kb_status check_pattern(kb_ctx* ctx, const kb_pattern& pt) {
    const kb_term* ts[3] = {&pt.s, &pt.p, &pt.o};
    for (auto* t : ts) {
        if (t->is_var > 1) return fail(ctx, KB_E_INVALID, "kb_term.is_var must be 0 or 1");
        if (!t->is_var && t->value == KB_ID_NONE) return fail(ctx, KB_E_INVALID, "constant id 0xFFFFFFFF is reserved (KB_ID_NONE)");
        if (t->is_var && t->value >= 4096) return fail(ctx, KB_E_LIMIT, "variable slot %u too large (max 4095)", t->value);
    }
    return KB_OK;
}

kb_status empty_rel(kb_ctx* ctx, const std::vector<u32>& slots, std::unique_ptr<kb_rel>* out) {
    auto r = std::make_unique<kb_rel>();
    r->slots = slots;
    for (size_t c = 0; c < slots.size(); c++) { Col col; KB_TRY(alloc_col(ctx, 0, &col)); r->cols.push_back(col); }
    *out = std::move(r);
    return KB_OK;
}

u32 pow2_at_least(u64 x) {
    u64 p = 1024;
    while (p < x) p <<= 1;
    return (u32)std::min<u64>(p, 1ull << 31);
}

}  // namespace kb

// =================================================================================================================
// C ABI
extern "C" {

const char* kb_version(void) { return "kolibrie_b200 0.1.0 (sm_90a)"; }

kb_status kb_ctx_create(int device, kb_ctx** out) {
    if (!out) return KB_E_INVALID;
    *out = nullptr;
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0) {
        cudaGetLastError();
        return kb::fail(nullptr, KB_E_CUDA, "no CUDA device available (%s): this library has no CPU fallback", cudaGetErrorString(e));
    }
    if (device < 0 || device >= n_dev) return kb::fail(nullptr, KB_E_INVALID, "device %d out of range (0..%d)", device, n_dev - 1);
    kb::DeviceGuard guard(device);
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return kb::fail(nullptr, KB_E_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    // sm_90a code (TMA bulk copies, mbarrier) loads on compute capability 9.0 only: the 'a' features are not forward compatible
    if (prop.major != 9 || prop.minor != 0)
        return kb::fail(nullptr, KB_E_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
    kb_ctx* ctx = new kb_ctx;
    ctx->device = device;
    ctx->n_sms = prop.multiProcessorCount;
    ctx->life->max_bytes = prop.totalGlobalMem / 8 * 3;
    auto bail = [&](const char* what, cudaError_t err) {
        kb::fail(nullptr, KB_E_CUDA, "%s: %s", what, cudaGetErrorString(err));
        delete ctx;
        return KB_E_CUDA;
    };
    if ((e = cudaStreamCreateWithFlags(&ctx->st, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    if ((e = cudaStreamCreateWithFlags(&ctx->st_copy, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    if ((e = cudaEventCreateWithFlags(&ctx->ev_copy, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaStreamCreateWithFlags(&ctx->st2, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    if ((e = cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        uint64_t thr = UINT64_MAX;  // keep freed blocks cached: steady-state queries never hit cudaMalloc
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    if (const char* ord = getenv("KOLIBRIE_ORDERED")) ctx->ordered = (ord[0] == '0') ? 0u : 1u;
    if (const char* ui = getenv("KOLIBRIE_USE_INDEX")) ctx->use_index = ui[0] != '0';
    if (const char* fk = getenv("KOLIBRIE_INDEX_KERNEL")) ctx->fast_index_kernel = fk[0] != '0';
    if (const char* cj = getenv("KOLIBRIE_CSR_JOIN")) ctx->csr_join = cj[0] != '0';
    if (const char* im = getenv("KOLIBRIE_INDEX_MAINTAIN")) ctx->index_maintain = im[0] != '0';
    if (const char* tm = getenv("KOLIBRIE_PROBE_TABLE")) ctx->probe_table_mode = tm[0] != '0';
    if (const char* dp = getenv("KOLIBRIE_DERIVE_PART")) ctx->derive_part = dp[0] != '0';
    if (const char* ds = getenv("KOLIBRIE_DERIVE_SLICE")) ctx->derive_slice_bytes = std::max<u64>(64, strtoull(ds, nullptr, 10));
    if (const char* dk = getenv("KOLIBRIE_DERIVE_SLACK")) ctx->derive_bucket_slack = strtoull(dk, nullptr, 10);
    if (const char* dr = getenv("KOLIBRIE_DERIVE_MIN_ROWS")) ctx->derive_min_part_rows = std::max<u64>(1, strtoull(dr, nullptr, 10));
    if (const char* sm = getenv("KOLIBRIE_SMS")) {  // grid cap for tests: every persistent CTA then runs many tiles
        const long n = strtol(sm, nullptr, 10);
        if (n > 0) ctx->n_sms = (int)std::min<long>(n, prop.multiProcessorCount);
    }
    if ((e = cudaMalloc(&ctx->ctrl, kb_ctx::CTRL_WORDS * sizeof(u32))) != cudaSuccess) return bail("cudaMalloc(ctrl)", e);
    if ((e = cudaMallocHost(&ctx->h_ctrl, kb_ctx::CTRL_WORDS * sizeof(u32))) != cudaSuccess) return bail("cudaMallocHost(ctrl)", e);
    if ((e = cudaMalloc(&ctx->fast_cb, 64)) != cudaSuccess) return bail("cudaMalloc(fast_cb)", e);
    if ((e = cudaMemset(ctx->fast_cb, 0, 64)) != cudaSuccess) return bail("cudaMemset(fast_cb)", e);
    if ((e = cudaHostAlloc(&ctx->h_fast, 64, cudaHostAllocMapped)) != cudaSuccess) return bail("cudaHostAlloc(h_fast)", e);
    if ((e = cudaHostGetDevicePointer(&ctx->d_fast, ctx->h_fast, 0)) != cudaSuccess) return bail("cudaHostGetDevicePointer", e);
    *out = ctx;
    return KB_OK;
}

void kb_ctx_destroy(kb_ctx* ctx) {
    if (!ctx) return;
    kb::DeviceGuard guard(ctx->device);
    cudaStreamSynchronize(ctx->st);
    cudaStreamSynchronize(ctx->st_copy);
    kb::timers_flush(ctx);
    kb::store_replace(ctx, {});
    ctx->num.reset();
    ctx->isnum.reset();
    ctx->numv.reset();
    ctx->i32val.reset();
    ctx->isi32.reset();
    ctx->dict_off.reset();
    ctx->dict_bytes.reset();
    ctx->tile_state.reset();
    ctx->block_state.reset();
    for (auto& cb : ctx->life->cache) cudaFreeAsync(cb.p, ctx->st);
    ctx->life->cache.clear();
    ctx->life->cached_bytes = 0;
    cudaStreamSynchronize(ctx->st);
    ctx->life->alive = false;  // buffers still referenced by live relations fall back to cudaFree
    for (auto e : ctx->ev_pool) cudaEventDestroy(e);
    if (ctx->ctrl) cudaFree(ctx->ctrl);
    if (ctx->h_ctrl) cudaFreeHost(ctx->h_ctrl);
    if (ctx->fast_cb) cudaFree(ctx->fast_cb);
    if (ctx->h_fast) cudaFreeHost(ctx->h_fast);
    if (ctx->pinned) cudaFreeHost(ctx->pinned);
    cudaEventDestroy(ctx->ev_copy);
    cudaEventDestroy(ctx->ev_fork);
    cudaEventDestroy(ctx->ev_join);
    cudaStreamSynchronize(ctx->st2);
    cudaStreamDestroy(ctx->st2);
    cudaStreamDestroy(ctx->st);
    cudaStreamDestroy(ctx->st_copy);
    delete ctx;
}

const char* kb_last_error(const kb_ctx* ctx) { return ctx ? ctx->err.c_str() : kb::g_create_err.c_str(); }

kb_status kb_set_timing(kb_ctx* ctx, int enabled) {
    if (!ctx) return KB_E_INVALID;
    ctx->timing = enabled != 0;
    return KB_OK;
}
kb_status kb_get_stats(kb_ctx* ctx, kb_stats* out, int reset) {
    if (!ctx || !out) return KB_E_INVALID;
    kb::DeviceGuard guard(ctx->device);
    cudaStreamSynchronize(ctx->st);
    kb::timers_flush(ctx);
    *out = ctx->stats;
    if (reset) ctx->stats = kb_stats{};
    return KB_OK;
}
kb_status kb_synchronize(kb_ctx* ctx) {
    if (!ctx) return KB_E_INVALID;
    kb::DeviceGuard guard(ctx->device);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st_copy));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    kb::timers_flush(ctx);
    return KB_OK;
}

kb_status kb_dict_numeric_load(kb_ctx* ctx, const double* num_or0, const uint8_t* is_num, uint32_t n_ids) {
    KB_ENTER(ctx);
    ctx->num.reset();
    ctx->isnum.reset();
    ctx->n_ids = 0;
    ctx->num_version++;
    if (n_ids == 0) return KB_OK;
    if (!num_or0 || !is_num) return kb::fail(ctx, KB_E_INVALID, "NULL numeric table");
    KB_TRY(kb::alloc_buf(ctx, (size_t)n_ids * sizeof(double), &ctx->num));
    KB_TRY(kb::alloc_buf(ctx, (size_t)n_ids, &ctx->isnum));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->num->p, num_or0, (size_t)n_ids * sizeof(double), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->isnum->p, is_num, (size_t)n_ids, cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->n_ids = n_ids;
    ctx->num_version++;
    return KB_OK;
}

kb_status kb_dict_legacy_i32_load(kb_ctx* ctx, const int32_t* val, const uint8_t* is_i32, uint32_t n_ids) {
    KB_ENTER(ctx);
    ctx->i32val.reset();
    ctx->isi32.reset();
    ctx->n_i32 = 0;
    if (n_ids == 0) return KB_OK;
    if (!val || !is_i32) return kb::fail(ctx, KB_E_INVALID, "NULL table");
    KB_TRY(kb::alloc_buf(ctx, (size_t)n_ids * sizeof(int32_t), &ctx->i32val));
    KB_TRY(kb::alloc_buf(ctx, (size_t)n_ids, &ctx->isi32));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->i32val->p, val, (size_t)n_ids * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->isi32->p, is_i32, (size_t)n_ids, cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.h2d_bytes += (u64)n_ids * 5;
    ctx->n_i32 = n_ids;
    return KB_OK;
}

// ------------------------------------------------------------------ relations
kb_status kb_rel_info(const kb_rel* r, uint64_t* n_rows, uint32_t* n_cols, uint32_t* slots) {
    if (!r) return KB_E_INVALID;
    if (n_rows) *n_rows = r->n;
    if (n_cols) *n_cols = (uint32_t)r->slots.size();
    if (slots) for (size_t i = 0; i < r->slots.size() && i < KB_MAX_COLS; i++) slots[i] = r->slots[i];
    return KB_OK;
}
kb_status kb_rel_download(kb_ctx* ctx, const kb_rel* r, uint32_t col, uint32_t* dst) {
    if (!ctx || !r) return KB_E_INVALID;
    kb::DeviceGuard guard(ctx->device);
    if (col >= r->cols.size()) return kb::fail(ctx, KB_E_INVALID, "column %u out of range", col);
    if (r->n == 0) return KB_OK;
    if (!dst) return kb::fail(ctx, KB_E_INVALID, "NULL destination");
    KB_CUDA(ctx, cudaMemcpyAsync(dst, r->cols[col].ptr, r->n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += r->n * sizeof(u32);
    return KB_OK;
}
kb_status kb_rel_device_col(const kb_rel* r, uint32_t col, const uint32_t** d_ptr) {
    if (!r || !d_ptr || col >= r->cols.size()) return KB_E_INVALID;
    *d_ptr = r->cols[col].ptr;
    return KB_OK;
}
static kb_status rel_from(kb_ctx* ctx, const uint32_t* slots, uint32_t n_cols, const uint32_t* const* cols, uint64_t n_rows, cudaMemcpyKind kind, kb_rel** out) {
    if (!out || (n_cols && (!slots || !cols))) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_cols > KB_MAX_COLS) return kb::fail(ctx, KB_E_LIMIT, "more than %d columns", KB_MAX_COLS);
    if (n_rows >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "relation too large");
    auto r = std::make_unique<kb_rel>();
    r->n = n_rows;
    for (u32 c = 0; c < n_cols; c++) {
        for (u32 d = 0; d < c; d++) if (slots[d] == slots[c]) return kb::fail(ctx, KB_E_INVALID, "duplicate slot %u", slots[c]);
        kb::Col col;
        KB_TRY(kb::alloc_col(ctx, n_rows, &col));
        if (n_rows) KB_CUDA(ctx, cudaMemcpyAsync(col.ptr, cols[c], n_rows * sizeof(u32), kind, ctx->st));
        r->slots.push_back(slots[c]);
        r->cols.push_back(col);
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    if (kind == cudaMemcpyHostToDevice) ctx->stats.h2d_bytes += (u64)n_cols * n_rows * sizeof(u32);
    *out = r.release();
    return KB_OK;
}
kb_status kb_rel_from_host(kb_ctx* ctx, const uint32_t* slots, uint32_t n_cols, const uint32_t* const* cols, uint64_t n_rows, kb_rel** out) {
    KB_ENTER(ctx);
    return rel_from(ctx, slots, n_cols, cols, n_rows, cudaMemcpyHostToDevice, out);
}
kb_status kb_rel_from_device(kb_ctx* ctx, const uint32_t* slots, uint32_t n_cols, const uint32_t* const* cols, uint64_t n_rows, kb_rel** out) {
    KB_ENTER(ctx);
    return rel_from(ctx, slots, n_cols, cols, n_rows, cudaMemcpyDeviceToDevice, out);
}
void kb_rel_free(kb_ctx* ctx, kb_rel* r) {
    if (!r) return;
    if (ctx) {
        kb::DeviceGuard guard(ctx->device);
        delete r;
    } else delete r;
}

// ------------------------------------------------------------------ operators
kb_status kb_filter(kb_ctx* ctx, const kb_rel* in, const kb_filter_op* prog, uint32_t n_ops, kb_rel** out) {
    KB_ENTER(ctx);
    if (!in || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    KB_TRY(kb::validate_filter(ctx, prog, n_ops));
    kb::FilterProg f;
    if (n_ops) f.ops.assign(prog, prog + n_ops);
    for (u32 s : kb::filter_slots(f)) if (in->col_of(s) < 0)
        return kb::fail(ctx, KB_E_UNSUPPORTED, "filter references slot %u which is not bound (the reference evaluates it to false, types.rs:149-151)", s);
    std::unique_ptr<kb_rel> r;
    KB_TRY(kb::filter_impl(ctx, *in, f, &r));
    ctx->stats.rows_out = r->n;
    *out = r.release();
    return KB_OK;
}

kb_status kb_project(kb_ctx* ctx, const kb_rel* in, const uint32_t* slots, uint32_t n_slots, kb_rel** out) {
    if (!ctx || !in || !out || (n_slots && !slots)) return KB_E_INVALID;
    std::vector<u32> v(slots, slots + n_slots);
    *out = kb::select_cols(*in, v).release();
    return KB_OK;
}

kb_status kb_hash_join(kb_ctx* ctx, const kb_rel* left, const kb_rel* right, kb_rel** out) {
    KB_ENTER(ctx);
    if (!left || !right || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    std::unique_ptr<kb_rel> r;
    KB_TRY(kb::hash_join_impl(ctx, *left, *right, nullptr, &r));
    ctx->stats.rows_out = r->n;
    *out = r.release();
    return KB_OK;
}

// BindJoin (engine.rs:840-885): every row of `left` is extended by the matches of ONE store pattern. With the store index valid, the
// pattern (?x P ?y) and `left` binding exactly one of its variables through a unique, dense column, this is one probe kernel against the
// persistent table of the index (spo[x][P] / pos[P][y] lookups, no scan, no build); every other shape = scan of the pattern + natural join.
kb_status kb_bind_join(kb_ctx* ctx, const kb_rel* left, const kb_pattern* pat, kb_rel** out) {
    KB_ENTER(ctx);
    if (!left || !pat || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    KB_TRY(kb::check_pattern(ctx, *pat));
    std::unique_ptr<kb_rel> r;
    KB_TRY(kb::bind_join_impl(ctx, *left, *pat, &r));
    ctx->stats.rows_out = r->n;
    *out = r.release();
    return KB_OK;
}

kb_status kb_star_join(kb_ctx* ctx, uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter, uint32_t n_ops, kb_rel** out) {
    KB_ENTER(ctx);
    if (!pats || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    std::unique_ptr<kb_rel> r;
    KB_TRY(kb::star_join_impl(ctx, join_slot, pats, n_pats, filter, n_ops, &r));
    ctx->stats.rows_out = r->n;
    *out = r.release();
    return KB_OK;
}

kb_status kb_bgp_execute(kb_ctx* ctx, const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter, uint32_t n_ops,
                         const uint32_t* project, uint32_t n_project, kb_rel** out) {
    KB_ENTER(ctx);
    if (!out) return kb::fail(ctx, KB_E_INVALID, "NULL or empty BGP");
    std::unique_ptr<kb_rel> cur;
    KB_TRY(kb::bgp_execute_impl(ctx, pats, n_pats, filter, n_ops, project, n_project, &cur));
    ctx->stats.rows_out = cur->n;
    *out = cur.release();
    return KB_OK;
}

}  // extern "C"

kb_status kb::bgp_execute_impl(kb_ctx* ctx, const kb_pattern* pats, u32 n_pats, const kb_filter_op* filter, u32 n_ops, const u32* project,
                               u32 n_project, std::unique_ptr<kb_rel>* out) {
    if (!pats || n_pats == 0) return kb::fail(ctx, KB_E_INVALID, "NULL or empty BGP");
    if (n_pats > KB_BGP_MAX_PATTERNS) return kb::fail(ctx, KB_E_LIMIT, "more than %d patterns", KB_BGP_MAX_PATTERNS);
    KB_TRY(kb::validate_filter(ctx, filter, n_ops));
    std::vector<std::vector<u32>> pv(n_pats), ps(n_pats);
    std::vector<u32> all_slots;
    for (u32 k = 0; k < n_pats; k++) {
        kb::pattern_vars(pats[k], &pv[k], &ps[k]);
        for (u32 s : pv[k]) if (std::find(all_slots.begin(), all_slots.end(), s) == all_slots.end()) all_slots.push_back(s);
    }
    // a variable shared by every pattern -> star join (optimizer.rs:84-152); prefer the subject position
    int star = -1;
    for (size_t i = 0; n_pats <= (u32)kb::MAXP && i < pv[0].size() && star < 0; i++) {
        bool all = true;
        for (u32 k = 1; k < n_pats; k++) if (std::find(pv[k].begin(), pv[k].end(), pv[0][i]) == pv[k].end()) all = false;
        if (all) star = (int)pv[0][i];
    }
    std::unique_ptr<kb_rel> cur;
    if (star >= 0) {
        KB_TRY(kb::star_join_impl(ctx, (u32)star, pats, n_pats, filter, n_ops, &cur));
        ctx->bgp_last = kb_bgp_plan_info{};
        ctx->bgp_last.route = KB_BGP_STAR;
        ctx->bgp_last.n_patterns = n_pats;
        ctx->bgp_last.n_components = 1;
        ctx->bgp_last.rows_unprojected = cur->n;
    } else {
        KB_TRY(kb::bgp_components(ctx, pats, n_pats, filter, n_ops, pv, all_slots, &cur));
    }
    if (project) {
        std::vector<u32> v(project, project + n_project);
        cur = kb::select_cols(*cur, v);
    }
    *out = std::move(cur);
    return KB_OK;
}

extern "C" {

// ------------------------------------------------------------------ multi-GPU helpers
uint32_t kb_shard_of(uint32_t key, uint32_t n_shards) { return n_shards ? kb::shard_of(key, n_shards) : 0; }

kb_status kb_set_sharding(kb_ctx* ctx, uint32_t rank, uint32_t world) {
    if (!ctx) return KB_E_INVALID;
    if (world == 0 || rank >= world) return kb::fail(ctx, KB_E_INVALID, "rank %u / world %u", rank, world);
    ctx->shard_rank = rank;
    ctx->shard_world = world;
    return KB_OK;
}

kb_status kb_partition_counts(kb_ctx* ctx, const kb_rel* in, uint32_t key_slot, uint32_t n_parts, uint64_t* counts) {
    KB_ENTER(ctx);
    if (!in || !counts) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_parts == 0 || n_parts > 64) return kb::fail(ctx, KB_E_LIMIT, "1..64 partitions");
    const int kc = in->col_of(key_slot);
    if (kc < 0) return kb::fail(ctx, KB_E_INVALID, "partition key slot %u is not a column", key_slot);
    if (in->n >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "relation too large");
    const u32 off = kb::ctrl_alloc(ctx, 64);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 64 * sizeof(u32), ctx->st));
    kb::timer_begin(ctx, kb::F_OTHER);
    kb::launch_part_count(in->cols[kc].ptr, (u32)in->n, n_parts, ctx->ctrl + off, ctx->n_sms, ctx->st);
    kb::timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(kb::ctrl_read(ctx));
    for (u32 i = 0; i < n_parts; i++) counts[i] = ctx->h_ctrl[off + i];
    return KB_OK;
}

static kb_status shuffle_common(kb_ctx* ctx, const kb_rel* in, uint32_t key_slot, uint32_t n_parts, uint32_t* const* peer_cols, const uint64_t* base,
                                uint32_t* const* peer_cursors, uint64_t capacity_rows) {
    if (!in || !peer_cols || (!base && !peer_cursors)) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_parts == 0 || n_parts > 64) return kb::fail(ctx, KB_E_LIMIT, "1..64 partitions");
    const int kc = in->col_of(key_slot);
    if (kc < 0) return kb::fail(ctx, KB_E_INVALID, "partition key slot %u is not a column", key_slot);
    if (in->n >= 0xFFFFFFF0ull || capacity_rows >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "relation too large");
    const u32 n_cols = (u32)in->cols.size();
    for (u32 i = 0; i < n_parts * n_cols; i++) if (!peer_cols[i]) return kb::fail(ctx, KB_E_INVALID, "peer column %u is NULL", i);
    if (peer_cursors) for (u32 i = 0; i < n_parts; i++) if (!peer_cursors[i]) return kb::fail(ctx, KB_E_INVALID, "peer cursor %u is NULL", i);
    // device-side tables: peer column addresses | cursor addresses | bases | local cursors | overflow flag, ticket
    kb::Buf tab;
    const size_t col_bytes = (size_t)n_parts * n_cols * sizeof(u32*);
    const size_t cur_bytes = 64 * sizeof(u32*);
    KB_TRY(kb::alloc_buf(ctx, col_bytes + cur_bytes + 3 * 64 * sizeof(u32), &tab));
    char* tb = static_cast<char*>(tab->p);
    u32* d_base = reinterpret_cast<u32*>(tb + col_bytes + cur_bytes);
    u32* d_cursors = d_base + 64;
    u32* d_flags = d_cursors + 64;  // [0] overflow, [1] tile ticket
    std::vector<u32> hbase(64, 0);
    std::vector<u32*> hcur(64, nullptr);
    for (u32 i = 0; i < n_parts; i++) {
        if (base) {
            if (base[i] > capacity_rows) return kb::fail(ctx, KB_E_INVALID, "base[%u] beyond the receive capacity", i);
            hbase[i] = (u32)base[i];
        }
        hcur[i] = peer_cursors ? peer_cursors[i] : d_cursors + i;
    }
    KB_CUDA(ctx, cudaMemcpyAsync(tb, peer_cols, col_bytes, cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(tb + col_bytes, hcur.data(), cur_bytes, cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(d_base, hbase.data(), 64 * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(d_cursors, 0, 2 * 64 * sizeof(u32), ctx->st));
    kb::ShuffleParams P{};
    P.key = in->cols[kc].ptr;
    P.n = (u32)in->n;
    P.n_parts = n_parts;
    P.n_cols = n_cols;
    for (u32 c = 0; c < n_cols; c++) P.in[c] = in->cols[c].ptr;
    P.peer_cols = reinterpret_cast<u32* const*>(tb);
    P.cursor_ptrs = reinterpret_cast<u32* const*>(tb + col_bytes);
    P.base = d_base;
    P.overflow = d_flags;
    P.ticket = d_flags + 1;
    P.capacity = (u32)capacity_rows;
    kb::timer_begin(ctx, kb::F_OTHER);
    kb::launch_shuffle_scatter(P, ctx->n_sms, ctx->st);
    kb::timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    u32 ovf = 0;
    KB_CUDA(ctx, cudaMemcpyAsync(&ovf, P.overflow, sizeof ovf, cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    kb::timers_flush(ctx);
    if (ovf) return kb::fail(ctx, KB_E_LIMIT, "a receive buffer is smaller than the rows sent to it (capacity %llu rows)", (unsigned long long)capacity_rows);
    return KB_OK;
}

kb_status kb_shuffle_scatter(kb_ctx* ctx, const kb_rel* in, uint32_t key_slot, uint32_t n_parts, uint32_t* const* peer_cols, const uint64_t* base,
                             uint64_t capacity_rows) {
    KB_ENTER(ctx);
    if (!base) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    return shuffle_common(ctx, in, key_slot, n_parts, peer_cols, base, nullptr, capacity_rows);
}

kb_status kb_shuffle_push(kb_ctx* ctx, const kb_rel* in, uint32_t key_slot, uint32_t n_parts, uint32_t* const* peer_cols, uint32_t* const* peer_cursors,
                          uint64_t capacity_rows) {
    KB_ENTER(ctx);
    if (!peer_cursors) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    return shuffle_common(ctx, in, key_slot, n_parts, peer_cols, nullptr, peer_cursors, capacity_rows);
}

kb_status kb_rel_wrap_device(kb_ctx* ctx, const uint32_t* slots, uint32_t n_cols, uint32_t* const* d_cols, uint64_t n_rows, kb_rel** out) {
    if (!ctx) return KB_E_INVALID;
    if (!out || (n_cols && (!slots || !d_cols))) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_cols > KB_MAX_COLS) return kb::fail(ctx, KB_E_LIMIT, "more than %d columns", KB_MAX_COLS);
    if (n_rows >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "relation too large");
    auto r = std::make_unique<kb_rel>();
    r->n = n_rows;
    for (u32 c = 0; c < n_cols; c++) {
        for (u32 d = 0; d < c; d++) if (slots[d] == slots[c]) return kb::fail(ctx, KB_E_INVALID, "duplicate slot %u", slots[c]);
        if (!d_cols[c] || (reinterpret_cast<uintptr_t>(d_cols[c]) & 15u)) return kb::fail(ctx, KB_E_INVALID, "column %u must be a 16-byte aligned device pointer", c);
        kb::Col col;  // no owner: the caller keeps the memory alive (and readable to the next 256-byte boundary) while the relation is used
        col.ptr = d_cols[c];
        r->slots.push_back(slots[c]);
        r->cols.push_back(col);
    }
    *out = r.release();
    return KB_OK;
}

kb_status kb_partition(kb_ctx* ctx, const kb_rel* in, uint32_t key_slot, uint32_t n_parts, kb_rel** out, uint64_t* part_offsets) {
    KB_ENTER(ctx);
    if (!in || !out || !part_offsets) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_parts == 0 || n_parts > 64) return kb::fail(ctx, KB_E_LIMIT, "1..64 partitions");
    const int kc = in->col_of(key_slot);
    if (kc < 0) return kb::fail(ctx, KB_E_INVALID, "partition key slot %u is not a column", key_slot);
    if (in->n >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "relation too large");
    auto r = std::make_unique<kb_rel>();
    r->slots = in->slots;
    r->n = in->n;
    const u32 off = kb::ctrl_alloc(ctx, 128);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 128 * sizeof(u32), ctx->st));
    kb::timer_begin(ctx, kb::F_OTHER);
    kb::launch_part_count(in->cols[kc].ptr, (u32)in->n, n_parts, ctx->ctrl + off, ctx->n_sms, ctx->st);
    kb::timer_end(ctx);
    KB_TRY(kb::ctrl_read(ctx));
    u64 run = 0;
    std::vector<u32> cursors(n_parts);
    for (u32 i = 0; i < n_parts; i++) { part_offsets[i] = run; cursors[i] = (u32)run; run += ctx->h_ctrl[off + i]; }
    part_offsets[n_parts] = run;
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->ctrl + off + 64, cursors.data(), n_parts * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    std::vector<const u32*> ic;
    std::vector<u32*> oc;
    for (auto& c : in->cols) {
        kb::Col col;
        KB_TRY(kb::alloc_col(ctx, in->n, &col));
        r->cols.push_back(col);
        ic.push_back(c.ptr);
        oc.push_back(col.ptr);
    }
    kb::timer_begin(ctx, kb::F_OTHER);
    kb::launch_part_scatter(in->cols[kc].ptr, (u32)in->n, n_parts, ctx->ctrl + off + 64, ic.data(), oc.data(), (u32)ic.size(), ctx->n_sms, ctx->st);
    kb::timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    kb::timers_flush(ctx);
    *out = r.release();
    return KB_OK;
}

// ------------------------------------------------------------------ one-shot host-buffer star join
static constexpr u64 HOST_UPLOAD_CHUNK = 8ull << 20;  // triples per upload chunk (one store segment each): 32 MiB per column
static kb_status star_join_host_common(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint32_t join_slot,
                                       const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter, uint32_t n_ops, uint32_t* n_cols,
                                       uint32_t* slots, uint32_t** cols, uint64_t* n_rows, bool caller_bufs, uint64_t caller_cap) {
    if (!pats || !n_cols || !slots || !cols || !n_rows) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (n && (!s || !p || !o)) return kb::fail(ctx, KB_E_INVALID, "NULL column pointer");
    if (n >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "too many triples");
    // everything that can be rejected without looking at the data is rejected BEFORE the upload starts: an early return must not
    // leave copies in flight that still read the caller's (borrowed) buffers
    if (n_pats == 0 || n_pats > (u32)kb::MAXP) return kb::fail(ctx, KB_E_LIMIT, "a star join takes 1..%d patterns (got %u)", kb::MAXP, n_pats);
    KB_TRY(kb::validate_filter(ctx, filter, n_ops));
    for (u32 k = 0; k < n_pats; k++) {
        KB_TRY(kb::check_pattern(ctx, pats[k]));
        std::vector<u32> vs, src;
        kb::pattern_vars(pats[k], &vs, &src);
        if (std::find(vs.begin(), vs.end(), join_slot) == vs.end())
            return kb::fail(ctx, KB_E_INVALID, "star join: pattern %u does not contain the join variable (slot %u)", k, join_slot);
    }
    // upload in chunks on the copy stream; each chunk is a store segment the scan starts on as soon as its copy has landed. The
    // previous store goes first: its memory is free for the upload.
    kb::store_replace(ctx, {});
    kb::Col cs, cp, co;
    KB_TRY(kb::alloc_col(ctx, n, &cs));
    KB_TRY(kb::alloc_col(ctx, n, &cp));
    KB_TRY(kb::alloc_col(ctx, n, &co));
    const u32 soff = kb::ctrl_alloc(ctx, 8);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + soff, 0xFF, 4 * sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + soff + 4, 0, 4 * sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));  // allocations are stream-ordered on st; the copy stream must see them
    const u64 chunk = HOST_UPLOAD_CHUNK;
    std::vector<cudaEvent_t> evs;
    std::vector<kb::Segment> segs;
    // whatever happens from here on, the caller's buffers are not read after this function returns and a failed call leaves an
    // EMPTY store (never segments whose copies did not complete)
    auto finish = [&](kb_status rc) -> kb_status {
        cudaStreamSynchronize(ctx->st_copy);
        for (auto& sg : ctx->segs) sg.ready = nullptr;
        ctx->upload_stats_off = -1;
        for (auto ev : evs) cudaEventDestroy(ev);
        if (rc != KB_OK) {
            cudaStreamSynchronize(ctx->st);
            kb::store_replace(ctx, {});
        }
        return rc;
    };
#define KB_HOST_CUDA(call)                                                                                                    \
    do {                                                                                                                      \
        cudaError_t _e = (call);                                                                                              \
        if (_e != cudaSuccess) return finish(kb::fail(ctx, KB_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__)); \
    } while (0)
    for (u64 b = 0; b < n; b += chunk) {
        const u64 m = std::min(chunk, n - b);
        KB_HOST_CUDA(cudaMemcpyAsync(cs.ptr + b, s + b, m * sizeof(u32), cudaMemcpyHostToDevice, ctx->st_copy));
        KB_HOST_CUDA(cudaMemcpyAsync(cp.ptr + b, p + b, m * sizeof(u32), cudaMemcpyHostToDevice, ctx->st_copy));
        KB_HOST_CUDA(cudaMemcpyAsync(co.ptr + b, o + b, m * sizeof(u32), cudaMemcpyHostToDevice, ctx->st_copy));
        {  // column ranges of this chunk, on the copy stream right behind its copies (the direct tables need the key range)
            const u32* cc[3] = {cs.ptr + b, cp.ptr + b, co.ptr + b};
            for (int c = 0; c < 3; c++) kb::launch_col_minmax(cc[c], (u32)m, ctx->ctrl + soff + c, ctx->ctrl + soff + 4 + c, ctx->n_sms, ctx->st_copy);
            ctx->stats.kernel_launches += 3;
        }
        cudaEvent_t ev;
        KB_HOST_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        evs.push_back(ev);
        KB_HOST_CUDA(cudaEventRecord(ev, ctx->st_copy));
        kb::Segment sg;
        sg.tag = 0; sg.n = m;
        sg.ready = ev;
        sg.s.buf = cs.buf; sg.s.ptr = cs.ptr + b;
        sg.p.buf = cp.buf; sg.p.ptr = cp.ptr + b;
        sg.o.buf = co.buf; sg.o.ptr = co.ptr + b;
        segs.push_back(sg);
    }
    kb::store_replace(ctx, std::move(segs));
    ctx->stats.h2d_bytes += 3 * n * sizeof(u32);
    ctx->upload_stats_off = (int)soff;
    // scan_segments makes st wait on each segment's `ready` event right before that segment's scan kernel: copy i+1 overlaps scan i
    std::unique_ptr<kb_rel> r;
    kb_status rc = kb::star_join_impl(ctx, join_slot, pats, n_pats, filter, n_ops, &r);
    if (rc != KB_OK) return finish(rc);
    if (n) {  // a column holding KB_ID_NONE (reserved) is refused like kb_store_load refuses it: the store is left empty, nothing returned
        // the scan stage took the upload's column ranges into the segments; a join that ended before it reads them from the
        // control words the copy stream filled
        u32 mx[3];
        if (!ctx->segs.empty() && ctx->segs[0].has_stats) {
            for (int c = 0; c < 3; c++) mx[c] = ctx->segs[0].cmax[c];
        } else {
            KB_HOST_CUDA(cudaStreamSynchronize(ctx->st_copy));
            KB_HOST_CUDA(cudaMemcpy(mx, ctx->ctrl + soff + 4, sizeof mx, cudaMemcpyDeviceToHost));
        }
        rc = kb::refuse_reserved_id(ctx, mx);
        if (rc != KB_OK) return finish(rc);
    }
    *n_cols = (u32)r->slots.size();
    *n_rows = r->n;
    for (size_t c = 0; c < r->slots.size(); c++) slots[c] = r->slots[c];
    if (caller_bufs && caller_cap < r->n)
        return finish(kb::fail(ctx, KB_E_LIMIT, "caller buffers hold %llu rows, result has %llu", (unsigned long long)caller_cap, (unsigned long long)r->n));
    if (!caller_bufs) for (size_t c = 0; c < KB_MAX_COLS; c++) cols[c] = nullptr;
    for (size_t c = 0; c < r->slots.size(); c++) {
        if (!caller_bufs) {
            cols[c] = (uint32_t*)malloc(std::max<size_t>(r->n * sizeof(u32), 4));
            if (!cols[c]) {
                for (size_t d = 0; d < c; d++) { free(cols[d]); cols[d] = nullptr; }
                return finish(kb::fail(ctx, KB_E_OOM, "malloc failed"));
            }
        } else if (!cols[c]) return finish(kb::fail(ctx, KB_E_INVALID, "caller-provided column buffer %zu is NULL", c));
        if (r->n) KB_HOST_CUDA(cudaMemcpyAsync(cols[c], r->cols[c].ptr, r->n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    }
    KB_HOST_CUDA(cudaStreamSynchronize(ctx->st));
#undef KB_HOST_CUDA
    ctx->stats.d2h_bytes += r->slots.size() * r->n * sizeof(u32);
    ctx->stats.rows_out = r->n;
    return finish(KB_OK);
}

kb_status kb_star_join_host(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint32_t join_slot,
                            const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter, uint32_t n_ops, uint32_t* n_cols,
                            uint32_t* slots, uint32_t** cols, uint64_t* n_rows) {
    KB_ENTER(ctx);
    return star_join_host_common(ctx, s, p, o, n, join_slot, pats, n_pats, filter, n_ops, n_cols, slots, cols, n_rows, false, 0);
}

kb_status kb_star_join_host_into(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint32_t join_slot,
                                 const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter, uint32_t n_ops, uint32_t* n_cols,
                                 uint32_t* slots, uint32_t* const* cols, uint64_t capacity_rows, uint64_t* n_rows) {
    KB_ENTER(ctx);
    return star_join_host_common(ctx, s, p, o, n, join_slot, pats, n_pats, filter, n_ops, n_cols, slots, const_cast<uint32_t**>(cols), n_rows, true,
                                 capacity_rows);
}

}  // extern "C"
