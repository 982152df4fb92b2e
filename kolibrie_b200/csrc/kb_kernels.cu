// kb_kernels.cu — hand-written sm_90a kernels of the Kolibrie hot path (see kb_kernels.cuh for what each replaces).
// All of them are HBM-bound integer kernels: column tiles are staged global->shared with TMA bulk copies (cp.async.bulk +
// mbarrier), matches are compacted with warp ballots, and output positions come from a single-pass decoupled look-back
// prefix over tiles, so every kernel reads its input exactly once and writes a deterministic, input-ordered output.
#include "kb_kernels.cuh"

#include <math_constants.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <type_traits>

namespace kb {

static inline u64 umin64(u64 a, u64 b) { return a < b ? a : b; }
// grid-stride utility kernels are capped at a few CTAs per SM of an H100; the persistent kernels size their grids from the device's count
constexpr u64 H100_SMS = 132;

static inline int grid_for(const void* kernel, int threads, size_t smem, int n_sms, u32 n_tiles) {
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem);
    if (per_sm < 1) per_sm = 1;
    long long g = (long long)per_sm * n_sms;  // persistent: a whole number of resident CTAs per SM, on every SM
    if (g > (long long)n_tiles) g = n_tiles;
    if (g < 1) g = 1;
    return (int)g;
}

// =================================================================================================================
// K_scan
// Thread t owns the 8 consecutive triples [8t, 8t+8) of a 2048-triple tile. The tile is TMA-staged into shared memory, pulled
// into registers with six LDS.128, and the shared buffer is immediately handed back to TMA for the NEXT tile (single buffer,
// register-staged double buffering). K is a template parameter so every pattern field is a constant-bank operand.
__device__ __forceinline__ u32 eq8(const uint4& a, const uint4& b, u32 c) {
    return (a.x == c ? 1u : 0u) | (a.y == c ? 2u : 0u) | (a.z == c ? 4u : 0u) | (a.w == c ? 8u : 0u) | (b.x == c ? 16u : 0u) | (b.y == c ? 32u : 0u) |
           (b.z == c ? 64u : 0u) | (b.w == c ? 128u : 0u);
}
__device__ __forceinline__ u32 eqv8(const uint4& a0, const uint4& a1, const uint4& b0, const uint4& b1) {
    return (a0.x == b0.x ? 1u : 0u) | (a0.y == b0.y ? 2u : 0u) | (a0.z == b0.z ? 4u : 0u) | (a0.w == b0.w ? 8u : 0u) | (a1.x == b1.x ? 16u : 0u) |
           (a1.y == b1.y ? 32u : 0u) | (a1.z == b1.z ? 64u : 0u) | (a1.w == b1.w ? 128u : 0u);
}
#define KB_ELEM(v0, v1, j) ((j) == 0 ? v0.x : (j) == 1 ? v0.y : (j) == 2 ? v0.z : (j) == 3 ? v0.w : (j) == 4 ? v1.x : (j) == 5 ? v1.y : (j) == 6 ? v1.z : v1.w)

template <int K>
__global__ void __launch_bounds__(SCAN_THREADS, (K <= 4 ? 1024 / SCAN_THREADS : 512 / SCAN_THREADS)) scan_kernel(const __grid_constant__ ScanParams P) {
    // two shared stages of three column tiles each: tile i+1 is in flight while tile i is processed; the stage of tile i is handed
    // back to TMA (for tile i+2) right after the first compaction barrier — every thread has its triples in registers by then, so
    // the hand-over costs no barrier of its own
    extern __shared__ __align__(128) u32 smem_all[];
    constexpr u32 STAGE_WORDS = 3u * SCAN_TILE;
    __shared__ __align__(8) u64 bars[2];
    __shared__ u32 s_nexts[2];
    __shared__ u32 s_wcnt[SCAN_THREADS / 32][MAXP];
    __shared__ u32 s_excl[MAXP];
    constexpr int NW = (K + 2) / 3;  // packed count words: three 10-bit fields each (a warp holds at most 256 matches per pattern)
    __shared__ u32 s_tcnt[2], s_tindex[2];  // triples in the staged tile, global index of its first triple
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // one thread: take the next tile, find its segment, start the three column copies into `stage`
    auto issue_next = [&](u32 stage) {
        const u32 t = atomicAdd(P.ticket, 1u);
        s_nexts[stage] = t;
        if (t < P.n_tiles) {
            u32 g = 0;
            while (g + 1u < P.n_seg && t >= P.seg[g + 1u].tile0) g++;
            const ScanSeg& sg = P.seg[g];
            const u32 b = (t - sg.tile0) * (u32)SCAN_TILE;
            const u32 c = min((u32)SCAN_TILE, sg.n - b);
            const u32 bytes = (c * 4u + 15u) & ~15u;  // columns are padded to 256 B: the rounded-up read stays in bounds
            s_tcnt[stage] = c;
            s_tindex[stage] = sg.index_base + b;
            u32* dst = smem_all + stage * STAGE_WORDS;
            mbar_arrive_expect_tx(&bars[stage], bytes * 3u);
            tma_load_1d(dst, sg.s + b, bytes, &bars[stage]);
            tma_load_1d(dst + SCAN_TILE, sg.p + b, bytes, &bars[stage]);
            tma_load_1d(dst + 2 * SCAN_TILE, sg.o + b, bytes, &bars[stage]);
        }
    };
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_mbar_init();
        issue_next(0);
        issue_next(1);
    }
    __syncthreads();
    u32 tile = s_nexts[0];
    u32 it = 0;

    while (tile < P.n_tiles) {
        const u32 stage = it & 1u;
        mbar_wait(&bars[stage], (it >> 1) & 1u);
        const uint4* sS4 = reinterpret_cast<const uint4*>(smem_all + stage * STAGE_WORDS);
        const uint4* sP4 = sS4 + SCAN_TILE / 4;
        const uint4* sO4 = sS4 + 2 * (SCAN_TILE / 4);
        const uint4 s0 = sS4[2 * tid], s1 = sS4[2 * tid + 1];
        const uint4 p0 = sP4[2 * tid], p1 = sP4[2 * tid + 1];
        const uint4 o0 = sO4[2 * tid], o1 = sO4[2 * tid + 1];
        const u32 cnt = s_tcnt[stage], tindex = s_tindex[stage];
        // ---- match: bit j of mk[k] = triple 8*tid+j matches pattern k
        const u32 first = (u32)tid * 8u;
        const u32 vmask = first >= cnt ? 0u : (cnt - first >= 8u ? 0xFFu : ((1u << (cnt - first)) - 1u));
        u32 mk[K];
#pragma unroll
        for (int k = 0; k < K; k++) {
            const u32 f = P.pat[k].flags;
            u32 m = vmask;
            if (f & SP_HAS_P) m &= eq8(p0, p1, P.pat[k].cp);
            if (f & SP_HAS_S) m &= eq8(s0, s1, P.pat[k].cs);
            if (f & SP_HAS_O) m &= eq8(o0, o1, P.pat[k].co);
            if (f & (SP_EQ_SP | SP_EQ_SO | SP_EQ_PO)) {
                if (f & SP_EQ_SP) m &= eqv8(s0, s1, p0, p1);
                if (f & SP_EQ_SO) m &= eqv8(s0, s1, o0, o1);
                if (f & SP_EQ_PO) m &= eqv8(p0, p1, o0, o1);
            }
            if (P.pat[k].f_len != 0u && m != 0u) {
                const FilterOp* fo = P.ops + P.pat[k].f_begin;
                if (P.pat[k].f_len == 1u && fo[0].op == KB_F_CMP_NUM) {  // FILTER(?x <cmp> c): gather the 8 numeric values, then compare
                    const u32 slot = fo[0].slot, cmp = fo[0].cmp;
                    const double cv = fo[0].value;
                    // the column is chosen once (two vector selects), not once per element
                    const uint4 x0 = slot == 0u ? s0 : (slot == 1u ? p0 : o0);
                    const uint4 x1 = slot == 0u ? s1 : (slot == 1u ? p1 : o1);
                    double a[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) a[j] = ((m >> j) & 1u) ? num_of(P.nt, KB_ELEM(x0, x1, j)) : 0.0;
                    u32 pass = 0;
#pragma unroll
                    for (int j = 0; j < 8; j++) pass |= (cmp_num(cmp, a[j], cv) ? 1u : 0u) << j;
                    m &= pass;
                } else {
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if ((m >> j) & 1u) {
                            u32 vals[3] = {KB_ELEM(s0, s1, j), KB_ELEM(p0, p1, j), KB_ELEM(o0, o1, j)};
                            if (!eval_filter(fo, P.pat[k].f_len, vals, P.nt)) m &= ~(1u << j);
                        }
                    }
                }
            }
            mk[k] = m;
        }
        // ---- ranks: one packed warp scan per three patterns
        u32 wex[K];
#pragma unroll
        for (int w = 0; w < NW; w++) {
            u32 packed = 0;
#pragma unroll
            for (int q = 0; q < 3; q++) if (w * 3 + q < K) packed |= (u32)__popc(mk[w * 3 + q]) << (10 * q);
            u32 incl = packed;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            const u32 excl = incl - packed;
            const u32 tot = __shfl_sync(0xffffffffu, incl, 31);
#pragma unroll
            for (int q = 0; q < 3; q++) if (w * 3 + q < K) {
                wex[w * 3 + q] = (excl >> (10 * q)) & 1023u;
                if (lane == 0) s_wcnt[warp][w * 3 + q] = (tot >> (10 * q)) & 1023u;
            }
        }
        __syncthreads();
        const u32 following = s_nexts[stage ^ 1u];  // the next iteration's tile (its copies are already in flight)
        if (tid == SCAN_THREADS - 1) issue_next(stage);
        if (warp < K) {  // warp k owns counter k: cross-warp prefix of its per-warp totals, then the look-back across tiles
            const u32 c = lane < SCAN_THREADS / 32 ? s_wcnt[lane][warp] : 0u;
            u32 incl = c;
#pragma unroll
            for (int o = 1; o < SCAN_THREADS / 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            const u32 total = __shfl_sync(0xffffffffu, incl, SCAN_THREADS / 32 - 1);
            if (lane < SCAN_THREADS / 32) s_wcnt[lane][warp] = incl - c;
            const u32 ex = tile_prefix_2level(P.tile_state, P.block_state, tile, P.n_tiles, (u32)warp, P.epoch, total, P.totals_in, P.totals_out, P.ordered, lane);
            if (lane == 0) s_excl[warp] = ex;
        }
        __syncthreads();
        // ---- write: rank = tile prefix + warp prefix + thread prefix, then a running rank over this thread's 8 triples
#pragma unroll
        for (int k = 0; k < K; k++) {
            const u32 m = mk[k];
            if (m == 0u) continue;
            const u32 f = P.pat[k].flags;
            if (f & SP_TABLE) {  // fused build: insert into the direct table of this pattern
                u32* tab = P.pat[k].outp[0];
                const u32 kbase = P.pat[k].cs, krange = P.pat[k].co;
                // key / value columns chosen once; offsets computed for all eight triples, stores predicated (no branch per triple).
                // Plain fire-and-forget stores: a returning atomic here stalls the tile loop (slower than a separate
                // scan + build); duplicate keys are detected afterwards by counting the occupied slots
                const bool key_o = (f & SP_TKEY_O) != 0u;
                const uint4 k0 = key_o ? o0 : s0, k1 = key_o ? o1 : s1;
                const uint4 v0 = key_o ? s0 : o0, v1 = key_o ? s1 : o1;
                u32 bad = 0;
                if (P.cshift == 0u) {
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const u32 off = KB_ELEM(k0, k1, j) - kbase;
                        const bool on = (m >> j) & 1u;
                        if (on && off < krange) tab[off] = KB_ELEM(v0, v1, j);
                        bad |= (on && off >= krange) ? 1u : 0u;
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const u32 off = compact_key(KB_ELEM(k0, k1, j), P.cshift) - kbase;
                        const bool on = (m >> j) & 1u;
                        if (on && off < krange) tab[off] = KB_ELEM(v0, v1, j);
                        bad |= (on && off >= krange) ? 1u : 0u;
                    }
                }
                const bool dup = bad != 0u;
                if (dup) *P.pat[k].outp[1] = 1u;
                continue;
            }
            const u32 pos = s_excl[k] + s_wcnt[warp][k] + wex[k];
            if (f & SP_PAIR) {
                uint2* out = reinterpret_cast<uint2*>(P.pat[k].outp[0]) + pos;
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    if ((m >> j) & 1u) *out = make_uint2(KB_ELEM(s0, s1, j), KB_ELEM(o0, o1, j));
                    out += (m >> j) & 1u;
                }
                continue;
            }
            if (f & SP_EMIT_S) {
                u32* out = P.pat[k].outp[0] + pos;
#pragma unroll
                for (int j = 0; j < 8; j++) { if ((m >> j) & 1u) *out = KB_ELEM(s0, s1, j); out += (m >> j) & 1u; }
            }
            if (f & SP_EMIT_P) {
                u32* out = P.pat[k].outp[1] + pos;
#pragma unroll
                for (int j = 0; j < 8; j++) { if ((m >> j) & 1u) *out = KB_ELEM(p0, p1, j); out += (m >> j) & 1u; }
            }
            if (f & SP_EMIT_O) {
                u32* out = P.pat[k].outp[2] + pos;
#pragma unroll
                for (int j = 0; j < 8; j++) { if ((m >> j) & 1u) *out = KB_ELEM(o0, o1, j); out += (m >> j) & 1u; }
            }
            if (f & SP_EMIT_IDX) {
                u32* out = P.pat[k].outp[3] + pos;
#pragma unroll
                for (int j = 0; j < 8; j++) { if ((m >> j) & 1u) *out = tindex + first + (u32)j; out += (m >> j) & 1u; }
            }
        }
        tile = following;
        it++;
    }
}

// K_scan, STAR shape: every pattern is (?s P ?o) with a constant predicate and distinct variables, its output goes to a direct join
// table (fused build) or to an interleaved (s,o) pair relation, and its pushed-down FILTER — if any — is one numeric comparison on the
// subject or the object. That is what a star join's scan looks like (engine.rs:587-691 over engine.rs:1364-1378), and knowing it at
// compile time removes what made the general kernel issue-bound (2.8 warp instructions per triple): no per-tile flag tests, no
// comparison switch per element (a < c is evaluated as -a > -c, so every operator is one DSETP), no divergent branches — every store is
// predicated — and no rank computation for patterns whose matches go to a table.
#ifndef KB_STAR_THREADS
#define KB_STAR_THREADS 256
#endif
constexpr int STAR_THREADS = KB_STAR_THREADS;  // K <= 4 patterns need 4 prefix warps: 128 threads suffice (smaller CTAs, cheaper barriers)
constexpr int STAR_TILE = STAR_THREADS * SCAN_ITEMS;
template <int K>
__global__ void __launch_bounds__(STAR_THREADS, 1024 / STAR_THREADS) scan_star_kernel(const __grid_constant__ ScanParams P) {
    extern __shared__ __align__(128) u32 smem_all[];
    constexpr u32 STAGE_WORDS = 3u * STAR_TILE;
    __shared__ __align__(8) u64 bars[2];
    __shared__ u32 s_nexts[2];
    __shared__ u32 s_wcnt[STAR_THREADS / 32][MAXP];
    __shared__ u32 s_excl[MAXP];
    __shared__ u32 s_tcnt[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    auto issue_next = [&](u32 stage) {
        const u32 t = atomicAdd(P.ticket, 1u);
        s_nexts[stage] = t;
        if (t < P.n_tiles) {
            u32 g = 0;
            while (g + 1u < P.n_seg && t >= P.seg[g + 1u].tile0) g++;
            const ScanSeg& sg = P.seg[g];
            const u32 b = (t - sg.tile0) * (u32)STAR_TILE;
            const u32 c = min((u32)STAR_TILE, sg.n - b);
            const u32 bytes = (c * 4u + 15u) & ~15u;
            s_tcnt[stage] = c;
            u32* dst = smem_all + stage * STAGE_WORDS;
            mbar_arrive_expect_tx(&bars[stage], bytes * 3u);
            tma_load_1d(dst, sg.s + b, bytes, &bars[stage]);
            tma_load_1d(dst + STAR_TILE, sg.p + b, bytes, &bars[stage]);
            tma_load_1d(dst + 2 * STAR_TILE, sg.o + b, bytes, &bars[stage]);
        }
    };
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_mbar_init();
        issue_next(0);
        issue_next(1);
    }
    if (P.n_clear) {
        // the tables this scan inserts into are cleared by the grid itself while the first tiles are in flight, then every CTA waits
        // until all have finished (the grid is sized to residency, so all of them are running)
        const uint4 ones = make_uint4(EMPTY32, EMPTY32, EMPTY32, EMPTY32);
        for (u32 t = 0; t < P.n_clear; t++) {
            uint4* t4 = reinterpret_cast<uint4*>(P.clear_tab[t]);
            const u32 n4 = P.clear_words[t] >> 2;
            for (u32 i = blockIdx.x * STAR_THREADS + (u32)tid; i < n4; i += gridDim.x * STAR_THREADS) t4[i] = ones;
            if (blockIdx.x == 0) for (u32 i = (n4 << 2) + (u32)tid; i < P.clear_words[t]; i += STAR_THREADS) P.clear_tab[t][i] = EMPTY32;
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            atomicAdd(P.clear_barrier, 1u);
            u32 spins = 0;
            while (*reinterpret_cast<volatile u32*>(P.clear_barrier) < gridDim.x) {
                __nanosleep(100);
                if (++spins > (1u << 24)) { P.clear_barrier[1] = 1u; break; }  // ~2 s: reported by the host as an error
            }
            __threadfence();
        }
    }
    __syncthreads();
    u32 tile = s_nexts[0];
    u32 it = 0;
    u32 bad_any = 0;
    while (tile < P.n_tiles) {
        const u32 stage = it & 1u;
        mbar_wait(&bars[stage], (it >> 1) & 1u);
        const uint4* sS4 = reinterpret_cast<const uint4*>(smem_all + stage * STAGE_WORDS);
        const uint4* sP4 = sS4 + STAR_TILE / 4;
        const uint4* sO4 = sS4 + 2 * (STAR_TILE / 4);
        // thread t owns triples [4t, 4t+4) of EACH half of the tile: consecutive threads read consecutive 16-byte words (LDS.128 without
        // bank conflicts; 8 consecutive triples per thread put two threads of a quarter-warp on the same banks). The rows of a tile
        // therefore come out in a fixed permutation of store order — fine for tables and for completion-order results; ordered
        // contexts take the general kernel.
        constexpr u32 HALF4 = STAR_TILE / 8;  // uint4 words per half column
        const uint4 s0 = sS4[tid], s1 = sS4[HALF4 + tid];
        const uint4 p0 = sP4[tid], p1 = sP4[HALF4 + tid];
        const uint4 o0 = sO4[tid], o1 = sO4[HALF4 + tid];
        const u32 cnt = s_tcnt[stage];
        const u32 first = (u32)tid * 4u;
        const u32 lo = first >= cnt ? 0u : (cnt - first >= 4u ? 0xFu : ((1u << (cnt - first)) - 1u));
        const u32 first2 = (u32)STAR_TILE / 2u + first;
        const u32 hi = first2 >= cnt ? 0u : (cnt - first2 >= 4u ? 0xFu : ((1u << (cnt - first2)) - 1u));
        const u32 vmask = lo | (hi << 4);
        u32 mk[K];
#pragma unroll
        for (int k = 0; k < K; k++) {
            u32 m = eq8(p0, p1, P.pat[k].cp) & vmask;
            if (P.pat[k].f_len != 0u) {  // uniform per pattern: FILTER(?x <cmp> c) on the subject (slot 0) or the object (slot 2)
                // the launcher canonicalised the comparison to >= or <= (a > c is a >= nextup(c)): one DSETP per triple, no operator switch
                const FilterOp fo = P.ops[P.pat[k].f_begin];
                const bool on_s = fo.slot == 0u;
                const double cv = fo.value;
                const uint4 x0 = on_s ? s0 : o0, x1 = on_s ? s1 : o1;
                double a[8];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const u32 id = KB_ELEM(x0, x1, j);
                    a[j] = 0.0;
                    if (((m >> j) & 1u) && id < P.nt.n_ids) a[j] = __ldg(P.nt.num_or0 + id);
                }
                u32 pass = 0;
                if (fo.cmp == KB_CMP_GE) {
#pragma unroll
                    for (int j = 0; j < 8; j++) pass |= (a[j] >= cv ? 1u : 0u) << j;
                } else {
#pragma unroll
                    for (int j = 0; j < 8; j++) pass |= (a[j] <= cv ? 1u : 0u) << j;
                }
                m &= pass;
            }
            mk[k] = m;
        }
        // ---- counts: a packed warp scan per three patterns (ranks are only consumed by pair outputs; totals by every pattern)
        constexpr int NW = (K + 2) / 3;
        u32 wex[K];
#pragma unroll
        for (int w = 0; w < NW; w++) {
            u32 packed = 0;
#pragma unroll
            for (int q = 0; q < 3; q++) if (w * 3 + q < K) packed |= (u32)__popc(mk[w * 3 + q]) << (10 * q);
            u32 incl = packed;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            const u32 excl = incl - packed;
            const u32 tot = __shfl_sync(0xffffffffu, incl, 31);
#pragma unroll
            for (int q = 0; q < 3; q++) if (w * 3 + q < K) {
                wex[w * 3 + q] = (excl >> (10 * q)) & 1023u;
                if (lane == 0) s_wcnt[warp][w * 3 + q] = (tot >> (10 * q)) & 1023u;
            }
        }
        __syncthreads();
        const u32 following = s_nexts[stage ^ 1u];
        if (tid == STAR_THREADS - 1) issue_next(stage);  // every thread holds its triples in registers: the stage takes the tile after next
        if (warp < K) {
            const u32 c = lane < STAR_THREADS / 32 ? s_wcnt[lane][warp] : 0u;
            u32 incl = c;
#pragma unroll
            for (int o = 1; o < STAR_THREADS / 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            const u32 total = __shfl_sync(0xffffffffu, incl, STAR_THREADS / 32 - 1);
            if (lane < STAR_THREADS / 32) s_wcnt[lane][warp] = incl - c;
            const u32 ex = tile_prefix_2level(P.tile_state, P.block_state, tile, P.n_tiles, (u32)warp, P.epoch, total, P.totals_in, P.totals_out, P.ordered, lane);
            if (lane == 0) s_excl[warp] = ex;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < K; k++) {
            const u32 m = mk[k];
            if (P.pat[k].flags & SP_TABLE) {  // uniform: the matches go straight into this pattern's direct table
                u32* tab = P.pat[k].outp[0];
                const u32 kbase = P.pat[k].cs, krange = P.pat[k].co;
                auto stores = [&](const uint4& k0, const uint4& k1, const uint4& v0, const uint4& v1, auto with_cshift) {
                    u32 worst = 0;  // largest offset of a matching triple: one range test per pattern and tile instead of one flag update per triple
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const u32 key = KB_ELEM(k0, k1, j);
                        const u32 off = (with_cshift.value ? compact_key(key, P.cshift) : key) - kbase;
                        const bool on = (m >> j) & 1u;  // (the compiler folds this with the predicate comparison the bit came from)
                        if (on && off < krange) tab[off] = KB_ELEM(v0, v1, j);
                        worst = max(worst, on ? off : 0u);
                    }
                    bad_any |= worst >= krange ? (1u << k) : 0u;
                };
                const bool key_o = (P.pat[k].flags & SP_TKEY_O) != 0u;
                if (P.cshift == 0u) {
                    if (key_o) stores(o0, o1, s0, s1, std::false_type{});
                    else stores(s0, s1, o0, o1, std::false_type{});
                } else {
                    if (key_o) stores(o0, o1, s0, s1, std::true_type{});
                    else stores(s0, s1, o0, o1, std::true_type{});
                }
            } else {
                u32 pos = s_excl[k] + s_wcnt[warp][k] + wex[k];
                uint2* out = reinterpret_cast<uint2*>(P.pat[k].outp[0]);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const bool on = (m >> j) & 1u;
                    if (on) out[pos] = make_uint2(KB_ELEM(s0, s1, j), KB_ELEM(o0, o1, j));
                    pos += on ? 1u : 0u;
                }
            }
        }
        tile = following;
        it++;
    }
    if (bad_any) {  // a key outside the table range (cannot happen with load-time statistics): reported like a duplicate
#pragma unroll
        for (int k = 0; k < K; k++) if ((bad_any >> k) & 1u) *P.pat[k].outp[1] = 1u;
    }
}

// does the star-shape kernel apply?
static bool scan_is_star(const ScanParams& p) {
    if (p.K > 4 || p.ordered) return false;  // store-order output (KOLIBRIE_ORDERED, legacy FFI): the general kernel
    for (u32 k = 0; k < p.K; k++) {
        const ScanPat& sp = p.pat[k];
        const u32 shape = sp.flags & ~(SP_TABLE | SP_TKEY_O | SP_TTRUSTED | SP_PAIR);
        if (shape != SP_HAS_P) return false;                       // constant predicate only, nothing emitted column-wise
        if (!(sp.flags & (SP_TABLE | SP_PAIR))) return false;
        if ((sp.flags & SP_TABLE) && (sp.flags & SP_PAIR)) return false;
        if (sp.f_len > 1u) return false;
        if (sp.f_len == 1u) {
            const FilterOp& fo = p.ops[sp.f_begin];
            if (fo.op != KB_F_CMP_NUM || (fo.slot != 0u && fo.slot != 2u) || fo.cmp < KB_CMP_GT || fo.cmp > KB_CMP_LE) return false;
        }
    }
    return true;
}
template <int K>
static void launch_scan_star_k(const ScanParams& p_in, int n_sms, cudaStream_t st) {
    ScanParams p = p_in;
    for (u32 k = 0; k < (u32)K; k++) {
        if (p.pat[k].f_len != 1u) continue;
        // strict comparisons become non-strict ones against the neighbouring double: a > c <=> a >= nextup(c) (c = +inf: never true -> NaN)
        FilterOp& fo = p.ops[p.pat[k].f_begin];
        if (fo.cmp == KB_CMP_GT) { fo.value = fo.value == HUGE_VAL ? NAN : nextafter(fo.value, HUGE_VAL); fo.cmp = KB_CMP_GE; }
        else if (fo.cmp == KB_CMP_LT) { fo.value = fo.value == -HUGE_VAL ? NAN : nextafter(fo.value, -HUGE_VAL); fo.cmp = KB_CMP_LE; }
    }
    // the kernel walks the store in STAR_TILE-triple tiles: renumber the segments' first tiles
    p.n_tiles = 0;
    for (u32 g = 0; g < p.n_seg; g++) {
        p.seg[g].tile0 = p.n_tiles;
        p.n_tiles += (p.seg[g].n + (u32)STAR_TILE - 1u) / (u32)STAR_TILE;
    }
    const size_t smem = 2 * 3 * STAR_TILE * sizeof(u32);
    static int grid_max = 0;
    if (grid_max == 0) {
        cudaFuncSetAttribute(scan_star_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int per_sm = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, scan_star_kernel<K>, STAR_THREADS, smem);
        grid_max = (per_sm < 1 ? 1 : per_sm) * n_sms;
    }
    const int grid = (int)umin64((u64)grid_max, (u64)p.n_tiles);
    scan_star_kernel<K><<<grid, STAR_THREADS, smem, st>>>(p);
}

template <int K>
static void launch_scan_k(const ScanParams& p, int n_sms, cudaStream_t st) {
    const size_t smem = 2 * 3 * SCAN_TILE * sizeof(u32);  // two stages: 48 KB, above the default dynamic limit
    cudaFuncSetAttribute(scan_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int grid = grid_for((const void*)scan_kernel<K>, SCAN_THREADS, smem, n_sms, p.n_tiles);
    scan_kernel<K><<<grid, SCAN_THREADS, smem, st>>>(p);
}
static bool scan_star_enabled() {
    static const bool star_off = getenv("KOLIBRIE_SCAN_STAR") && getenv("KOLIBRIE_SCAN_STAR")[0] == '0';  // A/B switch
    return !star_off;
}
bool scan_clears_tables(const ScanParams& p) {
    static const bool fold_off = getenv("KOLIBRIE_SCAN_CLEAR_FOLD") && getenv("KOLIBRIE_SCAN_CLEAR_FOLD")[0] == '0';  // A/B switch
    return !fold_off && p.n_tiles != 0 && scan_star_enabled() && scan_is_star(p);
}
void launch_scan(const ScanParams& p, int n_sms, cudaStream_t st) {
    if (p.n_tiles == 0) return;
    if (scan_star_enabled() && scan_is_star(p)) {
        switch (p.K) {
            case 1: launch_scan_star_k<1>(p, n_sms, st); return;
            case 2: launch_scan_star_k<2>(p, n_sms, st); return;
            case 3: launch_scan_star_k<3>(p, n_sms, st); return;
            default: launch_scan_star_k<4>(p, n_sms, st); return;
        }
    }
    switch (p.K) {
        case 1: launch_scan_k<1>(p, n_sms, st); break;
        case 2: launch_scan_k<2>(p, n_sms, st); break;
        case 3: launch_scan_k<3>(p, n_sms, st); break;
        case 4: launch_scan_k<4>(p, n_sms, st); break;
        case 5: launch_scan_k<5>(p, n_sms, st); break;
        case 6: launch_scan_k<6>(p, n_sms, st); break;
        case 7: launch_scan_k<7>(p, n_sms, st); break;
        default: launch_scan_k<8>(p, n_sms, st); break;
    }
}

// =================================================================================================================
// K_build
__global__ void __launch_bounds__(256) build_direct_kernel(const u32* __restrict__ keys, const u32* __restrict__ vals, u32 n,
                                                           u32* __restrict__ table, u32 kmin, u32 range, u32 cshift, u32* dup_flag) {
    const u32 stride = gridDim.x * blockDim.x;
    bool dup = false;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u32 off = compact_key(keys[i], cshift) - kmin;
        const u32 v = vals ? vals[i] : i;
        if (off < range) {
            const u32 old = atomicExch(&table[off], v);
            dup = dup || (old != EMPTY32);
        } else {
            dup = true;  // cannot happen when kmin/range come from the scan statistics; treated like a duplicate -> rebuild chained
        }
    }
    if (__any_sync(0xffffffffu, dup) && (threadIdx.x & 31) == 0) *dup_flag = 1u;
}
void launch_build_direct(const u32* keys, const u32* vals, u32 n, u32* table, u32 kmin, u32 range, u32 cshift, u32* dup_flag, int n_sms,
                         cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    build_direct_kernel<<<grid, 256, 0, st>>>(keys, vals, n, table, kmin, range, cshift, dup_flag);
}

__device__ __forceinline__ u32 key_tag(u32 n_keys, u32 k0, u32 k1, u32 k2, u32 k3) {
    if (n_keys == 1u) return k0;  // ids are never EMPTY32
    u32 h = mix32(k0) * 0x9E3779B1u ^ mix32(k1 + 0x7F4A7C15u);
    if (n_keys > 2u) h = mix32(h ^ k2) * 0x85EBCA77u;
    if (n_keys > 3u) h = mix32(h ^ k3) * 0xC2B2AE3Du;
    return h == EMPTY32 ? 0x7FFFFFFEu : h;
}

__global__ void __launch_bounds__(256) build_chained_kernel(const ChainTab T, u32 n) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 mask = T.n_slots - 1u;
    u32* words = reinterpret_cast<u32*>(T.slots);  // little-endian: word 2*slot = key tag, 2*slot+1 = head row
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u32 k0 = T.bkey[0][i];
        const u32 k1 = T.n_keys > 1u ? T.bkey[1][i] : 0u;
        const u32 k2 = T.n_keys > 2u ? T.bkey[2][i] : 0u;
        const u32 k3 = T.n_keys > 3u ? T.bkey[3][i] : 0u;
        const u32 tag = key_tag(T.n_keys, k0, k1, k2, k3);
        u32 slot = mix32(tag) & mask;
        for (;;) {
            u32 cur = *reinterpret_cast<volatile u32*>(&words[2u * slot]);
            if (cur == tag) break;
            if (cur == EMPTY32) {
                const u32 old = atomicCAS(&words[2u * slot], EMPTY32, tag);
                if (old == EMPTY32 || old == tag) break;
            }
            slot = (slot + 1u) & mask;
        }
        T.next[i] = atomicExch(&words[2u * slot + 1u], i);
    }
}
void launch_build_chained(const ChainTab& t, u32 n, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    build_chained_kernel<<<grid, 256, 0, st>>>(t, n);
}

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
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    if (trusted) build_direct_pairs_kernel<true><<<grid, 256, 0, st>>>(kv, key_is_y, n, table, kmin, range, cshift, dup_flag);
    else build_direct_pairs_kernel<false><<<grid, 256, 0, st>>>(kv, key_is_y, n, table, kmin, range, cshift, dup_flag);
}

// 4 rows per thread and iteration: the slice loads, the FILTER's numeric gathers and the table stores of the four rows are all
// independent, so each thread keeps 4 memory operations in flight at every stage (the 1-row version was latency-bound on
// two 16.7 M-row builds that move 0.5 GB).
template <bool TRUSTED>
__global__ void __launch_bounds__(256) build_pairs_filtered_kernel(const __grid_constant__ BuildPairsParams P) {
    constexpr int U = 4;
    const u32 stride = gridDim.x * blockDim.x;
    bool dup = false;
    u32 cnt = 0;
    const bool fast = P.n_ops == 1u && P.ops[0].op == KB_F_CMP_NUM;
    for (u32 i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < P.n; i0 += stride * U) {
        uint2 e[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const u32 i = i0 + (u32)u * stride;
            ok[u] = i < P.n;
            e[u] = ok[u] ? P.kv[i] : make_uint2(0u, 0u);
        }
        if (P.n_ops) {
            if (fast) {
                const u32 slot = P.ops[0].slot, cmp = P.ops[0].cmp;
                const double cv = P.ops[0].value;
                double a[U];
#pragma unroll
                for (int u = 0; u < U; u++) a[u] = ok[u] ? num_of(P.nt, slot == 0u ? e[u].x : (slot == 1u ? P.pred : e[u].y)) : 0.0;
#pragma unroll
                for (int u = 0; u < U; u++) ok[u] = ok[u] && cmp_num(cmp, a[u], cv);
            } else {
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (ok[u]) {
                        u32 vals[3] = {e[u].x, P.pred, e[u].y};
                        ok[u] = eval_filter(P.ops, P.n_ops, vals, P.nt);
                    }
                }
            }
        }
        u32 old[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            old[u] = EMPTY32;
            if (!ok[u]) continue;
            cnt++;
            const u32 off = compact_key(P.key_is_y ? e[u].y : e[u].x, P.cshift) - P.kmin;
            const u32 v = P.key_is_y ? e[u].x : e[u].y;
            if (off < P.range) {
                if (TRUSTED) P.table[off] = v;
                else old[u] = atomicExch(&P.table[off], v);
            } else dup = true;
        }
#pragma unroll
        for (int u = 0; u < U; u++) dup = dup || (old[u] != EMPTY32);
    }
    if (__any_sync(0xffffffffu, dup) && (threadIdx.x & 31) == 0) *P.dup_flag = 1u;
    cnt = warp_sum(cnt);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(P.count, cnt);
}
void launch_build_direct_pairs_filtered(const BuildPairsParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)p.n + 1023ull) / 1024ull);
    if (p.trusted) build_pairs_filtered_kernel<true><<<grid, 256, 0, st>>>(p);
    else build_pairs_filtered_kernel<false><<<grid, 256, 0, st>>>(p);
}

__global__ void __launch_bounds__(256) distinct_kernel(const u32* __restrict__ col, u32 n, u32* set, u32 set_slots, u32* overflow) {
    const int lane = threadIdx.x & 31;
    const u32 mask = set_slots - 1u;
    const u32 n_round = (n + 31u) & ~31u;
    u32 last = EMPTY32;  // values come in long runs in real stores: skip what this lane just inserted
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += gridDim.x * blockDim.x) {
        const bool valid = i < n;
        const u32 v = valid ? col[i] : EMPTY32;
        const unsigned act = __ballot_sync(0xffffffffu, valid && v != last);
        if (!(valid && v != last)) continue;
        const unsigned peers = __match_any_sync(act, v);
        last = v;
        if (lane != __ffs(peers) - 1) continue;
        u32 slot = mix32(v) & mask;
        for (u32 probes = 0;; probes++) {
            if (probes >= set_slots) { *overflow = 1u; break; }
            const u32 cur = *reinterpret_cast<volatile u32*>(&set[slot]);
            if (cur == v) break;
            if (cur == EMPTY32) {
                const u32 old = atomicCAS(&set[slot], EMPTY32, v);
                if (old == EMPTY32 || old == v) break;
            }
            slot = (slot + 1u) & mask;
        }
    }
}
void launch_distinct(const u32* col, u32 n, u32* set, u32 set_slots, u32* overflow, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
    distinct_kernel<<<grid, 256, 0, st>>>(col, n, set, set_slots, overflow);
}

// One pass over a new segment: id range of the three columns, subjects that belong to another shard, and the segment's distinct
// predicates with their row counts (32 open-addressing slots in the control words; a 33rd predicate raises the overflow word and the
// caller takes the batched scan path). Predicates come in short runs (one employee = six consecutive triples), so a warp holds a
// handful of distinct values: one probe sequence and one count atomic per (warp, value).
__global__ void __launch_bounds__(256) segment_profile_kernel(const u32* __restrict__ s, const u32* __restrict__ p, const u32* __restrict__ o, u32 n, u32 rank,
                                                              u32 world, u32* ctrl) {
    // per CTA: its own 32-slot table (value, rows) in shared memory, merged into the control words once at the end — the global table
    // sees one probe sequence and one add per (CTA, predicate) instead of one per (warp, predicate) and iteration
    __shared__ u32 s_key[SEGP_SLOTS], s_cnt[SEGP_SLOTS];
    __shared__ u32 s_over, s_foreign, s_mn[3], s_mx[3];
    const int lane = threadIdx.x & 31;
    if (threadIdx.x < SEGP_SLOTS) { s_key[threadIdx.x] = EMPTY32; s_cnt[threadIdx.x] = 0u; }
    if (threadIdx.x < 3) { s_mn[threadIdx.x] = EMPTY32; s_mx[threadIdx.x] = 0u; }
    if (threadIdx.x == 0) { s_over = 0u; s_foreign = 0u; }
    __syncthreads();
    u32 mn[3] = {EMPTY32, EMPTY32, EMPTY32}, mx[3] = {0u, 0u, 0u}, foreign = 0u;
    constexpr u32 U = 4;  // independent loads in flight per thread
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (n + 31u) & ~31u;
    for (u32 i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < n_round; i0 += stride * U) {
        u32 vs[U], vp[U], vo[U];
        bool valid[U];
#pragma unroll
        for (u32 u = 0; u < U; u++) {
            const u32 i = i0 + u * stride;
            valid[u] = i < n;
            vs[u] = valid[u] ? s[i] : 0u; vp[u] = valid[u] ? p[i] : 0u; vo[u] = valid[u] ? o[i] : 0u;
        }
#pragma unroll
        for (u32 u = 0; u < U; u++) {
            const unsigned act = __ballot_sync(0xffffffffu, valid[u]);  // (i0 + u * stride is warp-uniform in being below n_round or not)
            if (!valid[u]) continue;
            mn[0] = min(mn[0], vs[u]); mx[0] = max(mx[0], vs[u]);
            mn[1] = min(mn[1], vp[u]); mx[1] = max(mx[1], vp[u]);
            mn[2] = min(mn[2], vo[u]); mx[2] = max(mx[2], vo[u]);
            if (world > 1u) foreign += shard_of(vs[u], world) != rank;
            const unsigned peers = __match_any_sync(act, vp[u]);
            if (lane != __ffs(peers) - 1) continue;
            u32 slot = mix32(vp[u]) & (SEGP_SLOTS - 1u);
            for (u32 probes = 0;; probes++) {
                if (probes >= SEGP_SLOTS) { s_over = 1u; break; }
                u32 cur = *reinterpret_cast<volatile u32*>(&s_key[slot]);
                if (cur == EMPTY32) cur = atomicCAS(&s_key[slot], EMPTY32, vp[u]);
                if (cur == EMPTY32 || cur == vp[u]) { atomicAdd(&s_cnt[slot], (u32)__popc(peers)); break; }
                slot = (slot + 1u) & (SEGP_SLOTS - 1u);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
        mn[c] = __reduce_min_sync(0xffffffffu, mn[c]);
        mx[c] = __reduce_max_sync(0xffffffffu, mx[c]);
    }
    foreign = warp_sum(foreign);
    if (lane == 0) {  // CTA-level reduction in shared memory first: 6 global atomics per CTA, not per warp
#pragma unroll
        for (int c = 0; c < 3; c++) { atomicMin(&s_mn[c], mn[c]); atomicMax(&s_mx[c], mx[c]); }
        if (foreign) atomicAdd(&s_foreign, foreign);
    }
    __syncthreads();
    if (threadIdx.x < SEGP_SLOTS && s_key[threadIdx.x] != EMPTY32) {
        const u32 vp = s_key[threadIdx.x];
        u32 slot = mix32(vp) & (SEGP_SLOTS - 1u);
        for (u32 probes = 0;; probes++) {
            if (probes >= SEGP_SLOTS) { ctrl[SEGP_OVERFLOW] = 1u; break; }
            u32 cur = *reinterpret_cast<volatile u32*>(&ctrl[SEGP_SLOT + slot]);
            if (cur == EMPTY32) cur = atomicCAS(&ctrl[SEGP_SLOT + slot], EMPTY32, vp);
            if (cur == EMPTY32 || cur == vp) { atomicAdd(&ctrl[SEGP_COUNT + slot], s_cnt[threadIdx.x]); break; }
            slot = (slot + 1u) & (SEGP_SLOTS - 1u);
        }
    }
    if (threadIdx.x == 0 && s_over) ctrl[SEGP_OVERFLOW] = 1u;
    if (threadIdx.x < 3) { atomicMin(&ctrl[SEGP_MIN + threadIdx.x], s_mn[threadIdx.x]); atomicMax(&ctrl[SEGP_MAX + threadIdx.x], s_mx[threadIdx.x]); }
    if (threadIdx.x == 0 && s_foreign) atomicAdd(&ctrl[SEGP_FOREIGN], s_foreign);
}
void launch_segment_profile(const u32* s, const u32* p, const u32* o, u32 n, u32 rank, u32 world, u32* ctrl, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
    segment_profile_kernel<<<grid, 256, 0, st>>>(s, p, o, n, rank, world, ctrl);
}

// One pass over a new segment that files every triple under its predicate's slice: the (subject, object) pair goes to the slice's new
// chunk (one cursor reservation per warp and predicate), the object's f64 value to the chunk's typed column, both ids into the slice's
// persistent tables (atomicExch: a previous occupant = the column is not unique; a key outside the table = the table has to be
// rebuilt; both reported through control words), id ranges reduced per CTA in shared memory. Replaces, per slide, a scan + copy + range
// pass + two table builds + a typed column pass PER PREDICATE (~30 launches and 4 host round trips for six predicates).
constexpr u32 SPLIT_ITEMS = 4, SPLIT_TILE = 256 * SPLIT_ITEMS;
__global__ void __launch_bounds__(256) segment_split_kernel(const __grid_constant__ SplitParams P) {
    // Tile of 1024 triples per CTA and iteration. Positions: rank inside the tile from warp-aggregated SHARED atomics, then ONE global
    // cursor reservation per (tile, predicate) — with one global atomic per (warp, predicate) the six cursors of the employee shape
    // took 31 K same-address atomics each for 1 M triples.
    __shared__ u32 s_mm[MAXP][4];
    __shared__ u32 s_flag[MAXP][4];
    __shared__ u32 s_nnum[MAXP];
    __shared__ u32 s_cnt[MAXP], s_base[MAXP];
    const int lane = threadIdx.x & 31;
    if (threadIdx.x < MAXP) {
        s_mm[threadIdx.x][0] = EMPTY32; s_mm[threadIdx.x][1] = EMPTY32; s_mm[threadIdx.x][2] = 0u; s_mm[threadIdx.x][3] = 0u;
        s_flag[threadIdx.x][0] = 0u; s_flag[threadIdx.x][1] = 0u; s_flag[threadIdx.x][2] = 0u; s_flag[threadIdx.x][3] = 0u;
        s_nnum[threadIdx.x] = 0u;
        s_cnt[threadIdx.x] = 0u;
    }
    __syncthreads();
    const u32 n_tiles = (P.n + SPLIT_TILE - 1u) / SPLIT_TILE;
    for (u32 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const u32 row0 = tile * SPLIT_TILE;
        u32 vs[SPLIT_ITEMS], vo[SPLIT_ITEMS], which[SPLIT_ITEMS], rank[SPLIT_ITEMS];
#pragma unroll
        for (u32 j = 0; j < SPLIT_ITEMS; j++) {  // independent loads first
            const u32 i = row0 + j * 256u + threadIdx.x;
            u32 vp = EMPTY32;
            vs[j] = 0u; vo[j] = 0u;
            if (i < P.n) { vp = P.p[i]; vs[j] = P.s[i]; vo[j] = P.o[i]; }
            which[j] = EMPTY32;
#pragma unroll
            for (u32 e = 0; e < MAXP; e++) if (e < P.k && P.e[e].pred == vp && i < P.n) which[j] = e;
        }
#pragma unroll
        for (u32 j = 0; j < SPLIT_ITEMS; j++) {
            const unsigned act = __ballot_sync(0xffffffffu, which[j] != EMPTY32);
            rank[j] = 0u;
            if (which[j] == EMPTY32) continue;
            const u32 w = which[j];
            const unsigned peers = __match_any_sync(act, w);
            const int leader = __ffs(peers) - 1;
            u32 b = 0;
            const u32 xlo = __reduce_min_sync(peers, vs[j]), ylo = __reduce_min_sync(peers, vo[j]);
            const u32 xhi = __reduce_max_sync(peers, vs[j]), yhi = __reduce_max_sync(peers, vo[j]);
            const unsigned nm = __ballot_sync(peers, P.e[w].ynum != nullptr && isnum_of(P.nt, vo[j]));
            if (lane == leader) {
                b = atomicAdd(&s_cnt[w], (u32)__popc(peers));
                atomicMin(&s_mm[w][0], xlo); atomicMin(&s_mm[w][1], ylo); atomicMax(&s_mm[w][2], xhi); atomicMax(&s_mm[w][3], yhi);
                if (nm) atomicAdd(&s_nnum[w], (u32)__popc(nm));
            }
            b = __shfl_sync(peers, b, leader);
            rank[j] = b + (u32)__popc(peers & ((1u << lane) - 1u));
        }
        __syncthreads();
        if (threadIdx.x < P.k) {
            const u32 c = s_cnt[threadIdx.x];
            s_base[threadIdx.x] = c ? atomicAdd(&P.ctrl[threadIdx.x * SPLIT_WORDS + SPLIT_CURSOR], c) : 0u;
            s_cnt[threadIdx.x] = 0u;
        }
        __syncthreads();
#pragma unroll
        for (u32 j = 0; j < SPLIT_ITEMS; j++) {
            if (which[j] == EMPTY32) continue;
            const u32 w = which[j];
            const SplitEntry& E = P.e[w];
            const u32 pos = s_base[w] + rank[j];
            if (pos < E.n) {  // (always: the capacities are the profile pass's exact counts)
                E.pairs[pos] = make_uint2(vs[j], vo[j]);
                if (E.ynum) E.ynum[pos] = num_of(P.nt, vo[j]);
            }
            if (E.xtab) {
                const u32 off = compact_key(vs[j], E.cshift) - E.xtab_min;
                if (off < E.xtab_range) {
                    if (atomicExch(&E.xtab[off], vo[j]) != EMPTY32) s_flag[w][0] = 1u;
                    if (E.xnum) E.xnum[off] = num_of(P.nt, vo[j]);
                } else s_flag[w][2] = 1u;
            }
            if (E.ytab) {
                const u32 off = vo[j] - E.ytab_min;
                if (off < E.ytab_range) {
                    if (atomicExch(&E.ytab[off], vs[j]) != EMPTY32) s_flag[w][1] = 1u;
                } else s_flag[w][3] = 1u;
            }
        }
        // (s_base is rewritten only after the next tile's first barrier, which every thread reaches after these reads)
    }
    __syncthreads();
    if (threadIdx.x < P.k) {
        const u32 j = threadIdx.x;
        u32* c = P.ctrl + j * SPLIT_WORDS;
        if (s_mm[j][0] != EMPTY32 || s_mm[j][2] != 0u) {  // minima are kept complemented so that every control word starts at 0
            atomicMax(&c[SPLIT_XMIN], ~s_mm[j][0]); atomicMax(&c[SPLIT_YMIN], ~s_mm[j][1]);
            atomicMax(&c[SPLIT_XMAX], s_mm[j][2]); atomicMax(&c[SPLIT_YMAX], s_mm[j][3]);
        }
        if (s_nnum[j]) atomicAdd(&c[SPLIT_NNUM], s_nnum[j]);
        if (s_flag[j][0]) c[SPLIT_XDUP] = 1u;
        if (s_flag[j][1]) c[SPLIT_YDUP] = 1u;
        if (s_flag[j][2]) c[SPLIT_XOUT] = 1u;
        if (s_flag[j][3]) c[SPLIT_YOUT] = 1u;
    }
}
void launch_segment_split(const SplitParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0 || p.k == 0) return;
    const int grid = (int)umin64((u64)n_sms * 6ull, ((u64)p.n + SPLIT_TILE - 1ull) / SPLIT_TILE);
    segment_split_kernel<<<grid, 256, 0, st>>>(p);
}

// the keys of up to CLEAR_MAX evicted chunks leave their slices' persistent tables in one launch (blockIdx.y = chunk)
__global__ void __launch_bounds__(256) clear_chunks_kernel(const __grid_constant__ ClearParams P) {
    const ClearEntry& E = P.e[blockIdx.y];
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < E.n; i += stride) {
        const uint2 v = E.pairs[i];
        if (E.xtab) {
            const u32 off = compact_key(v.x, E.cshift) - E.xtab_min;
            if (off < E.xtab_range) E.xtab[off] = EMPTY32;
        }
        if (E.ytab) {
            const u32 off = v.y - E.ytab_min;
            if (off < E.ytab_range) E.ytab[off] = EMPTY32;
        }
    }
}
void launch_clear_chunks(const ClearParams& p, int n_sms, cudaStream_t st) {
    if (p.k == 0) return;
    u32 n_max = 0;
    for (u32 j = 0; j < p.k; j++) n_max = p.e[j].n > n_max ? p.e[j].n : n_max;
    if (n_max == 0) return;
    const u32 gx = (u32)umin64((u64)n_sms * 8ull / p.k + 1ull, ((u64)n_max + 255ull) / 256ull);
    clear_chunks_kernel<<<dim3(gx, p.k), 256, 0, st>>>(p);
}

__global__ void __launch_bounds__(256) pair_minmax_kernel(const uint2* __restrict__ kv, u32 n, u32* out4) {
    u32 mnx = EMPTY32, mny = EMPTY32, mxx = 0u, mxy = 0u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint2 e = kv[i];
        mnx = min(mnx, e.x); mxx = max(mxx, e.x);
        mny = min(mny, e.y); mxy = max(mxy, e.y);
    }
    mnx = __reduce_min_sync(0xffffffffu, mnx); mny = __reduce_min_sync(0xffffffffu, mny);
    mxx = __reduce_max_sync(0xffffffffu, mxx); mxy = __reduce_max_sync(0xffffffffu, mxy);
    if ((threadIdx.x & 31) == 0) { atomicMin(&out4[0], mnx); atomicMin(&out4[1], mny); atomicMax(&out4[2], mxx); atomicMax(&out4[3], mxy); }
}
__global__ void __launch_bounds__(256) pair_numcol_kernel(const uint2* __restrict__ kv, u32 n, NumTab nt, double* __restrict__ out, u32* n_numeric) {
    u32 c = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 id = kv[i].y;
        out[i] = num_of(nt, id);
        c += isnum_of(nt, id) ? 1u : 0u;
    }
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(n_numeric, c);
}
__global__ void __launch_bounds__(256) pair_numtab_kernel(const uint2* __restrict__ kv, u32 n, NumTab nt, double* __restrict__ out, u32 kmin, u32 range, u32 cshift) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint2 v = kv[i];
        const u32 off = compact_key(v.x, cshift) - kmin;
        if (off < range) out[off] = num_of(nt, v.y);
    }
}
void launch_pair_numtab(const uint2* kv, u32 n, NumTab nt, double* out, u32 kmin, u32 range, u32 cshift, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    pair_numtab_kernel<<<grid, 256, 0, st>>>(kv, n, nt, out, kmin, range, cshift);
}
void launch_pair_numcol(const uint2* kv, u32 n, NumTab nt, double* out, u32* n_numeric, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    pair_numcol_kernel<<<grid, 256, 0, st>>>(kv, n, nt, out, n_numeric);
}
void launch_pair_minmax(const uint2* kv, u32 n, u32* out4, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
    pair_minmax_kernel<<<grid, 256, 0, st>>>(kv, n, out4);
}

__global__ void unpair_kernel(const uint2* __restrict__ kv, u32 n, u32* __restrict__ x, u32* __restrict__ y) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint2 e = kv[i];
        x[i] = e.x;
        y[i] = e.y;
    }
}
void launch_unpair(const uint2* kv, u32 n, u32* x, u32* y, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64(H100_SMS * 8, ((u64)n + 255) / 256);
    unpair_kernel<<<grid, 256, 0, st>>>(kv, n, x, y);
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
__global__ void __launch_bounds__(256) count_nonempty_kernel(const uint4* __restrict__ t4, u32 n4, const u32* __restrict__ tail, u32 n_tail, u32* out) {
    u32 c = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
        const uint4 v = t4[i];
        c += (v.x != EMPTY32) + (v.y != EMPTY32) + (v.z != EMPTY32) + (v.w != EMPTY32);
    }
    if (blockIdx.x == 0 && threadIdx.x < n_tail) c += tail[threadIdx.x] != EMPTY32;
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
__global__ void __launch_bounds__(256) clear_direct_pairs_kernel(const uint2* __restrict__ kv, u32 key_is_y, u32 n, u32* __restrict__ table, u32 kmin, u32 range,
                                                                 u32 cshift) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint2 v = kv[i];
        const u32 off = compact_key(key_is_y ? v.y : v.x, cshift) - kmin;
        if (off < range) table[off] = EMPTY32;
    }
}
void launch_clear_direct_pairs(const uint2* kv, u32 key_is_y, u32 n, u32* table, u32 kmin, u32 range, u32 cshift, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    clear_direct_pairs_kernel<<<grid, 256, 0, st>>>(kv, key_is_y, n, table, kmin, range, cshift);
}
void launch_count_nonempty(const u32* table, u32 n, u32* out_count, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const u32 n4 = n / 4;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n4 + 255ull) / 256ull + 1ull);
    count_nonempty_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(table), n4, table + (u64)n4 * 4, n - n4 * 4, out_count);
}
__global__ void __launch_bounds__(256) count_foreign_kernel(const u32* __restrict__ col, u32 n, u32 rank, u32 world, u32* out) {
    u32 c = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) c += shard_of(col[i], world) != rank;
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
void launch_count_foreign(const u32* col, u32 n, u32 rank, u32 world, u32* out, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
    count_foreign_kernel<<<grid, 256, 0, st>>>(col, n, rank, world, out);
}
void launch_col_minmax(const u32* col, u32 n, u32* out_min, u32* out_max, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
    col_minmax_kernel<<<grid, 256, 0, st>>>(col, n, out_min, out_max);
}

// =================================================================================================================
// K_probe (direct, FAST)
template <int T>
__global__ void __launch_bounds__(PROBEF_THREADS, (PROBEF_ITEMS <= 4 ? 4 : 3)) probe_fast_kernel(const __grid_constant__ ProbeFParams P) {
    constexpr int R = PROBEF_ITEMS;  // rows per thread, consecutive
    extern __shared__ __align__(128) u32 smem_all[];  // two stages of PROBEF_TILE pairs (see probe_index_kernel)
    constexpr u32 STAGE_WORDS = 2u * PROBEF_TILE;
    __shared__ __align__(8) u64 bars[2];
    __shared__ u32 s_nexts[2];
    __shared__ u32 s_wcnt[PROBEF_THREADS / 32];
    __shared__ u32 s_excl1;
    if (P.abort_flag != nullptr) {
        for (int t = 0; t < T; t++) if (reinterpret_cast<const volatile u32*>(P.abort_flag)[t] != 0u) return;
    }
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    auto issue_next = [&](u32 stage) {
        const u32 t = atomicAdd(P.ticket, 1u);
        s_nexts[stage] = t;
        if (t < P.n_tiles) {
            const u32 b = t * (u32)PROBEF_TILE;
            const u32 c = min((u32)PROBEF_TILE, P.n - b);
            const u32 bytes = (c * 8u + 15u) & ~15u;
            mbar_arrive_expect_tx(&bars[stage], bytes);
            tma_load_1d(smem_all + stage * STAGE_WORDS, P.pairs + b, bytes, &bars[stage]);
        }
    };
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_mbar_init();
        issue_next(0);
        issue_next(1);
    }
    __syncthreads();
    u32 tile = s_nexts[0];
    u32 it = 0;
    while (tile < P.n_tiles) {
        const u32 stage = it & 1u;
        const u32* smem = smem_all + stage * STAGE_WORDS;
        const u32 base = tile * (u32)PROBEF_TILE;
        const u32 cnt = min((u32)PROBEF_TILE, P.n - base);
        mbar_wait(&bars[stage], (it >> 1) & 1u);
        // striped: row j of this thread is row (warp*32*R + j*32 + lane) of the tile — one warp instruction touches 32 consecutive rows, so
        // lookups by a sorted key hit 4 sectors instead of 16 and the compacted stores of one j form one contiguous run
        u32 rx[R], ry[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            const uint2 v = reinterpret_cast<const uint2*>(smem)[(u32)warp * (32u * R) + (u32)j * 32u + (u32)lane];
            rx[j] = v.x; ry[j] = v.y;
        }
        const u32 row0 = (u32)warp * (32u * R) + (u32)lane;  // row j = row0 + 32*j
        u32 vmask = 0;
#pragma unroll
        for (int j = 0; j < R; j++) vmask |= (row0 + 32u * (u32)j < cnt ? 1u : 0u) << j;
        // FILTER conjuncts over the probe row alone. The common shape FILTER(?x <cmp> c) needs one numeric gather per row: it is issued
        // together with the table lookups (independent loads, one memory round trip) and resolved afterwards — gating the lookups on
        // it would put two dependent round trips on the critical path of a latency-bound kernel.
        const bool pre_fast = P.n_pre == 1u && P.pre_ops[0].op == KB_F_CMP_NUM;
        double pa[R];
        if (pre_fast) {
            const u32 slot = P.pre_ops[0].slot;
#pragma unroll
            for (int j = 0; j < R; j++) {
                if (P.pre_num != nullptr && slot == 1u) pa[j] = ((vmask >> j) & 1u) ? __ldg(P.pre_num + base + row0 + 32u * (u32)j) : 0.0;
                else pa[j] = ((vmask >> j) & 1u) ? num_of(P.nt, slot == 0u ? rx[j] : ry[j]) : 0.0;
            }
        } else if (P.n_pre != 0u && vmask != 0u) {
#pragma unroll
            for (int j = 0; j < R; j++) {
                if ((vmask >> j) & 1u) {
                    u32 vals[2] = {rx[j], ry[j]};
                    if (!eval_filter(P.pre_ops, P.n_pre, vals, P.nt)) vmask &= ~(1u << j);
                }
            }
        }
        u32 tv[R][T > 0 ? T : 1];
#pragma unroll
        for (int j = 0; j < R; j++) {
            const u32 key = P.key_is_y ? ry[j] : rx[j];
#pragma unroll
            for (int t = 0; t < T; t++) {
                const u32 off = compact_key(key, P.tab[t].cshift) - P.tab[t].kmin;
                tv[j][t] = (((vmask >> j) & 1u) && off < P.tab[t].range) ? __ldg(P.tab[t].tab + off) : EMPTY32;
            }
        }
        if (pre_fast) {
            const u32 cmp = P.pre_ops[0].cmp;
            const double cv = P.pre_ops[0].value;
            u32 pass = 0;
#pragma unroll
            for (int j = 0; j < R; j++) pass |= (cmp_num(cmp, pa[j], cv) ? 1u : 0u) << j;
            vmask &= pass;
        }
        u32 m = 0;
#pragma unroll
        for (int j = 0; j < R; j++) {
            bool hit = (vmask >> j) & 1u;
#pragma unroll
            for (int t = 0; t < T; t++) hit = hit && (tv[j][t] != EMPTY32);
            m |= (hit ? 1u : 0u) << j;
        }
        if (P.n_ops != 0u && m != 0u) {
            if (P.n_ops == 1u && P.ops[0].op == KB_F_CMP_NUM) {
                const OutCol oc = P.oc[P.ops[0].slot];
                const u32 cmp = P.ops[0].cmp;
                const double cv = P.ops[0].value;
                double a[R];
#pragma unroll
                for (int j = 0; j < R; j++) {
                    u32 id = oc.kind == OUT_PROBE ? (oc.a == 0u ? rx[j] : ry[j]) : 0u;
#pragma unroll
                    for (int t = 0; t < T; t++) if (oc.kind == OUT_TABVAL && oc.a == (u32)t) id = tv[j][t];
                    a[j] = ((m >> j) & 1u) ? num_of(P.nt, id) : 0.0;
                }
                u32 pass = 0;
#pragma unroll
                for (int j = 0; j < R; j++) pass |= (cmp_num(cmp, a[j], cv) ? 1u : 0u) << j;
                m &= pass;
            } else {
#pragma unroll
                for (int j = 0; j < R; j++) {
                    if ((m >> j) & 1u) {
                        u32 vals[KB_MAX_COLS];
                        for (u32 c = 0; c < P.n_out; c++) {
                            const OutCol oc = P.oc[c];
                            u32 x = oc.kind == OUT_PROBE ? (oc.a == 0u ? rx[j] : ry[j]) : 0u;
#pragma unroll
                            for (int t = 0; t < T; t++) if (oc.kind == OUT_TABVAL && oc.a == (u32)t) x = tv[j][t];
                            vals[c] = x;
                        }
                        if (!eval_filter(P.ops, P.n_ops, vals, P.nt)) m &= ~(1u << j);
                    }
                }
            }
        }
        u32 bal[R];
        u32 wtot = 0;
#pragma unroll
        for (int j = 0; j < R; j++) {
            bal[j] = __ballot_sync(0xffffffffu, (m >> j) & 1u);
            wtot += (u32)__popc(bal[j]);
        }
        if (lane == 0) s_wcnt[warp] = wtot;
        __syncthreads();
        const u32 following = s_nexts[stage ^ 1u];
        if (tid == 32) issue_next(stage);  // every thread holds its rows in registers: refill this stage with the tile after next
        if (warp == 0) {
            const u32 wc = lane < PROBEF_THREADS / 32 ? s_wcnt[lane] : 0u;
            u32 wi = wc;
#pragma unroll
            for (int o = 1; o < PROBEF_THREADS / 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += y;
            }
            const u32 total = __shfl_sync(0xffffffffu, wi, PROBEF_THREADS / 32 - 1);
            if (lane < PROBEF_THREADS / 32) s_wcnt[lane] = wi - wc;
            const u32 ex = tile_prefix_2level(P.tile_state, P.block_state, tile, P.n_tiles, 0u, P.epoch, total, P.zero_word, P.total, P.ordered, lane);
            if (lane == 0) s_excl1 = ex;
        }
        __syncthreads();
        {
            const u32 lt = (1u << lane) - 1u;
            const u32 wbase = s_excl1 + s_wcnt[warp];
            for (u32 cidx = 0; cidx < P.n_out; cidx++) {
                const OutCol oc = P.oc[cidx];
                u32* out = P.out[cidx];
                u32 run = wbase;
#pragma unroll
                for (int j = 0; j < R; j++) {
                    u32 x = oc.kind == OUT_PROBE ? (oc.a == 0u ? rx[j] : ry[j]) : 0u;
#pragma unroll
                    for (int t = 0; t < T; t++) if (oc.kind == OUT_TABVAL && oc.a == (u32)t) x = tv[j][t];
                    const u32 pos = run + (u32)__popc(bal[j] & lt);
                    if (((m >> j) & 1u) && pos < P.cap) out[pos] = x;
                    run += (u32)__popc(bal[j]);
                }
            }
        }
        tile = following;
        it++;
    }
}

void launch_probe_fast(const ProbeFParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    const size_t smem = 2 * (size_t)PROBEF_TILE * sizeof(uint2);
    const void* fn = nullptr;
    switch (p.T) {
        case 1: fn = (const void*)probe_fast_kernel<1>; break;
        case 2: fn = (const void*)probe_fast_kernel<2>; break;
        case 3: fn = (const void*)probe_fast_kernel<3>; break;
        default: fn = (const void*)probe_fast_kernel<4>; break;
    }
    const int grid = grid_for(fn, PROBEF_THREADS, smem, n_sms, p.n_tiles);
    switch (p.T) {
        case 1: probe_fast_kernel<1><<<grid, PROBEF_THREADS, smem, st>>>(p); break;
        case 2: probe_fast_kernel<2><<<grid, PROBEF_THREADS, smem, st>>>(p); break;
        case 3: probe_fast_kernel<3><<<grid, PROBEF_THREADS, smem, st>>>(p); break;
        default: probe_fast_kernel<4><<<grid, PROBEF_THREADS, smem, st>>>(p); break;
    }
}

// =================================================================================================================
// K_probe (INDEX)
#ifndef KB_PI_MINB
#define KB_PI_MINB 4
#endif
// AGG = true: the joined rows are not written; GROUP BY one output column with at most one aggregate is folded in the kernel
// (execute_query.rs:1150-1227 over the rows of engine.rs:587-691): per warp __match_any_sync on the key, a 64-entry CTA table in shared
// memory, flushed to the global group table when the CTA is done. Only the row count and the groups leave the kernel.
constexpr int PI_GROUP_SMEM = 64;
__device__ void group_update_global(const GroupParams& P, const u32* k, unsigned long long cnt, const double* val);
__device__ void atomic_min_f64(double* addr, double v);
__device__ void atomic_max_f64(double* addr, double v);
// TAB = true: the probe stream is not the slice but the probe pattern's own persistent TABLE, walked slot by slot: slot i holds the
// other half of the triple whose key is (table base + i), EMPTY32 where no triple has that key. The keys then come in ascending order
// whatever the order of the store and of the dictionary ids, so the lookups into the other patterns' tables are sequential too — a
// direct table over dense ids IS the slice sorted by that column (with the gaps of the id space). With a FILTER on the other half's
// numeric value the typed column is read from a second table in the same order.
template <int T, int PRE, bool AGG, bool TAB>
__global__ void __launch_bounds__(PROBEF_THREADS, KB_PI_MINB) probe_index_kernel(const __grid_constant__ ProbeIParams P, const __grid_constant__ GroupParams G) {
    constexpr int R = 4;  // rows per thread (striped over the warp's 128-row chunk, see below)
    constexpr u32 TILE = PROBEF_THREADS * R;
    extern __shared__ __align__(128) u32 smem_all[];  // per stage: TILE pairs [+ TILE doubles]
    constexpr u32 STAGE_WORDS = TAB ? (PRE == 1 ? 3u : 1u) * TILE : (PRE == 1 ? 4u : 2u) * TILE;  // TAB: TILE values [+ TILE doubles]
    __shared__ __align__(8) u64 bars[2];
    __shared__ u32 s_nexts[2];
    __shared__ u32 s_wcnt[PROBEF_THREADS / 32];
    __shared__ u32 s_excl1;
    __shared__ u32 a_key[AGG ? PI_GROUP_SMEM : 1];
    __shared__ u32 a_cnt[AGG ? PI_GROUP_SMEM : 1];
    __shared__ double a_val[AGG ? PI_GROUP_SMEM : 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    u32 my_rows = 0;  // AGG: joined rows seen by this thread
    if (AGG) {
        for (int i = tid; i < PI_GROUP_SMEM; i += PROBEF_THREADS) {
            a_key[i] = EMPTY32;
            a_cnt[i] = 0u;
            a_val[i] = agg_identity(P.akind);
        }
    }
    __shared__ u32 s_tcnt[2];  // rows in the staged tile
    auto issue = [&](u32 t, u32 stage) {
        u32* smem = smem_all + stage * STAGE_WORDS;
        u64& bar = bars[stage];
        if constexpr (TAB) {
            const u32 b = t * TILE;
            const u32 c = min(TILE, P.ptab_range - b);
            const u32 bytes = (c * 4u + 15u) & ~15u;
            s_tcnt[stage] = c;
            mbar_arrive_expect_tx(&bar, PRE == 1 ? 3u * bytes : bytes);
            tma_load_1d(smem, P.ptab + b, bytes, &bar);
            if (PRE == 1) tma_load_1d(smem + TILE, P.pnum + b, 2u * bytes, &bar);
            return;
        }
        u32 g = 0;  // the chunk (store segment) this tile belongs to
        while (g + 1u < P.n_seg && t >= P.seg[g + 1u].tile0) g++;
        const ProbeISeg& sg = P.seg[g];
        const u32 b = (t - sg.tile0) * TILE;
        const u32 c = min(TILE, sg.n - b);
        const u32 bytes = (c * 8u + 15u) & ~15u;
        s_tcnt[stage] = c;
        mbar_arrive_expect_tx(&bar, PRE == 1 ? 2u * bytes : bytes);
        tma_load_1d(smem, sg.pairs + b, bytes, &bar);
        if (PRE == 1) tma_load_1d(smem + 2 * TILE, sg.ynum + b, bytes, &bar);
    };
    // two shared stages: tile i+1 is in flight while tile i is processed, and the stage of tile i is refilled (tile i+2) right after
    // the first compaction barrier — by then every thread has its rows in registers, so no barrier is spent on the hand-over
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        fence_mbar_init();
        for (u32 st = 0; st < 2; st++) {
            const u32 t0 = atomicAdd(&P.cb[0], 1u);
            s_nexts[st] = t0;
            if (t0 < P.n_tiles) issue(t0, st);
        }
    }
    __syncthreads();
    u32 tile = s_nexts[0];
    u32 it = 0;
    while (tile < P.n_tiles) {
        const u32 stage = it & 1u;
        const u32* smem = smem_all + stage * STAGE_WORDS;
        mbar_wait(&bars[stage], (it >> 1) & 1u);
        const u32 cnt = s_tcnt[stage];
        u32 rx[R], ry[R];
        double pa[R];
        // striped: row j of this thread is row (warp*128 + j*32 + lane) of the tile, so one warp instruction touches 32 CONSECUTIVE
        // rows: lookups into a table indexed by a sorted key hit 4 sectors instead of 16, and the compacted stores of one j are
        // one contiguous run
        u32 vmask = 0;
        if constexpr (TAB) {
#pragma unroll
            for (int j = 0; j < R; j++) {
                const u32 idx = (u32)warp * (32u * R) + (u32)j * 32u + (u32)lane;
                const u32 v = smem[idx];
                // the key of slot (tile base + idx): the inverse of compact_key for this shard's keys
                const u32 ck = P.ptab_min + tile * TILE + idx;
                const u32 key = P.ptab_cshift ? (((((ck >> SHARD_B) << P.ptab_cshift) | P.shard_rank) << SHARD_B) | (ck & ((1u << SHARD_B) - 1u))) : ck;
                rx[j] = P.key_is_y ? v : key;
                ry[j] = P.key_is_y ? key : v;
                if (PRE == 1) pa[j] = reinterpret_cast<const double*>(smem + TILE)[idx];
                vmask |= ((idx < cnt && v != EMPTY32) ? 1u : 0u) << j;
            }
        } else {
#pragma unroll
            for (int j = 0; j < R; j++) {
                const u32 idx = (u32)warp * (32u * R) + (u32)j * 32u + (u32)lane;
                const uint2 v = reinterpret_cast<const uint2*>(smem)[idx];
                rx[j] = v.x; ry[j] = v.y;
                if (PRE == 1) pa[j] = reinterpret_cast<const double*>(smem + 2 * TILE)[idx];
            }
#pragma unroll
            for (int j = 0; j < R; j++) vmask |= (((u32)warp * (32u * R) + (u32)j * 32u + (u32)lane) < cnt ? 1u : 0u) << j;
        }
        if (PRE == 1) {
            u32 pass = 0;
#pragma unroll
            for (int j = 0; j < R; j++) pass |= (cmp_num(P.pre_cmp, pa[j], P.pre_val) ? 1u : 0u) << j;
            vmask &= pass;
        } else if (P.pre_mode == 2u && vmask != 0u) {
#pragma unroll
            for (int j = 0; j < R; j++) {
                if ((vmask >> j) & 1u) {
                    u32 vals[2] = {rx[j], ry[j]};
                    if (!eval_filter(P.pre_ops, P.n_pre, vals, P.nt)) vmask &= ~(1u << j);
                }
            }
        }
        u32 tv[R][T];
#pragma unroll
        for (int j = 0; j < R; j++) {
            const u32 key = P.key_is_y ? ry[j] : rx[j];
#pragma unroll
            for (int t = 0; t < T; t++) {
                const u32 off = compact_key(key, P.tab[t].cshift) - P.tab[t].kmin;
                tv[j][t] = (((vmask >> j) & 1u) && off < P.tab[t].range) ? __ldg(P.tab[t].tab + off) : EMPTY32;
            }
        }
        u32 m = 0;
#pragma unroll
        for (int j = 0; j < R; j++) {
            bool hit = (vmask >> j) & 1u;
#pragma unroll
            for (int t = 0; t < T; t++) hit = hit && (tv[j][t] != EMPTY32);
            m |= (hit ? 1u : 0u) << j;
        }
        if (P.n_ops != 0u && m != 0u) {
#pragma unroll
            for (int j = 0; j < R; j++) {
                if ((m >> j) & 1u) {
                    u32 vals[KB_MAX_COLS];
                    vals[0] = rx[j]; vals[1] = ry[j];
#pragma unroll
                    for (int t = 0; t < T; t++) vals[2 + t] = tv[j][t];
                    if (!eval_filter(P.ops, P.n_ops, vals, P.nt)) m &= ~(1u << j);
                }
            }
        }
        if constexpr (AGG) {
            __syncthreads();  // every thread holds its rows in registers: the stage can take the tile after next
            const u32 following_a = s_nexts[stage ^ 1u];
            if (tid == 32) {
                const u32 nt = atomicAdd(&P.cb[0], 1u);
                s_nexts[stage] = nt;
                if (nt < P.n_tiles) issue(nt, stage);
            }
            my_rows += (u32)__popc(m);
#pragma unroll
            for (int j = 0; j < R; j++) {
                const bool on = (m >> j) & 1u;
                const unsigned act = __ballot_sync(0xffffffffu, on);
                if (act == 0u || !on) continue;
                u32 key = P.gsel == 0u ? rx[j] : ry[j];
                u32 vid = P.asel == 0u ? rx[j] : ry[j];
#pragma unroll
                for (int t = 0; t < T; t++) {
                    if (P.gsel == 2u + (u32)t) key = tv[j][t];
                    if (P.asel == 2u + (u32)t) vid = tv[j][t];
                }
                const unsigned peers = __match_any_sync(act, key);
                const int leader = __ffs(peers) - 1;
                double acc = 0.0;
                if (P.akind != KB_AGG_COUNT) {
                    const double mine = num_of(P.nt, vid);
                    acc = mine;
                    unsigned rest = peers & ~(1u << leader);
                    while (rest) {  // every lane of the group runs the same shuffles
                        const int src = __ffs(rest) - 1;
                        rest &= rest - 1u;
                        const double o = __shfl_sync(peers, mine, src);
                        if (P.akind == KB_AGG_MIN) acc = fmin(acc, o);
                        else if (P.akind == KB_AGG_MAX) acc = fmax(acc, o);
                        else acc += o;
                    }
                }
                if (lane != leader) continue;
                const u32 cnt_g = (u32)__popc(peers);
                u32 slot = mix32(key) & (PI_GROUP_SMEM - 1);
                bool done = false;
                for (int probes = 0; probes < PI_GROUP_SMEM && !done && key != EMPTY32; probes++) {  // EMPTY32 marks a free entry
                    u32 cur = *reinterpret_cast<volatile u32*>(&a_key[slot]);
                    if (cur == EMPTY32) cur = atomicCAS(&a_key[slot], EMPTY32, key);
                    if (cur == EMPTY32 || cur == key) {
                        atomicAdd(&a_cnt[slot], cnt_g);
                        if (P.akind == KB_AGG_MIN) atomic_min_f64(&a_val[slot], acc);
                        else if (P.akind == KB_AGG_MAX) atomic_max_f64(&a_val[slot], acc);
                        else if (P.akind != KB_AGG_COUNT) atomicAdd(&a_val[slot], acc);
                        done = true;
                    } else slot = (slot + 1u) & (PI_GROUP_SMEM - 1);
                }
                if (!done) {  // more than 64 distinct groups in this CTA
                    u32 kk[4] = {key, 0u, 0u, 0u};
                    double vv[8] = {acc, 0, 0, 0, 0, 0, 0, 0};
                    group_update_global(G, kk, (unsigned long long)cnt_g, vv);
                }
            }
            tile = following_a;
            it++;
            continue;
        }
        u32 bal[R];
        u32 wtot = 0;
#pragma unroll
        for (int j = 0; j < R; j++) {
            bal[j] = __ballot_sync(0xffffffffu, (m >> j) & 1u);
            wtot += (u32)__popc(bal[j]);
        }
        if (lane == 0) s_wcnt[warp] = wtot;
        __syncthreads();
        const u32 following = s_nexts[stage ^ 1u];  // tile of the next iteration (its copy is in flight)
        if (tid == 32) {  // a lane outside the prefix warp refills this stage with the tile after that one
            const u32 nt = atomicAdd(&P.cb[0], 1u);
            s_nexts[stage] = nt;
            if (nt < P.n_tiles) issue(nt, stage);
        }
        if (warp == 0) {
            const u32 wc = lane < PROBEF_THREADS / 32 ? s_wcnt[lane] : 0u;
            u32 wi = wc;
#pragma unroll
            for (int o = 1; o < PROBEF_THREADS / 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += y;
            }
            const u32 total = __shfl_sync(0xffffffffu, wi, PROBEF_THREADS / 32 - 1);
            if (lane < PROBEF_THREADS / 32) s_wcnt[lane] = wi - wc;
            const u32 ex = tile_prefix_2level(P.tile_state, P.block_state, tile, P.n_tiles, 0u, P.epoch, total, P.cb + 2, P.cb + 1, P.ordered, lane);
            if (lane == 0) s_excl1 = ex;
        }
        __syncthreads();
        {
            u32 run = s_excl1 + s_wcnt[warp];
            const u32 lt = (1u << lane) - 1u;
#pragma unroll
            for (int j = 0; j < R; j++) {
                const u32 pos = run + (u32)__popc(bal[j] & lt);
                if (((m >> j) & 1u) && pos < P.cap) {
                    P.out[0][pos] = rx[j];
                    P.out[1][pos] = ry[j];
#pragma unroll
                    for (int t = 0; t < T; t++) P.out[2 + t][pos] = tv[j][t];
                }
                run += (u32)__popc(bal[j]);
            }
        }
        tile = following;
        it++;
    }
    if constexpr (AGG) {
        __syncthreads();
        for (int i = tid; i < PI_GROUP_SMEM; i += PROBEF_THREADS) {
            if (a_key[i] == EMPTY32) continue;
            u32 kk[4] = {a_key[i], 0u, 0u, 0u};
            double vv[8] = {a_val[i], 0, 0, 0, 0, 0, 0, 0};
            group_update_global(G, kk, (unsigned long long)a_cnt[i], vv);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) my_rows += __shfl_xor_sync(0xffffffffu, my_rows, o);
        if (lane == 0 && my_rows) atomicAdd(&P.cb[1], my_rows);
    }
    // the last CTA to get here publishes the row count and leaves the control block zeroed for the next launch
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        const u32 prev = atomicAdd(&P.cb[3], 1u);
        if (prev == gridDim.x - 1u) {
            __threadfence();
            const u32 total = atomicExch(&P.cb[1], 0u);
            *reinterpret_cast<volatile u32*>(P.host_total) = total;
            P.cb[0] = 0u;
            P.cb[3] = 0u;
            __threadfence_system();
        }
    }
}

template <int T, int PRE, bool AGG, bool TAB>
static void launch_probe_index_tp(const ProbeIParams& p, const GroupParams& g, int n_sms, cudaStream_t st) {
    static int per_sm = 0;  // occupancy is a property of the kernel image: asked once per instantiation
    const size_t smem = TAB ? (size_t)PROBEF_THREADS * 4 * (PRE == 1 ? 12 : 4) * 2 : (size_t)PROBEF_THREADS * 4 * (PRE == 1 ? 16 : 8) * 2;
    if (per_sm == 0) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, probe_index_kernel<T, PRE, AGG, TAB>, PROBEF_THREADS, smem);
        if (per_sm < 1) per_sm = 1;
    }
    long long grid = (long long)per_sm * n_sms;
    if (grid > (long long)p.n_tiles) grid = p.n_tiles;
    probe_index_kernel<T, PRE, AGG, TAB><<<(int)grid, PROBEF_THREADS, smem, st>>>(p, g);
}
template <int T, bool TAB>
static void launch_probe_index_t(const ProbeIParams& p, const GroupParams* g, int n_sms, cudaStream_t st) {
    static const GroupParams none{};
    if (g) {
        if (p.pre_mode == 1u) launch_probe_index_tp<T, 1, true, TAB>(p, *g, n_sms, st);
        else launch_probe_index_tp<T, 0, true, TAB>(p, *g, n_sms, st);
    } else {
        if (p.pre_mode == 1u) launch_probe_index_tp<T, 1, false, TAB>(p, none, n_sms, st);
        else launch_probe_index_tp<T, 0, false, TAB>(p, none, n_sms, st);
    }
}
void launch_probe_index(const ProbeIParams& p, const GroupParams* agg, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    if (p.ptab) {
        switch (p.T) {
            case 1: launch_probe_index_t<1, true>(p, agg, n_sms, st); break;
            case 2: launch_probe_index_t<2, true>(p, agg, n_sms, st); break;
            case 3: launch_probe_index_t<3, true>(p, agg, n_sms, st); break;
            default: launch_probe_index_t<4, true>(p, agg, n_sms, st); break;
        }
        return;
    }
    switch (p.T) {
        case 1: launch_probe_index_t<1, false>(p, agg, n_sms, st); break;
        case 2: launch_probe_index_t<2, false>(p, agg, n_sms, st); break;
        case 3: launch_probe_index_t<3, false>(p, agg, n_sms, st); break;
        default: launch_probe_index_t<4, false>(p, agg, n_sms, st); break;
    }
}

// =================================================================================================================
// K_probe (direct, fused multiway)
template <int T>
__global__ void __launch_bounds__(PROBE_THREADS) probe_direct_kernel(const __grid_constant__ ProbeDParams P) {
    extern __shared__ __align__(128) u32 smem[];  // n_pcols tiles of PROBE_TILE
    __shared__ __align__(8) u64 bar;
    __shared__ u32 s_tile;
    __shared__ u32 s_wcnt[PROBE_THREADS / 32];
    __shared__ u32 s_cnt[MAXP], s_excl[MAXP];
    if (P.abort_flag != nullptr) {  // a direct build met duplicate keys: the host will redo this join with the chained operator
        for (int t = 0; t < T; t++) if (reinterpret_cast<const volatile u32*>(P.abort_flag)[t] != 0u) return;
    }

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    u32 parity = 0;
    const unsigned lt_mask = (1u << lane) - 1u;
    const u32* sKey = smem + P.key_col * PROBE_TILE;

    for (;;) {
        if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= P.n_tiles) break;
        const u32 base = tile * (u32)PROBE_TILE;
        const u32 cnt = min((u32)PROBE_TILE, P.n - base);
        if (tid == 0) {
            const u32 bytes = (cnt * 4u + 15u) & ~15u;
            mbar_arrive_expect_tx(&bar, bytes * P.n_pcols);
            for (u32 c = 0; c < P.n_pcols; c++) tma_load_1d(smem + c * PROBE_TILE, P.pcol[c] + base, bytes, &bar);
        }
        mbar_wait(&bar, parity);
        parity ^= 1u;

        // all table loads of this thread's rows are issued before any is consumed (ITEMS*T independent loads in flight)
        u32 v[PROBE_ITEMS][T > 0 ? T : 1];
#pragma unroll
        for (int j = 0; j < PROBE_ITEMS; j++) {
            const u32 idx = (u32)warp * (32u * PROBE_ITEMS) + (u32)j * 32u + (u32)lane;
            const bool valid = idx < cnt;
            const u32 key = sKey[idx];
#pragma unroll
            for (int t = 0; t < T; t++) {
                const u32 off = compact_key(key, P.tab[t].cshift) - P.tab[t].kmin;
                v[j][t] = (valid && off < P.tab[t].range) ? __ldg(P.tab[t].tab + off) : EMPTY32;
            }
            if (T == 0) v[j][0] = valid ? 0u : EMPTY32;
        }
        u32 mbits = 0;
#pragma unroll
        for (int j = 0; j < PROBE_ITEMS; j++) {
            const u32 idx = (u32)warp * (32u * PROBE_ITEMS) + (u32)j * 32u + (u32)lane;
            bool hit = true;
#pragma unroll
            for (int t = 0; t < (T > 0 ? T : 1); t++) hit = hit && (v[j][t] != EMPTY32);
            if (hit && P.n_ops != 0u) {
                u32 vals[KB_MAX_COLS];
                for (u32 c = 0; c < P.n_out; c++) {
                    const OutCol oc = P.oc[c];
                    u32 x;
                    if (oc.kind == OUT_PROBE) x = smem[oc.a * PROBE_TILE + idx];
                    else {
                        u32 tv = 0;
#pragma unroll
                        for (int t = 0; t < T; t++) if ((u32)t == oc.a) tv = v[j][t];
                        x = oc.kind == OUT_TABVAL ? tv : __ldg(P.tab[oc.a].pay[oc.b] + tv);
                    }
                    vals[c] = x;
                }
                hit = eval_filter(P.ops, P.n_ops, vals, P.nt);
            }
            mbits |= (hit ? 1u : 0u) << j;
        }
        {
            const u32 c = warp_sum((u32)__popc(mbits));
            if (lane == 0) s_wcnt[warp] = c;
        }
        __syncthreads();
        if (warp == 0) {
            if (lane == 0) {
                u32 run = 0;
#pragma unroll
                for (int w = 0; w < PROBE_THREADS / 32; w++) {
                    const u32 c = s_wcnt[w];
                    s_wcnt[w] = run;
                    run += c;
                }
                s_cnt[0] = run;
            }
            __syncwarp();
            const u32 total = __shfl_sync(0xffffffffu, s_cnt[0], 0);
            const u32 ex = tile_prefix_2level(P.tile_state, P.block_state, tile, P.n_tiles, 0u, P.epoch, total, P.zero_word, P.total, P.ordered, lane);
            if (lane == 0) {
                s_excl[0] = ex;
            }
        }
        __syncthreads();
        if (__ballot_sync(0xffffffffu, mbits != 0u) != 0u) {
            u32 pos = s_excl[0] + s_wcnt[warp];
#pragma unroll
            for (int j = 0; j < PROBE_ITEMS; j++) {
                const bool m = (mbits >> j) & 1u;
                const unsigned b = __ballot_sync(0xffffffffu, m);
                if (b == 0u) continue;
                const u32 r = pos + (u32)__popc(b & lt_mask);
                if (m && r < P.cap) {
                    const u32 idx = (u32)warp * (32u * PROBE_ITEMS) + (u32)j * 32u + (u32)lane;
                    for (u32 c = 0; c < P.n_out; c++) {
                        const OutCol oc = P.oc[c];
                        u32 x;
                        if (oc.kind == OUT_PROBE) x = smem[oc.a * PROBE_TILE + idx];
                        else {
                            u32 tv = 0;
#pragma unroll
                            for (int t = 0; t < T; t++) if ((u32)t == oc.a) tv = v[j][t];
                            x = oc.kind == OUT_TABVAL ? tv : __ldg(P.tab[oc.a].pay[oc.b] + tv);
                        }
                        P.out[c][r] = x;
                    }
                }
                pos += (u32)__popc(b);
            }
        }
    }
}

void launch_probe_direct(const ProbeDParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    const size_t smem = (size_t)p.n_pcols * PROBE_TILE * sizeof(u32);
    const void* fn = nullptr;
    switch (p.T) {
        case 0: fn = (const void*)probe_direct_kernel<0>; break;
        case 1: fn = (const void*)probe_direct_kernel<1>; break;
        case 2: fn = (const void*)probe_direct_kernel<2>; break;
        case 3: fn = (const void*)probe_direct_kernel<3>; break;
        default: fn = (const void*)probe_direct_kernel<4>; break;
    }
    if (smem > 48 * 1024) cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int grid = grid_for(fn, PROBE_THREADS, smem, n_sms, p.n_tiles);
    switch (p.T) {
        case 0: probe_direct_kernel<0><<<grid, PROBE_THREADS, smem, st>>>(p); break;
        case 1: probe_direct_kernel<1><<<grid, PROBE_THREADS, smem, st>>>(p); break;
        case 2: probe_direct_kernel<2><<<grid, PROBE_THREADS, smem, st>>>(p); break;
        case 3: probe_direct_kernel<3><<<grid, PROBE_THREADS, smem, st>>>(p); break;
        default: probe_direct_kernel<4><<<grid, PROBE_THREADS, smem, st>>>(p); break;
    }
}

// =================================================================================================================
// K_probe (chained, binary, 1:N)
__device__ __forceinline__ u32 warp_excl_scan(u32 v, int lane, u32* total) {
    u32 x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u32 y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    *total = __shfl_sync(0xffffffffu, x, 31);
    return x - v;
}

// Walks the chain of probe row `idx` (tile-local) and calls emit(build_row) for every build row whose key columns equal the
// probe row's and whose joined row passes the FILTER.
template <class Emit>
__device__ __forceinline__ void chain_walk(const ProbeCParams& P, const u32* smem, u32 idx, Emit&& emit) {
    const ChainTab& T = P.tab;
    u32 pk[4];
#pragma unroll
    for (int q = 0; q < 4; q++) pk[q] = (u32)q < T.n_keys ? smem[P.pkey[q] * PROBEC_TILE + idx] : 0u;
    const u32 tag = key_tag(T.n_keys, pk[0], pk[1], pk[2], pk[3]);
    const u32 mask = T.n_slots - 1u;
    u32 slot = mix32(tag) & mask;
    u32 head = EMPTY32;
    for (;;) {
        const u64 w = __ldg(reinterpret_cast<const unsigned long long*>(T.slots) + slot);
        const u32 key = (u32)w;
        if (key == tag) { head = (u32)(w >> 32); break; }
        if (key == EMPTY32) break;
        slot = (slot + 1u) & mask;
    }
    for (u32 r = head; r != EMPTY32; r = __ldg(T.next + r)) {
        bool ok = true;
        if (T.n_keys > 1u) {
#pragma unroll
            for (int q = 0; q < 4; q++) if ((u32)q < T.n_keys) ok = ok && (__ldg(T.bkey[q] + r) == pk[q]);
        }
        if (ok && P.n_ops != 0u) {
            u32 vals[KB_MAX_COLS];
            for (u32 c = 0; c < P.n_pcols; c++) vals[c] = smem[c * PROBEC_TILE + idx];
            for (u32 c = 0; c < P.n_bpay; c++) vals[P.n_pcols + c] = __ldg(P.bpay[c] + r);
            ok = eval_filter(P.ops, P.n_ops, vals, P.nt);
        }
        if (ok) emit(r);
    }
}

__global__ void __launch_bounds__(PROBEC_THREADS) probe_chained_kernel(const __grid_constant__ ProbeCParams P) {
    extern __shared__ __align__(128) u32 smem[];
    __shared__ __align__(8) u64 bar;
    __shared__ u32 s_tile;
    __shared__ u32 s_wcnt[PROBEC_THREADS / 32];
    __shared__ u32 s_cnt[MAXP], s_excl[MAXP];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    u32 parity = 0;
    for (;;) {
        if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= P.n_tiles) break;
        const u32 base = tile * (u32)PROBEC_TILE;
        const u32 cnt = min((u32)PROBEC_TILE, P.n - base);
        if (tid == 0) {
            const u32 bytes = (cnt * 4u + 15u) & ~15u;
            mbar_arrive_expect_tx(&bar, bytes * P.n_pcols);
            for (u32 c = 0; c < P.n_pcols; c++) tma_load_1d(smem + c * PROBEC_TILE, P.pcol[c] + base, bytes, &bar);
        }
        mbar_wait(&bar, parity);
        parity ^= 1u;

        u32 mc[PROBEC_ITEMS];
        u32 tsum = 0;
#pragma unroll
        for (int j = 0; j < PROBEC_ITEMS; j++) {
            const u32 idx = (u32)warp * (32u * PROBEC_ITEMS) + (u32)j * 32u + (u32)lane;
            u32 c = 0;
            if (idx < cnt) chain_walk(P, smem, idx, [&](u32) { c++; });
            mc[j] = c;
            tsum += c;
        }
        {
            const u32 c = warp_sum(tsum);
            if (lane == 0) s_wcnt[warp] = c;
        }
        __syncthreads();
        if (warp == 0) {
            if (lane == 0) {
                u32 run = 0;
#pragma unroll
                for (int w = 0; w < PROBEC_THREADS / 32; w++) {
                    const u32 c = s_wcnt[w];
                    s_wcnt[w] = run;
                    run += c;
                }
                s_cnt[0] = run;
            }
            __syncwarp();
            const u32 total = __shfl_sync(0xffffffffu, s_cnt[0], 0);
            const u32 ex = tile_prefix_2level(P.tile_state, P.block_state, tile, P.n_tiles, 0u, P.epoch, total, P.zero_word, P.total, P.ordered, lane);
            if (lane == 0) {
                s_excl[0] = ex;
                if (total) atomicAdd(P.total64, (unsigned long long)total);
            }
        }
        __syncthreads();
        u32 pos = s_excl[0] + s_wcnt[warp];
#pragma unroll
        for (int j = 0; j < PROBEC_ITEMS; j++) {
            u32 tot;
            const u32 ex = warp_excl_scan(mc[j], lane, &tot);
            if (mc[j] != 0u) {
                const u32 idx = (u32)warp * (32u * PROBEC_ITEMS) + (u32)j * 32u + (u32)lane;
                u32 r = pos + ex;
                chain_walk(P, smem, idx, [&](u32 br) {
                    if (r < P.cap) {
                        for (u32 c = 0; c < P.n_pcols; c++) P.out[c][r] = smem[c * PROBEC_TILE + idx];
                        for (u32 c = 0; c < P.n_bpay; c++) P.out[P.n_pcols + c][r] = __ldg(P.bpay[c] + br);
                    }
                    r++;
                });
            }
            pos += tot;
        }
    }
}

void launch_probe_chained(const ProbeCParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    const size_t smem = (size_t)p.n_pcols * PROBEC_TILE * sizeof(u32);
    const int grid = grid_for((const void*)probe_chained_kernel, PROBEC_THREADS, smem, n_sms, p.n_tiles);
    probe_chained_kernel<<<grid, PROBEC_THREADS, smem, st>>>(p);
}

// =================================================================================================================
// K_build / K_probe (grouped by key, CSR directory)
// Directory builds (count, then fill) go tile by tile through a shared-memory hash of the tile's keys: the rows of a tile that carry the
// same key are counted / ranked with SHARED atomics and the global counter of a key is touched once per (tile, key). A Datalog
// closure's subClassOf facts name the root class a million times, in no particular order: one global atomic per row (and per warp-level
// group of equal keys, which random order leaves at size one) made the 2 M-row build of the transitive rule's join take
// longer than the 331 M-row join next to it.
constexpr u32 CSR_ITEMS = 8, CSR_TILE = 256 * CSR_ITEMS, CSR_HASH = 4096;
struct CsrTileHash {
    u32 key[CSR_HASH], cnt[CSR_HASH], base[CSR_HASH];
};
// slot of k in the tile's table (claimed when absent); the table is at most half full (2048 rows, 4096 slots)
__device__ __forceinline__ u32 csr_slot(CsrTileHash& H, u32 k) {
    u32 slot = mix32(k) & (CSR_HASH - 1u);
    for (;;) {
        u32 cur = *reinterpret_cast<volatile u32*>(&H.key[slot]);
        if (cur == EMPTY32) cur = atomicCAS(&H.key[slot], EMPTY32, k);
        if (cur == EMPTY32 || cur == k) return slot;
        slot = (slot + 1u) & (CSR_HASH - 1u);
    }
}
__global__ void __launch_bounds__(256) csr_count_kernel(const u32* __restrict__ keys, u32 n, u32 kmin, u32* __restrict__ counts) {
    __shared__ CsrTileHash H;
    for (u32 i = threadIdx.x; i < CSR_HASH; i += 256u) { H.key[i] = EMPTY32; H.cnt[i] = 0u; }
    __syncthreads();
    const u32 n_tiles = (n + CSR_TILE - 1u) / CSR_TILE;
    for (u32 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const u32 row0 = tile * CSR_TILE;
        u32 k[CSR_ITEMS], slot[CSR_ITEMS];
        bool lead[CSR_ITEMS];
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) {
            const u32 i = row0 + j * 256u + threadIdx.x;
            k[j] = i < n ? keys[i] - kmin : EMPTY32;
        }
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) {
            lead[j] = false;
            if (k[j] == EMPTY32) continue;
            slot[j] = csr_slot(H, k[j]);
            lead[j] = atomicAdd(&H.cnt[slot[j]], 1u) == 0u;  // the first row of the key in this tile speaks for it
        }
        __syncthreads();
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) if (lead[j]) atomicAdd(&counts[k[j]], H.cnt[slot[j]]);
        __syncthreads();
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) if (lead[j]) { H.key[slot[j]] = EMPTY32; H.cnt[slot[j]] = 0u; }
        __syncthreads();
    }
}
void launch_csr_count(const u32* keys, u32 n, u32 kmin, u32* counts, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + CSR_TILE - 1ull) / CSR_TILE);
    csr_count_kernel<<<grid, 256, 0, st>>>(keys, n, kmin, counts);
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

struct CsrFillParams {
    const u32* keys;
    u32 n, kmin, n_pay;
    u32* cursor;
    const u32* pay_in[KB_MAX_COLS];
    u32* pay_out[KB_MAX_COLS];
};
__global__ void __launch_bounds__(256) csr_fill_kernel(const __grid_constant__ CsrFillParams P) {
    __shared__ CsrTileHash H;
    for (u32 i = threadIdx.x; i < CSR_HASH; i += 256u) { H.key[i] = EMPTY32; H.cnt[i] = 0u; }
    __syncthreads();
    const u32 n_tiles = (P.n + CSR_TILE - 1u) / CSR_TILE;
    for (u32 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const u32 row0 = tile * CSR_TILE;
        u32 k[CSR_ITEMS], slot[CSR_ITEMS], rank[CSR_ITEMS];
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) {
            const u32 i = row0 + j * 256u + threadIdx.x;
            k[j] = i < P.n ? P.keys[i] - P.kmin : EMPTY32;
        }
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) {
            rank[j] = EMPTY32;
            if (k[j] == EMPTY32) continue;
            slot[j] = csr_slot(H, k[j]);
            rank[j] = atomicAdd(&H.cnt[slot[j]], 1u);
        }
        __syncthreads();
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++)  // one range of the key's run per (tile, key)
            if (rank[j] == 0u) H.base[slot[j]] = atomicAdd(&P.cursor[k[j]], H.cnt[slot[j]]);
        __syncthreads();
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) {
            if (rank[j] == EMPTY32) continue;
            const u32 i = row0 + j * 256u + threadIdx.x;
            const u32 pos = H.base[slot[j]] + rank[j];
            for (u32 c = 0; c < P.n_pay; c++) P.pay_out[c][pos] = P.pay_in[c][i];
        }
        __syncthreads();
#pragma unroll
        for (u32 j = 0; j < CSR_ITEMS; j++) if (rank[j] == 0u) { H.key[slot[j]] = EMPTY32; H.cnt[slot[j]] = 0u; }
        __syncthreads();
    }
}
void launch_csr_fill(const u32* keys, u32 n, u32 kmin, u32* cursor, const u32* const* pay_in, u32* const* pay_out, u32 n_pay, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    CsrFillParams P{};
    P.keys = keys; P.n = n; P.kmin = kmin; P.n_pay = n_pay; P.cursor = cursor;
    for (u32 c = 0; c < n_pay; c++) { P.pay_in[c] = pay_in[c]; P.pay_out[c] = pay_out[c]; }
    const int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + CSR_TILE - 1ull) / CSR_TILE);
    csr_fill_kernel<<<grid, 256, 0, st>>>(P);
}

// Directory builds over a predicate slice. The key column may hold a handful of distinct values repeated millions of times (the objects
// of foaf:title, of ds:full_or_part_time ...): one global atomic per row serialises on three addresses. The lanes of a
// warp that carry the same key are therefore aggregated (__match_any_sync): one atomic per (warp, distinct key), ranks inside the group
// from the lane mask.
__global__ void __launch_bounds__(256) csr_count_pairs_kernel(const uint2* __restrict__ kv, u32 key_is_y, u32 n, u32 kmin, u32* __restrict__ counts) {
    const u32 stride = gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    const u32 n_round = (n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        const bool valid = i < n;
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (!valid) continue;
        const uint2 v = kv[i];
        const u32 key = (key_is_y ? v.y : v.x) - kmin;
        const unsigned peers = __match_any_sync(act, key);
        if (lane == __ffs(peers) - 1) atomicAdd(&counts[key], (u32)__popc(peers));
    }
}
void launch_csr_count_pairs(const uint2* kv, u32 key_is_y, u32 n, u32 kmin, u32* counts, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    csr_count_pairs_kernel<<<grid, 256, 0, st>>>(kv, key_is_y, n, kmin, counts);
}
__global__ void __launch_bounds__(256) csr_fill_pairs_kernel(const uint2* __restrict__ kv, u32 key_is_y, u32 n, u32 kmin, u32* __restrict__ cursor,
                                                             u32* __restrict__ val_out) {
    const u32 stride = gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31;
    const u32 n_round = (n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        const bool valid = i < n;
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (!valid) continue;
        const uint2 v = kv[i];
        const u32 key = (key_is_y ? v.y : v.x) - kmin;
        const unsigned peers = __match_any_sync(act, key);
        const int leader = __ffs(peers) - 1;
        u32 base = 0;
        if (lane == leader) base = atomicAdd(&cursor[key], (u32)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        val_out[base + (u32)__popc(peers & ((1u << lane) - 1u))] = key_is_y ? v.x : v.y;
    }
}
void launch_csr_fill_pairs(const uint2* kv, u32 key_is_y, u32 n, u32 kmin, u32* cursor, u32* val_out, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    csr_fill_pairs_kernel<<<grid, 256, 0, st>>>(kv, key_is_y, n, kmin, cursor, val_out);
}

__global__ void __launch_bounds__(256) csr_total_kernel(const u32* __restrict__ pk, u32 n, const u32* __restrict__ off, u32 kmin, u32 range,
                                                        unsigned long long* total) {
    const u32 stride = gridDim.x * blockDim.x;
    unsigned long long t = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u32 o = pk[i] - kmin;
        if (o < range) t += (unsigned long long)(__ldg(off + o + 1) - __ldg(off + o));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(total, t);
}
void launch_csr_total(const u32* pkeys, u32 n, const CsrTab& tab, unsigned long long* total, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    csr_total_kernel<<<grid, 256, 0, st>>>(pkeys, n, tab.off, tab.kmin, tab.range, total);
}

// One tile = 1024 probe rows staged by TMA. Pass 1: every row reads its directory entry (begin, count); the counts are scanned over the
// tile. Pass 2: output row r of the tile belongs to the probe row whose prefix range holds r (binary search in shared memory), so
// consecutive threads write consecutive output rows and read consecutive payload rows.
// Skew: a probe row may match 10^5 build rows (the closure of a class tree joined on the ancestor), and a tile of such rows used to be
// expanded by the ONE CTA that scanned it — the 2 M x 5 M-row join of the transitive rule ran on a handful of SMs. A tile whose
// expansion exceeds PROBEG_HEAVY rows is now only recorded by the first launch (HEAVY = false); the second launch (HEAVY = true) walks
// the recorded tiles, every CTA re-stages the tile and expands its share of PROBEG_CHUNK-row pieces.
template <bool HEAVY>
__global__ void __launch_bounds__(PROBEG_THREADS) probe_grouped_kernel(const __grid_constant__ ProbeGParams P) {
    extern __shared__ __align__(128) u32 smem[];  // n_pcols tiles, then begin[TILE], pref[TILE]
    u32* s_begin = smem + P.n_pcols * PROBEG_TILE;
    u32* s_pref = s_begin + PROBEG_TILE;
    __shared__ __align__(8) u64 bar;
    __shared__ u32 s_tile;
    __shared__ u32 s_w[PROBEG_THREADS / 32 + 1];
    __shared__ u32 s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        mbar_init(&bar, 1);
        fence_mbar_init();
    }
    u32 parity = 0;
    const u32* sKey = smem + P.pkey * PROBEG_TILE;
    const u32 n_heavy = HEAVY ? *reinterpret_cast<volatile u32*>(P.heavy_count) : 0u;
    u32 h_next = 0;  // HEAVY: next recorded tile to look at
    for (;;) {
        __syncthreads();  // the previous tile's expansion has finished reading shared memory
        u32 h_gbase = 0, h_total = 0;
        if constexpr (HEAVY) {
            // the recorded tiles in list order; a CTA takes part in a tile when it has at least one piece of it
            u32 t = EMPTY32;
            while (h_next < n_heavy) {
                const ProbeGParams::Heavy e = P.heavy[h_next++];
                const u32 pieces = (e.total + PROBEG_CHUNK - 1u) / PROBEG_CHUNK;
                if (blockIdx.x < pieces) { t = e.tile; h_gbase = e.gbase; h_total = e.total; break; }
            }
            if (tid == 0) s_tile = t;
        } else if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= P.n_tiles) break;
        if (tid == 0) {
            const u32 b = tile * (u32)PROBEG_TILE;
            const u32 c = min((u32)PROBEG_TILE, P.n - b);
            const u32 bytes = (c * 4u + 15u) & ~15u;
            mbar_arrive_expect_tx(&bar, bytes * P.n_pcols);
            for (u32 q = 0; q < P.n_pcols; q++) tma_load_1d(smem + q * PROBEG_TILE, P.pcol[q] + b, bytes, &bar);
        }
        const u32 cnt = min((u32)PROBEG_TILE, P.n - tile * (u32)PROBEG_TILE);
        mbar_wait(&bar, parity);
        parity ^= 1u;
        // pass 1: directory reads (all of a thread's rows in flight together), warp-local exclusive scan in row order
        u32 b[PROBEG_ITEMS], c[PROBEG_ITEMS];
#pragma unroll
        for (int j = 0; j < PROBEG_ITEMS; j++) {
            const u32 idx = (u32)warp * (32u * PROBEG_ITEMS) + (u32)j * 32u + (u32)lane;
            const u32 o = sKey[idx] - P.tab.kmin;
            const bool ok = idx < cnt && o < P.tab.range;
            b[j] = ok ? __ldg(P.tab.off + o) : 0u;
            c[j] = ok ? __ldg(P.tab.off + o + 1) : 0u;
        }
        u32 run = 0;
#pragma unroll
        for (int j = 0; j < PROBEG_ITEMS; j++) {
            const u32 idx = (u32)warp * (32u * PROBEG_ITEMS) + (u32)j * 32u + (u32)lane;
            const u32 n_match = c[j] - b[j];
            u32 incl = n_match;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
            }
            s_begin[idx] = b[j];
            s_pref[idx] = run + incl - n_match;  // exclusive within the warp's 128 rows; the warp base is added below
            run += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) s_w[warp] = run;
        __syncthreads();
        if (warp == 0) {
            const u32 w = lane < PROBEG_THREADS / 32 ? s_w[lane] : 0u;
            u32 wi = w;
#pragma unroll
            for (int o = 1; o < PROBEG_THREADS / 32; o <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += y;
            }
            const u32 total = __shfl_sync(0xffffffffu, wi, PROBEG_THREADS / 32 - 1);
            if (lane < PROBEG_THREADS / 32) s_w[lane] = wi - w;
            if (lane == 0) s_w[PROBEG_THREADS / 32] = total;
            if (!HEAVY) {
                const u32 ex = tile_prefix_2level(P.tile_state, P.block_state, tile, P.n_tiles, 0u, P.epoch, total, P.zero_word, P.total, P.ordered, lane);
                if (lane == 0) {
                    s_base = ex;
                    if (P.heavy && total > PROBEG_HEAVY) {  // recorded for the second launch
                        ProbeGParams::Heavy e;
                        e.tile = tile; e.gbase = ex; e.total = total; e.pad = 0u;
                        P.heavy[atomicAdd(P.heavy_count, 1u)] = e;
                    }
                }
            }
        }
        __syncthreads();
        {
            const u32 wb = s_w[warp];
#pragma unroll
            for (int j = 0; j < PROBEG_ITEMS; j++) s_pref[(u32)warp * (32u * PROBEG_ITEMS) + (u32)j * 32u + (u32)lane] += wb;
        }
        __syncthreads();
        // pass 2: load-balanced expansion
        const u32 total = s_w[PROBEG_THREADS / 32];
        const u32 gbase = HEAVY ? h_gbase : s_base;
        if (!HEAVY && P.heavy && total > PROBEG_HEAVY) continue;
        const u32 pieces = HEAVY ? (h_total + PROBEG_CHUNK - 1u) / PROBEG_CHUNK : 1u;
        for (u32 piece = HEAVY ? blockIdx.x : 0u; piece < pieces; piece += gridDim.x) {
            const u32 r0 = HEAVY ? piece * PROBEG_CHUNK : 0u;
            const u32 r1 = HEAVY ? min(total, r0 + PROBEG_CHUNK) : total;
            for (u32 r = r0 + (u32)tid; r < r1; r += PROBEG_THREADS) {
                u32 lo = 0, hi = PROBEG_TILE - 1;  // largest idx with pref[idx] <= r
#pragma unroll
                for (int step = 0; step < 10; step++) {
                    const u32 mid = (lo + hi + 1u) >> 1;
                    if (s_pref[mid] <= r) lo = mid; else hi = mid - 1u;
                }
                const u32 src = lo;
                const u32 brow = s_begin[src] + (r - s_pref[src]);
                const u32 pos = gbase + r;
                if (pos < P.cap) {
                    for (u32 q = 0; q < P.n_pcols; q++) P.out[q][pos] = smem[q * PROBEG_TILE + src];
                    for (u32 q = 0; q < P.tab.n_pay; q++) P.out[P.n_pcols + q][pos] = __ldg(P.tab.pay[q] + brow);
                }
            }
        }
    }
}
void launch_probe_grouped(const ProbeGParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    const size_t smem = (size_t)(p.n_pcols + 2) * PROBEG_TILE * sizeof(u32);
    if (smem > 48 * 1024) {
        cudaFuncSetAttribute(probe_grouped_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cudaFuncSetAttribute(probe_grouped_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    }
    const int grid = grid_for((const void*)probe_grouped_kernel<false>, PROBEG_THREADS, smem, n_sms, p.n_tiles);
    probe_grouped_kernel<false><<<grid, PROBEG_THREADS, smem, st>>>(p);
    if (p.heavy) {  // the recorded heavy tiles (usually none: the launch then finds an empty list and ends)
        const int grid2 = grid_for((const void*)probe_grouped_kernel<true>, PROBEG_THREADS, smem, n_sms, 1u << 20);
        probe_grouped_kernel<true><<<grid2, PROBEG_THREADS, smem, st>>>(p);
    }
}

// cartesian product: output row (i*nr + j) = left row i ++ right row j (engine.rs:1054-1071)
struct CartParams {
    const u32* l[KB_MAX_COLS];
    const u32* r[KB_MAX_COLS];
    u32* out[KB_MAX_COLS];
    u32 nl, nr, n_l, n_r;
};
__global__ void cartesian_kernel(const CartParams P) {
    const u64 total = (u64)P.nl * P.nr;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (u64)gridDim.x * blockDim.x) {
        const u32 li = (u32)(i / P.nr), ri = (u32)(i % P.nr);
        for (u32 c = 0; c < P.n_l; c++) P.out[c][i] = P.l[c][li];
        for (u32 c = 0; c < P.n_r; c++) P.out[P.n_l + c][i] = P.r[c][ri];
    }
}
void launch_cartesian(const u32* const* lcols, u32 nl, u32 n_lcols, const u32* const* rcols, u32 nr, u32 n_rcols, u32* const* out,
                      cudaStream_t st) {
    CartParams P;
    P.nl = nl; P.nr = nr; P.n_l = n_lcols; P.n_r = n_rcols;
    for (u32 c = 0; c < n_lcols; c++) P.l[c] = lcols[c];
    for (u32 c = 0; c < n_rcols; c++) P.r[c] = rcols[c];
    for (u32 c = 0; c < n_lcols + n_rcols; c++) P.out[c] = out[c];
    const u64 total = (u64)nl * nr;
    if (total == 0) return;
    int grid = (int)umin64(H100_SMS * 8, (total + 255) / 256);
    cartesian_kernel<<<grid, 256, 0, st>>>(P);
}

// =================================================================================================================
// K_group
__device__ void atomic_min_f64(double* addr, double v) {
    unsigned long long* a = reinterpret_cast<unsigned long long*>(addr);
    unsigned long long old = *a;
    while (v < __longlong_as_double((long long)old) || __longlong_as_double((long long)old) != __longlong_as_double((long long)old)) {
        const unsigned long long assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)__double_as_longlong(v));
        if (old == assumed) break;
    }
}
__device__ void atomic_max_f64(double* addr, double v) {
    unsigned long long* a = reinterpret_cast<unsigned long long*>(addr);
    unsigned long long old = *a;
    while (v > __longlong_as_double((long long)old) || __longlong_as_double((long long)old) != __longlong_as_double((long long)old)) {
        const unsigned long long assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)__double_as_longlong(v));
        if (old == assumed) break;
    }
}


__global__ void group_init_kernel(const GroupParams P) {
    const u32 stride = gridDim.x * blockDim.x;
    if (P.overflow != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *P.overflow = 0u;  // prepared plans: the flag lives behind the table
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n_slots; i += stride) {
        P.gstate[i] = 0u;
        P.gcnt[i] = 0ull;
        for (u32 a = 0; a < P.n_aggs; a++) P.gval[(u64)i * 8 + a] = agg_identity(P.akind[a]);
    }
}
void launch_group_init(const GroupParams& p, cudaStream_t st) {
    int grid = (int)umin64(H100_SMS * 4, ((u64)p.n_slots + 255) / 256);
    group_init_kernel<<<grid, 256, 0, st>>>(p);
}

// find-or-insert the group of key k[] in the global table; returns slot or EMPTY32 on overflow
__device__ __forceinline__ u32 group_slot(const GroupParams& P, const u32* k) {
    u32 h = 0x9E3779B9u;
    for (u32 c = 0; c < P.n_gcols; c++) h = mix32(h ^ k[c]) * 0x85EBCA77u + c;
    const u32 mask = P.n_slots - 1u;
    u32 slot = mix32(h) & mask;
    for (u32 probes = 0; probes < P.n_slots; probes++) {
        u32 st = *reinterpret_cast<volatile u32*>(&P.gstate[slot]);  // read first: a ready slot must not cost an atomic
        if (st == 0u) st = atomicCAS(&P.gstate[slot], 0u, 1u);
        else if (st == 2u) st = 3u;  // ready, skip the claim path
        if (st == 0u) {
            for (u32 c = 0; c < P.n_gcols; c++) P.gkeys[(u64)slot * 4 + c] = k[c];
            __threadfence();
            atomicExch(&P.gstate[slot], 2u);
            return slot;
        }
        while (st == 1u) st = *reinterpret_cast<volatile u32*>(&P.gstate[slot]);
        __threadfence();
        bool eq = true;
        for (u32 c = 0; c < P.n_gcols; c++) eq = eq && (*reinterpret_cast<volatile u32*>(&P.gkeys[(u64)slot * 4 + c]) == k[c]);
        if (eq) return slot;
        slot = (slot + 1u) & mask;
    }
    return EMPTY32;
}

// Two levels of pre-aggregation keep a GROUP BY with a handful of groups from serialising on a handful of addresses:
// (1) a warp folds its 32 rows per distinct group (__match_any_sync), (2) leaders accumulate into a 64-entry shared-memory
// table of the CTA, flushed to the global table once per CTA. Rows whose group does not fit the CTA table go straight to global.
constexpr int GROUP_SMEM = 64;
__device__ void group_update_global(const GroupParams& P, const u32* k, unsigned long long cnt, const double* val) {
    const u32 slot = group_slot(P, k);
    if (slot == EMPTY32) { *P.overflow = 1u; return; }
    atomicAdd(&P.gcnt[slot], cnt);
    for (u32 a = 0; a < P.n_aggs; a++) {
        double* dst = &P.gval[(u64)slot * 8 + a];
        if (P.akind[a] == KB_AGG_MIN) atomic_min_f64(dst, val[a]);
        else if (P.akind[a] == KB_AGG_MAX) atomic_max_f64(dst, val[a]);
        else if (P.akind[a] != KB_AGG_COUNT) atomicAdd(dst, val[a]);
    }
}

__global__ void __launch_bounds__(256) group_merge_kernel(const __grid_constant__ GroupParams P, const GroupRecord* __restrict__ recs, u32 n) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const GroupRecord r = recs[i];
        if (r.count == 0ull) continue;
        group_update_global(P, r.keys, r.count, r.raw);
    }
}
void launch_group_merge(const GroupParams& p, const GroupRecord* recs, u32 n, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
    group_merge_kernel<<<grid, 256, 0, st>>>(p, recs, n);
}

__global__ void __launch_bounds__(1024) group_compact_kernel(const __grid_constant__ GroupParams P, GroupRecord* __restrict__ out, u32* header, u32 cap) {
    __shared__ u32 s_n;
    if (threadIdx.x == 0) s_n = 0u;
    __syncthreads();
    for (u32 i = threadIdx.x; i < P.n_slots; i += blockDim.x) {
        if (P.gstate[i] != 2u) continue;
        const u32 at = atomicAdd(&s_n, 1u);
        if (at >= cap) continue;
        GroupRecord r;
#pragma unroll
        for (int c = 0; c < 4; c++) r.keys[c] = (u32)c < P.n_gcols ? P.gkeys[(u64)i * 4 + c] : 0u;
        r.count = P.gcnt[i];
#pragma unroll
        for (int a = 0; a < 8; a++) r.raw[a] = (u32)a < P.n_aggs ? P.gval[(u64)i * 8 + a] : 0.0;
        out[at] = r;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        header[1] = (P.overflow ? *P.overflow : 0u) | (s_n > cap ? 1u : 0u);
        header[0] = min(s_n, cap);
        __threadfence_system();
    }
}
void launch_group_compact(const GroupParams& p, GroupRecord* out, u32* header, u32 cap, cudaStream_t st) {
    group_compact_kernel<<<1, 1024, 0, st>>>(p, out, header, cap);
}

// ---- cross-rank GROUP BY over peer memory
__device__ __forceinline__ void st_release_sys(u32* p, u32 v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ u32 ld_acquire_sys(const u32* p) {
    u32 v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
template <class T>
__device__ __forceinline__ T ld_sys(const T* p) { return *reinterpret_cast<const volatile T*>(p); }

__global__ void __launch_bounds__(64) peer_barrier_kernel(const __grid_constant__ PeerTables T, u32 epoch) {
    const u32 r = threadIdx.x;
    __threadfence_system();
    if (r < T.world) {
        st_release_sys(T.flags[r] + T.rank, epoch);                                  // "I have arrived" in r's array
        const u32* mine = T.flags[T.rank] + r;
        unsigned long long t0, now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        while ((int)(ld_acquire_sys(mine) - epoch) < 0) {                            // r has arrived (epochs only grow; wrap-safe compare)
            __nanosleep(100);
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (now - t0 > 5000000000ull) {  // 5 s: a rank never submitted this query — give up loudly instead of hanging the GPU
                atomicExch(T.flags[T.rank] + 63, 1u);
                break;
            }
        }
    }
    __syncthreads();
    __threadfence_system();
}
void launch_peer_barrier(const PeerTables& t, u32 epoch, cudaStream_t st) { peer_barrier_kernel<<<1, 64, 0, st>>>(t, epoch); }

__global__ void __launch_bounds__(256) group_merge_peers_kernel(const __grid_constant__ GroupParams P, const __grid_constant__ PeerTables T) {
    const u32 total = T.world * T.n_slots;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const u32 r = i / T.n_slots, s = i - r * T.n_slots;
        const char* tb = T.table[r];
        if (s == 0u && ld_sys(reinterpret_cast<const u32*>(tb + T.o_overflow)) != 0u) *P.overflow = 1u;  // a partial overflowed: so does the merge
        if (i == 0u && ld_sys(T.flags[T.rank] + 63) != 0u) *P.overflow = 2u;                               // the barrier before this kernel timed out
        if (ld_sys(reinterpret_cast<const u32*>(tb + T.o_state) + s) != 2u) continue;
        u32 k[4];
        double v[8];
#pragma unroll
        for (int c = 0; c < 4; c++) k[c] = ld_sys(reinterpret_cast<const u32*>(tb + T.o_keys) + (u64)s * 4 + c);
        const unsigned long long cnt = ld_sys(reinterpret_cast<const unsigned long long*>(tb + T.o_cnt) + s);
#pragma unroll
        for (int a = 0; a < 8; a++) v[a] = (u32)a < P.n_aggs ? ld_sys(reinterpret_cast<const double*>(tb + T.o_val) + (u64)s * 8 + a) : 0.0;
        group_update_global(P, k, cnt, v);
    }
}
void launch_group_merge_peers(const GroupParams& p, const PeerTables& t, int n_sms, cudaStream_t st) {
    const u64 total = (u64)t.world * t.n_slots;
    const int grid = (int)umin64((u64)n_sms * 2ull, (total + 255ull) / 256ull);
    group_merge_peers_kernel<<<grid, 256, 0, st>>>(p, t);
}

__global__ void __launch_bounds__(256) group_kernel(const __grid_constant__ GroupParams P) {
    __shared__ u32 sk[GROUP_SMEM][4];
    __shared__ u32 sstate[GROUP_SMEM];  // 0 free, 1 being written, 2 ready
    __shared__ unsigned long long scnt[GROUP_SMEM];
    __shared__ double sval[GROUP_SMEM][8];
    for (int i = threadIdx.x; i < GROUP_SMEM; i += blockDim.x) {
        sstate[i] = 0u;
        scnt[i] = 0ull;
        for (u32 a = 0; a < 8; a++) sval[i][a] = agg_identity(a < P.n_aggs ? P.akind[a] : (u32)KB_AGG_COUNT);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (P.n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        const bool valid = i < P.n;
        u32 k[4] = {0, 0, 0, 0};
        u32 h = 0;
        if (valid) for (u32 c = 0; c < P.n_gcols; c++) { k[c] = P.gcol[c][i]; h = mix32(h ^ k[c]) + c; }
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (!valid) continue;
        // lanes with the same full key form a group: match on the hash, then confirm equality with the leader
        unsigned peers = __match_any_sync(act, h);
        int leader = __ffs(peers) - 1;
        bool same = true;
        for (u32 c = 0; c < P.n_gcols; c++) {  // every lane of `peers` must reach every shuffle: no short-circuit around it
            const u32 lk = __shfl_sync(peers, k[c], leader);
            same = same && lk == k[c];
        }
        const unsigned agree = __ballot_sync(act, same);
        peers = same ? (peers & agree) : (1u << lane);  // rare hash collision inside a warp: the odd lanes go alone
        leader = __ffs(peers) - 1;
        double val[8];
        for (u32 a = 0; a < P.n_aggs; a++) val[a] = P.acol[a] ? num_of(P.nt, P.acol[a][i]) : 0.0;
        const unsigned long long cnt = (unsigned long long)__popc(peers);
        for (u32 a = 0; a < P.n_aggs; a++) {
            if (P.akind[a] == KB_AGG_COUNT) continue;  // COUNT needs no values: popc(peers) is the fold
            double acc = val[a];
            unsigned rest = peers & ~(1u << leader);
            while (rest) {  // every lane of the group runs the same shuffles
                const int src = __ffs(rest) - 1;
                rest &= rest - 1u;
                const double o = __shfl_sync(peers, val[a], src);
                if (P.akind[a] == KB_AGG_MIN) acc = fmin(acc, o);
                else if (P.akind[a] == KB_AGG_MAX) acc = fmax(acc, o);
                else acc += o;
            }
            val[a] = acc;
        }
        if (lane != leader) continue;
        // CTA table: find or claim
        u32 slot = mix32(h) & (GROUP_SMEM - 1);
        bool done = false;
        for (int probes = 0; probes < GROUP_SMEM && !done; probes++) {
            u32 st = *reinterpret_cast<volatile u32*>(&sstate[slot]);
            if (st == 0u) st = atomicCAS(&sstate[slot], 0u, 1u);
            else if (st == 2u) st = 3u;
            if (st == 0u) {
                for (u32 c = 0; c < 4; c++) sk[slot][c] = k[c];
                __threadfence_block();
                atomicExch(&sstate[slot], 2u);
                st = 3u;
            }
            while (st == 1u) st = *reinterpret_cast<volatile u32*>(&sstate[slot]);
            __threadfence_block();
            bool eq = true;
            for (u32 c = 0; c < P.n_gcols; c++) eq = eq && (*reinterpret_cast<volatile u32*>(&sk[slot][c]) == k[c]);
            if (eq) {
                atomicAdd(&scnt[slot], cnt);
                for (u32 a = 0; a < P.n_aggs; a++) {
                    if (P.akind[a] == KB_AGG_MIN) atomic_min_f64(&sval[slot][a], val[a]);
                    else if (P.akind[a] == KB_AGG_MAX) atomic_max_f64(&sval[slot][a], val[a]);
                    else if (P.akind[a] != KB_AGG_COUNT) atomicAdd(&sval[slot][a], val[a]);
                }
                done = true;
            } else slot = (slot + 1u) & (GROUP_SMEM - 1);
        }
        if (!done) group_update_global(P, k, cnt, val);  // more than 64 distinct groups in this CTA
    }
    __syncthreads();
    for (int i = threadIdx.x; i < GROUP_SMEM; i += blockDim.x) {
        if (sstate[i] != 2u) continue;
        u32 k[4] = {sk[i][0], sk[i][1], sk[i][2], sk[i][3]};
        double v[8];
        for (u32 a = 0; a < 8; a++) v[a] = sval[i][a];
        group_update_global(P, k, scnt[i], v);
    }
}
// GROUP BY one variable with at most one aggregate (GROUP BY ?t COUNT, SUM/AVG/MIN/MAX(?x) GROUP BY ?t — execute_query.rs:1150-1227):
// the key itself is the match value, four rows per thread are loaded before any is folded (the loop is load-latency bound), the CTA
// table is keyed by a CAS on the key word and counts are 32-bit shared atomics.
template <int AGG>  // 0: COUNT only, else the kb_agg kind of the single value aggregate
__global__ void __launch_bounds__(256) group1_kernel(const __grid_constant__ GroupParams P) {
    constexpr int IT = 4;
    __shared__ u32 sk[GROUP_SMEM];
    __shared__ u32 scnt[GROUP_SMEM];
    __shared__ double sval[GROUP_SMEM];
    for (int i = threadIdx.x; i < GROUP_SMEM; i += blockDim.x) {
        sk[i] = EMPTY32;
        scnt[i] = 0u;
        sval[i] = agg_identity((u32)AGG);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (P.n + 31u) & ~31u;
    const u32* __restrict__ kc = P.gcol[0];
    const u32* __restrict__ ac = P.acol[0];
    for (u32 i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < n_round; i0 += IT * stride) {
        u32 key[IT];
        double val[IT];
#pragma unroll
        for (int j = 0; j < IT; j++) {
            const u32 i = i0 + (u32)j * stride;
            key[j] = i < P.n ? __ldg(kc + i) : EMPTY32;
            if (AGG != 0) val[j] = i < P.n ? num_of(P.nt, __ldg(ac + i)) : 0.0;
        }
#pragma unroll
        for (int j = 0; j < IT; j++) {
            const u32 i = i0 + (u32)j * stride;
            if (i - (u32)lane >= P.n) continue;  // the whole warp is past the end (warp-uniform)
            const bool valid = i < P.n;
            const unsigned act = __ballot_sync(0xffffffffu, valid);
            if (!valid) continue;
            const unsigned peers = __match_any_sync(act, key[j]);
            const int leader = __ffs(peers) - 1;
            double acc = 0.0;
            if (AGG != 0) {
                acc = val[j];
                unsigned rest = peers & ~(1u << leader);
                while (rest) {
                    const int src = __ffs(rest) - 1;
                    rest &= rest - 1u;
                    const double o = __shfl_sync(peers, val[j], src);
                    if (AGG == KB_AGG_MIN) acc = fmin(acc, o);
                    else if (AGG == KB_AGG_MAX) acc = fmax(acc, o);
                    else acc += o;
                }
            }
            if (lane != leader) continue;
            const u32 cnt = (u32)__popc(peers);
            u32 slot = mix32(key[j]) & (GROUP_SMEM - 1);
            bool done = false;
            for (int probes = 0; probes < GROUP_SMEM && !done && key[j] != EMPTY32; probes++) {  // EMPTY32 marks a free entry
                u32 cur = *reinterpret_cast<volatile u32*>(&sk[slot]);
                if (cur == EMPTY32) cur = atomicCAS(&sk[slot], EMPTY32, key[j]);
                if (cur == EMPTY32 || cur == key[j]) {
                    atomicAdd(&scnt[slot], cnt);
                    if (AGG == KB_AGG_MIN) atomic_min_f64(&sval[slot], acc);
                    else if (AGG == KB_AGG_MAX) atomic_max_f64(&sval[slot], acc);
                    else if (AGG != 0) atomicAdd(&sval[slot], acc);
                    done = true;
                } else slot = (slot + 1u) & (GROUP_SMEM - 1);
            }
            if (!done) {  // more than 64 distinct groups in this CTA
                u32 k[4] = {key[j], 0u, 0u, 0u};
                double v[8] = {acc, 0, 0, 0, 0, 0, 0, 0};
                group_update_global(P, k, (unsigned long long)cnt, v);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < GROUP_SMEM; i += blockDim.x) {
        if (sk[i] == EMPTY32) continue;
        u32 k[4] = {sk[i], 0u, 0u, 0u};
        double v[8] = {sval[i], 0, 0, 0, 0, 0, 0, 0};
        group_update_global(P, k, (unsigned long long)scnt[i], v);
    }
}
void launch_group(const GroupParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    if (p.n_gcols == 1 && p.n_aggs <= 1) {
        // a CTA's 32-bit shared counters see at most n / grid * ... rows: far below 2^32
        int grid = (int)umin64((u64)n_sms * 8ull, ((u64)p.n + 1023ull) / 1024ull);
        const u32 kind = (p.n_aggs == 0 || p.akind[0] == KB_AGG_COUNT) ? 0u : p.akind[0];
        switch (kind) {
            case 0: group1_kernel<0><<<grid, 256, 0, st>>>(p); break;
            case KB_AGG_SUM: group1_kernel<KB_AGG_SUM><<<grid, 256, 0, st>>>(p); break;
            case KB_AGG_AVG: group1_kernel<KB_AGG_AVG><<<grid, 256, 0, st>>>(p); break;
            case KB_AGG_MIN: group1_kernel<KB_AGG_MIN><<<grid, 256, 0, st>>>(p); break;
            default: group1_kernel<KB_AGG_MAX><<<grid, 256, 0, st>>>(p); break;
        }
        return;
    }
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)p.n + 255ull) / 256ull);
    group_kernel<<<grid, 256, 0, st>>>(p);
}

// =================================================================================================================
// Datalog: known-fact set with 96-bit keys in 16-byte slots {s,p,o,state}
__device__ __forceinline__ u32 set_hash(u32 s, u32 p, u32 o) { return mix32(mix32(s) * 0x9E3779B1u ^ mix32(o + 0x632BE5ABu) ^ (p * 0x85EBCA77u)); }

// returns 1 if (s,p,o) was inserted now, 0 if it was already there, 2 on overflow
__device__ __forceinline__ u32 set_insert(uint4* set, u32 n_slots, u32 s, u32 p, u32 o) {
    const u32 mask = n_slots - 1u;
    u32 slot = set_hash(s, p, o) & mask;
    for (u32 probes = 0; probes < n_slots; probes++) {
        u32* st_ptr = &reinterpret_cast<u32*>(&set[slot])[3];
        u32 st = atomicCAS(st_ptr, 0u, 1u);
        if (st == 0u) {
            u32* w = reinterpret_cast<u32*>(&set[slot]);
            w[0] = s; w[1] = p; w[2] = o;
            __threadfence();
            atomicExch(st_ptr, 2u);
            return 1u;
        }
        while (st == 1u) st = *reinterpret_cast<volatile u32*>(st_ptr);
        __threadfence();
        const volatile u32* w = reinterpret_cast<const volatile u32*>(&set[slot]);
        if (w[0] == s && w[1] == p && w[2] == o) return 0u;
        slot = (slot + 1u) & mask;
    }
    return 2u;
}

__global__ void __launch_bounds__(256) set_insert_kernel(uint4* set, u32 set_slots, const u32* s, const u32* p, u32 p_const, const u32* o,
                                                         u32 n, u32* overflow) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        if (set_insert(set, set_slots, s[i], p ? p[i] : p_const, o[i]) == 2u) *overflow = 1u;
}
void launch_set_insert(uint4* set, u32 set_slots, const u32* s, const u32* p, u32 p_const, const u32* o, u32 n, u32* overflow, int n_sms,
                       cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    set_insert_kernel<<<grid, 256, 0, st>>>(set, set_slots, s, p, p_const, o, n, overflow);
}

// 64-bit (s,o) set of one predicate: returns 1 inserted now, 0 already present, 2 table full
__device__ __forceinline__ u32 set64_insert(u64* set, u32 n_slots, u32 s, u32 o) {
    const u64 key = ((u64)s << 32) | (u64)o;
    const u32 mask = n_slots - 1u;
    u32 slot = mix32(mix32(s) * 0x9E3779B1u ^ mix32(o + 0x632BE5ABu)) & mask;
    for (u32 probes = 0; probes < n_slots; probes++) {
        const u64 cur = *reinterpret_cast<volatile u64*>(&set[slot]);
        if (cur == key) return 0u;
        if (cur == EMPTY64) {
            const u64 old = atomicCAS(reinterpret_cast<unsigned long long*>(&set[slot]), (unsigned long long)EMPTY64, (unsigned long long)key);
            if (old == EMPTY64) return 1u;
            if (old == key) return 0u;
        }
        slot = (slot + 1u) & mask;
    }
    return 2u;
}
__global__ void __launch_bounds__(256) set64_insert_kernel(u64* set, u32 set_slots, const u32* s, const u32* o, u32 n, u32* overflow) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        if (set64_insert(set, set_slots, s[i], o[i]) == 2u) *overflow = 1u;
}
void launch_set64_insert(u64* set, u32 set_slots, const u32* s, const u32* o, u32 n, u32* overflow, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    set64_insert_kernel<<<grid, 256, 0, st>>>(set, set_slots, s, o, n, overflow);
}

__device__ __forceinline__ bool rule_filters_pass(const DeriveParams& P, u32 i) {
    for (u32 f = 0; f < P.n_filt; f++) {
        const RuleFilterDev fl = P.filt[f];
        const u32 lhs = P.bcol[fl.lhs_col][i];
        if (fl.rhs_is_var) {  // rules.rs:141-146 — ids of two bound variables; only = / != act
            const u32 rhs = P.bcol[fl.rhs_col][i];
            if (fl.cmp == KB_CMP_NE && lhs == rhs) return false;
            if (fl.cmp == KB_CMP_EQ && lhs != rhs) return false;
        } else {  // rules.rs:148-160
            const double a = num_of(P.nt, lhs), c = fl.rhs_value;
            const double eps = 2.220446049250313e-16;
            switch (fl.cmp) {
                case KB_CMP_GT: if (a <= c) return false; break;
                case KB_CMP_LT: if (a >= c) return false; break;
                case KB_CMP_GE: if (a < c) return false; break;
                case KB_CMP_LE: if (a > c) return false; break;
                case KB_CMP_EQ: if (fabs(a - c) > eps) return false; break;
                case KB_CMP_NE: if (fabs(a - c) <= eps) return false; break;
                default: break;
            }
        }
    }
    return true;
}

__global__ void __launch_bounds__(256) derive_kernel(const __grid_constant__ DeriveParams P) {
    const int lane = threadIdx.x & 31;
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (P.n + 31u) & ~31u;
    unsigned long long nd = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        bool pass = i < P.n && rule_filters_pass(P, i);
        bool fresh = false;
        u32 s = 0, o = 0;
        if (pass) nd++;
        if (pass && *reinterpret_cast<volatile u32*>(P.out_count) >= P.budget) {  // the set must grow first; this launch is run again
            *P.overflow = 2u;
            pass = false;
        }
        if (pass) {
            s = P.head_s.is_var ? P.bcol[P.head_s.value][i] : P.head_s.value;
            o = P.head_o.is_var ? P.bcol[P.head_o.value][i] : P.head_o.value;
            const u32 r = set64_insert(P.set, P.set_slots, s, o);
            if (r == 2u) atomicMax(P.overflow, 1u);
            fresh = r == 1u;
        }
        const unsigned b = __ballot_sync(0xffffffffu, fresh);  // warp-aggregated append of the facts that were new
        if (b) {
            u32 basepos = 0;
            if (lane == __ffs(b) - 1) basepos = atomicAdd(P.out_count, (u32)__popc(b));
            basepos = __shfl_sync(0xffffffffu, basepos, __ffs(b) - 1);
            if (fresh) {
                const u32 r = basepos + (u32)__popc(b & ((1u << lane) - 1u));
                if (r < P.out_cap) { P.out_s[r] = s; P.out_o[r] = o; }
                else *P.overflow = 1u;
            }
        }
    }
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 16);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 8);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 4);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 2);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 1);
    if (lane == 0 && nd) atomicAdd(P.n_deriv, nd);
}
// ---- radix-partitioned variant
constexpr int DPART_THREADS = 256;
constexpr int DPART_ITEMS = 16;
constexpr int DPART_TILE = DPART_THREADS * DPART_ITEMS;  // 4096 candidates: 32 KB of keys + 8 KB of partition ids in shared memory
constexpr int DPART_MAXP = 1024;
__device__ __forceinline__ u32 set64_home(u32 n_slots, u32 s, u32 o) { return mix32(mix32(s) * 0x9E3779B1u ^ mix32(o + 0x632BE5ABu)) & (n_slots - 1u); }

// insert + append of ONE candidate outside any warp-cooperative section (bucket overflow path of the partition pass)
__device__ __noinline__ void derive_one(const DeriveParams& P, u32 s, u32 o) {
    if (*reinterpret_cast<volatile u32*>(P.out_count) >= P.budget) { *P.overflow = 2u; return; }
    const u32 r = set64_insert(P.set, P.set_slots, s, o);
    if (r == 2u) *P.overflow = 2u;
    if (r == 1u) {
        const u32 at = atomicAdd(P.out_count, 1u);
        if (at < P.out_cap) { P.out_s[at] = s; P.out_o[at] = o; }
        else *P.overflow = 1u;
    }
}

__global__ void __launch_bounds__(DPART_THREADS) derive_partition_kernel(const __grid_constant__ DerivePartParams Q) {
    extern __shared__ __align__(16) u64 sh_keys[];  // [DPART_TILE] keys sorted by partition, then u16 partition ids
    __shared__ u32 s_cnt[DPART_MAXP], s_off[DPART_MAXP], s_gbase[DPART_MAXP];
    __shared__ u32 s_tile;
    const DeriveParams& P = Q.d;
    unsigned short* s_dest = reinterpret_cast<unsigned short*>(sh_keys + DPART_TILE);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 n_tiles = (P.n + DPART_TILE - 1u) / DPART_TILE;
    unsigned long long nd = 0;
    for (;;) {
        if (tid == 0) s_tile = atomicAdd(&Q.tickets[0], 1u);
        for (u32 d = (u32)tid; d < Q.n_parts; d += DPART_THREADS) s_cnt[d] = 0u;
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= n_tiles) break;
        const u32 row0 = tile * (u32)DPART_TILE;
        const u32 cnt = min((u32)DPART_TILE, P.n - row0);
        // ---- 1. head instantiation + rule filters; partition = high bits of the key's home slot; histogram
        u64 key[DPART_ITEMS];
        u32 part[DPART_ITEMS], rank[DPART_ITEMS];
#pragma unroll
        for (int j = 0; j < DPART_ITEMS; j++) {
            const u32 r = (u32)j * DPART_THREADS + (u32)tid;
            const u32 i = row0 + r;
            bool pass = r < cnt && rule_filters_pass(P, i);
            u32 s = 0, o = 0;
            if (pass) {
                nd++;
                s = P.head_s.is_var ? __ldg(P.bcol[P.head_s.value] + i) : P.head_s.value;
                o = P.head_o.is_var ? __ldg(P.bcol[P.head_o.value] + i) : P.head_o.value;
            }
            key[j] = ((u64)s << 32) | (u64)o;
            part[j] = pass ? (set64_home(P.set_slots, s, o) >> Q.slice_bits) : 0xFFFFu;
            rank[j] = pass ? atomicAdd(&s_cnt[part[j]], 1u) : 0u;  // the key's place among the tile's keys of its partition (kept for step 3)
        }
        __syncthreads();
        // ---- 2. offsets inside the tile (one warp scans the histogram), one range reservation per partition
        if (warp == 0) {
            u32 run = 0;
            for (u32 d0 = 0; d0 < Q.n_parts; d0 += 32u) {
                const u32 d = d0 + (u32)lane;
                const u32 c = d < Q.n_parts ? s_cnt[d] : 0u;
                u32 incl = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += y;
                }
                if (d < Q.n_parts) {
                    s_off[d] = run + incl - c;
                    s_gbase[d] = c ? atomicAdd(&Q.cursors[d], c) : 0u;
                }
                run += __shfl_sync(0xffffffffu, incl, 31);
            }
        }
        __syncthreads();
        // ---- 3. keys staged in partition order
#pragma unroll
        for (int j = 0; j < DPART_ITEMS; j++) {
            if (part[j] == 0xFFFFu) continue;
            const u32 pos = s_off[part[j]] + rank[j];
            sh_keys[pos] = key[j];
            s_dest[pos] = (unsigned short)part[j];
        }
        __syncthreads();
        // ---- 4. flush: staged position q belongs to partition s_dest[q]; consecutive q of one partition are consecutive in its bucket
        const u32 staged = s_off[Q.n_parts - 1u] + s_cnt[Q.n_parts - 1u];
        for (u32 q = (u32)tid; q < staged; q += DPART_THREADS) {
            const u32 d = s_dest[q];
            const u32 at = s_gbase[d] + (q - s_off[d]);
            const u64 k = sh_keys[q];
            if (at < Q.bucket_cap) Q.buckets[(u64)d * Q.bucket_cap + at] = k;
            else derive_one(P, (u32)(k >> 32), (u32)k);  // the bucket is full (skewed hash): probe directly
        }
        __syncthreads();
    }
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 16);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 8);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 4);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 2);
    nd = nd + __shfl_xor_sync(0xffffffffu, nd, 1);
    if (lane == 0 && nd) atomicAdd(P.n_deriv, nd);
}

constexpr int DPROBE_TILE = 2048;
__global__ void __launch_bounds__(1024) derive_tile_starts_kernel(const __grid_constant__ DerivePartParams Q) {
    __shared__ u32 s_tiles[DPART_MAXP];
    const int tid = threadIdx.x;
    if ((u32)tid < Q.n_parts) s_tiles[tid] = (min(Q.cursors[tid], Q.bucket_cap) + DPROBE_TILE - 1u) / DPROBE_TILE;
    __syncthreads();
    if (tid == 0) {
        u32 run = 0;
        for (u32 d = 0; d < Q.n_parts; d++) { Q.tile_start[d] = run; run += s_tiles[d]; }
        Q.tile_start[Q.n_parts] = run;
    }
}

__global__ void __launch_bounds__(256) derive_probe_kernel(const __grid_constant__ DerivePartParams Q) {
    __shared__ u32 s_tile, s_base;
    __shared__ u32 s_wcnt[8];
    const DeriveParams& P = Q.d;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 n_tiles = Q.tile_start[Q.n_parts];
    constexpr int R = DPROBE_TILE / 256;
    for (;;) {
        __syncthreads();
        if (tid == 0) s_tile = atomicAdd(&Q.tickets[1], 1u);  // tickets are handed out in partition order: the CTAs walk the slices together
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= n_tiles) break;
        u32 lo = 0, hi = Q.n_parts;  // partition of this tile: last d with tile_start[d] <= tile
        while (hi - lo > 1u) {
            const u32 mid = (lo + hi) >> 1;
            if (Q.tile_start[mid] <= tile) lo = mid; else hi = mid;
        }
        const u32 d = lo;
        const u32 n_keys = min(Q.cursors[d], Q.bucket_cap);
        const u32 first = (tile - Q.tile_start[d]) * (u32)DPROBE_TILE;
        const u64* keys = Q.buckets + (u64)d * Q.bucket_cap;
        // the set must not fill past its budget: checked once per tile (a tile adds at most DPROBE_TILE facts: the budget leaves that room)
        const bool room = *reinterpret_cast<volatile u32*>(P.out_count) < P.budget;
        if (!room && tid == 0) *P.overflow = 2u;
        u64 k[R];
        u32 fresh = 0;
#pragma unroll
        for (int j = 0; j < R; j++) {
            const u32 q = first + (u32)j * 256u + (u32)tid;
            k[j] = (room && q < n_keys) ? __ldg(keys + q) : EMPTY64;
        }
#pragma unroll
        for (int j = 0; j < R; j++) {
            if (k[j] == EMPTY64) continue;  // (s = o = 0xFFFFFFFF is the reserved id: never a fact)
            const u32 r = set64_insert(P.set, P.set_slots, (u32)(k[j] >> 32), (u32)k[j]);
            if (r == 2u) *P.overflow = 2u;  // table full (the per-tile budget check lets a small table overshoot): grow and run again
            fresh |= (r == 1u ? 1u : 0u) << j;
        }
        // ONE reservation per tile for the facts that were new (a single global cursor serialises: per-warp reservations
        // dominated the pass on 1.4e8 new facts), then ranked writes
        const u32 c = (u32)__popc(fresh);
        u32 incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const u32 y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) s_wcnt[warp] = incl;
        __syncthreads();
        if (tid == 0) {
            u32 run = 0;
#pragma unroll
            for (int w = 0; w < 8; w++) { const u32 x = s_wcnt[w]; s_wcnt[w] = run; run += x; }
            s_base = run ? atomicAdd(P.out_count, run) : 0u;
        }
        __syncthreads();
        u32 pos = s_base + s_wcnt[warp] + incl - c;
#pragma unroll
        for (int j = 0; j < R; j++) {
            if ((fresh >> j) & 1u) {
                if (pos < P.out_cap) { P.out_s[pos] = (u32)(k[j] >> 32); P.out_o[pos] = (u32)k[j]; }
                else *P.overflow = 1u;
                pos++;
            }
        }
    }
}

void launch_derive_partitioned(const DerivePartParams& p, int n_sms, cudaStream_t st) {
    if (p.d.n == 0) return;
    const size_t smem = (size_t)DPART_TILE * (sizeof(u64) + sizeof(unsigned short));
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(derive_partition_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr = true; }
    const u32 n_tiles = (p.d.n + DPART_TILE - 1u) / DPART_TILE;
    const int grid1 = grid_for((const void*)derive_partition_kernel, DPART_THREADS, smem, n_sms, n_tiles);
    static const bool trace = getenv("KOLIBRIE_TRACE") != nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr;
    if (trace) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventCreate(&e2); cudaEventRecord(e0, st); }
    derive_partition_kernel<<<grid1, DPART_THREADS, smem, st>>>(p);
    if (trace) cudaEventRecord(e1, st);
    derive_tile_starts_kernel<<<1, 1024, 0, st>>>(p);
    const int grid2 = grid_for((const void*)derive_probe_kernel, 256, 0, n_sms, (p.d.n + DPROBE_TILE - 1u) / DPROBE_TILE + p.n_parts);
    derive_probe_kernel<<<grid2, 256, 0, st>>>(p);
    if (trace) {
        cudaEventRecord(e2, st);
        cudaEventSynchronize(e2);
        float a = 0.f, b = 0.f;
        cudaEventElapsedTime(&a, e0, e1);
        cudaEventElapsedTime(&b, e1, e2);
        fprintf(stderr, "[kb trace]     derive partitioned: %u candidates, %u partitions: partition pass %.3f ms, probe pass %.3f ms\n", p.d.n, p.n_parts, a, b);
        cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(e2);
    }
}

void launch_derive(const DeriveParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)p.n + 255ull) / 256ull);
    derive_kernel<<<grid, 256, 0, st>>>(p);
}

// =================================================================================================================
// dictionary decode
__global__ void __launch_bounds__(256) decode_lengths_kernel(const u32* __restrict__ ids, u32 n, const unsigned long long* __restrict__ dict_off, u32 dict_ids,
                                                             u32* __restrict__ len, unsigned long long* total, u32* quoted) {
    const u32 stride = gridDim.x * blockDim.x;
    unsigned long long t = 0;
    bool q = false;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u32 id = ids[i];
        q = q || (id & 0x80000000u) != 0u;
        const u32 l = id < dict_ids ? (u32)(__ldg(dict_off + id + 1) - __ldg(dict_off + id)) : 7u;  // "unknown"
        len[i] = l;
        t += l;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(total, t);
    if (q) *quoted = 1u;
}
void launch_decode_lengths(const u32* ids, u32 n, const unsigned long long* dict_off, u32 dict_ids, u32* len, unsigned long long* total, u32* quoted,
                           int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    decode_lengths_kernel<<<grid, 256, 0, st>>>(ids, n, dict_off, dict_ids, len, total, quoted);
}
__global__ void __launch_bounds__(256) decode_gather_kernel(const u32* __restrict__ ids, u32 n, const unsigned long long* __restrict__ dict_off,
                                                            const unsigned char* __restrict__ dict_bytes, u32 dict_ids, const u32* __restrict__ off,
                                                            unsigned char* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const u32 warps = (gridDim.x * blockDim.x) >> 5;
    const u32 n_chunks = (n + 31u) >> 5;
    for (u32 chunk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; chunk < n_chunks; chunk += warps) {
        const u32 i = chunk * 32u + (u32)lane;
        u32 id = 0, dst = 0, l = 0;
        unsigned long long src = 0;
        bool known = false;
        if (i < n) {
            id = ids[i];
            dst = off[i];
            l = off[i + 1] - dst;
            known = id < dict_ids;
            if (known) src = __ldg(dict_off + id);
        }
        for (int r = 0; r < 32; r++) {  // the warp copies row r of its chunk: consecutive lanes, consecutive bytes
            const u32 rl = __shfl_sync(0xffffffffu, l, r);
            if (rl == 0u) continue;
            const u32 rdst = __shfl_sync(0xffffffffu, dst, r);
            const unsigned long long rsrc = __shfl_sync(0xffffffffu, src, r);
            const bool rknown = __shfl_sync(0xffffffffu, known ? 1 : 0, r) != 0;
            for (u32 b = (u32)lane; b < rl; b += 32u) out[rdst + b] = rknown ? __ldg(dict_bytes + rsrc + b) : (unsigned char)"unknown"[b];
        }
    }
}
void launch_decode_gather(const u32* ids, u32 n, const unsigned long long* dict_off, const unsigned char* dict_bytes, u32 dict_ids, const u32* off,
                          unsigned char* out, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    decode_gather_kernel<<<grid, 256, 0, st>>>(ids, n, dict_off, dict_bytes, dict_ids, off, out);
}

// =================================================================================================================
// utilities
__global__ void fill_kernel(u32* p, u32 v, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) p[i] = v;
}
void launch_fill_u32(u32* p, u32 v, u64 n, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64(H100_SMS * 8, (n + 255) / 256);
    fill_kernel<<<grid, 256, 0, st>>>(p, v, n);
}
void launch_fill_const_col(u32* p, u32 v, u64 n, cudaStream_t st) { launch_fill_u32(p, v, n, st); }

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
void launch_part_count(const u32* key, u32 n, u32 n_parts, u32* counts, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
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
void launch_part_scatter(const u32* key, u32 n, u32 n_parts, u32* cursors, const u32* const* in_cols, u32* const* out_cols, u32 n_cols,
                         int n_sms, cudaStream_t st) {
    if (n == 0) return;
    PartScatterParams P;
    P.n_cols = n_cols;
    for (u32 c = 0; c < n_cols; c++) { P.in[c] = in_cols[c]; P.out[c] = out_cols[c]; }
    int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
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
void launch_shuffle_scatter(const ShuffleParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    static const int threads_env = getenv("KOLIBRIE_SHUFFLE_THREADS") ? atoi(getenv("KOLIBRIE_SHUFFLE_THREADS")) : 0;
    const bool wide = threads_env ? threads_env >= 512 : true;  // 4096-row tiles (512 threads) for the register-resident cases
    if (p.n_cols == 1) { if (wide) launch_shuffle_t<1, 512>(p, n_sms, st); else launch_shuffle_t<1, 256>(p, n_sms, st); }
    else if (p.n_cols == 2) { if (wide) launch_shuffle_t<2, 512>(p, n_sms, st); else launch_shuffle_t<2, 256>(p, n_sms, st); }
    else if (p.n_cols <= 6) launch_shuffle_t<0, 512>(p, n_sms, st);  // <= 6 x (4096 + 768) x 4 B = 114 KB of staging
    else launch_shuffle_t<0, 128>(p, n_sms, st);                    // 16 columns x (1024 + 768) x 4 B = 112 KB
}

// kb_store_delete: p_out[i] = p[i], or EMPTY32 when (s,p,o)[i] is in the delete set; a scan with a variable predicate and
// NE_ID(EMPTY32)... is not needed: the store compaction simply rescans with pattern (?s ?p ?o) over (s, p_out, o) and drops
// rows whose predicate became EMPTY32 (KB_ID_NONE is never a real predicate).
__global__ void __launch_bounds__(256) delete_mark_kernel(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots,
                                                          u32* p_out) {
    const u32 mask = set_slots - 1u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 vs = s[i], vp = p[i], vo = o[i];
        u32 slot = set_hash(vs, vp, vo) & mask;
        bool found = false;
        for (u32 probes = 0; probes < set_slots; probes++) {
            const uint4 e = set[slot];
            if (e.w == 0u) break;
            if (e.x == vs && e.y == vp && e.z == vo) { found = true; break; }
            slot = (slot + 1u) & mask;
        }
        p_out[i] = found ? EMPTY32 : vp;
    }
}
void launch_delete_mark(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots, u32* p_out, int n_sms,
                        cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    delete_mark_kernel<<<grid, 256, 0, st>>>(s, p, o, n, set, set_slots, p_out);
}

}  // namespace kb
