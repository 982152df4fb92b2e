// kb_scan.cu — the fused triple scan: its launch format, the general and the star-shape scan kernel, IndexScan over the store index,
// and kb_scan. scan_segments, scan_store and scan_predicates (kb_internal.hpp) are what the rest of the library calls; the launch
// format and everything behind it stay in this file.
#include "kb_internal.hpp"

#include <cmath>
#include <cstdlib>
#include <type_traits>

using namespace kb;

namespace kb {
namespace {

// ---------------------------------------------------------------------------------------------------------------
// K_scan: fused multi-pattern triple scan + constant filter + pushed-down FILTER + ordered compaction.
// Replaces execute_table_scan_with_ids (engine.rs:510-584), the index scans (engine.rs:1192-1407), QueryBuilder's
// Exact filter scan (query_builder.rs:486-531) and the reference's hash_join_kernel (cuda_join.cu:26-45).
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;  // 2048 triples = 24 KB of shared memory per CTA

enum : u32 {
    SP_HAS_S = 1, SP_HAS_P = 2, SP_HAS_O = 4,      // constant in that position
    SP_EQ_SP = 8, SP_EQ_SO = 16, SP_EQ_PO = 32,    // same variable twice in one pattern (quirk Q4: enforced)
    SP_EMIT_S = 64, SP_EMIT_P = 128, SP_EMIT_O = 256,  // positions written to the output (columns come out in s,p,o order)
    SP_EMIT_IDX = 512,                              // global triple index (legacy FFI)
    SP_PAIR = 1024,  // emit (subject, object) interleaved as uint2 into outp[0]: one 8-byte store per match (2-variable patterns)
    // scan + build fused: the match goes straight into a direct join table, table[key - cs] = other half (cs = key base, co = key
    // range, outp[0] = table, outp[1] = duplicate flag); no intermediate relation is written or re-read
    SP_TABLE = 2048,
    SP_TKEY_O = 4096     // the join key is the object (default: the subject)
};
struct ScanPat {
    u32 cs, cp, co;
    u32 flags;
    u32* outp[4];        // output column of position s / p / o / index (null when not emitted)
    u32 f_begin, f_len;  // pushed-down FILTER program (slots = positions 0/1/2)
};
constexpr int SCAN_MAXSEG = 16;  // store segments one launch can walk (an RSP window of slides is scanned in ONE launch)
struct ScanSeg {
    const u32 *s, *p, *o;
    u32 n;           // triples
    u32 tile0;       // first tile of this segment in the launch's tile numbering
    u32 index_base;  // global index of the segment's first triple
};
struct ScanParams {
    ScanSeg seg[SCAN_MAXSEG];
    u32 n_seg;
    u32 n_tiles, K;  // n_tiles: over all segments of the launch
    u32 cshift;      // SP_TABLE patterns: log2(world) key compaction of a subject-sharded store (0 = none)
    ScanPat pat[MAXP];
    FilterOp ops[KB_MAX_FILTER_OPS];
    NumTab nt;
    // direct tables the FIRST launch of a scan clears itself (scan_star_kernel: every CTA fills a slice with 0xFF, then the grid meets
    // at clear_barrier[0] before any insert; clear_barrier[1] is raised when the meeting timed out) — two 67 MB cudaMemsetAsync calls
    // in front of the kernel cost two launch gaps and more time than the same bytes written by the resident grid
    u32* clear_tab[4];
    u32 clear_words[4];
    u32 n_clear;
    u32* clear_barrier;
    Compact c;         // total / zero_word unused: the scan counts per pattern in totals_in / totals_out
    u32* ticket;
    const u32* totals_in;  // [MAXP] rows written by earlier segments
    u32* totals_out;       // [MAXP] rows written so far (ordered: a different array than totals_in; unordered: the same, used as atomic cursor)
};

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
            const u32 ex = tile_prefix_2level(P.c.tile_state, P.c.block_state, tile, P.n_tiles, (u32)warp, P.c.epoch, total, P.totals_in, P.totals_out, P.c.ordered, lane);
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
            const u32 ex = tile_prefix_2level(P.c.tile_state, P.c.block_state, tile, P.n_tiles, (u32)warp, P.c.epoch, total, P.totals_in, P.totals_out, P.c.ordered, lane);
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
    if (p.K > 4 || p.c.ordered) return false;  // store-order output (KOLIBRIE_ORDERED, legacy FFI): the general kernel
    for (u32 k = 0; k < p.K; k++) {
        const ScanPat& sp = p.pat[k];
        const u32 shape = sp.flags & ~(SP_TABLE | SP_TKEY_O | SP_PAIR);
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
    static int per_sm = 0;  // occupancy is a property of the kernel image; the grid follows each caller's n_sms
    if (per_sm == 0) {
        cudaFuncSetAttribute(scan_star_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int occ = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, scan_star_kernel<K>, STAR_THREADS, smem);
        per_sm = occ < 1 ? 1 : occ;
    }
    const int grid = (int)umin64((u64)per_sm * (u64)n_sms, (u64)p.n_tiles);
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
// true when launch_scan(p) runs the kernel that honours clear_tab / n_clear
bool scan_clears_tables(const ScanParams& p) { return p.n_tiles != 0 && scan_star_enabled() && scan_is_star(p); }
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

// IndexScan proper (engine.rs:1192-1407, the 8-case lookup of index_manager.rs:253-340 for a constant predicate): with a valid store
// index a pattern whose predicate is constant is answered from the predicate's slice — (c P ?o) from the subject table / directory,
// (?s P c) from the object table / directory, (?s P ?o) is the slice itself — without touching the 12-byte/triple store.
// *out stays null when the index cannot answer the pattern (the caller scans).
kb_status index_lookup(kb_ctx* ctx, const kb_pattern& pt, std::unique_ptr<kb_rel>* out) {
    out->reset();
    if (!ctx->use_index || ctx->index_version != ctx->store_version || pt.p.is_var) return KB_OK;
    std::vector<u32> slots, src;
    pattern_vars(pt, &slots, &src);
    auto it = ctx->index.find(pt.p.value);
    if (it == ctx->index.end() || it->second.n == 0) return empty_rel(ctx, slots, out);  // the predicate does not occur: empty answer
    auto rel = std::make_unique<kb_rel>();
    rel->slots = slots;
    const PredSlice& ps = it->second;
    if (pt.s.is_var && pt.o.is_var) {
        if (pt.s.value == pt.o.value) return KB_OK;  // ?x P ?x: the scan enforces the equality
        Col x, y;  // the slice itself, de-interleaved (all chunks)
        KB_TRY(alloc_col(ctx, ps.n, &x));
        KB_TRY(alloc_col(ctx, ps.n, &y));
        u64 at = 0;
        timer_begin(ctx, F_SCAN, (int)ps.chunks.size());
        for (auto& ch : ps.chunks) {
            // (chunk boundaries keep 16-byte alignment only by luck: unpair writes element-wise, no TMA on the output side)
            launch_unpair(reinterpret_cast<const uint2*>(ch.pairs.ptr), (u32)ch.n, x.ptr + at, y.ptr + at, ctx->st);
            at += ch.n;
        }
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        rel->cols = {x, y};
        rel->n = ps.n;
        ctx->stats.index_joins++;
        *out = std::move(rel);
        return KB_OK;
    }
    if (pt.s.is_var == pt.o.is_var) return KB_OK;  // both constant: left to the scan
    const bool by_y = !pt.o.is_var;                // the bound position is the object
    const u32 key = by_y ? pt.o.value : pt.s.value;
    const Buf& tab = by_y ? ps.ytab : ps.xtab;
    const Buf& off = by_y ? ps.yoff : ps.xoff;
    const Buf& val = by_y ? ps.yval : ps.xval;
    if (tab) {  // unique column: one table slot
        const u32 cs = by_y ? 0u : ps.tab_cshift;
        if (cs != 0u && shard_of(key, ctx->shard_world) != ctx->shard_rank) return empty_rel(ctx, slots, out);  // a key of another shard: not in this store
        const u32 o = compact_key(key, cs) - (by_y ? ps.ytab_min : ps.xtab_min);
        u32 v = EMPTY32;
        if (o < (by_y ? ps.ytab_range : ps.xtab_range)) {
            KB_CUDA(ctx, cudaMemcpyAsync(&v, static_cast<const u32*>(tab->p) + o, sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
            KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
            ctx->stats.d2h_bytes += 4;
        }
        Col col;
        KB_TRY(alloc_col(ctx, v == EMPTY32 ? 0 : 1, &col));
        if (v != EMPTY32) KB_CUDA(ctx, cudaMemcpyAsync(col.ptr, &v, sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        rel->cols.push_back(col);
        rel->n = v == EMPTY32 ? 0 : 1;
        ctx->stats.index_joins++;
        *out = std::move(rel);
        return KB_OK;
    }
    if (off && val) {  // multi-valued column: the key's run in the directory
        const u32 kmin = by_y ? ps.ycsr_min : ps.xcsr_min, range = by_y ? ps.ycsr_range : ps.xcsr_range;
        u32 be[2] = {0, 0};
        if (key >= kmin && key - kmin < range) {
            KB_CUDA(ctx, cudaMemcpyAsync(be, static_cast<const u32*>(off->p) + (key - kmin), 2 * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
            KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
            ctx->stats.d2h_bytes += 8;
        }
        const u64 n = be[1] - be[0];
        Col col;
        if ((be[0] & 3u) == 0 && n) {  // 16-byte aligned run: a view of the directory's values, no copy
            col.buf = val;
            col.ptr = static_cast<u32*>(val->p) + be[0];
        } else {
            KB_TRY(alloc_col(ctx, n, &col));
            if (n) KB_CUDA(ctx, cudaMemcpyAsync(col.ptr, static_cast<const u32*>(val->p) + be[0], n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        }
        rel->cols.push_back(col);
        rel->n = n;
        ctx->stats.index_joins++;
        *out = std::move(rel);
        return KB_OK;
    }
    return KB_OK;
}

}  // namespace

kb_status unpair_rel(kb_ctx* ctx, std::unique_ptr<kb_rel>* r) {
    if (!(*r)->pair) return KB_OK;
    auto c = std::make_unique<kb_rel>();
    c->slots = (*r)->slots;
    c->n = (*r)->n;
    Col x, y;
    KB_TRY(alloc_col(ctx, c->n, &x));
    KB_TRY(alloc_col(ctx, c->n, &y));
    timer_begin(ctx, F_OTHER);
    launch_unpair(reinterpret_cast<const uint2*>((*r)->cols[0].ptr), (u32)c->n, x.ptr, y.ptr, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    c->cols = {x, y};
    *r = std::move(c);
    return KB_OK;
}

kb_status scan_segments(kb_ctx* ctx, const std::vector<Segment>& segs, const kb_pattern* pats, u32 K, const std::vector<FilterProg>& pushdown,
                        ScanOut mode, std::vector<std::unique_ptr<kb_rel>>* out, const std::vector<ScanTable>* tables) {
    if (K == 0 || K > (u32)MAXP) return fail(ctx, KB_E_LIMIT, "a fused scan takes 1..%d patterns (got %u)", MAXP, K);
    u64 N = 0;
    for (auto& sg : segs) N += sg.n;
    if (N >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "store holds %llu triples; row positions are 32-bit", (unsigned long long)N);
    ScanParams P{};
    P.K = K;
    P.nt = numtab(ctx);
    std::vector<FilterOp> ops;
    out->clear();
    for (u32 k = 0; k < K; k++) {
        KB_TRY(check_pattern(ctx, pats[k]));
        const kb_pattern& pt = pats[k];
        ScanPat& sp = P.pat[k];
        sp.flags = 0;
        if (!pt.s.is_var) { sp.flags |= SP_HAS_S; sp.cs = pt.s.value; }
        if (!pt.p.is_var) { sp.flags |= SP_HAS_P; sp.cp = pt.p.value; }
        if (!pt.o.is_var) { sp.flags |= SP_HAS_O; sp.co = pt.o.value; }
        if (pt.s.is_var && pt.p.is_var && pt.s.value == pt.p.value) sp.flags |= SP_EQ_SP;
        if (pt.s.is_var && pt.o.is_var && pt.s.value == pt.o.value) sp.flags |= SP_EQ_SO;
        if (pt.p.is_var && pt.o.is_var && pt.p.value == pt.o.value) sp.flags |= SP_EQ_PO;
        std::vector<u32> slots, src;
        pattern_vars(pt, &slots, &src);
        auto rel = std::make_unique<kb_rel>();
        if (mode == ScanOut::RowIndex) {
            slots.assign(1, 0u);
            src.assign(1, 3u);
        }
        rel->slots = slots;
        for (int q = 0; q < 4; q++) sp.outp[q] = nullptr;
        if (tables && k < tables->size() && (*tables)[k].tab) {  // fused build: no output relation, the table is the output
            const ScanTable& tb = (*tables)[k];
            rel->pair = true;
            sp.outp[0] = tb.tab;
            sp.outp[1] = tb.dup_flag;
            sp.cs = tb.kmin;
            sp.co = tb.range;
            sp.flags |= SP_TABLE | (tb.key_is_o ? SP_TKEY_O : 0u);
            P.cshift = tb.cshift;
        } else if (mode == ScanOut::Pairs && slots.size() == 2 && src[0] == 0 && src[1] == 2) {
            Col col;  // interleaved (subject, object) rows: one 8-byte store per match
            KB_TRY(alloc_col(ctx, 2 * N, &col));
            rel->cols.push_back(col);
            rel->pair = true;
            sp.outp[0] = col.ptr;
            sp.flags |= SP_PAIR;
        } else {
            for (size_t c = 0; c < slots.size(); c++) {  // columns come out in s,p,o order = order of first appearance
                Col col;
                KB_TRY(alloc_col(ctx, N, &col));
                rel->cols.push_back(col);
                sp.outp[src[c]] = col.ptr;
                sp.flags |= src[c] == 0 ? SP_EMIT_S : src[c] == 1 ? SP_EMIT_P : src[c] == 2 ? SP_EMIT_O : SP_EMIT_IDX;
            }
        }
        sp.f_begin = (u32)ops.size();
        sp.f_len = 0;
        if (k < pushdown.size() && !pushdown[k].ops.empty()) {
            std::vector<u32> vs, vsrc;
            pattern_vars(pt, &vs, &vsrc);
            std::vector<FilterOp> local;
            KB_TRY(compile_prog(ctx, pushdown[k], vs, &local, &vsrc));
            if (ops.size() + local.size() > KB_MAX_FILTER_OPS) return fail(ctx, KB_E_LIMIT, "pushed-down filters exceed %d ops", KB_MAX_FILTER_OPS);
            ops.insert(ops.end(), local.begin(), local.end());
            sp.f_len = (u32)local.size();
        }
        out->push_back(std::move(rel));
    }
    for (size_t i = 0; i < ops.size(); i++) P.ops[i] = ops[i];

    const u32 n_seg = (u32)segs.size();
    // the guard depends on the segment count alone: where the arena cursor stands is irrelevant, ctrl_alloc wraps (an index build
    // over hundreds of predicates hands out ~76 words per 8-predicate batch and every consumer clears its own words)
    if (std::max(n_seg, 1u) + 2u * MAXP > kb_ctx::CTRL_WORDS - 64u) return fail(ctx, KB_E_LIMIT, "too many store segments (%u)", n_seg);
    const u32 off_tot = ctrl_alloc(ctx, 2 * MAXP);
    const u32 off_ticket = ctrl_alloc(ctx, std::max(n_seg, 1u));
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off_tot, 0, 2 * MAXP * sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off_ticket, 0, std::max(n_seg, 1u) * sizeof(u32), ctx->st));
    u64 all_tiles = 0;
    for (auto& sg : segs) all_tiles += (sg.n + SCAN_TILE - 1) / SCAN_TILE;
    // One launch walks up to SCAN_MAXSEG consecutive segments (an RSP window is ~10 slides). A segment whose upload is still in
    // flight (chunked kb_star_join_host) closes the group before it, so the scan of the chunks that already landed can start.
    u64 index_base = 0;
    u32 n_launched = 0;
    u32 g = 0;
    // tables that still have to be set to 0xFF: by the first launch itself when it is the star-shape kernel, else by memsets here
    std::vector<std::pair<u32*, u32>> pending_clear;
    if (tables) for (auto& tb : *tables) if (tb.tab && tb.clear) pending_clear.push_back({tb.tab, tb.range});
    u32 off_clear = 0;
    bool clear_folded = false;
    while (g < n_seg) {
        P.n_seg = 0;
        P.n_tiles = 0;
        cudaEvent_t wait_ev = nullptr;
        while (g < n_seg && P.n_seg < (u32)SCAN_MAXSEG) {
            const Segment& sg = segs[g];
            if (sg.n == 0) { g++; continue; }
            if (sg.ready && P.n_seg > 0) break;  // starts its own group
            ScanSeg& d = P.seg[P.n_seg++];
            d.s = sg.s.ptr; d.p = sg.p.ptr; d.o = sg.o.ptr;
            d.n = (u32)sg.n;
            d.tile0 = P.n_tiles;
            d.index_base = (u32)index_base;
            P.n_tiles += (u32)((sg.n + SCAN_TILE - 1) / SCAN_TILE);
            index_base += sg.n;
            g++;
            if (sg.ready) { wait_ev = sg.ready; break; }
        }
        if (P.n_seg == 0) break;
        P.ticket = ctx->ctrl + off_ticket + n_launched;
        if (ctx->ordered) {  // ping-pong: a launch never writes the word its tiles read their base from
            P.totals_in = ctx->ctrl + off_tot + (n_launched & 1u) * MAXP;
            P.totals_out = ctx->ctrl + off_tot + ((n_launched + 1u) & 1u) * MAXP;
        } else {
            P.totals_in = P.totals_out = ctx->ctrl + off_tot;
        }
        n_launched++;
        // (the star-shape kernel may walk the store in smaller tiles than SCAN_TILE)
        KB_TRY(compact_setup(ctx, all_tiles * 4, nullptr, &P.c));
        P.n_clear = 0;
        if (!pending_clear.empty()) {
            if (pending_clear.size() <= 4 && scan_clears_tables(P)) {
                off_clear = ctrl_alloc(ctx, 4);
                KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off_clear, 0, 4 * sizeof(u32), ctx->st));
                for (auto& pc : pending_clear) { P.clear_tab[P.n_clear] = pc.first; P.clear_words[P.n_clear] = pc.second; P.n_clear++; }
                P.clear_barrier = ctx->ctrl + off_clear;
                clear_folded = true;
            } else {
                timer_begin(ctx, F_BUILD, 0);
                for (auto& pc : pending_clear) KB_CUDA(ctx, cudaMemsetAsync(pc.first, 0xFF, (size_t)pc.second * sizeof(u32), ctx->st));
                timer_end(ctx);
            }
            pending_clear.clear();
        }
        if (wait_ev) KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, wait_ev, 0));  // chunked upload: start as soon as this chunk landed
        timer_begin(ctx, F_SCAN);
        launch_scan(P, ctx->n_sms, ctx->st);
        timer_end(ctx);
    }
    for (auto& pc : pending_clear) KB_CUDA(ctx, cudaMemsetAsync(pc.first, 0xFF, (size_t)pc.second * sizeof(u32), ctx->st));  // (nothing was launched)
    KB_CUDA(ctx, cudaGetLastError());
    ctx->stats.rows_scanned += N;
    KB_TRY(ctrl_read(ctx));
    if (clear_folded && ctx->h_ctrl[off_clear + 1]) return fail(ctx, KB_E_CUDA, "scan: the grid did not meet at the table-clear barrier (another kernel holds SMs?)");
    for (u32 k = 0; k < K; k++) (*out)[k]->n = ctx->h_ctrl[off_tot + (ctx->ordered ? (n_launched & 1u) * MAXP : 0u) + k];
    return KB_OK;
}

kb_status scan_store(kb_ctx* ctx, const kb_pattern* pats, u32 K, const std::vector<FilterProg>& pushdown, std::vector<std::unique_ptr<kb_rel>>* out) {
    if (K == 0 || K > (u32)MAXP) return fail(ctx, KB_E_LIMIT, "a fused scan takes 1..%d patterns (got %u)", MAXP, K);
    if (!ctx->use_index || ctx->index_version != ctx->store_version) return scan_segments(ctx, ctx->segs, pats, K, pushdown, ScanOut::Cols, out);
    // patterns the index answers are not scanned; the rest (if any) go through one fused scan
    std::vector<std::unique_ptr<kb_rel>> got(K);
    std::vector<u32> rest;
    for (u32 k = 0; k < K; k++) {
        KB_TRY(check_pattern(ctx, pats[k]));
        KB_TRY(index_lookup(ctx, pats[k], &got[k]));
        if (!got[k]) { rest.push_back(k); continue; }
        if (k < pushdown.size() && !pushdown[k].ops.empty()) {  // the pattern's own FILTER, applied to the looked-up rows
            std::unique_ptr<kb_rel> f;
            KB_TRY(filter_impl(ctx, *got[k], pushdown[k], &f));
            got[k] = std::move(f);
        }
    }
    if (rest.size() == K) return scan_segments(ctx, ctx->segs, pats, K, pushdown, ScanOut::Cols, out);
    if (!rest.empty()) {
        std::vector<kb_pattern> rp;
        std::vector<FilterProg> rf;
        for (u32 k : rest) { rp.push_back(pats[k]); rf.push_back(k < pushdown.size() ? pushdown[k] : FilterProg{}); }
        std::vector<std::unique_ptr<kb_rel>> sub;
        KB_TRY(scan_segments(ctx, ctx->segs, rp.data(), (u32)rp.size(), rf, ScanOut::Cols, &sub));
        for (size_t i = 0; i < rest.size(); i++) got[rest[i]] = std::move(sub[i]);
    }
    out->clear();
    for (u32 k = 0; k < K; k++) out->push_back(std::move(got[k]));
    return KB_OK;
}

kb_status scan_predicates(kb_ctx* ctx, const std::vector<Segment>& segs, const u32* preds, u32 k, ScanOut mode,
                          std::vector<std::unique_ptr<kb_rel>>* out) {
    std::vector<kb_pattern> pats(k);
    for (u32 i = 0; i < k; i++) { pats[i].s = kb_term{1, 0}; pats[i].p = kb_term{0, preds[i]}; pats[i].o = kb_term{1, 1}; }
    return scan_segments(ctx, segs, pats.data(), k, {}, mode, out);
}

}  // namespace kb

extern "C" {

kb_status kb_scan(kb_ctx* ctx, const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* const* pushdown, const uint32_t* pushdown_len, kb_rel** out) {
    KB_ENTER(ctx);
    if (!pats || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    std::vector<kb::FilterProg> pd(n_pats);
    if (pushdown && pushdown_len)
        for (u32 k = 0; k < n_pats; k++) if (pushdown[k] && pushdown_len[k]) {
            KB_TRY(kb::validate_filter(ctx, pushdown[k], pushdown_len[k]));
            pd[k].ops.assign(pushdown[k], pushdown[k] + pushdown_len[k]);
        }
    std::vector<std::unique_ptr<kb_rel>> rels;
    KB_TRY(kb::scan_store(ctx, pats, n_pats, pd, &rels));
    for (u32 k = 0; k < n_pats; k++) out[k] = rels[k].release();
    if (n_pats) ctx->stats.rows_out = out[n_pats - 1]->n;
    return KB_OK;
}

}  // extern "C"
