// kb_store.cu — the device triple store: its segments, the version that everything derived from it is keyed to (prepared plans, the
// seeded fixpoint's state, kb_datalog_maintain's closed token), the per-version hints of the star-join builds and the
// predicate-partitioned index. This file is the only writer of that state: every change to the store goes through store_replace,
// store_add_device_segment, store_evict_tag or store_swap, which bump the version, drop the hints and maintain or drop the index.
// The kernels behind those changes (the index's profile, split, clear, table, code and rank passes, the key sets of INSERT and DELETE,
// the DELETE-template fill) and their launch formats are in this file too.
#include <algorithm>
#include <chrono>
#include <cstdlib>

#include "kb_internal.hpp"
#include "kb_numrank.cuh"

using namespace kb;

namespace kb {

// ctrl = {overflow, values inserted}. A value already in the set costs a plain load, never an atomic: a column of a few values
// repeated millions of times does not serialise on their slots. Every warp stops at its next row once the overflow word is set.
__global__ void __launch_bounds__(256) distinct_kernel(const u32* __restrict__ col, u32 n, u32* set, u32 set_slots, u32 limit, u32* ctrl) {
    const int lane = threadIdx.x & 31;
    const u32 mask = set_slots - 1u;
    const u32 n_round = (n + 31u) & ~31u;
    u32 last = EMPTY32;  // values come in long runs in real stores: skip what this lane just inserted
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += gridDim.x * blockDim.x) {
        u32 stop = lane == 0 ? *reinterpret_cast<volatile u32*>(&ctrl[0]) : 0u;
        if (__shfl_sync(0xffffffffu, stop, 0)) break;
        const bool valid = i < n;
        const u32 v = valid ? col[i] : EMPTY32;
        const bool fresh = valid && v != EMPTY32 && v != last;
        const unsigned act = __ballot_sync(0xffffffffu, fresh);
        if (!fresh) continue;
        const unsigned peers = __match_any_sync(act, v);
        last = v;
        if (lane != __ffs(peers) - 1) continue;
        u32 slot = mix32(v) & mask;
        for (u32 probes = 0;; probes++) {
            if (probes >= set_slots) { ctrl[0] = 1u; break; }
            const u32 cur = *reinterpret_cast<volatile u32*>(&set[slot]);
            if (cur == v) break;
            if (cur == EMPTY32) {
                const u32 old = atomicCAS(&set[slot], EMPTY32, v);
                if (old == EMPTY32) {
                    if (atomicAdd(&ctrl[1], 1u) >= limit) ctrl[0] = 1u;
                    break;
                }
                if (old == v) break;
            }
            slot = (slot + 1u) & mask;
        }
    }
}
// distinct values of a column other than EMPTY32 into a small open-addressing set (EMPTY32 = free). ctrl = {overflow, count}, both 0
// at launch: the overflow word is set when the set fills up or when a value past the first `limit` arrives, and ends the pass
static void launch_distinct(const u32* col, u32 n, u32* set, u32 set_slots, u32 limit, u32* ctrl, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms, 256, 4);
    distinct_kernel<<<grid, 256, 0, st>>>(col, n, set, set_slots, limit, ctrl);
}

// one-byte codes of a subject table (PredSlice::xcode): code[i] = index of tab[i] in the ascending dictionary, 0xFF where tab[i] is
// EMPTY32; four slots per thread, one 16-byte load and one 4-byte store
__global__ void __launch_bounds__(256) tab_code_kernel(const u32* __restrict__ tab, u32 range, const u32* __restrict__ dict, u32 n_dict,
                                                       u8* __restrict__ code) {
    __shared__ u32 s_dict[CODE_MAX];
    for (u32 i = threadIdx.x; i < n_dict; i += blockDim.x) s_dict[i] = dict[i];
    __syncthreads();
    const u32 quads = (range + 3u) / 4u;
    for (u32 q = blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += gridDim.x * blockDim.x) {
        const uint4 v4 = __ldg(reinterpret_cast<const uint4*>(tab) + q);  // (the buffer is padded past the table's last slot)
        const u32 v[4] = {v4.x, v4.y, v4.z, v4.w};
        u32 packed = 0;
#pragma unroll
        for (u32 k = 0; k < 4; k++) {
            u32 c = 0xFFu;
            if (4u * q + k < range && v[k] != EMPTY32) {
                u32 lo = 0, hi = n_dict;  // the first entry >= v: v is in the dictionary
                while (lo < hi) {
                    const u32 mid = (lo + hi) / 2u;
                    if (s_dict[mid] < v[k]) lo = mid + 1u;
                    else hi = mid;
                }
                c = lo;
            }
            packed |= c << (8u * k);
        }
        reinterpret_cast<u32*>(code)[q] = packed;
    }
}
// code[i] = index of tab[i] in dict (ascending, every value of tab but EMPTY32, n_dict <= CODE_MAX), 0xFF where tab[i] is EMPTY32, for
// i < range; tab and code start 16-byte aligned and may be read / written up to the next multiple of 4 slots
static void launch_tab_code(const u32* tab, u32 range, const u32* dict, u32 n_dict, u8* code, int n_sms, cudaStream_t st) {
    if (range == 0) return;
    const int grid = grid_1d(range, n_sms, 1024);
    tab_code_kernel<<<grid, 256, 0, st>>>(tab, range, dict, n_dict, code);
}

// ---- window-slide maintenance of the store index: ONE pass profiles a new segment (column ranges, foreign subjects, its distinct
// predicates with their row counts), ONE pass splits it into the predicate slices' new chunks — pairs, id ranges, typed literal
// column, in-place inserts into the persistent tables — and ONE pass clears an evicted segment's keys from all of its slices' tables.
constexpr u32 SEGP_SLOTS = 32;  // open-addressing slots for a segment's distinct predicates (more than that: the batched scan path)
// control words of segment_profile: [0..2] min s/p/o, [3] unused, [4 .. 4+SLOTS) predicate slots (all 0xFF at launch);
// then (all 0 at launch) [P_MAX .. +3) max s/p/o, P_FOREIGN, P_OVERFLOW, [P_COUNT .. +SLOTS) rows per slot
constexpr u32 SEGP_MIN = 0, SEGP_SLOT = 4, SEGP_MAX = 4 + SEGP_SLOTS, SEGP_FOREIGN = SEGP_MAX + 3, SEGP_OVERFLOW = SEGP_MAX + 4, SEGP_COUNT = SEGP_MAX + 8,
              SEGP_WORDS = SEGP_COUNT + SEGP_SLOTS;
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
static void launch_segment_profile(const u32* s, const u32* p, const u32* o, u32 n, u32 rank, u32 world, u32* ctrl, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms, 256, 4);
    segment_profile_kernel<<<grid, 256, 0, st>>>(s, p, o, n, rank, world, ctrl);
}

struct SplitEntry {
    u32 pred;
    u32 n;              // rows of the predicate in the segment (capacity of pairs / ynum)
    uint2* pairs;       // the new chunk
    double* ynum;       // its typed literal column (null: no numeric side table loaded)
    u32* xtab; u32 xtab_min, xtab_range, cshift;   // subject table to insert into (null: none)
    u16* xkey;          // value ranks in table order (kb_numrank.cuh: rank16), maintained with xtab (null: none)
    u32* ytab; u32 ytab_min, ytab_range;           // object table (null: none)
};
// control words per entry (all 0 at launch): cursor, n_numeric, xdup, ydup, xout, yout, pad, pad, ~xmin, ~ymin, xmax, ymax
constexpr u32 SPLIT_CURSOR = 0, SPLIT_NNUM = 1, SPLIT_XDUP = 2, SPLIT_YDUP = 3, SPLIT_XOUT = 4, SPLIT_YOUT = 5, SPLIT_XMIN = 8, SPLIT_YMIN = 9, SPLIT_XMAX = 10,
              SPLIT_YMAX = 11, SPLIT_WORDS = 12;
struct SplitParams {
    const u32 *s, *p, *o;
    u32 n, k;
    SplitEntry e[MAXP];
    u32* ctrl;  // k * SPLIT_WORDS words
    NumTab nt;
    const double* numv;  // value order of the numeric side table (kb_numrank.cuh), for the entries' xkey (n_numv = 0: no entry has one)
    u32 n_numv;
};

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
        u32 xk[SPLIT_ITEMS];  // value ranks for the rank columns (xkey): the SPLIT_ITEMS searches in V run side by side
        if (P.n_numv) {
            double xv[SPLIT_ITEMS];
#pragma unroll
            for (u32 j = 0; j < SPLIT_ITEMS; j++) xv[j] = which[j] != EMPTY32 && P.e[which[j]].xkey ? kb_nr::fold(num_of(P.nt, vo[j])) : 0.0;
            kb_nr::rank_of_n<SPLIT_ITEMS>(P.numv, P.n_numv, xv, xk);
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
                    if (E.xkey) E.xkey[off] = kb_nr::rank16(xk[j], kb_nr::rank_shift(P.n_numv));
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
static void launch_segment_split(const SplitParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0 || p.k == 0) return;
    const int grid = grid_1d(p.n, n_sms, SPLIT_TILE, 6);
    segment_split_kernel<<<grid, 256, 0, st>>>(p);
}

constexpr u32 CLEAR_MAX = 16;
struct ClearEntry {
    const uint2* pairs; u32 n;
    u32* xtab; u32 xtab_min, xtab_range, cshift;
    u32* ytab; u32 ytab_min, ytab_range;
};
struct ClearParams { ClearEntry e[CLEAR_MAX]; u32 k; };
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
static void launch_clear_chunks(const ClearParams& p, int n_sms, cudaStream_t st) {
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
// RANKTAB_ITEMS rows per thread (striped over the CTA's chunk): their searches in V run side by side
constexpr u32 RANKTAB_ITEMS = 4;
__global__ void __launch_bounds__(256) pair_ranktab_kernel(const uint2* __restrict__ kv, u32 n, NumTab nt, const double* __restrict__ numv, u32 n_numv,
                                                          u16* __restrict__ out, u32 kmin, u32 range, u32 cshift) {
    for (u32 row0 = blockIdx.x * 256u * RANKTAB_ITEMS; row0 < n; row0 += gridDim.x * 256u * RANKTAB_ITEMS) {
        double x[RANKTAB_ITEMS];
        u32 off[RANKTAB_ITEMS], r[RANKTAB_ITEMS];
#pragma unroll
        for (u32 j = 0; j < RANKTAB_ITEMS; j++) {
            const u32 i = row0 + j * 256u + threadIdx.x;
            off[j] = EMPTY32;
            x[j] = 0.0;
            if (i < n) {
                const uint2 v = kv[i];
                off[j] = compact_key(v.x, cshift) - kmin;
                x[j] = kb_nr::fold(num_of(nt, v.y));
            }
        }
        kb_nr::rank_of_n<RANKTAB_ITEMS>(numv, n_numv, x, r);
        const u32 shift = kb_nr::rank_shift(n_numv);
#pragma unroll
        for (u32 j = 0; j < RANKTAB_ITEMS; j++) if (off[j] < range) out[off[j]] = kb_nr::rank16(r[j], shift);
    }
}
// the ranks of those values in the value order numv[0 .. n_numv) (kb_numrank.cuh), laid out like the subject-keyed direct table:
// out[compact(subject) - kmin] = rank_of(num_of(object))
static void launch_pair_ranktab(const uint2* kv, u32 n, NumTab nt, const double* numv, u32 n_numv, u16* out, u32 kmin, u32 range, u32 cshift, int n_sms,
                                cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms, 256 * RANKTAB_ITEMS);
    pair_ranktab_kernel<<<grid, 256, 0, st>>>(kv, n, nt, numv, n_numv, out, kmin, range, cshift);
}
// typed literal column of a predicate slice: out[i] = num_or0[kv[i].y]; *n_numeric += rows whose object is numeric
static void launch_pair_numcol(const uint2* kv, u32 n, NumTab nt, double* out, u32* n_numeric, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms);
    pair_numcol_kernel<<<grid, 256, 0, st>>>(kv, n, nt, out, n_numeric);
}
// min/max of both halves of a pair relation: out[0..3] = min x, min y, max x, max y
static void launch_pair_minmax(const uint2* kv, u32 n, u32* out4, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms, 256, 4);
    pair_minmax_kernel<<<grid, 256, 0, st>>>(kv, n, out4);
}

// the CSR directory of a grouped join (CsrTab, kb_join.cu) built from an interleaved (subject, object) slice of the store index: key = one
// half, payload = the other half.
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
static void launch_csr_count_pairs(const uint2* kv, u32 key_is_y, u32 n, u32 kmin, u32* counts, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
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
static void launch_csr_fill_pairs(const uint2* kv, u32 key_is_y, u32 n, u32 kmin, u32* cursor, u32* val_out, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    csr_fill_pairs_kernel<<<grid, 256, 0, st>>>(kv, key_is_y, n, kmin, cursor, val_out);
}

// the store's 96-bit (s,p,o) key set
__global__ void __launch_bounds__(256) set_insert_kernel(uint4* set, u32 set_slots, const u32* s, const u32* p, const u32* o, u32 n,
                                                         u32* overflow) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        if (set_insert(set, set_slots, s[i], p[i], o[i]) == 2u) *overflow = 1u;
}
static void launch_set_insert(uint4* set, u32 set_slots, const u32* s, const u32* p, const u32* o, u32 n, u32* overflow, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    set_insert_kernel<<<grid_1d(n, n_sms), 256, 0, st>>>(set, set_slots, s, p, o, n, overflow);
}

// kb_store_delete: p_out[i] = p[i], or EMPTY32 when (s,p,o)[i] is in the delete set; a scan with a variable predicate and
// NE_ID(EMPTY32)... is not needed: the store compaction simply rescans with pattern (?s ?p ?o) over (s, p_out, o) and drops
// rows whose predicate became EMPTY32 (KB_ID_NONE is never a real predicate).
__global__ void __launch_bounds__(256) delete_mark_kernel(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots,
                                                          u32* p_out) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 vp = p[i];
        p_out[i] = set_find(set, set_slots, s[i], vp, o[i]) != EMPTY32 ? EMPTY32 : vp;
    }
}
// mark rows of a segment that equal any triple of a (small) delete set held in a 96-bit set; then compaction is a scan with flags
static void launch_delete_mark(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots, u32* p_out, int n_sms,
                               cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms);
    delete_mark_kernel<<<grid, 256, 0, st>>>(s, p, o, n, set, set_slots, p_out);
}

// ---- kb_store_insert / kb_store_remove: the batch as a key set (the layout of set_insert, so that delete_mark reads it too), the
// batch index of each key's first occurrence, and a found bit per key set by one pass over the store
__global__ void __launch_bounds__(256) batch_set_kernel(uint4* set, u32 set_slots, const u32* s, const u32* p, const u32* o, u32 n, u32* first,
                                                        u32* slot_of, u32* overflow) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        u32 slot = EMPTY32;  // stays EMPTY32 when the set is full
        set_insert_at(set, set_slots, s[i], p[i], o[i], &slot);
        slot_of[i] = slot;
        if (slot == EMPTY32) *overflow = 1u;
        else atomicMin(&first[slot], i);
    }
}
// kb_store_insert / kb_store_remove (kb_store.cu). The batch's keys go into a set laid out as launch_set_insert's (set_slots a power of
// two, zeroed); slot_of[i] = the slot of triple i, first[slot] (set to EMPTY32 before) = the smallest batch index holding that key;
// *overflow = 1 when the set is full
static void launch_batch_set(uint4* set, u32 set_slots, const u32* s, const u32* p, const u32* o, u32 n, u32* first, u32* slot_of, u32* overflow,
                             int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    batch_set_kernel<<<grid, 256, 0, st>>>(set, set_slots, s, p, o, n, first, slot_of, overflow);
}

__global__ void __launch_bounds__(256) batch_mark_kernel(const u32* __restrict__ s, const u32* __restrict__ p, const u32* __restrict__ o, u32 n,
                                                         const uint4* __restrict__ set, u32 set_slots, u32* found, u32* hits) {
    u32 mine = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 slot = set_find(set, set_slots, s[i], p[i], o[i]);
        if (slot != EMPTY32) { found[slot] = 1u; mine++; }
    }
    if (mine) atomicAdd(hits, mine);
}
// one stored segment against the batch set: found[slot] = 1 for every key the segment holds, *hits += its triples that match a key
static void launch_batch_mark(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots, u32* found, u32* hits, int n_sms,
                              cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    batch_mark_kernel<<<grid, 256, 0, st>>>(s, p, o, n, set, set_slots, found, hits);
}

__global__ void __launch_bounds__(256) batch_flags_kernel(u32 n, const u32* slot_of, const u32* first, const u32* found, u32 want_found, u8* flag8,
                                                          u32* flag32, u32* count) {
    u32 mine = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 slot = slot_of[i];
        const bool f = slot != EMPTY32 && first[slot] == i && (found[slot] != 0u) == (want_found != 0u);
        flag8[i] = f ? 1 : 0;
        flag32[i] = f ? 1u : 0u;
        mine += f ? 1u : 0u;
    }
    if (mine) atomicAdd(count, mine);
}
// flag[i] = 1 iff triple i is the first of its key in the batch and found[its slot] equals want_found; *count += the flags set.
// flag8 is what the caller reads back, flag32 what an exclusive scan turns into output positions
static void launch_batch_flags(u32 n, const u32* slot_of, const u32* first, const u32* found, bool want_found, u8* flag8, u32* flag32, u32* count, int n_sms,
                               cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    batch_flags_kernel<<<grid, 256, 0, st>>>(n, slot_of, first, found, want_found ? 1u : 0u, flag8, flag32, count);
}

__global__ void __launch_bounds__(256) batch_gather_kernel(const u32* s, const u32* p, const u32* o, u32 n, const u8* flag8, const u32* pos, u32* out_s,
                                                           u32* out_p, u32* out_o) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (!flag8[i]) continue;
        const u32 k = pos[i];
        out_s[k] = s[i]; out_p[k] = p[i]; out_o[k] = o[i];
    }
}
// out[pos[i]] = triple i for every flagged i (batch order is kept: pos is the exclusive scan of the flags)
static void launch_batch_gather(const u32* s, const u32* p, const u32* o, u32 n, const u8* flag8, const u32* pos, u32* out_s, u32* out_p, u32* out_o, int n_sms,
                                cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    batch_gather_kernel<<<grid, 256, 0, st>>>(s, p, o, n, flag8, pos, out_s, out_p, out_o);
}

// kb_store_remove_template: one triple per (relation row, template pattern); col[t][c] null: position c of pattern t is the constant
// cval[t][c]. bad[0] += the variable cells that are unbound, bad[1] += those whose term would not re-encode to the same id
constexpr u32 TEMPLATE_MAX = 16;
struct TemplateFillParams {
    const u32* col[TEMPLATE_MAX][3];
    u32 cval[TEMPLATE_MAX][3];
    u32 n_tmpl, rows;
    u32 *s, *p, *o;
    DictTab dict;
    u32* bad;
};
// kb_store_remove_template: triple (row r, template pattern t) at r * n_tmpl + t. bad[0] counts unbound cells; bad[1] the cells whose
// term the reference would not re-encode to the same id (execute_query.rs:398-403 decodes every binding and encodes it again with
// encode_term_star): a quoted id (its rendering is re-parsed), an id the device dictionary does not hold, or a string that
// encode_term_star changes: surrounding whitespace, '<' ... '>' (and so "<< ... >>"), a leading '"'
__device__ __forceinline__ bool reencodes_to_itself(u32 id, const DictTab& d) {
    if ((id & 0x80000000u) || id >= d.ids) return false;
    const unsigned long long a = d.off[id], b = d.off[id + 1];
    if (a == b) return true;
    const unsigned char c0 = d.bytes[a], c1 = d.bytes[b - 1];
    // Rust's str::trim: char::is_whitespace (U+0009..U+000D, U+0020, U+0085, U+00A0, U+1680, U+2000..U+200A, U+2028, U+2029, U+202F,
    // U+205F, U+3000) at either end
    const auto ws_cp = [](u32 cp) {
        return (cp >= 0x09 && cp <= 0x0D) || cp == 0x20 || cp == 0x85 || cp == 0xA0 || cp == 0x1680 || (cp >= 0x2000 && cp <= 0x200A) ||
               cp == 0x2028 || cp == 0x2029 || cp == 0x202F || cp == 0x205F || cp == 0x3000;
    };
    const auto cp_at = [&](unsigned long long i, u32 len) {  // the code point of the len-byte UTF-8 sequence at i (EMPTY32: not one)
        if (i + len > b) return EMPTY32;
        const unsigned char x = d.bytes[i];
        u32 cp = len == 1 ? x : len == 2 ? (x & 0x1Fu) : (x & 0x0Fu);
        for (u32 k = 1; k < len; k++) cp = (cp << 6) | (d.bytes[i + k] & 0x3Fu);
        return cp;
    };
    const u32 lead = c0 < 0x80 ? 1u : (c0 & 0xE0) == 0xC0 ? 2u : (c0 & 0xF0) == 0xE0 ? 3u : 4u;
    if (lead <= 3 && ws_cp(cp_at(a, lead))) return false;
    u32 tail = 1;  // the last character starts at the last byte that is not a continuation byte
    while (tail < 4 && tail < b - a && (d.bytes[b - tail] & 0xC0) == 0x80) tail++;
    if (tail <= 3 && ws_cp(cp_at(b - tail, tail))) return false;
    if (c0 == '<' && c1 == '>') return false;
    return c0 != '"';
}
__global__ void __launch_bounds__(256) template_fill_kernel(const __grid_constant__ TemplateFillParams P) {
    const u64 total = (u64)P.rows * P.n_tmpl;
    u32 unbound = 0, changes = 0;
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (u64)gridDim.x * blockDim.x) {
        const u32 r = (u32)(k / P.n_tmpl), t = (u32)(k % P.n_tmpl);
        u32 v[3];
        for (int c = 0; c < 3; c++) {
            const u32* col = P.col[t][c];
            v[c] = col ? col[r] : P.cval[t][c];
            if (!col) continue;
            if (v[c] == EMPTY32) unbound++;
            else if (!reencodes_to_itself(v[c], P.dict)) changes++;
        }
        P.s[k] = v[0]; P.p[k] = v[1]; P.o[k] = v[2];
    }
    if (unbound) atomicAdd(&P.bad[0], unbound);
    if (changes) atomicAdd(&P.bad[1], changes);
}
static void launch_template_fill(const TemplateFillParams& P, int n_sms, cudaStream_t st) {
    const u64 total = (u64)P.rows * P.n_tmpl;
    if (total == 0) return;
    const int grid = grid_1d(total, n_sms);
    template_fill_kernel<<<grid, 256, 0, st>>>(P);
}

kb_status segment_stats(kb_ctx* ctx, Segment* sg) {
    if ((sg->has_stats && sg->stats_world == ctx->shard_world) || sg->n == 0) { sg->has_stats = true; sg->stats_world = ctx->shard_world; return KB_OK; }
    // one pass: column ranges, foreign subjects, distinct predicates + their row counts (segment_profile_kernel)
    const u32 off = ctrl_alloc(ctx, SEGP_WORDS);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0xFF, SEGP_MAX * sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off + SEGP_MAX, 0, (SEGP_WORDS - SEGP_MAX) * sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER);
    launch_segment_profile(sg->s.ptr, sg->p.ptr, sg->o.ptr, (u32)sg->n, ctx->shard_rank, ctx->shard_world, ctx->ctrl + off, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32* h = ctx->h_ctrl + off;
    for (int c = 0; c < 3; c++) { sg->cmin[c] = h[SEGP_MIN + c]; sg->cmax[c] = h[SEGP_MAX + c]; }
    sg->sharded_ok = h[SEGP_FOREIGN] == 0;  // key compaction is only sound when every subject is ours
    sg->pred_rows.clear();
    sg->preds_overflow = h[SEGP_OVERFLOW] != 0;
    sg->has_preds = true;
    if (!sg->preds_overflow) {
        for (u32 i = 0; i < SEGP_SLOTS; i++) if (h[SEGP_SLOT + i] != EMPTY32) sg->pred_rows.push_back({h[SEGP_SLOT + i], h[SEGP_COUNT + i]});
        std::sort(sg->pred_rows.begin(), sg->pred_rows.end());
    }
    sg->stats_world = ctx->shard_world;
    sg->has_stats = true;
    return KB_OK;
}

kb_status refuse_reserved_id(kb_ctx* ctx, const u32 cmax[3]) {
    static const char* const pos[3] = {"subject", "predicate", "object"};
    for (int c = 0; c < 3; c++)
        if (cmax[c] == KB_ID_NONE) return fail(ctx, KB_E_INVALID, "a triple's %s is 0xFFFFFFFF, which is reserved (KB_ID_NONE)", pos[c]);
    return KB_OK;
}

// ---- store index, one chunk per (predicate, store segment)
// the rank column of a slice's subject table: xkey[compact(subject) - xtab_min] = rank of the object's value in the value order (slots
// without a key are never read: they stay unset)
static kb_status build_rank_column(kb_ctx* ctx, PredSlice& ps) {
    bool ok = false;
    KB_TRY(ensure_num_order(ctx, &ok));
    if (!ok) return KB_OK;
    KB_TRY(alloc_buf(ctx, (size_t)ps.xtab_range * sizeof(u16), &ps.xkey));
    for (auto& ch : ps.chunks) {
        if (!ch.n) continue;
        launch_pair_ranktab(reinterpret_cast<const uint2*>(ch.pairs.ptr), (u32)ch.n, numtab(ctx), static_cast<const double*>(ctx->numv->p),
                            (u32)ctx->h_numv.size(), static_cast<u16*>(ps.xkey->p), ps.xtab_min, ps.xtab_range, ps.tab_cshift, ctx->n_sms, ctx->st);
        ctx->stats.kernel_launches++;
    }
    ps.xkey_version = ctx->num_version;
    return KB_OK;
}

// the one-byte codes of every subject table that holds at most CODE_MAX distinct objects (PredSlice::xcode): one distinct pass per
// table, which ends early past CODE_MAX values, one read-back for all of them, the dictionaries sorted here (codes ascend with the
// object ids), one code pass per coded table
static kb_status build_subject_codes(kb_ctx* ctx) {
    constexpr u32 SLOTS = 512;  // the distinct set: at most half full below the limit
    std::vector<PredSlice*> tabs;
    for (auto& kv : ctx->index) if (kv.second.xtab) tabs.push_back(&kv.second);
    if (tabs.empty()) return KB_OK;
    const size_t n = tabs.size();  // <= 4096 slices: 2 control words each fit the arena
    Buf sets;
    KB_TRY(alloc_buf(ctx, n * SLOTS * sizeof(u32), &sets));
    KB_CUDA(ctx, cudaMemsetAsync(sets->p, 0xFF, n * SLOTS * sizeof(u32), ctx->st));
    const u32 off = ctrl_alloc(ctx, 2 * (u32)n);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 2 * n * sizeof(u32), ctx->st));
    for (size_t i = 0; i < n; i++) {
        launch_distinct(static_cast<const u32*>(tabs[i]->xtab->p), tabs[i]->xtab_range, static_cast<u32*>(sets->p) + i * SLOTS, SLOTS, CODE_MAX,
                        ctx->ctrl + off + 2 * i, ctx->n_sms, ctx->st);
        ctx->stats.kernel_launches++;
    }
    KB_CUDA(ctx, cudaGetLastError());
    std::vector<u32> h(n * SLOTS);
    KB_CUDA(ctx, cudaMemcpyAsync(h.data(), sets->p, n * SLOTS * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    ctx->stats.d2h_bytes += n * SLOTS * sizeof(u32);
    KB_TRY(ctrl_read(ctx));
    for (size_t i = 0; i < n; i++) {
        if (ctx->h_ctrl[off + 2 * i]) continue;  // more than CODE_MAX objects
        std::vector<u32> dict;
        for (u32 k = 0; k < SLOTS; k++) if (h[i * SLOTS + k] != EMPTY32) dict.push_back(h[i * SLOTS + k]);
        if (dict.empty()) continue;
        std::sort(dict.begin(), dict.end());
        PredSlice& ps = *tabs[i];
        KB_TRY(alloc_buf(ctx, dict.size() * sizeof(u32), &ps.xdict));
        KB_CUDA(ctx, cudaMemcpyAsync(ps.xdict->p, dict.data(), dict.size() * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
        ctx->stats.h2d_bytes += dict.size() * sizeof(u32);
        KB_TRY(alloc_buf(ctx, ps.xtab_range, &ps.xcode));
        launch_tab_code(static_cast<const u32*>(ps.xtab->p), ps.xtab_range, static_cast<const u32*>(ps.xdict->p), (u32)dict.size(),
                        static_cast<u8*>(ps.xcode->p), ctx->n_sms, ctx->st);
        ctx->stats.kernel_launches++;
        ps.n_xdict = (u32)dict.size();
    }
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

// (re)build or extend the persistent table of one column of a slice after `added` (index into ps.chunks; -1: all chunks) arrived.
// flag_word: control word the insert kernels raise on a duplicate key. Returns through *touched whether a flag has to be read.
// full_build: called by kb_store_build_index, which builds the rank columns itself once every chunk is in.
static kb_status slice_table_update(kb_ctx* ctx, PredSlice& ps, u32 y, int added, u32 cshift, u32 flag_off, bool full_build, bool* touched) {
    Buf& tab = y ? ps.ytab : ps.xtab;
    u32& tmin = y ? ps.ytab_min : ps.xtab_min;
    u32& tcap = y ? ps.ytab_range : ps.xtab_range;
    bool& tried = y ? ps.y_tried : ps.x_tried;
    bool& unique = y ? ps.y_unique : ps.x_unique;
    *touched = false;
    if (tried && !tab) return KB_OK;  // the column was found multi-valued or too sparse: no table, nothing to maintain
    const u32 cs = y ? 0u : cshift;    // only subjects are sharded
    const u32 lo = compact_key(y ? ps.ymin : ps.xmin, cs), hi = compact_key(y ? ps.ymax : ps.xmax, cs);
    const u64 range = (u64)hi - lo + 1;
    const bool fits = tab && lo >= tmin && (u64)hi < (u64)tmin + tcap && (y || ps.tab_cshift == cshift);
    if (!fits) {
        // (re)build over every chunk, with headroom above the largest key: dictionary ids grow, so appended segments bring larger ones
        tab.reset();
        if (!y) ps.xkey.reset();
        tried = true;
        unique = false;
        if (range > std::max<u64>(4 * ps.n + 65536, 1ull << 16) || range > (1ull << 28)) return KB_OK;  // not dense: keep no table
        // headroom: half the range for large tables, twice the range for small ones (a sliding window's ids move up by a slide per
        // slide: a 10-slide window then re-bases its tables every ~20 slides instead of every ~5)
        const u64 cap = std::min<u64>(range + (range <= (4ull << 20) ? 2 * range : range / 2) + 65536, 1ull << 29);
        KB_TRY(alloc_buf(ctx, cap * sizeof(u32), &tab));
        KB_CUDA(ctx, cudaMemsetAsync(tab->p, 0xFF, cap * sizeof(u32), ctx->st));
        tmin = lo;
        tcap = (u32)cap;
        if (!y) ps.tab_cshift = cshift;
        added = -1;
        unique = true;  // until a flag says otherwise
    }
    for (size_t c = 0; c < ps.chunks.size(); c++) {
        if (added >= 0 && (int)c != added) continue;
        const SliceChunk& ch = ps.chunks[c];
        if (!ch.n) continue;
        launch_build_direct_pairs(reinterpret_cast<const uint2*>(ch.pairs.ptr), y, (u32)ch.n, static_cast<u32*>(tab->p), tmin, tcap, cs, ctx->ctrl + flag_off, 0u,
                                  ctx->n_sms, ctx->st);
        ctx->stats.kernel_launches++;
        *touched = true;
    }
    // a subject table rebuilt outside the full build takes its rank column along (the table-mode probe filters on it)
    if (!y && !fits && !full_build && ctx->n_ids && ps.typed(ctx->num_version)) KB_TRY(build_rank_column(ctx, ps));
    return KB_OK;
}

// index the triples of ONE store segment: a chunk per predicate it carries, ranges, persistent tables, typed literal columns
// the slide-sized case of index_add_segment: the segment's predicates and their row counts are known from its profile pass, so the
// chunks are allocated exactly and ONE kernel files every triple (segment_split_kernel); one read-back
static kb_status index_add_segment_split(kb_ctx* ctx, const Segment& sg, u32 cshift) {
    const u32 k = (u32)sg.pred_rows.size();
    SplitParams P{};
    P.s = sg.s.ptr; P.p = sg.p.ptr; P.o = sg.o.ptr;
    P.n = (u32)sg.n;
    P.k = k;
    P.nt = numtab(ctx);
    const u32 off = ctrl_alloc(ctx, k * SPLIT_WORDS);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, k * SPLIT_WORDS * sizeof(u32), ctx->st));
    P.ctrl = ctx->ctrl + off;
    std::vector<SliceChunk> chs(k);
    bool rebuild[MAXP][2];
    for (u32 i = 0; i < k; i++) {
        PredSlice& ps = ctx->index[sg.pred_rows[i].first];
        SliceChunk& ch = chs[i];
        ch.tag = sg.tag;
        ch.seg = sg.id;
        ch.n = sg.pred_rows[i].second;
        KB_TRY(alloc_col(ctx, 2 * ch.n, &ch.pairs));
        if (ctx->n_ids) KB_TRY(alloc_buf(ctx, ch.n * sizeof(double), &ch.ynum));
        SplitEntry& e = P.e[i];
        e.pred = sg.pred_rows[i].first;
        e.n = (u32)ch.n;
        e.pairs = reinterpret_cast<uint2*>(ch.pairs.ptr);
        e.ynum = ch.ynum ? static_cast<double*>(ch.ynum->p) : nullptr;
        const bool xok = ps.xtab && ps.tab_cshift == cshift;
        rebuild[i][0] = ps.xtab ? !xok : !ps.x_tried;
        rebuild[i][1] = !ps.ytab && !ps.y_tried;
        if (xok) { e.xtab = static_cast<u32*>(ps.xtab->p); e.xtab_min = ps.xtab_min; e.xtab_range = ps.xtab_range; e.cshift = cshift; }
        if (xok && ps.xkey && ps.xkey_version == ctx->num_version && ctx->numv_version == ctx->num_version && ctx->n_ids) {
            e.xkey = static_cast<u16*>(ps.xkey->p);
            P.numv = static_cast<const double*>(ctx->numv->p);
            P.n_numv = (u32)ctx->h_numv.size();
        } else ps.xkey.reset();
        if (ps.ytab) { e.ytab = static_cast<u32*>(ps.ytab->p); e.ytab_min = ps.ytab_min; e.ytab_range = ps.ytab_range; }
    }
    timer_begin(ctx, F_OTHER);
    launch_segment_split(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches++;
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32 uoff = ctrl_alloc(ctx, 2 * MAXP);
    bool any_touched = false;
    std::vector<char> touched(2 * k, 0);
    std::vector<int> chunk_of(k, -1);
    for (u32 i = 0; i < k; i++) {
        const u32* h = ctx->h_ctrl + off + i * SPLIT_WORDS;
        PredSlice& ps = ctx->index[sg.pred_rows[i].first];
        SliceChunk& ch = chs[i];
        if (h[SPLIT_CURSOR] != ch.n) return fail(ctx, KB_E_CUDA, "index maintenance: predicate %u has %u rows, its profile said %llu", sg.pred_rows[i].first,
                                                  h[SPLIT_CURSOR], (unsigned long long)ch.n);
        ch.xmin = ~h[SPLIT_XMIN]; ch.ymin = ~h[SPLIT_YMIN]; ch.xmax = h[SPLIT_XMAX]; ch.ymax = h[SPLIT_YMAX];
        if (ch.ynum && h[SPLIT_NNUM] > 0) ch.ynum_version = ctx->num_version;
        else { ch.ynum.reset(); ps.xkey.reset(); }
        ps.xmin = std::min(ps.xmin, ch.xmin); ps.ymin = std::min(ps.ymin, ch.ymin);
        ps.xmax = std::max(ps.xmax, ch.xmax); ps.ymax = std::max(ps.ymax, ch.ymax);
        chunk_of[i] = (int)ps.chunks.size();
        ps.chunks.push_back(ch);
        ps.n += ch.n;
        if (ps.chunks.size() > 1) { ps.xoff.reset(); ps.xval.reset(); ps.yoff.reset(); ps.yval.reset(); }  // the directories describe one chunk
        if (h[SPLIT_XDUP]) { ps.x_unique = false; ps.xtab.reset(); ps.xkey.reset(); }  // a subject occurs twice
        if (h[SPLIT_YDUP]) { ps.y_unique = false; ps.ytab.reset(); }
        if (h[SPLIT_XOUT] && ps.xtab) rebuild[i][0] = true;  // a key outside the table: rebuild it over every chunk, with new headroom
        if (h[SPLIT_YOUT] && ps.ytab) rebuild[i][1] = true;
    }
    for (u32 i = 0; i < k; i++) {
        PredSlice& ps = ctx->index[sg.pred_rows[i].first];
        for (u32 y = 0; y < 2; y++) {
            if (!rebuild[i][y]) continue;
            if (!any_touched) { KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + uoff, 0, 2 * MAXP * sizeof(u32), ctx->st)); any_touched = true; }
            Buf& tab = y ? ps.ytab : ps.xtab;
            tab.reset();  // slice_table_update sees no table: a rebuild over all chunks (the new one included)
            if (y) ps.y_tried = false; else ps.x_tried = false;
            bool t = false;
            KB_TRY(slice_table_update(ctx, ps, y, chunk_of[i], cshift, uoff + 2 * i + y, /*full_build=*/false, &t));
            touched[2 * i + y] = t ? 1 : 0;
        }
    }
    if (any_touched) {
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        for (u32 i = 0; i < k; i++) {
            PredSlice& ps = ctx->index[sg.pred_rows[i].first];
            if (touched[2 * i] && ctx->h_ctrl[uoff + 2 * i]) { ps.x_unique = false; ps.xtab.reset(); }
            if (touched[2 * i + 1] && ctx->h_ctrl[uoff + 2 * i + 1]) { ps.y_unique = false; ps.ytab.reset(); }
        }
    }
    return KB_OK;
}

// full_build: kb_store_build_index indexes the store segment by segment
static kb_status index_add_segment(kb_ctx* ctx, size_t seg_idx, bool full_build, bool* indexable) {
    *indexable = true;
    Segment sg = ctx->segs[seg_idx];
    if (sg.n == 0) return KB_OK;
    static const bool split_ok = !(getenv("KOLIBRIE_INDEX_SPLIT") && getenv("KOLIBRIE_INDEX_SPLIT")[0] == '0');
    if (split_ok && !full_build && sg.has_stats && sg.stats_world == ctx->shard_world && sg.has_preds && !sg.preds_overflow &&
        sg.pred_rows.size() <= MAXP) {
        size_t n_new = 0;
        for (auto& pr : sg.pred_rows) n_new += ctx->index.count(pr.first) ? 0 : 1;
        if (ctx->index.size() + n_new <= 4096) {
            u32 cshift = 0;  // subject-sharded store: compact the subject keys (see compact_key)
            bool sharded = ctx->shard_world > 1 && (ctx->shard_world & (ctx->shard_world - 1)) == 0;
            for (auto& g : ctx->segs) if (g.n && g.has_stats && !g.sharded_ok) sharded = false;
            if (sharded) while ((1u << cshift) < ctx->shard_world) cshift++;
            return index_add_segment_split(ctx, sg, cshift);
        }
    }
    // 1. distinct predicates of the segment
    const u32 set_slots = 8192;
    Buf set;
    KB_TRY(alloc_buf(ctx, set_slots * sizeof(u32), &set));
    KB_CUDA(ctx, cudaMemsetAsync(set->p, 0xFF, set_slots * sizeof(u32), ctx->st));
    const u32 off = ctrl_alloc(ctx, 4);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 4 * sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER);
    launch_distinct(sg.p.ptr, (u32)sg.n, static_cast<u32*>(set->p), set_slots, set_slots, ctx->ctrl + off, ctx->n_sms, ctx->st);
    timer_end(ctx);
    std::vector<u32> hset(set_slots);
    KB_CUDA(ctx, cudaMemcpyAsync(hset.data(), set->p, set_slots * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    KB_TRY(ctrl_read(ctx));
    std::vector<u32> preds;
    for (u32 v : hset) if (v != EMPTY32) preds.push_back(v);
    std::sort(preds.begin(), preds.end());
    {
        std::set<u32> all(preds.begin(), preds.end());
        for (auto& kv : ctx->index) all.insert(kv.first);
        if (ctx->h_ctrl[off] || all.size() > 4096) { *indexable = false; return KB_OK; }  // too many predicates: keep scanning
    }
    if (!sg.has_stats || sg.stats_world != ctx->shard_world) { KB_TRY(segment_stats(ctx, &ctx->segs[seg_idx])); sg = ctx->segs[seg_idx]; }
    u32 cshift = 0;  // subject-sharded store: compact the subject keys (see compact_key)
    {
        bool sharded = ctx->shard_world > 1 && (ctx->shard_world & (ctx->shard_world - 1)) == 0;
        for (auto& g : ctx->segs) if (g.n && g.has_stats && !g.sharded_ok) sharded = false;
        if (sharded) while ((1u << cshift) < ctx->shard_world) cshift++;
    }
    // 2. one fused scan of THIS segment per 8 predicates, pair output, shrunk to a chunk; id ranges of both halves
    const std::vector<Segment> one{sg};
    for (size_t b = 0; b < preds.size(); b += MAXP) {
        const u32 k = (u32)std::min<size_t>(MAXP, preds.size() - b);
        std::vector<std::unique_ptr<kb_rel>> rels;
        KB_TRY(scan_predicates(ctx, one, preds.data() + b, k, ScanOut::Pairs, &rels));
        const u32 soff = ctrl_alloc(ctx, 4 * MAXP);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + soff, 0, 4 * MAXP * sizeof(u32), ctx->st));
        for (u32 i = 0; i < k; i++) KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + soff + 4 * i, 0xFF, 2 * sizeof(u32), ctx->st));
        std::vector<int> chunk_of(k, -1);
        for (u32 i = 0; i < k; i++) {
            if (rels[i]->n == 0) continue;
            PredSlice& ps = ctx->index[preds[b + i]];
            SliceChunk ch;
            ch.tag = sg.tag;
            ch.seg = sg.id;
            ch.n = rels[i]->n;
            KB_TRY(alloc_col(ctx, 2 * ch.n, &ch.pairs));
            KB_CUDA(ctx, cudaMemcpyAsync(ch.pairs.ptr, rels[i]->cols[0].ptr, ch.n * sizeof(uint2), cudaMemcpyDeviceToDevice, ctx->st));
            launch_pair_minmax(reinterpret_cast<const uint2*>(ch.pairs.ptr), (u32)ch.n, ctx->ctrl + soff + 4 * i, ctx->n_sms, ctx->st);
            ctx->stats.kernel_launches++;
            chunk_of[i] = (int)ps.chunks.size();
            ps.chunks.push_back(ch);
            ps.n += ch.n;
            if (ps.chunks.size() > 1) { ps.xoff.reset(); ps.xval.reset(); ps.yoff.reset(); ps.yval.reset(); }  // the directories describe one chunk
            if (!full_build) ps.xkey.reset();  // (kept in table order by the full build only)
        }
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        // 3. persistent tables (inserted in place; a duplicate key or a key outside the table ends / rebuilds it) and the typed literal
        //    column of the new chunk: the f64 value of every object, so that FILTER(?o <cmp> c) reads it sequentially instead of
        //    gathering num_or0[object] at random
        const u32 uoff = ctrl_alloc(ctx, 2 * MAXP);
        const u32 noff = ctrl_alloc(ctx, MAXP);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + uoff, 0, 2 * MAXP * sizeof(u32), ctx->st));
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + noff, 0, MAXP * sizeof(u32), ctx->st));
        std::vector<char> touched(2 * k, 0);
        for (u32 i = 0; i < k; i++) {
            if (chunk_of[i] < 0) continue;
            PredSlice& ps = ctx->index[preds[b + i]];
            {
                SliceChunk& ch = ps.chunks[chunk_of[i]];
                ch.xmin = ctx->h_ctrl[soff + 4 * i]; ch.ymin = ctx->h_ctrl[soff + 4 * i + 1];
                ch.xmax = ctx->h_ctrl[soff + 4 * i + 2]; ch.ymax = ctx->h_ctrl[soff + 4 * i + 3];
                ps.xmin = std::min(ps.xmin, ch.xmin); ps.ymin = std::min(ps.ymin, ch.ymin);
                ps.xmax = std::max(ps.xmax, ch.xmax); ps.ymax = std::max(ps.ymax, ch.ymax);
            }
            for (u32 y = 0; y < 2; y++) {
                bool t = false;
                KB_TRY(slice_table_update(ctx, ps, y, chunk_of[i], cshift, uoff + 2 * i + y, full_build, &t));
                touched[2 * i + y] = t ? 1 : 0;
            }
            if (ctx->n_ids) {
                SliceChunk& ch = ps.chunks[chunk_of[i]];
                KB_TRY(alloc_buf(ctx, ch.n * sizeof(double), &ch.ynum));
                launch_pair_numcol(reinterpret_cast<const uint2*>(ch.pairs.ptr), (u32)ch.n, numtab(ctx), static_cast<double*>(ch.ynum->p), ctx->ctrl + noff + i,
                                   ctx->n_sms, ctx->st);
                ctx->stats.kernel_launches++;
            }
        }
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        for (u32 i = 0; i < k; i++) {
            if (chunk_of[i] < 0) continue;
            PredSlice& ps = ctx->index[preds[b + i]];
            SliceChunk& ch = ps.chunks[chunk_of[i]];
            if (ch.ynum && ctx->h_ctrl[noff + i] > 0) ch.ynum_version = ctx->num_version;
            else ch.ynum.reset();
            if (touched[2 * i] && ctx->h_ctrl[uoff + 2 * i]) { ps.x_unique = false; ps.xtab.reset(); }      // a subject occurs twice
            if (touched[2 * i + 1] && ctx->h_ctrl[uoff + 2 * i + 1]) { ps.y_unique = false; ps.ytab.reset(); }
        }
    }
    return KB_OK;
}

// eviction of the chunks `dies` selects (those of the segments tagged `tag`, or of given segments): they leave the slices, their keys
// leave the persistent tables
template <class Dies>
static kb_status index_evict(kb_ctx* ctx, Dies dies) {
    ClearParams C{};
    std::vector<SliceChunk> dying;  // kept until the clears are queued: their buffers are released stream-ordered behind them
    auto flush = [&]() {
        if (C.k) { launch_clear_chunks(C, ctx->n_sms, ctx->st); ctx->stats.kernel_launches++; }
        C.k = 0;
    };
    for (auto it = ctx->index.begin(); it != ctx->index.end();) {
        PredSlice& ps = it->second;
        bool hit = false;
        for (size_t c = 0; c < ps.chunks.size();) {
            SliceChunk& ch = ps.chunks[c];
            if (!dies(ch)) { c++; continue; }
            hit = true;
            if ((ps.xtab || ps.ytab) && ch.n) {
                ClearEntry& e = C.e[C.k++];
                e = ClearEntry{};
                e.pairs = reinterpret_cast<const uint2*>(ch.pairs.ptr);
                e.n = (u32)ch.n;
                if (ps.xtab) { e.xtab = static_cast<u32*>(ps.xtab->p); e.xtab_min = ps.xtab_min; e.xtab_range = ps.xtab_range; e.cshift = ps.tab_cshift; }
                if (ps.ytab) { e.ytab = static_cast<u32*>(ps.ytab->p); e.ytab_min = ps.ytab_min; e.ytab_range = ps.ytab_range; }
                if (C.k == CLEAR_MAX) flush();
            }
            ps.n -= ch.n;
            dying.push_back(ch);
            ps.chunks.erase(ps.chunks.begin() + c);
            ps.xoff.reset(); ps.xval.reset(); ps.yoff.reset(); ps.yval.reset();  // (xkey stays: its slots are only read where xtab holds a key)
        }
        if (hit) {  // the slice's id ranges shrink to the surviving chunks': a long-running window does not walk its whole past
            ps.xmin = ps.ymin = 0xFFFFFFFFu;
            ps.xmax = ps.ymax = 0u;
            for (auto& ch : ps.chunks) {
                ps.xmin = std::min(ps.xmin, ch.xmin); ps.ymin = std::min(ps.ymin, ch.ymin);
                ps.xmax = std::max(ps.xmax, ch.xmax); ps.ymax = std::max(ps.ymax, ch.ymax);
            }
        }
        if (ps.chunks.empty()) it = ctx->index.erase(it);
        else ++it;
    }
    flush();
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

// ---- changes to the store: the only code that writes ctx->segs, n_triples, store_version, the hint sets and the index
static bool index_maintainable(const kb_ctx* ctx) {
    return ctx->index_maintain && ctx->index_version == ctx->store_version && !ctx->index.empty();
}
// a new store version: everything keyed to the old one is void, and what the star-join builds learnt about its predicates is forgotten.
// The subject codes go too: they are built by kb_store_build_index only, never maintained.
static void bump_version(kb_ctx* ctx) {
    ctx->store_version++;
    ctx->multi_valued.clear();
    ctx->single_valued.clear();
    for (auto& kv : ctx->index) {
        kv.second.xcode.reset();
        kv.second.xdict.reset();
        kv.second.n_xdict = 0;
    }
}
static void drop_index(kb_ctx* ctx) {
    ctx->index.clear();
    ctx->index_version = ~0ull;
}

void store_replace(kb_ctx* ctx, std::vector<Segment> segs) {
    ctx->segs = std::move(segs);
    for (auto& sg : ctx->segs) sg.id = ++ctx->seg_ids;
    ctx->n_triples = 0;
    for (auto& sg : ctx->segs) ctx->n_triples += sg.n;
    bump_version(ctx);
    drop_index(ctx);  // a replaced store: nothing to maintain
}

kb_status store_add_device_segment(kb_ctx* ctx, Segment& sg, bool keep_index) {
    if (keep_index && sg.n && !sg.has_stats) KB_TRY(segment_stats(ctx, &sg));
    const bool maintain = keep_index && index_maintainable(ctx);
    sg.id = ++ctx->seg_ids;
    ctx->segs.push_back(sg);
    ctx->n_triples += sg.n;
    bump_version(ctx);
    if (maintain) {
        // the index stays alive across the mutation: the new segment becomes one more chunk of every predicate slice it touches and
        // its keys are inserted into the persistent tables in place (an RSP window slide keeps the one-kernel index path)
        bool indexable = true;
        const kb_status rc = index_add_segment(ctx, ctx->segs.size() - 1, /*full_build=*/false, &indexable);
        if (rc == KB_OK && indexable) { ctx->index_version = ctx->store_version; return KB_OK; }
        drop_index(ctx);
        return rc;
    }
    drop_index(ctx);  // the predicate-partitioned index describes the previous store version
    return KB_OK;
}

bool store_evict_tag(kb_ctx* ctx, u64 tag, bool keep_index) {
    bool found = false;
    for (size_t i = 0; i < ctx->segs.size();) {
        if (ctx->segs[i].tag == tag) {
            ctx->n_triples -= ctx->segs[i].n;
            ctx->segs.erase(ctx->segs.begin() + i);
            found = true;
        } else i++;
    }
    const bool maintain = keep_index && index_maintainable(ctx);
    bump_version(ctx);
    if (maintain && index_evict(ctx, [tag](const SliceChunk& ch) { return ch.tag == tag; }) == KB_OK) ctx->index_version = ctx->store_version;
    else drop_index(ctx);
    return found;
}

// one new store version in which the segments at `out` (indices into ctx->segs) are replaced by `in` (empty ones are left out). The
// index is maintained when it describes the store: the chunks of the replaced segments leave it as an eviction's do and every new
// segment comes in as a slide's does; a slice it cannot maintain drops the whole index.
static kb_status store_swap(kb_ctx* ctx, std::vector<size_t> out, std::vector<Segment> in) {
    for (auto& sg : in) if (sg.n && !sg.has_stats) KB_TRY(segment_stats(ctx, &sg));
    bool maintain = index_maintainable(ctx);
    std::set<u64> gone;
    std::sort(out.rbegin(), out.rend());
    for (size_t i : out) {
        gone.insert(ctx->segs[i].id);
        ctx->n_triples -= ctx->segs[i].n;
        ctx->segs.erase(ctx->segs.begin() + i);
    }
    bump_version(ctx);
    kb_status rc = KB_OK;
    if (maintain && !gone.empty()) maintain = index_evict(ctx, [&gone](const SliceChunk& ch) { return gone.count(ch.seg) != 0; }) == KB_OK;
    for (auto& sg : in) {
        if (!sg.n) continue;
        sg.id = ++ctx->seg_ids;
        ctx->segs.push_back(sg);
        ctx->n_triples += sg.n;
        if (!maintain) continue;
        bool indexable = true;
        rc = index_add_segment(ctx, ctx->segs.size() - 1, /*full_build=*/false, &indexable);
        maintain = rc == KB_OK && indexable;
    }
    if (maintain) ctx->index_version = ctx->store_version;
    else drop_index(ctx);
    return rc;
}

// the triples of `sg` that are not in the 96-bit set (kb_store_delete's compaction): a copy of the predicate column with KB_ID_NONE
// where a triple is in the set, then a rescan with (?s ?p ?o) — a row whose predicate is KB_ID_NONE can never equal a real constant,
// and the pattern's pushed-down filter NE_ID drops it
static kb_status segment_without(kb_ctx* ctx, const Segment& sg, const Buf& set, u32 set_slots, Segment* out) {
    static const kb_pattern pt{{1, 0}, {1, 1}, {1, 2}};
    FilterProg keep;
    kb_filter_op ne{};
    ne.op = KB_F_NE_ID; ne.slot = 1; ne.id = KB_ID_NONE;  // true for every bound predicate; a marked one reads as unbound: false
    keep.ops.push_back(ne);
    const std::vector<FilterProg> pd{keep};
    Segment marked = sg;
    if (sg.n) {
        KB_TRY(alloc_col(ctx, sg.n, &marked.p));
        launch_delete_mark(sg.s.ptr, sg.p.ptr, sg.o.ptr, (u32)sg.n, static_cast<const uint4*>(set->p), set_slots, marked.p.ptr, ctx->n_sms, ctx->st);
    }
    std::vector<std::unique_ptr<kb_rel>> rels;
    KB_TRY(scan_segments(ctx, {marked}, &pt, 1, pd, ScanOut::Cols, &rels));
    *out = Segment{};
    out->tag = sg.tag;
    out->n = rels[0]->n;
    out->s = rels[0]->cols[0]; out->p = rels[0]->cols[1]; out->o = rels[0]->cols[2];
    return KB_OK;
}

// ---- set-semantic writes (kb_store_insert, kb_store_remove, kb_store_remove_template) over a batch in device memory
// the batch's key set has a power of two >= 2n slots and pow2_at_least stops at 2^31: larger batches are refused up front
constexpr u64 BATCH_MAX = 1ull << 30;
struct BatchMark {
    Buf set, first, slot_of, found, flag8, flag32;
    u32 slots = 0, n = 0;
    u32 n_flagged = 0;                // triples of the batch the call acts on
    std::vector<u32> seg_hits;        // per segment of ctx->segs: its triples that equal a key of the batch
};

// The batch's key set, one mark pass over every segment, and the per-triple flags: want_found = false flags each triple that is in
// neither the store nor an earlier entry of the batch (BTreeSet::insert), true each that is in the store and not earlier in the batch
// (BTreeSet::remove).
static kb_status batch_mark(kb_ctx* ctx, const u32* s, const u32* p, const u32* o, u32 n, bool want_found, BatchMark* b) {
    b->n = n;
    b->slots = pow2_at_least((u64)n * 2);
    KB_TRY(alloc_buf(ctx, (size_t)b->slots * sizeof(uint4), &b->set));
    KB_TRY(alloc_buf(ctx, (size_t)b->slots * sizeof(u32), &b->first));
    KB_TRY(alloc_buf(ctx, (size_t)b->slots * sizeof(u32), &b->found));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &b->slot_of));
    KB_TRY(alloc_buf(ctx, (size_t)n, &b->flag8));
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &b->flag32));
    KB_CUDA(ctx, cudaMemsetAsync(b->set->p, 0, (size_t)b->slots * sizeof(uint4), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(b->first->p, 0xFF, (size_t)b->slots * sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(b->found->p, 0, (size_t)b->slots * sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(static_cast<u32*>(b->flag32->p) + n, 0, sizeof(u32), ctx->st));
    const size_t nseg = ctx->segs.size();
    Buf hits;
    KB_TRY(alloc_buf(ctx, (nseg + 1) * sizeof(u32), &hits));
    KB_CUDA(ctx, cudaMemsetAsync(hits->p, 0, (nseg + 1) * sizeof(u32), ctx->st));
    const u32 c = ctrl_alloc(ctx, 2);  // [0] set overflow, [1] flagged triples
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 2 * sizeof(u32), ctx->st));
    int launches = 2;  // the set and the flags, and one mark pass per non-empty segment
    for (auto& sg : ctx->segs) launches += sg.n ? 1 : 0;
    timer_begin(ctx, F_OTHER, launches);
    launch_batch_set(static_cast<uint4*>(b->set->p), b->slots, s, p, o, n, static_cast<u32*>(b->first->p), static_cast<u32*>(b->slot_of->p), ctx->ctrl + c,
                     ctx->n_sms, ctx->st);
    for (size_t g = 0; g < nseg; g++) {
        const Segment& sg = ctx->segs[g];
        if (sg.ready) KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, sg.ready, 0));
        launch_batch_mark(sg.s.ptr, sg.p.ptr, sg.o.ptr, (u32)sg.n, static_cast<const uint4*>(b->set->p), b->slots, static_cast<u32*>(b->found->p),
                          static_cast<u32*>(hits->p) + g, ctx->n_sms, ctx->st);
    }
    launch_batch_flags(n, static_cast<const u32*>(b->slot_of->p), static_cast<const u32*>(b->first->p), static_cast<const u32*>(b->found->p), want_found,
                       static_cast<u8*>(b->flag8->p), static_cast<u32*>(b->flag32->p), ctx->ctrl + c + 1, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    b->seg_hits.assign(nseg, 0);
    if (nseg) KB_CUDA(ctx, cudaMemcpyAsync(b->seg_hits.data(), hits->p, nseg * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    KB_TRY(ctrl_read(ctx));  // (synchronises the stream: seg_hits has arrived too)
    if (ctx->h_ctrl[c]) return fail(ctx, KB_E_CUDA, "update batch set overflow");
    b->n_flagged = ctx->h_ctrl[c + 1];
    return KB_OK;
}

static kb_status batch_flags_out(kb_ctx* ctx, const BatchMark& b, uint8_t* flags) {
    if (!flags || !b.n) return KB_OK;
    KB_CUDA(ctx, cudaMemcpyAsync(flags, b.flag8->p, b.n, cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += b.n;
    return KB_OK;
}

// kb_store_insert over a batch in device memory
static kb_status store_insert_device(kb_ctx* ctx, const u32* s, const u32* p, const u32* o, u32 n, u64 tag, uint8_t* inserted, uint64_t* n_inserted) {
    BatchMark b;
    KB_TRY(batch_mark(ctx, s, p, o, n, /*want_found=*/false, &b));
    const u32 n_new = b.n_flagged;
    if (ctx->n_triples + n_new >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "store would exceed 2^32-16 triples");
    KB_TRY(batch_flags_out(ctx, b, inserted));
    if (n_inserted) *n_inserted = n_new;
    if (n_new == 0) return KB_OK;  // nothing changes: no new version
    // geometric merge: the new triples absorb the latest segments of the same tag while each holds at most twice what is gathered so
    // far, so that a run of small inserts leaves O(log n) segments and every triple is copied O(log n) times
    std::vector<size_t> absorbed;
    u64 total = n_new;
    for (size_t g = ctx->segs.size(); g-- > 0;) {
        const Segment& sg = ctx->segs[g];
        if (sg.tag != tag || sg.ready) continue;
        if (sg.n > 2 * total) break;
        absorbed.push_back(g);
        total += sg.n;
    }
    Segment ns;
    ns.tag = tag;
    ns.n = total;
    KB_TRY(alloc_col(ctx, total, &ns.s));
    KB_TRY(alloc_col(ctx, total, &ns.p));
    KB_TRY(alloc_col(ctx, total, &ns.o));
    u64 at = 0;
    for (size_t k = absorbed.size(); k-- > 0;) {  // the absorbed segments in store order, then the new triples in batch order
        const Segment& sg = ctx->segs[absorbed[k]];
        KB_CUDA(ctx, cudaMemcpyAsync(ns.s.ptr + at, sg.s.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(ns.p.ptr + at, sg.p.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(ns.o.ptr + at, sg.o.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        at += sg.n;
    }
    Buf scratch;
    KB_TRY(alloc_buf(ctx, (((size_t)n + 1) / 2048 + 4) * sizeof(u32), &scratch));
    u32* pos = static_cast<u32*>(b.flag32->p);
    timer_begin(ctx, F_OTHER, 4);  // the scan's three kernels and the gather
    launch_exclusive_scan_u32(pos, n + 1, static_cast<u32*>(scratch->p), ctx->st);
    launch_batch_gather(s, p, o, n, static_cast<const u8*>(b.flag8->p), pos, ns.s.ptr + at, ns.p.ptr + at, ns.o.ptr + at, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    return store_swap(ctx, std::move(absorbed), {ns});
}

// kb_store_remove over a batch in device memory
static kb_status store_remove_device(kb_ctx* ctx, const u32* s, const u32* p, const u32* o, u32 n, uint8_t* removed, uint64_t* n_removed) {
    BatchMark b;
    KB_TRY(batch_mark(ctx, s, p, o, n, /*want_found=*/true, &b));
    KB_TRY(batch_flags_out(ctx, b, removed));
    if (n_removed) *n_removed = b.n_flagged;
    if (b.n_flagged == 0) return KB_OK;  // nothing stored matches: no new version
    // segments without a hit stay as they are (their buffers and index chunks); the others are compacted
    std::vector<size_t> hit;
    std::vector<Segment> kept;
    for (size_t g = 0; g < ctx->segs.size(); g++) {
        if (!b.seg_hits[g]) continue;
        Segment ns;
        KB_TRY(segment_without(ctx, ctx->segs[g], b.set, b.slots, &ns));
        hit.push_back(g);
        kept.push_back(ns);
    }
    return store_swap(ctx, std::move(hit), std::move(kept));
}

// a host batch checked as the appends check theirs (NULL columns, KB_ID_NONE) and copied to the device
static kb_status upload_batch(kb_ctx* ctx, const u32* s, const u32* p, const u32* o, u64 n, Buf* d) {
    if (!s || !p || !o) return fail(ctx, KB_E_INVALID, "NULL column pointer");
    if (n > BATCH_MAX) return fail(ctx, KB_E_LIMIT, "a batch of %llu triples: at most 2^30", (unsigned long long)n);
    u32 cmax[3] = {0, 0, 0};
    const u32* col[3] = {s, p, o};
    for (int c = 0; c < 3; c++)
        for (u64 i = 0; i < n; i++) if (col[c][i] == KB_ID_NONE) { cmax[c] = KB_ID_NONE; break; }
    KB_TRY(refuse_reserved_id(ctx, cmax));
    KB_TRY(alloc_buf(ctx, 3 * n * sizeof(u32), d));
    u32* dst = static_cast<u32*>((*d)->p);
    for (int c = 0; c < 3; c++) KB_CUDA(ctx, cudaMemcpyAsync(dst + c * n, col[c], n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    ctx->stats.h2d_bytes += 3 * n * sizeof(u32);
    return KB_OK;
}
}  // namespace kb

extern "C" {

// ------------------------------------------------------------------ store
static kb_status store_add_segment(kb_ctx* ctx, const u32* s, const u32* p, const u32* o, u64 n, u64 tag, cudaMemcpyKind kind) {
    if (n && (!s || !p || !o)) return kb::fail(ctx, KB_E_INVALID, "NULL column pointer");
    if (ctx->n_triples + n >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "store would exceed 2^32-16 triples");
    kb::Segment sg;
    sg.tag = tag;
    sg.n = n;
    KB_TRY(kb::alloc_col(ctx, n, &sg.s));
    KB_TRY(kb::alloc_col(ctx, n, &sg.p));
    KB_TRY(kb::alloc_col(ctx, n, &sg.o));
    if (n) {
        static const bool trace = getenv("KOLIBRIE_TRACE") != nullptr;
        const auto t0 = std::chrono::steady_clock::now();
        // one stream, back to back: three concurrent H2D copies on three streams were several times SLOWER at 16 MB per column
        // and no faster at 4 MB
        KB_CUDA(ctx, cudaMemcpyAsync(sg.s.ptr, s, n * sizeof(u32), kind, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(sg.p.ptr, p, n * sizeof(u32), kind, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(sg.o.ptr, o, n * sizeof(u32), kind, ctx->st));
        if (trace) KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        const auto t1 = std::chrono::steady_clock::now();
        if (kind == cudaMemcpyHostToDevice) ctx->stats.h2d_bytes += 3 * n * sizeof(u32);
        // the statistics pass ends with a read-back on the same stream: when it returns the copies are done too (the caller's
        // buffers are borrowed for this call only)
        KB_TRY(kb::segment_stats(ctx, &sg));
        KB_TRY(kb::refuse_reserved_id(ctx, sg.cmax));
        if (trace)
            fprintf(stderr, "[kb trace] segment of %llu triples: copies %.3f ms, statistics %.3f ms\n", (unsigned long long)n,
                    std::chrono::duration<double, std::milli>(t1 - t0).count(),
                    std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count());
    }
    return kb::store_add_device_segment(ctx, sg);
}

kb_status kb_store_clear(kb_ctx* ctx) {
    KB_ENTER(ctx);
    kb::store_replace(ctx, {});
    return KB_OK;
}
// a load empties the store first: a rejected load (a NULL column, a triple holding KB_ID_NONE) leaves it empty, at a new version;
// a rejected append leaves the store as it was
kb_status kb_store_load(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n) {
    KB_ENTER(ctx);
    kb::store_replace(ctx, {});
    return store_add_segment(ctx, s, p, o, n, 0, cudaMemcpyHostToDevice);
}
kb_status kb_store_load_device(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n) {
    KB_ENTER(ctx);
    kb::store_replace(ctx, {});
    return store_add_segment(ctx, s, p, o, n, 0, cudaMemcpyDeviceToDevice);
}
kb_status kb_store_append(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t tag) {
    KB_ENTER(ctx);
    return store_add_segment(ctx, s, p, o, n, tag, cudaMemcpyHostToDevice);
}
kb_status kb_store_append_device(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t tag) {
    KB_ENTER(ctx);
    return store_add_segment(ctx, s, p, o, n, tag, cudaMemcpyDeviceToDevice);
}
kb_status kb_store_evict(kb_ctx* ctx, uint64_t tag) {
    KB_ENTER(ctx);
    const bool found = kb::store_evict_tag(ctx, tag, /*keep_index=*/true);
    return found ? KB_OK : kb::fail(ctx, KB_E_NOT_FOUND, "no segment with tag %llu", (unsigned long long)tag);
}
kb_status kb_set_use_index(kb_ctx* ctx, int enabled) {
    if (!ctx) return KB_E_INVALID;
    ctx->use_index = enabled != 0;
    return KB_OK;
}

kb_status kb_store_build_index(kb_ctx* ctx, uint32_t* n_predicates, double* build_ms) {
    KB_ENTER(ctx);
    if (n_predicates) *n_predicates = 0;
    if (build_ms) *build_ms = 0.0;
    kb::drop_index(ctx);
    if (ctx->n_triples == 0) return KB_OK;
    kb::ScopedEvent e0, e1;
    cudaEventRecord(e0, ctx->st);
    for (auto& sg : ctx->segs) if (sg.n && (!sg.has_stats || sg.stats_world != ctx->shard_world)) KB_TRY(kb::segment_stats(ctx, &sg));
    for (size_t g = 0; g < ctx->segs.size(); g++) {
        bool indexable = true;
        const kb_status rc = kb::index_add_segment(ctx, g, /*full_build=*/true, &indexable);
        if (rc != KB_OK || !indexable) {
            ctx->index.clear();
            if (rc != KB_OK) return rc;
            return KB_OK;  // too many predicates: keep scanning (n_predicates = 0)
        }
    }
    // value ranks in table order for subject tables whose slice is numeric: the table-mode probe reads FILTER operands sequentially
    for (auto& kv : ctx->index) {
        kb::PredSlice& ps = kv.second;
        if (!ps.xtab || !ctx->n_ids || !ps.typed(ctx->num_version)) continue;
        KB_TRY(kb::build_rank_column(ctx, ps));
    }
    // one-byte codes for the subject tables of few distinct objects: the index probe looks them up 1 byte a slot instead of 4
    KB_TRY(kb::build_subject_codes(ctx));
    // key-grouped directories (counting sort by the dense key) for the columns that did not get a direct table
    for (auto& kv : ctx->index) {
        kb::PredSlice& ps = kv.second;
        const kb::SliceChunk* ch = ps.single();
        if (!ch || ch->n == 0) continue;
        for (u32 y = 0; y < 2; y++) {
            if (y ? (bool)ps.ytab : (bool)ps.xtab) continue;  // unique column: the direct table answers the lookup
            const u32 lo = y ? ps.ymin : ps.xmin, hi = y ? ps.ymax : ps.xmax;
            const u64 range = (u64)hi - lo + 1;
            if (range > std::max<u64>(8 * ps.n, 1ull << 20) || range > (1ull << 28)) continue;  // sparse ids: no directory
            kb::Buf off, val, cursor, scratch;
            KB_TRY(kb::alloc_buf(ctx, (range + 1) * sizeof(u32), &off));
            KB_TRY(kb::alloc_buf(ctx, ch->n * sizeof(u32), &val));
            KB_TRY(kb::alloc_buf(ctx, range * sizeof(u32), &cursor));
            KB_TRY(kb::alloc_buf(ctx, ((range + 1) / 2048 + 4) * sizeof(u32), &scratch));
            KB_CUDA(ctx, cudaMemsetAsync(off->p, 0, (range + 1) * sizeof(u32), ctx->st));
            const uint2* pairs = reinterpret_cast<const uint2*>(ch->pairs.ptr);
            kb::launch_csr_count_pairs(pairs, y, (u32)ch->n, lo, static_cast<u32*>(off->p), ctx->n_sms, ctx->st);
            kb::launch_exclusive_scan_u32(static_cast<u32*>(off->p), (u32)range + 1, static_cast<u32*>(scratch->p), ctx->st);
            KB_CUDA(ctx, cudaMemcpyAsync(cursor->p, off->p, range * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
            kb::launch_csr_fill_pairs(pairs, y, (u32)ch->n, lo, static_cast<u32*>(cursor->p), static_cast<u32*>(val->p), ctx->n_sms, ctx->st);
            ctx->stats.kernel_launches += 5;
            if (y) { ps.yoff = off; ps.yval = val; ps.ycsr_min = lo; ps.ycsr_range = (u32)range; }
            else { ps.xoff = off; ps.xval = val; ps.xcsr_min = lo; ps.xcsr_range = (u32)range; }
        }
    }
    KB_CUDA(ctx, cudaGetLastError());
    cudaEventRecord(e1, ctx->st);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    ctx->index_version = ctx->store_version;
    if (n_predicates) *n_predicates = (uint32_t)ctx->index.size();
    if (build_ms) *build_ms = ms;
    return KB_OK;
}

kb_status kb_store_size(kb_ctx* ctx, uint64_t* n, uint32_t* n_seg) {
    if (!ctx) return KB_E_INVALID;
    if (n) *n = ctx->n_triples;
    if (n_seg) *n_seg = (uint32_t)ctx->segs.size();
    return KB_OK;
}

kb_status kb_store_delete(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n) {
    KB_ENTER(ctx);
    if (n == 0 || ctx->n_triples == 0) return KB_OK;
    if (!s || !p || !o) return kb::fail(ctx, KB_E_INVALID, "NULL column pointer");
    // the delete set (96-bit keys), then every segment without its triples (segment_without)
    const u32 set_slots = kb::pow2_at_least(n * 2);
    kb::Buf set, ds, dp, dob;
    KB_TRY(kb::alloc_buf(ctx, (size_t)set_slots * sizeof(uint4), &set));
    KB_TRY(kb::alloc_buf(ctx, n * sizeof(u32), &ds));
    KB_TRY(kb::alloc_buf(ctx, n * sizeof(u32), &dp));
    KB_TRY(kb::alloc_buf(ctx, n * sizeof(u32), &dob));
    KB_CUDA(ctx, cudaMemsetAsync(set->p, 0, (size_t)set_slots * sizeof(uint4), ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(ds->p, s, n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(dp->p, p, n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(dob->p, o, n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    const u32 off = kb::ctrl_alloc(ctx, 4);
    kb::launch_set_insert(static_cast<uint4*>(set->p), set_slots, (const u32*)ds->p, (const u32*)dp->p, (const u32*)dob->p, (u32)n,
                          ctx->ctrl + off, ctx->n_sms, ctx->st);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    // the new segments are built aside: the store changes only when all of them are (a failure leaves it as it was)
    std::vector<kb::Segment> kept;
    for (auto& sg : ctx->segs) {
        kb::Segment ns;
        KB_TRY(kb::segment_without(ctx, sg, set, set_slots, &ns));
        kept.push_back(ns);
    }
    kb::store_replace(ctx, std::move(kept));
    return KB_OK;
}

kb_status kb_store_insert(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t segment_tag, uint8_t* inserted,
                          uint64_t* n_inserted) {
    KB_ENTER(ctx);
    if (n_inserted) *n_inserted = 0;
    if (n == 0) return KB_OK;
    kb::Buf d;
    KB_TRY(kb::upload_batch(ctx, s, p, o, n, &d));
    const u32* b = static_cast<const u32*>(d->p);
    return kb::store_insert_device(ctx, b, b + n, b + 2 * n, (u32)n, segment_tag, inserted, n_inserted);
}

kb_status kb_store_remove(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint8_t* removed, uint64_t* n_removed) {
    KB_ENTER(ctx);
    if (n_removed) *n_removed = 0;
    if (n == 0) return KB_OK;
    kb::Buf d;
    KB_TRY(kb::upload_batch(ctx, s, p, o, n, &d));
    const u32* b = static_cast<const u32*>(d->p);
    return kb::store_remove_device(ctx, b, b + n, b + 2 * n, (u32)n, removed, n_removed);
}

kb_status kb_store_remove_template(kb_ctx* ctx, const kb_rel* rel, const kb_pattern* tmpl, uint32_t n_tmpl, uint64_t* n_removed) {
    KB_ENTER(ctx);
    if (n_removed) *n_removed = 0;
    if (!rel || (n_tmpl && !tmpl)) return kb::fail(ctx, KB_E_INVALID, "NULL relation or template");
    if (rel->pair) return kb::fail(ctx, KB_E_INVALID, "an internal pair relation");
    if (n_tmpl > kb::TEMPLATE_MAX) return kb::fail(ctx, KB_E_LIMIT, "%u template patterns: at most %u", n_tmpl, kb::TEMPLATE_MAX);
    static const char* const pos[3] = {"subject", "predicate", "object"};
    kb::TemplateFillParams P{};
    for (u32 t = 0; t < n_tmpl; t++) {
        const kb_term* term[3] = {&tmpl[t].s, &tmpl[t].p, &tmpl[t].o};
        for (int c = 0; c < 3; c++) {
            if (term[c]->is_var > 1) return kb::fail(ctx, KB_E_INVALID, "template pattern %u: the %s is not a variable or a constant", t, pos[c]);
            if (!term[c]->is_var) {
                if (term[c]->value == KB_ID_NONE)
                    return kb::fail(ctx, KB_E_INVALID, "template pattern %u: the %s is 0xFFFFFFFF, which is reserved (KB_ID_NONE)", t, pos[c]);
                P.cval[t][c] = term[c]->value;
                continue;
            }
            const int col = rel->col_of(term[c]->value);
            if (col < 0) return kb::fail(ctx, KB_E_UNSUPPORTED, "template pattern %u: the %s variable %u is not a column of the relation", t, pos[c], term[c]->value);
            P.col[t][c] = rel->cols[col].ptr;
        }
    }
    const u64 total = rel->n * n_tmpl;
    if (total == 0) return KB_OK;
    if (total > kb::BATCH_MAX) return kb::fail(ctx, KB_E_LIMIT, "%llu template triples (rows x patterns): at most 2^30", (unsigned long long)total);
    kb::Buf d;
    KB_TRY(kb::alloc_buf(ctx, 3 * total * sizeof(u32), &d));
    u32* b = static_cast<u32*>(d->p);
    P.n_tmpl = n_tmpl;
    P.rows = (u32)rel->n;
    P.s = b; P.p = b + total; P.o = b + 2 * total;
    P.dict = kb::dicttab(ctx);
    const u32 c = kb::ctrl_alloc(ctx, 2);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 2 * sizeof(u32), ctx->st));
    P.bad = ctx->ctrl + c;
    kb::timer_begin(ctx, kb::F_OTHER);
    kb::launch_template_fill(P, ctx->n_sms, ctx->st);
    kb::timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(kb::ctrl_read(ctx));
    if (ctx->h_ctrl[c])
        return kb::fail(ctx, KB_E_UNSUPPORTED, "%u template cells are unbound: the reference would delete the variable's name as a term", ctx->h_ctrl[c]);
    if (ctx->h_ctrl[c + 1])
        return kb::fail(ctx, KB_E_UNSUPPORTED,
                        "%u template cells hold a term that encode_term_star would not re-encode to the same id (a quoted id, an id without a "
                        "device dictionary string, or a string it strips or parses)", ctx->h_ctrl[c + 1]);
    return kb::store_remove_device(ctx, P.s, P.p, P.o, (u32)total, nullptr, n_removed);
}

kb_status kb_store_download(kb_ctx* ctx, uint32_t* s, uint32_t* p, uint32_t* o, uint64_t cap, uint64_t* n) {
    KB_ENTER(ctx);
    if (n) *n = ctx->n_triples;
    if (cap < ctx->n_triples) return kb::fail(ctx, KB_E_LIMIT, "buffer holds %llu triples, store has %llu", (unsigned long long)cap, (unsigned long long)ctx->n_triples);
    u64 off = 0;
    for (auto& sg : ctx->segs) {
        if (!sg.n) continue;
        KB_CUDA(ctx, cudaMemcpyAsync(s + off, sg.s.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(p + off, sg.p.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(o + off, sg.o.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        off += sg.n;
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    return KB_OK;
}

}  // extern "C"
