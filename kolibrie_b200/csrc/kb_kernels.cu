// kb_kernels.cu — hand-written sm_90a kernels of the Kolibrie hot path (see kb_kernels.cuh for what each replaces).
// All of them are HBM-bound integer kernels: column tiles are staged global->shared with TMA bulk copies (cp.async.bulk +
// mbarrier), matches are compacted with warp ballots, and output positions come from a single-pass decoupled look-back
// prefix over tiles, so every kernel reads its input exactly once and writes a deterministic, input-ordered output.
#include "kb_group.cuh"
#include "kb_internal.hpp"
#include "kb_numrank.cuh"

#include <math_constants.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>

namespace kb {

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
void launch_distinct(const u32* col, u32 n, u32* set, u32 set_slots, u32 limit, u32* ctrl, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = (int)umin64((u64)n_sms * 4ull, ((u64)n + 255ull) / 256ull);
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
void launch_tab_code(const u32* tab, u32 range, const u32* dict, u32 n_dict, u8* code, int n_sms, cudaStream_t st) {
    if (range == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)range + 1023ull) / 1024ull);
    tab_code_kernel<<<grid, 256, 0, st>>>(tab, range, dict, n_dict, code);
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
void launch_pair_ranktab(const uint2* kv, u32 n, NumTab nt, const double* numv, u32 n_numv, u16* out, u32 kmin, u32 range, u32 cshift, int n_sms,
                         cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 256ull * RANKTAB_ITEMS - 1ull) / (256ull * RANKTAB_ITEMS));
    pair_ranktab_kernel<<<grid, 256, 0, st>>>(kv, n, nt, numv, n_numv, out, kmin, range, cshift);
}
// the value order's keys (kb_numrank.cuh: order_key / order_value); id n is the extra 0.0
__global__ void __launch_bounds__(256) numorder_keys_kernel(const double* __restrict__ num, u32 n, unsigned long long* __restrict__ keys) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (u64)gridDim.x * blockDim.x) keys[i] = kb_nr::order_key(i < n ? num[i] : 0.0);
}
__global__ void __launch_bounds__(256) numorder_values_kernel(const unsigned long long* __restrict__ keys, u32 n, double* __restrict__ out) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = kb_nr::order_value(keys[i]);
}
void launch_numorder_keys(const double* num_or0, u32 n, unsigned long long* keys, int n_sms, cudaStream_t st) {
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 256ull) / 256ull);
    numorder_keys_kernel<<<grid, 256, 0, st>>>(num_or0, n, keys);
}
void launch_numorder_values(const unsigned long long* keys, u32 n, double* out, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    numorder_values_kernel<<<grid, 256, 0, st>>>(keys, n, out);
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
        const u32 t = atomicAdd(P.c.ticket, 1u);
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
            const u32 ex = tile_prefix_2level(P.c.tile_state, P.c.block_state, tile, P.n_tiles, 0u, P.c.epoch, total, P.c.zero_word, P.c.total, P.c.ordered, lane);
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
// TAB = true: the probe stream is not the slice but the probe pattern's own persistent TABLE, walked slot by slot: slot i holds the
// other half of the triple whose key is (table base + i), EMPTY32 where no triple has that key. The keys then come in ascending order
// whatever the order of the store and of the dictionary ids, so the lookups into the other patterns' tables are sequential too — a
// direct table over dense ids IS the slice sorted by that column (with the gaps of the id space). With a FILTER on the other half's
// numeric value the 2-byte value ranks are read from a second table in the same order (kb_numrank.cuh: the FILTER is a range of
// stored ranks; a slot whose stored rank is at an end of that range is decided on its value, num_of(object)).
template <int T, int PRE, bool AGG, bool TAB>
__global__ void __launch_bounds__(PROBEF_THREADS, KB_PI_MINB) probe_index_kernel(const __grid_constant__ ProbeIParams P, const __grid_constant__ GroupParams G) {
    constexpr int R = 4;  // rows per thread (striped over the warp's 128-row chunk, see below)
    constexpr u32 TILE = PROBEF_THREADS * R;
    extern __shared__ __align__(128) u32 smem_all[];  // per stage: TILE pairs [+ TILE doubles]
    constexpr u32 STAGE_WORDS = TAB ? (PRE == 1 ? 3u * TILE / 2u : TILE) : (PRE == 1 ? 4u : 2u) * TILE;  // TAB: TILE values [+ TILE u16 ranks]
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
    // dictionaries of the coded tables (DirectTab::code): entry 0xFF is EMPTY32, so a code decodes with one shared load (the barrier
    // after the stage set-up below publishes them)
    __shared__ u32 s_dict[T][256];
#pragma unroll
    for (int t = 0; t < T; t++)
        if (P.tab[t].code) s_dict[t][tid] = (u32)tid < P.tab[t].n_dict ? P.tab[t].dict[tid] : EMPTY32;
    static_assert(PROBEF_THREADS == 256, "one dictionary entry per thread");
    auto issue = [&](u32 t, u32 stage) {
        u32* smem = smem_all + stage * STAGE_WORDS;
        u64& bar = bars[stage];
        if constexpr (TAB) {
            const u32 b = t * TILE;
            const u32 c = min(TILE, P.ptab_range - b);
            const u32 bytes = (c * 4u + 15u) & ~15u;
            const u32 kbytes = (c * 2u + 15u) & ~15u;
            s_tcnt[stage] = c;
            mbar_arrive_expect_tx(&bar, PRE == 1 ? bytes + kbytes : bytes);
            tma_load_1d(smem, P.ptab + b, bytes, &bar);
            if (PRE == 1) tma_load_1d(smem + TILE, P.pkey + b, kbytes, &bar);
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
        double pa[R];  // PRE == 1: the FILTER operand (slice mode: the f64 value, table mode: its rank in pk)
        u32 pk[R];
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
                if (PRE == 1) pk[j] = reinterpret_cast<const u16*>(smem + TILE)[idx];
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
            u32 pass = 0, edge = 0;
#pragma unroll
            for (int j = 0; j < R; j++) {
                bool ok;
                if constexpr (TAB) {
                    ok = pk[j] >= P.key_lo && pk[j] <= P.key_hi;
                    edge |= ((ok && (pk[j] == P.key_lo || pk[j] == P.key_hi)) ? 1u : 0u) << j;
                } else ok = cmp_num(P.pre_cmp, pa[j], P.pre_val);
                pass |= (ok ? 1u : 0u) << j;
            }
            vmask &= pass;
            if (TAB && P.key_shift != 0u && (edge & vmask) != 0u) {  // a stored rank at an end of the range: its values straddle the constant
#pragma unroll
                for (int j = 0; j < R; j++) {
                    if (((edge & vmask) >> j) & 1u) {
                        if (!cmp_num(P.pre_cmp, num_of(P.nt, P.key_is_y ? rx[j] : ry[j]), P.pre_val)) vmask &= ~(1u << j);
                    }
                }
            }
        } else if (P.pre_mode == 2u && vmask != 0u) {
#pragma unroll
            for (int j = 0; j < R; j++) {
                if ((vmask >> j) & 1u) {
                    u32 vals[2] = {rx[j], ry[j]};
                    if (!eval_filter(P.pre_ops, P.n_pre, vals, P.nt)) vmask &= ~(1u << j);
                }
            }
        }
        // a coded table (warp-uniform) is read one byte a slot: a warp's 32 consecutive keys are one sector instead of four. Every
        // load is issued before the first code is decoded
        u32 tv[R][T];
#pragma unroll
        for (int t = 0; t < T; t++) {
            const DirectTab& D = P.tab[t];
            if (D.code) {
#pragma unroll
                for (int j = 0; j < R; j++) {
                    const u32 off = compact_key(P.key_is_y ? ry[j] : rx[j], D.cshift) - D.kmin;
                    tv[j][t] = (((vmask >> j) & 1u) && off < D.range) ? (u32)__ldg(D.code + off) : 0xFFu;
                }
            } else {
#pragma unroll
                for (int j = 0; j < R; j++) {
                    const u32 off = compact_key(P.key_is_y ? ry[j] : rx[j], D.cshift) - D.kmin;
                    tv[j][t] = (((vmask >> j) & 1u) && off < D.range) ? __ldg(D.tab + off) : EMPTY32;
                }
            }
        }
#pragma unroll
        for (int t = 0; t < T; t++)
            if (P.tab[t].code) {
#pragma unroll
                for (int j = 0; j < R; j++) tv[j][t] = s_dict[t][tv[j][t]];
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
            const u32 ex = tile_prefix_2level(P.c.tile_state, P.c.block_state, tile, P.n_tiles, 0u, P.c.epoch, total, P.c.zero_word, P.c.total, P.c.ordered, lane);
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
    const size_t smem = TAB ? (size_t)PROBEF_THREADS * 4 * (PRE == 1 ? 6 : 4) * 2 : (size_t)PROBEF_THREADS * 4 * (PRE == 1 ? 16 : 8) * 2;
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
        if (tid == 0) s_tile = atomicAdd(P.c.ticket, 1u);
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
            const u32 ex = tile_prefix_2level(P.c.tile_state, P.c.block_state, tile, P.n_tiles, 0u, P.c.epoch, total, P.c.zero_word, P.c.total, P.c.ordered, lane);
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
        if (tid == 0) s_tile = atomicAdd(P.c.ticket, 1u);
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
            const u32 ex = tile_prefix_2level(P.c.tile_state, P.c.block_state, tile, P.n_tiles, 0u, P.c.epoch, total, P.c.zero_word, P.c.total, P.c.ordered, lane);
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
        } else if (tid == 0) s_tile = atomicAdd(P.c.ticket, 1u);
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
                const u32 ex = tile_prefix_2level(P.c.tile_state, P.c.block_state, tile, P.n_tiles, 0u, P.c.epoch, total, P.c.zero_word, P.c.total, P.c.ordered, lane);
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
// the store's 96-bit (s,p,o) key set (kb_store.cu)
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

// ---- kb_store_insert / kb_store_remove: the batch as a key set (the layout of set_insert, so that delete_mark reads it too), the
// batch index of each key's first occurrence, and a found bit per key set by one pass over the store
// set_insert that returns the key's slot, whether it was inserted now or found (EMPTY32: the set is full)
__device__ __forceinline__ u32 set_insert_slot(uint4* set, u32 n_slots, u32 s, u32 p, u32 o) {
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
            return slot;
        }
        while (st == 1u) st = *reinterpret_cast<volatile u32*>(st_ptr);
        __threadfence();
        const volatile u32* w = reinterpret_cast<const volatile u32*>(&set[slot]);
        if (w[0] == s && w[1] == p && w[2] == o) return slot;
        slot = (slot + 1u) & mask;
    }
    return EMPTY32;
}
__global__ void __launch_bounds__(256) batch_set_kernel(uint4* set, u32 set_slots, const u32* s, const u32* p, const u32* o, u32 n, u32* first,
                                                        u32* slot_of, u32* overflow) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 slot = set_insert_slot(set, set_slots, s[i], p[i], o[i]);
        slot_of[i] = slot;
        if (slot == EMPTY32) *overflow = 1u;
        else atomicMin(&first[slot], i);
    }
}
void launch_batch_set(uint4* set, u32 set_slots, const u32* s, const u32* p, const u32* o, u32 n, u32* first, u32* slot_of, u32* overflow,
                      int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    batch_set_kernel<<<grid, 256, 0, st>>>(set, set_slots, s, p, o, n, first, slot_of, overflow);
}

__global__ void __launch_bounds__(256) batch_mark_kernel(const u32* __restrict__ s, const u32* __restrict__ p, const u32* __restrict__ o, u32 n,
                                                         const uint4* __restrict__ set, u32 set_slots, u32* found, u32* hits) {
    const u32 mask = set_slots - 1u;
    u32 mine = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u32 vs = s[i], vp = p[i], vo = o[i];
        u32 slot = set_hash(vs, vp, vo) & mask;
        for (u32 probes = 0; probes < set_slots; probes++) {
            const uint4 e = set[slot];
            if (e.w == 0u) break;
            if (e.x == vs && e.y == vp && e.z == vo) { found[slot] = 1u; mine++; break; }
            slot = (slot + 1u) & mask;
        }
    }
    if (mine) atomicAdd(hits, mine);
}
void launch_batch_mark(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots, u32* found, u32* hits, int n_sms,
                       cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
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
void launch_batch_flags(u32 n, const u32* slot_of, const u32* first, const u32* found, bool want_found, u8* flag8, u32* flag32, u32* count, int n_sms,
                        cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
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
void launch_batch_gather(const u32* s, const u32* p, const u32* o, u32 n, const u8* flag8, const u32* pos, u32* out_s, u32* out_p, u32* out_o, int n_sms,
                         cudaStream_t st) {
    if (n == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n + 255ull) / 256ull);
    batch_gather_kernel<<<grid, 256, 0, st>>>(s, p, o, n, flag8, pos, out_s, out_p, out_o);
}

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
void launch_template_fill(const TemplateFillParams& P, int n_sms, cudaStream_t st) {
    const u64 total = (u64)P.rows * P.n_tmpl;
    if (total == 0) return;
    const int grid = (int)umin64((u64)n_sms * 8ull, (total + 255ull) / 256ull);
    template_fill_kernel<<<grid, 256, 0, st>>>(P);
}

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
void launch_r2s_build(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.cur.n) r2s_build_kernel<<<grid_1d(p.cur.n, n_sms), 256, 0, st>>>(p);
}
void launch_r2s_mark(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.cur.n) r2s_mark_kernel<<<grid_1d(p.cur.n, n_sms), 256, 0, st>>>(p);
}
void launch_r2s_gone_mark(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.last.n) r2s_gone_mark_kernel<<<grid_1d(p.last.n, n_sms), 256, 0, st>>>(p);
}
void launch_r2s_write(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.cur.n) r2s_write_kernel<<<grid_1d(p.cur.n, n_sms), 256, 0, st>>>(p);
}
void launch_r2s_gone_write(const R2sParams& p, int n_sms, cudaStream_t st) {
    if (p.last.n) r2s_gone_write_kernel<<<grid_1d(p.last.n, n_sms), 256, 0, st>>>(p);
}

}  // namespace kb
