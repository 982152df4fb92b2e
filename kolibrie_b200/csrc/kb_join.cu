// kb_join.cu — the join operators: FILTER, the natural join (cartesian, grouped, chained), the star join's routes R1-R5, the
// one-kernel index plan and the bind join; and what every compacting launch shares (tile state, epoch, control words). The file owns
// the join's kernels (the direct, chained and filtered builds, the CSR directory, the direct, fast, index, chained and grouped probes,
// the cartesian product) and their launch formats. The index probe's launch format and launcher are declared in kb_kernels.cuh
// because a prepared plan (kb_plan.cu) holds and launches one; the direct-table build from a pair relation is in kb_kernels.cu because
// the store index builds the same tables.
#include <algorithm>

#include "kb_group.cuh"
#include "kb_internal.hpp"
#include "kb_numrank.cuh"

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
static void launch_build_direct(const u32* keys, const u32* vals, u32 n, u32* table, u32 kmin, u32 range, u32 cshift, u32* dup_flag, int n_sms,
                                cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms);
    build_direct_kernel<<<grid, 256, 0, st>>>(keys, vals, n, table, kmin, range, cshift, dup_flag);
}

// CHAINED multimap: open-addressing slots {key tag, head row} + next[] chains. Insert cost is O(1) whatever the key
// multiplicity (1:N joins and heavy hitters of the Datalog joins).
struct ChainTab {
    u64* slots;   // lo 32: key tag (EMPTY32 free), hi 32: head row index (EMPTY32 = end)
    u32 n_slots;  // power of two
    u32* next;    // [n_build]
    u32 n_keys;   // 1..4 key columns; tag = key itself when n_keys==1 else a 32-bit mix of all
    const u32* bkey[4];
};
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
static void launch_build_chained(const ChainTab& t, u32 n, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms);
    build_chained_kernel<<<grid, 256, 0, st>>>(t, n);
}

// direct build from a predicate slice of the store index, with the pattern's pushed-down FILTER evaluated on (s, P, o)
struct BuildPairsParams {
    const uint2* kv;
    u32 n, key_is_y, pred;
    u32* table;
    u32 kmin, range, cshift;
    u32* dup_flag;
    u32 trusted;
    FilterOp ops[KB_MAX_FILTER_OPS];  // slots = positions 0/1/2
    u32 n_ops;
    NumTab nt;
    u32* count;  // rows inserted (after the filter)
};
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
static void launch_build_direct_pairs_filtered(const BuildPairsParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    int grid = grid_1d(p.n, n_sms, 1024);
    if (p.trusted) build_pairs_filtered_kernel<true><<<grid, 256, 0, st>>>(p);
    else build_pairs_filtered_kernel<false><<<grid, 256, 0, st>>>(p);
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
// number of occupied (non-EMPTY32) slots of a direct table: equals the number of inserted rows iff the keys were single-valued
static void launch_count_nonempty(const u32* table, u32 n, u32* out_count, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const u32 n4 = n / 4;
    // one CTA more than the vectors need: n4 may be 0, and block 0 also counts the n % 4 tail slots
    int grid = (int)umin64((u64)n_sms * 8ull, ((u64)n4 + 255ull) / 256ull + 1ull);
    count_nonempty_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(table), n4, table + (u64)n4 * 4, n - n4 * 4, out_count);
}
__global__ void __launch_bounds__(256) count_foreign_kernel(const u32* __restrict__ col, u32 n, u32 rank, u32 world, u32* out) {
    u32 c = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) c += shard_of(col[i], world) != rank;
    c = warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
// number of keys that do NOT belong to shard `rank` of `world` (kb_shard_of): 0 for a correctly sharded column
static void launch_count_foreign(const u32* col, u32 n, u32 rank, u32 world, u32* out, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms, 256, 4);
    count_foreign_kernel<<<grid, 256, 0, st>>>(col, n, rank, world, out);
}

// =================================================================================================================
// K_probe (direct, fused multiway): one probe stream against T<=4 direct tables + FILTER + ordered compaction.
// Replaces execute_star_join_with_ids (engine.rs:587-691) / bind-join chains (engine.rs:840-885) on unique keys.
constexpr int PROBE_THREADS = 256;
constexpr int PROBE_ITEMS = 4;
constexpr int PROBE_TILE = PROBE_THREADS * PROBE_ITEMS;  // 1024 rows
enum : u32 { OUT_PROBE = 0, OUT_TABVAL = 1, OUT_TABPAY = 2 };
struct OutCol {
    u32 kind, a, b;  // OUT_PROBE: a = probe column; OUT_TABVAL: a = table; OUT_TABPAY: a = table, b = payload column
};
struct ProbeDParams {
    const u32* pcol[KB_MAX_COLS];
    u32 n_pcols, key_col, n, n_tiles, T;
    DirectTab tab[MAXT];
    u32 n_out;
    OutCol oc[KB_MAX_COLS];
    u32* out[KB_MAX_COLS];
    u32 cap;
    FilterOp ops[KB_MAX_FILTER_OPS];  // slots = output column indices
    u32 n_ops;
    NumTab nt;
    Compact c;
    const u32* abort_flag;  // non-null: exit immediately if *abort_flag != 0 (a direct build met duplicate keys)
};

// K_probe (direct, FAST): the probe side is a pair relation; each thread owns 4 consecutive rows held in registers, so the shared
// tile is refilled by TMA while the rows are probed (same register-staged double buffering as K_scan).
constexpr int PROBEF_THREADS = 256;
#ifndef KB_PROBEF_ITEMS
#define KB_PROBEF_ITEMS 4
#endif
constexpr int PROBEF_ITEMS = KB_PROBEF_ITEMS;  // rows per thread: 8 keeps twice the lookups in flight per thread (the kernel is latency-bound)
constexpr int PROBEF_TILE = PROBEF_THREADS * PROBEF_ITEMS;
struct ProbeFParams {
    const uint2* pairs;
    u32 key_is_y;  // which half of the pair is the join key
    u32 n, n_tiles, T;
    DirectTab tab[MAXT];  // mode 0 (value payload) or 2 (existence) only
    u32 n_out;
    OutCol oc[KB_MAX_COLS];  // OUT_PROBE: a = 0 (pair.x) / 1 (pair.y); OUT_TABVAL: a = table
    u32* out[KB_MAX_COLS];
    u32 cap;
    FilterOp ops[KB_MAX_FILTER_OPS];
    u32 n_ops;
    FilterOp pre_ops[8];  // conjuncts over the probe row alone (slot 0 = pair.x, 1 = pair.y): evaluated BEFORE any table lookup
    u32 n_pre;
    const double* pre_num;  // non-null: numeric value of pair.y per probe row (typed literal column of the index): a coalesced read
                            // replaces the random gather num_or0[pair.y] when the pre-filter is FILTER(?y <cmp> c)
    NumTab nt;
    Compact c;
    const u32* abort_flag;
};
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

static void launch_probe_fast(const ProbeFParams& p, int n_sms, cudaStream_t st) {
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

static void launch_probe_direct(const ProbeDParams& p, int n_sms, cudaStream_t st) {
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
// K_probe (chained, binary): general natural join with 1:N matches, multi-column keys, FILTER, ordered compaction.
// Replaces execute_optimized_hash_join_with_ids / execute_hash_join_with_ids / merge join (engine.rs:710-811, 970-1039) and
// perform_hash_join_for_rules (shared/src/join_algorithm.rs:499-677).
constexpr int PROBEC_THREADS = 256;
constexpr int PROBEC_ITEMS = 2;
constexpr int PROBEC_TILE = PROBEC_THREADS * PROBEC_ITEMS;
struct ProbeCParams {
    const u32* pcol[KB_MAX_COLS];
    u32 n_pcols, n, n_tiles;
    u32 pkey[4];  // probe columns matching tab.bkey[]
    ChainTab tab;
    u32 n_bpay;
    const u32* bpay[KB_MAX_COLS];  // build columns appended to the output
    u32 n_out;                      // = n_pcols + n_bpay
    u32* out[KB_MAX_COLS];
    u32 cap;
    FilterOp ops[KB_MAX_FILTER_OPS];
    u32 n_ops;
    NumTab nt;
    Compact c;
    unsigned long long* total64;  // exact output size in 64 bits (the 32-bit positions wrap past 2^32 rows: the host checks this one)
};
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

static void launch_probe_chained(const ProbeCParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    const size_t smem = (size_t)p.n_pcols * PROBEC_TILE * sizeof(u32);
    const int grid = grid_for((const void*)probe_chained_kernel, PROBEC_THREADS, smem, n_sms, p.n_tiles);
    probe_chained_kernel<<<grid, PROBEC_THREADS, smem, st>>>(p);
}

// =================================================================================================================
// K_build / K_probe (grouped): 1:N equi-join on ONE key column whose ids are dense. The build side is grouped by key into a CSR
// directory — off[key - kmin] .. off[key - kmin + 1] delimit the key's rows in payload columns permuted into key order — so a probe
// is two directory reads and a contiguous run of payload, and the expansion can hand consecutive OUTPUT rows to consecutive threads
// (coalesced stores). Replaces the (tag, head) + next[] chains wherever the key range allows; same bag of rows as
// perform_hash_join_for_rules (join_algorithm.rs:499-677) / execute_hash_join_with_ids (engine.rs:710-811).
struct CsrTab {
    const u32* off;  // [range + 1]
    u32 kmin, range;
    u32 n_pay;
    const u32* pay[KB_MAX_COLS];  // payload columns in key order
};
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
static void launch_csr_count(const u32* keys, u32 n, u32 kmin, u32* counts, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms, CSR_TILE, 4);
    csr_count_kernel<<<grid, 256, 0, st>>>(keys, n, kmin, counts);
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
static void launch_csr_fill(const u32* keys, u32 n, u32 kmin, u32* cursor, const u32* const* pay_in, u32* const* pay_out, u32 n_pay, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    CsrFillParams P{};
    P.keys = keys; P.n = n; P.kmin = kmin; P.n_pay = n_pay; P.cursor = cursor;
    for (u32 c = 0; c < n_pay; c++) { P.pay_in[c] = pay_in[c]; P.pay_out[c] = pay_out[c]; }
    const int grid = grid_1d(n, n_sms, CSR_TILE, 4);
    csr_fill_kernel<<<grid, 256, 0, st>>>(P);
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
static void launch_csr_total(const u32* pkeys, u32 n, const CsrTab& tab, unsigned long long* total, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    csr_total_kernel<<<grid, 256, 0, st>>>(pkeys, n, tab.off, tab.kmin, tab.range, total);
}

constexpr int PROBEG_THREADS = 256;
constexpr int PROBEG_ITEMS = 4;
constexpr int PROBEG_TILE = PROBEG_THREADS * PROBEG_ITEMS;
struct ProbeGParams {
    const u32* pcol[KB_MAX_COLS];
    u32 n_pcols, n, n_tiles;
    u32 pkey;  // probe column holding the key
    CsrTab tab;
    u32* out[KB_MAX_COLS];  // n_pcols probe columns, then tab.n_pay payload columns
    u32 cap;
    Compact c;
    // tiles whose expansion exceeds PROBEG_HEAVY output rows are not expanded by the CTA that scanned them: it appends them here
    // (heavy_count[0] entries) and a second launch spreads each one's output range over the whole grid in PROBEG_CHUNK-row pieces
    struct Heavy { u32 tile, gbase, total, pad; };
    Heavy* heavy;        // room for n_tiles entries (null: no splitting)
    u32* heavy_count;    // zeroed control word
};
constexpr u32 PROBEG_HEAVY = 32768, PROBEG_CHUNK = 4096;
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
static void launch_probe_grouped(const ProbeGParams& p, int n_sms, cudaStream_t st) {
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
static void launch_cartesian(const u32* const* lcols, u32 nl, u32 n_lcols, const u32* const* rcols, u32 nr, u32 n_rcols, u32* const* out,
                             cudaStream_t st) {
    CartParams P;
    P.nl = nl; P.nr = nr; P.n_l = n_lcols; P.n_r = n_rcols;
    for (u32 c = 0; c < n_lcols; c++) P.l[c] = lcols[c];
    for (u32 c = 0; c < n_rcols; c++) P.r[c] = rcols[c];
    for (u32 c = 0; c < n_lcols + n_rcols; c++) P.out[c] = out[c];
    const u64 total = (u64)nl * nr;
    if (total == 0) return;
    int grid = grid_1d(total, (int)H100_SMS);
    cartesian_kernel<<<grid, 256, 0, st>>>(P);
}

// AND the program `f` into `dst`
static void and_into(FilterProg* dst, const FilterProg& f) {
    if (f.ops.empty()) return;
    const bool had = !dst->ops.empty();
    dst->ops.insert(dst->ops.end(), f.ops.begin(), f.ops.end());
    if (had) { kb_filter_op a{}; a.op = KB_F_AND; dst->ops.push_back(a); }
}

// ---------------------------------------------------------------------------------------------------------------
// what every compacting launch shares

// The epoch tags a launch's tile-state words, so the buffers need no clearing between launches. When the epoch field
// (TS_EPOCH_BITS) would overflow, the count starts again at 1 and the buffers are zeroed first, on the stream, before the launch
// that reuses the epoch: a word an old launch left with that epoch must not pass for one of the new launch's.
static kb_status next_epoch(kb_ctx* ctx, u64* epoch) {
    if (ctx->epoch >= (1ull << TS_EPOCH_BITS)) {
        if (ctx->tile_state) {
            KB_CUDA(ctx, cudaMemsetAsync(ctx->tile_state->p, 0, ctx->tile_state->bytes, ctx->st));
            KB_CUDA(ctx, cudaMemsetAsync(ctx->block_state->p, 0, ctx->block_state->bytes, ctx->st));
        }
        ctx->epoch = 1;
    }
    *epoch = ctx->epoch++;
    return KB_OK;
}

kb_status compact_setup(kb_ctx* ctx, u64 n_tiles, u32* ctrl, Compact* c) {
    KB_TRY(ensure_tile_state(ctx, n_tiles));
    c->tile_state = static_cast<u64*>(ctx->tile_state->p);
    c->block_state = static_cast<u64*>(ctx->block_state->p);
    c->ordered = ctx->ordered;
    KB_TRY(next_epoch(ctx, &c->epoch));
    c->ticket = ctrl;
    c->total = ctrl ? ctrl + 1 : nullptr;
    c->zero_word = ctrl ? ctrl + 2 : nullptr;
    return KB_OK;
}

kb_status alloc_strided_cols(kb_ctx* ctx, u64 rows, u32 n_cols, std::vector<Col>* cols) {
    const size_t stride = round256((size_t)rows * sizeof(u32)) + 256;
    Buf b;
    KB_TRY(alloc_buf(ctx, stride * n_cols, &b));
    cols->clear();
    for (u32 c = 0; c < n_cols; c++) {
        Col col;
        col.buf = b;
        col.ptr = reinterpret_cast<u32*>(static_cast<char*>(b->p) + stride * c);
        cols->push_back(col);
    }
    return KB_OK;
}

// what every probe launch over a direct table shares: the output columns (`ocs`, n rows each, appended to res->cols), the FILTER
// over them and the compaction block with control words ctrl = {ticket, total, zero}
template <class Params>
static kb_status probe_setup(kb_ctx* ctx, Params* P, u64 n, const std::vector<OutCol>& ocs, const std::vector<FilterOp>& fops, u32* ctrl,
                             const u32* abort_flag, kb_rel* res) {
    P->n_out = (u32)ocs.size();
    std::vector<Col> cols;
    KB_TRY(alloc_strided_cols(ctx, n, P->n_out, &cols));
    for (u32 c = 0; c < P->n_out; c++) {
        res->cols.push_back(cols[c]);
        P->oc[c] = ocs[c];
        P->out[c] = cols[c].ptr;
    }
    P->cap = (u32)n;
    P->n_ops = (u32)fops.size();
    for (size_t i = 0; i < fops.size(); i++) P->ops[i] = fops[i];
    P->nt = numtab(ctx);
    P->abort_flag = abort_flag;
    return compact_setup(ctx, P->n_tiles, ctrl, &P->c);
}

// ---------------------------------------------------------------------------------------------------------------
// filter (= probe kernel with zero tables)
kb_status filter_impl(kb_ctx* ctx, const kb_rel& in, const FilterProg& f, std::unique_ptr<kb_rel>* out) {
    auto rel = std::make_unique<kb_rel>();
    rel->slots = in.slots;
    if (in.n == 0 || f.ops.empty()) {
        rel->cols = in.cols;
        rel->n = in.n;
        *out = std::move(rel);
        return KB_OK;
    }
    if (in.n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "relation too large");
    ProbeDParams P{};
    P.n_pcols = (u32)in.cols.size();
    if (P.n_pcols == 0) return fail(ctx, KB_E_UNSUPPORTED, "filter on a relation without columns");
    P.n = (u32)in.n;  // key_col 0, T = 0 tables
    P.n_tiles = (u32)((in.n + PROBE_TILE - 1) / PROBE_TILE);
    std::vector<OutCol> ocs;
    for (u32 c = 0; c < P.n_pcols; c++) {
        P.pcol[c] = in.cols[c].ptr;
        ocs.push_back(OutCol{OUT_PROBE, c, 0});
    }
    std::vector<FilterOp> ops;
    KB_TRY(compile_prog(ctx, f, in.slots, &ops));
    const u32 off = ctrl_alloc(ctx, 4);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 4 * sizeof(u32), ctx->st));
    KB_TRY(probe_setup(ctx, &P, in.n, ocs, ops, ctx->ctrl + off, nullptr, rel.get()));
    timer_begin(ctx, F_FILTER);
    launch_probe_direct(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    rel->n = ctx->h_ctrl[off + 1];
    *out = std::move(rel);
    return KB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// natural join: three strategies, tried in this order by hash_join_impl
//   cartesian  no common variable (engine.rs:1054-1071)
//   grouped    one key column over a dense id range, no post-filter: a CSR directory of the build side
//   chained    everything else: the multimap operator (1:N keys, up to 4 key columns, post-filter)
enum class Route { answered, declined, retry };

struct NatJoin {  // a natural join as hash_join_impl set it up
    const kb_rel &L, &R;
    const kb_rel &B, &Pr;   // build side: the smaller one (engine.rs:729-733); probe side: the other
    std::vector<u32> keys;  // the common variables
    std::vector<u32> slots; // result columns: L's, then R's new ones
};

// output columns of a kernel that writes the columns of `first`, then those of `second` that are not keys: `rows` rows each, placed at
// their variable's column of `rel` (whose slots are the join's); out[c] receives kernel column c
static kb_status alloc_join_out(kb_ctx* ctx, const NatJoin& j, const kb_rel& first, const kb_rel& second, u64 rows, kb_rel* rel, u32** out) {
    std::vector<u32> ks = first.slots;
    for (u32 s : second.slots) if (std::find(j.keys.begin(), j.keys.end(), s) == j.keys.end()) ks.push_back(s);
    rel->slots = j.slots;
    rel->cols.assign(j.slots.size(), Col{});
    for (size_t c = 0; c < ks.size(); c++) {
        Col col;
        KB_TRY(alloc_col(ctx, rows, &col));
        rel->cols[rel->col_of(ks[c])] = col;
        out[c] = col.ptr;
    }
    return KB_OK;
}

static kb_status join_cartesian(kb_ctx* ctx, const NatJoin& j, const FilterProg* post, std::unique_ptr<kb_rel>* out, Route* route) {
    *route = Route::declined;
    if (!j.keys.empty()) return KB_OK;
    *route = Route::answered;
    const u64 total = j.L.n * j.R.n;
    if (total > (1ull << 28)) return fail(ctx, KB_E_LIMIT, "cartesian product of %llu x %llu rows exceeds 2^28", (unsigned long long)j.L.n, (unsigned long long)j.R.n);
    std::vector<const u32*> lc, rc;
    for (auto& c : j.L.cols) lc.push_back(c.ptr);
    for (auto& c : j.R.cols) rc.push_back(c.ptr);
    auto rel = std::make_unique<kb_rel>();
    std::vector<u32*> oc(j.slots.size());
    KB_TRY(alloc_join_out(ctx, j, j.L, j.R, total, rel.get(), oc.data()));
    timer_begin(ctx, F_PROBE);
    launch_cartesian(lc.data(), (u32)j.L.n, (u32)lc.size(), rc.data(), (u32)j.R.n, (u32)rc.size(), oc.data(), ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    rel->n = total;
    if (post && !post->ops.empty()) return filter_impl(ctx, *rel, *post, out);
    *out = std::move(rel);
    return KB_OK;
}

// declines (after reading the key range back) when the range is too wide for a directory
static kb_status join_grouped(kb_ctx* ctx, const NatJoin& j, const FilterProg* post, std::unique_ptr<kb_rel>* out, Route* route) {
    *route = Route::declined;
    if (!ctx->csr_join || j.keys.size() != 1 || (post && !post->ops.empty())) return KB_OK;
    const kb_rel &B = j.B, &Pr = j.Pr;
    const u32* bk = B.cols[B.col_of(j.keys[0])].ptr;
    const u32 off = ctrl_alloc(ctx, 8);  // [0] min, [1] max, [2..3] u64 output rows, [4] ticket, [5] total, [6] zero, [7] heavy tiles
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0xFF, sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off + 1, 0, 7 * sizeof(u32), ctx->st));
    timer_begin(ctx, F_BUILD);
    launch_col_minmax(bk, (u32)B.n, ctx->ctrl + off, ctx->ctrl + off + 1, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_TRY(ctrl_read(ctx));
    const u32 kmin = ctx->h_ctrl[off], kmax = ctx->h_ctrl[off + 1];
    const u64 range = (u64)kmax - kmin + 1;
    if (!(kmax >= kmin && range <= std::max<u64>(16 * B.n, 1ull << 20) && range < (1ull << 31))) return KB_OK;
    *route = Route::answered;
    Buf dir, cursor, scratch;
    KB_TRY(alloc_buf(ctx, (range + 1) * sizeof(u32), &dir));
    KB_TRY(alloc_buf(ctx, range * sizeof(u32), &cursor));
    KB_TRY(alloc_buf(ctx, ((range + 1) / 2048 + 4) * sizeof(u32), &scratch));
    CsrTab tab{};
    tab.off = static_cast<const u32*>(dir->p);
    tab.kmin = kmin;
    tab.range = (u32)range;
    std::vector<const u32*> pay_in;
    std::vector<u32*> pay_out;
    std::vector<Col> pay_cols;
    for (size_t c = 0; c < B.slots.size(); c++) {
        if (B.slots[c] == j.keys[0]) continue;
        Col pc;
        KB_TRY(alloc_col(ctx, B.n, &pc));
        pay_cols.push_back(pc);
        pay_in.push_back(B.cols[c].ptr);
        pay_out.push_back(pc.ptr);
        tab.pay[tab.n_pay++] = pc.ptr;
    }
    timer_begin(ctx, F_BUILD, 5);
    KB_CUDA(ctx, cudaMemsetAsync(dir->p, 0, (range + 1) * sizeof(u32), ctx->st));
    launch_csr_count(bk, (u32)B.n, kmin, static_cast<u32*>(dir->p), ctx->n_sms, ctx->st);
    launch_exclusive_scan_u32(static_cast<u32*>(dir->p), (u32)range + 1, static_cast<u32*>(scratch->p), ctx->st);
    KB_CUDA(ctx, cudaMemcpyAsync(cursor->p, dir->p, range * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    launch_csr_fill(bk, (u32)B.n, kmin, static_cast<u32*>(cursor->p), pay_in.data(), pay_out.data(), tab.n_pay, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.rows_built += B.n;
    const u32* pk = Pr.cols[Pr.col_of(j.keys[0])].ptr;
    timer_begin(ctx, F_PROBE);
    launch_csr_total(pk, (u32)Pr.n, tab, reinterpret_cast<unsigned long long*>(ctx->ctrl + off + 2), ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    unsigned long long total = 0;
    memcpy(&total, ctx->h_ctrl + off + 2, sizeof total);
    if (total >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "join result of %llu rows exceeds 2^32", total);
    ProbeGParams G{};
    G.n_pcols = (u32)Pr.cols.size();
    G.n = (u32)Pr.n;
    G.n_tiles = (u32)((Pr.n + PROBEG_TILE - 1) / PROBEG_TILE);
    for (u32 c = 0; c < G.n_pcols; c++) G.pcol[c] = Pr.cols[c].ptr;
    G.pkey = (u32)Pr.col_of(j.keys[0]);
    G.tab = tab;
    auto rel = std::make_unique<kb_rel>();
    KB_TRY(alloc_join_out(ctx, j, Pr, B, total, rel.get(), G.out));
    G.cap = (u32)total;
    KB_TRY(compact_setup(ctx, G.n_tiles, ctx->ctrl + off + 4, &G.c));
    Buf heavy;  // tiles whose expansion is spread over the grid by the second launch (skewed keys)
    if (total > PROBEG_HEAVY) {
        KB_TRY(alloc_buf(ctx, (size_t)G.n_tiles * sizeof(ProbeGParams::Heavy), &heavy));
        G.heavy = static_cast<ProbeGParams::Heavy*>(heavy->p);
        G.heavy_count = ctx->ctrl + off + 7;
    }
    ctx->stats.rows_probed += Pr.n;
    if (total) {
        timer_begin(ctx, F_PROBE, G.heavy ? 2 : 1);
        launch_probe_grouped(G, ctx->n_sms, ctx->st);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
    }
    rel->n = total;
    // dir / cursor / payload copies are released stream-ordered (cudaFreeAsync on ctx->st), i.e. after the launch above
    *out = std::move(rel);
    return KB_OK;
}

// the first pass writes what fits in max(|L|, |R|) rows and counts all of them; a larger result takes a second pass of that size
static kb_status join_chained(kb_ctx* ctx, const NatJoin& j, const FilterProg* post, std::unique_ptr<kb_rel>* out) {
    const kb_rel &B = j.B, &Pr = j.Pr;
    ChainTab T{};
    T.n_slots = pow2_at_least(B.n * 2);
    T.n_keys = (u32)j.keys.size();
    Buf slots_buf, next_buf;
    KB_TRY(alloc_buf(ctx, (size_t)T.n_slots * sizeof(u64), &slots_buf));
    KB_TRY(alloc_buf(ctx, (size_t)B.n * sizeof(u32), &next_buf));
    T.slots = static_cast<u64*>(slots_buf->p);
    T.next = static_cast<u32*>(next_buf->p);
    for (u32 q = 0; q < T.n_keys; q++) T.bkey[q] = B.cols[B.col_of(j.keys[q])].ptr;
    timer_begin(ctx, F_BUILD);
    KB_CUDA(ctx, cudaMemsetAsync(T.slots, 0xFF, (size_t)T.n_slots * sizeof(u64), ctx->st));
    launch_build_chained(T, (u32)B.n, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.rows_built += B.n;

    ProbeCParams P{};
    P.tab = T;
    P.n_pcols = (u32)Pr.cols.size();
    P.n = (u32)Pr.n;
    P.n_tiles = (u32)((Pr.n + PROBEC_TILE - 1) / PROBEC_TILE);
    for (u32 c = 0; c < P.n_pcols; c++) P.pcol[c] = Pr.cols[c].ptr;
    for (u32 q = 0; q < T.n_keys; q++) P.pkey[q] = (u32)Pr.col_of(j.keys[q]);
    std::vector<u32> kernel_slots = Pr.slots;  // kernel output order: probe columns, then build payload columns
    for (size_t c = 0; c < B.slots.size(); c++) {
        if (std::find(j.keys.begin(), j.keys.end(), B.slots[c]) != j.keys.end()) continue;
        P.bpay[P.n_bpay++] = B.cols[c].ptr;
        kernel_slots.push_back(B.slots[c]);
    }
    P.n_out = (u32)kernel_slots.size();
    std::vector<FilterOp> ops;
    if (post) KB_TRY(compile_prog(ctx, *post, kernel_slots, &ops));
    P.n_ops = (u32)ops.size();
    for (size_t i = 0; i < ops.size(); i++) P.ops[i] = ops[i];
    P.nt = numtab(ctx);
    const u32 off = ctrl_alloc(ctx, 8);  // [0] ticket, [1] total (32-bit positions), [2] zero, [4..5] exact total in 64 bits
    P.total64 = reinterpret_cast<unsigned long long*>(ctx->ctrl + off + 4);
    u64 cap = std::max(Pr.n, B.n);
    ctx->stats.rows_probed += Pr.n;
    auto rel = std::make_unique<kb_rel>();
    for (int attempt = 0; attempt < 2; attempt++) {
        KB_TRY(alloc_join_out(ctx, j, Pr, B, cap, rel.get(), P.out));
        P.cap = (u32)std::min<u64>(cap, 0xFFFFFFF0ull);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 8 * sizeof(u32), ctx->st));
        KB_TRY(compact_setup(ctx, P.n_tiles, ctx->ctrl + off, &P.c));
        timer_begin(ctx, F_PROBE);
        launch_probe_chained(P, ctx->n_sms, ctx->st);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        unsigned long long total = 0;
        memcpy(&total, ctx->h_ctrl + off + 4, sizeof total);
        if (total >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "join result of %llu rows exceeds 2^32", total);
        rel->n = total;
        if (total <= cap) break;
        if (attempt == 1) return fail(ctx, KB_E_LIMIT, "join output did not fit after resizing");
        cap = total;  // the first pass doubled as the exact count
    }
    *out = std::move(rel);
    return KB_OK;
}

kb_status hash_join_impl(kb_ctx* ctx, const kb_rel& L, const kb_rel& R, const FilterProg* post, std::unique_ptr<kb_rel>* out) {
    const bool build_left = L.n <= R.n;
    NatJoin j{L, R, build_left ? L : R, build_left ? R : L, {}, L.slots};
    for (u32 s : R.slots) {
        if (L.col_of(s) >= 0) j.keys.push_back(s);
        else j.slots.push_back(s);
    }
    if (j.slots.size() > KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "join result has more than %d columns", KB_MAX_COLS);
    if (L.n == 0 || R.n == 0) return empty_rel(ctx, j.slots, out);  // engine.rs:714-716
    if (L.n >= 0xFFFFFFF0ull || R.n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "relation too large");
    Route r;
    KB_TRY(join_cartesian(ctx, j, post, out, &r));
    if (r == Route::answered) return KB_OK;
    if (j.keys.size() > 4) return fail(ctx, KB_E_LIMIT, "join on more than 4 common variables");
    KB_TRY(join_grouped(ctx, j, post, out, &r));
    if (r == Route::answered) return KB_OK;
    return join_chained(ctx, j, post, out);
}

std::unique_ptr<kb_rel> select_cols(const kb_rel& in, const std::vector<u32>& slots) {
    auto r = std::make_unique<kb_rel>();
    r->n = in.n;
    for (u32 s : slots) {
        int c = in.col_of(s);
        if (c < 0) continue;
        r->slots.push_back(s);
        r->cols.push_back(in.cols[c]);
    }
    return r;
}

// ---------------------------------------------------------------------------------------------------------------
// star join: five routes, tried in this order by star_join_impl
//   R1 one-kernel index join   every build side is a persistent table of the store index: one probe_index_kernel (fused GROUP BY)
//   R2 index join with builds  direct tables built from predicate slices, then the fused multiway probe
//   R3 fused scan + build      the scan fills the direct tables, then the fused multiway probe
//   R4 scan, then builds       direct tables in batches of at most MAXT per probe launch
//   R5 chained joins           natural joins on the multimap operator: 1:N keys, quirk Q3, sparse key ranges
struct StarQuery {  // a star join, validated once: what every route reads
    u32 join_slot = 0, K = 0;
    const kb_pattern* pats = nullptr;
    std::vector<std::vector<u32>> pv, psrc;  // variables of pattern k in order of appearance, and their positions (0 s, 1 p, 2 o)
    std::vector<u32> all_slots;              // column order of the result
    std::vector<FilterProg> pushdown;        // FILTER conjuncts over one pattern's variables, evaluated while that pattern is read
    FilterProg post;                         // the other conjuncts, evaluated on the joined row
    std::vector<u32> key_pos;                // position of the join variable in pattern k
    // fast path shape: every pattern binds exactly two variables in subject and object position (the join variable + one more)
    bool all_pairs = false;
    // no variable but the join variable occurs in two patterns (quirk Q3: the reference never checks the others — we must, so such
    // shapes take the natural-join chain)
    bool only_join_shared = true;
};

kb_status split_filter(kb_ctx* ctx, const kb_filter_op* filter, u32 n_ops, const std::vector<std::vector<u32>>& pv,
                       const std::vector<u32>& all_slots, std::vector<FilterProg>* pushdown, FilterProg* post) {
    std::vector<FilterProg> conj;
    if (!split_conjuncts(filter, n_ops, &conj)) return fail(ctx, KB_E_INVALID, "malformed filter program");
    pushdown->assign(pv.size(), FilterProg{});
    for (auto& c : conj) {
        std::set<u32> fs = filter_slots(c);
        for (u32 s : fs) if (std::find(all_slots.begin(), all_slots.end(), s) == all_slots.end())
            return fail(ctx, KB_E_UNSUPPORTED, "filter references slot %u which no pattern binds (the reference evaluates it to false, types.rs:149-151)", s);
        int target = -1;
        for (size_t k = 0; k < pv.size() && target < 0; k++) {
            bool all = true;
            for (u32 s : fs) if (std::find(pv[k].begin(), pv[k].end(), s) == pv[k].end()) all = false;
            if (all) target = (int)k;
        }
        and_into(target >= 0 ? &(*pushdown)[target] : post, c);
    }
    return KB_OK;
}

static kb_status star_query(kb_ctx* ctx, u32 join_slot, const kb_pattern* pats, u32 K, const kb_filter_op* filter, u32 n_ops, StarQuery* q) {
    if (K == 0 || K > (u32)MAXP) return fail(ctx, KB_E_LIMIT, "a star join takes 1..%d patterns (got %u)", MAXP, K);
    KB_TRY(validate_filter(ctx, filter, n_ops));
    q->join_slot = join_slot;
    q->K = K;
    q->pats = pats;
    q->pv.resize(K);
    q->psrc.resize(K);
    q->key_pos.resize(K);
    for (u32 k = 0; k < K; k++) {
        KB_TRY(check_pattern(ctx, pats[k]));
        pattern_vars(pats[k], &q->pv[k], &q->psrc[k]);
        const auto j = std::find(q->pv[k].begin(), q->pv[k].end(), join_slot);
        if (j == q->pv[k].end()) return fail(ctx, KB_E_INVALID, "star join: pattern %u does not contain the join variable (slot %u)", k, join_slot);
        q->key_pos[k] = q->psrc[k][j - q->pv[k].begin()];
        for (u32 s : q->pv[k]) if (std::find(q->all_slots.begin(), q->all_slots.end(), s) == q->all_slots.end()) q->all_slots.push_back(s);
    }
    if (q->all_slots.size() > KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "more than %d variables", KB_MAX_COLS);
    KB_TRY(split_filter(ctx, filter, n_ops, q->pv, q->all_slots, &q->pushdown, &q->post));
    q->all_pairs = K >= 2;
    for (u32 k = 0; k < K; k++) if (!(q->pv[k].size() == 2 && q->psrc[k][0] == 0 && q->psrc[k][1] == 2)) q->all_pairs = false;
    for (u32 a = 0; a < K; a++)
        for (u32 b = a + 1; b < K; b++)
            for (u32 s2 : q->pv[a]) if (s2 != join_slot && std::find(q->pv[b].begin(), q->pv[b].end(), s2) != q->pv[b].end()) q->only_join_shared = false;
    return KB_OK;
}

// What direct builds proved about the keys of a (predicate, key position) pair on this store version: a build that met a duplicate key
// makes the pair multi-valued (direct tables are not tried for it again); one that inserted the whole (?s P ?o) relation without
// meeting one makes it single-valued (later builds use plain stores). A filtered or non-pair build side proves nothing about the rest
// of the relation, and a pattern with a variable predicate names no pair.
enum class Keys { unknown, single, multi };

// the keys of pattern k's build side; `unique`: its slice of the store index says they are single-valued (x_unique / y_unique)
static Keys build_keys(const kb_ctx* ctx, const StarQuery& q, u32 k, bool unique = false) {
    const kb_pattern& pt = q.pats[k];
    if (pt.p.is_var) return Keys::unknown;
    const std::pair<u32, u32> pk{pt.p.value, q.key_pos[k]};
    if (ctx->multi_valued.count(pk)) return Keys::multi;
    return unique || ctx->single_valued.count(pk) ? Keys::single : Keys::unknown;
}

// records what a direct build of pattern k proved: `dup` a duplicate key; else, when the build side was pair-shaped, that it has none
static void build_proved(kb_ctx* ctx, const StarQuery& q, u32 k, bool dup, bool pair) {
    const kb_pattern& pt = q.pats[k];
    if (pt.p.is_var) return;
    const std::pair<u32, u32> pk{pt.p.value, q.key_pos[k]};
    if (dup) ctx->multi_valued.insert(pk);
    else if (pair && q.pushdown[k].ops.empty()) ctx->single_valued.insert(pk);
}

// key range of the join variable over the store, from the load-time column statistics of its segments
static kb_status store_key_range(kb_ctx* ctx, const StarQuery& q, u32* kmin, u32* kmax) {
    *kmin = 0xFFFFFFFFu;
    *kmax = 0;
    for (auto& sg : ctx->segs) {
        if (sg.n == 0) continue;
        if (!sg.has_stats) KB_TRY(segment_stats(ctx, &sg));
        for (u32 k = 0; k < q.K; k++) { const u32 c = q.key_pos[k]; *kmin = std::min(*kmin, sg.cmin[c]); *kmax = std::max(*kmax, sg.cmax[c]); }
    }
    return KB_OK;
}

// a subject-sharded store (kb_set_sharding) owns every world-th block of ids: subject keys are compacted by this shift so that the
// tables stay dense. 0 unless every key is a subject and no segment may hold a foreign subject (current_stats: the statistics that
// say so must have been taken under the current sharding)
static u32 subject_cshift(const kb_ctx* ctx, const StarQuery& q, bool current_stats) {
    bool subj = true;
    for (u32 k = 0; k < q.K; k++) if (q.key_pos[k] != 0) subj = false;
    for (auto& sg : ctx->segs)
        if (sg.n && (!sg.sharded_ok || (current_stats && (!sg.has_stats || sg.stats_world != ctx->shard_world)))) subj = false;
    u32 cshift = 0;
    const u32 w = ctx->shard_world;
    if (subj && w > 1 && (w & (w - 1)) == 0) while ((1u << cshift) < w) cshift++;
    return cshift;
}

// a persistent table of the store index, looked up like spo[s][P] (subject key) or pos[P][o] (object key)
static DirectTab persistent_tab(const PredSlice& s, bool key_is_y) {
    DirectTab D{};
    D.tab = static_cast<const u32*>(key_is_y ? s.ytab->p : s.xtab->p);
    D.kmin = key_is_y ? s.ytab_min : s.xtab_min;
    D.range = key_is_y ? s.ytab_range : s.xtab_range;
    D.cshift = key_is_y ? 0u : s.tab_cshift;
    if (!key_is_y && s.xcode) {
        D.code = static_cast<const u8*>(s.xcode->p);
        D.dict = static_cast<const u32*>(s.xdict->p);
        D.n_dict = s.n_xdict;
    }
    return D;
}

// the fused multiway probe over pair rows (probe_fast_kernel) against T direct tables; P may carry a pre-filter. The output columns
// (`ocs`, `n` rows each) are appended to res->cols; the row count lands in ctrl[1]
static kb_status probe_fast(kb_ctx* ctx, ProbeFParams& P, const uint2* pairs, u64 n, u32 key_is_y, const DirectTab* dt, u32 T,
                            const std::vector<OutCol>& ocs, const std::vector<FilterOp>& fops, u32* ctrl, const u32* abort_flag, kb_rel* res) {
    P.pairs = pairs;
    P.key_is_y = key_is_y;
    P.n = (u32)n;
    P.n_tiles = (u32)((n + PROBEF_TILE - 1) / PROBEF_TILE);
    P.T = T;
    for (u32 q = 0; q < T; q++) P.tab[q] = dt[q];
    KB_TRY(probe_setup(ctx, &P, n, ocs, fops, ctrl, abort_flag, res));
    timer_begin(ctx, F_PROBE);
    launch_probe_fast(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    ctx->stats.rows_probed += n;
    return KB_OK;
}

// what the store index says about a star of (?s P ?o) patterns
struct IndexSlices {
    bool shape = false;   // valid index, every pattern (?s P ?o), at most MAXT build sides
    bool empty = false;   // a pattern's predicate does not occur in the store: the answer is empty
    bool usable = false;  // every predicate constant and present, the patterns share only the join variable
    std::vector<const PredSlice*> sl;
    std::vector<bool> persistent;  // the key column of pattern k has a persistent table in the index: it needs no build
    bool all_persistent = false;
    u32 kmin = 0xFFFFFFFFu, kmax = 0, cshift = 0;
    int probe_k = -1;
};

static IndexSlices index_slices(const kb_ctx* ctx, const StarQuery& q) {
    IndexSlices ix;
    ix.shape = ctx->use_index && ctx->index_version == ctx->store_version && q.all_pairs && q.K - 1 <= (u32)MAXT;
    if (!ix.shape) return ix;
    const u32 K = q.K;
    bool ok = q.only_join_shared, empty = false;
    ix.sl.assign(K, nullptr);
    for (u32 k = 0; k < K; k++) {
        if (q.pats[k].p.is_var) { ok = false; break; }
        auto it = ctx->index.find(q.pats[k].p.value);
        if (it == ctx->index.end() || it->second.n == 0) { empty = true; continue; }  // predicate absent from the store
        ix.sl[k] = &it->second;
    }
    ix.empty = ok && empty;
    ix.usable = ok && !empty;
    if (!ix.usable) return ix;
    // key range of the join variable from the slices (its position is the same in every pattern that can take this path)
    for (u32 k = 0; k < K; k++) {
        const bool y = q.key_pos[k] == 2;
        ix.kmin = std::min(ix.kmin, y ? ix.sl[k]->ymin : ix.sl[k]->xmin);
        ix.kmax = std::max(ix.kmax, y ? ix.sl[k]->ymax : ix.sl[k]->xmax);
    }
    ix.cshift = subject_cshift(ctx, q, true);
    ix.kmin = compact_key(ix.kmin, ix.cshift);
    ix.kmax = compact_key(ix.kmax, ix.cshift);
    ix.persistent.resize(K);
    ix.all_persistent = true;
    for (u32 k = 0; k < K; k++) {
        ix.persistent[k] = q.key_pos[k] == 2 ? (bool)ix.sl[k]->ytab : ((bool)ix.sl[k]->xtab && ix.sl[k]->tab_cshift == ix.cshift);
        if (!ix.persistent[k]) ix.all_persistent = false;
    }
    // probe side: prefer a pattern WITHOUT a persistent table (it would need a build), then the smallest slice (fewest lookups);
    // when builds remain, the classic choice: the largest unfiltered slice probes, filtered sides build
    int& probe_k = ix.probe_k;
    if (ix.all_persistent) {
        // no builds at all: the probe side should be the most selective stream — a pattern that carries its own FILTER (evaluated
        // on the probe row before any lookup), else the smallest slice
        for (u32 k = 0; k < K; k++)
            if (!q.pushdown[k].ops.empty() && q.pushdown[k].ops.size() <= 8 && (probe_k < 0 || ix.sl[k]->n < ix.sl[probe_k]->n)) probe_k = (int)k;
        if (probe_k < 0) { probe_k = 0; for (u32 k = 1; k < K; k++) if (ix.sl[k]->n < ix.sl[probe_k]->n) probe_k = (int)k; }
    } else {
        for (u32 k = 0; k < K; k++) if (q.pushdown[k].ops.empty() && (probe_k < 0 || ix.sl[k]->n > ix.sl[probe_k]->n)) probe_k = (int)k;
        if (probe_k < 0) { probe_k = 0; for (u32 k = 1; k < K; k++) if (ix.sl[k]->n > ix.sl[probe_k]->n) probe_k = (int)k; }
    }
    return ix;
}

kb_status launch_index_rows(kb_ctx* ctx, ProbeIParams& P, const std::vector<Col>& cols) {
    for (size_t c = 0; c < cols.size(); c++) P.out[c] = cols[c].ptr;
    KB_TRY(compact_setup(ctx, P.n_tiles, ctx->fast_cb, &P.c));
    timer_begin(ctx, F_PROBE);
    launch_probe_index(P, nullptr, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

static kb_status resolve_index_plan(kb_ctx* ctx, const StarQuery& q, const IndexSlices& ix, const AggSpec* agg, IndexPlan* ip) {
    if (!ix.shape) { ip->why = "it needs a valid store index (kb_store_build_index) and (?s P ?o) patterns"; return KB_OK; }
    if (ix.empty) { ip->why = "a pattern's predicate does not occur in the store (the answer is empty)"; return KB_OK; }
    if (!ix.usable || !ix.all_persistent || !ctx->fast_index_kernel || ix.sl[ix.probe_k]->chunks.size() > (size_t)PROBEI_MAXSEG) {
        ip->why = "every pattern (?s P ?o) over a predicate whose key column has a persistent table in the store index";
        return KB_OK;
    }
    const u32 pk = (u32)ix.probe_k, T = q.K - 1;
    const PredSlice& PS = *ix.sl[pk];
    ProbeIParams& P = ip->P;
    ip->out_slots = q.pv[pk];
    FilterProg postp = q.post;  // filters of patterns that are not built (every one here) run on the joined row
    u32 t = 0;
    for (u32 k = 0; k < q.K; k++) {
        if (k == pk) continue;
        const bool y = q.key_pos[k] == 2;
        P.tab[t++] = persistent_tab(*ix.sl[k], y);
        and_into(&postp, q.pushdown[k]);
        ip->out_slots.push_back(q.pv[k][y ? 0 : 1]);
    }
    const FilterProg& pf = q.pushdown[pk];
    if (pf.ops.size() > 8) and_into(&postp, pf);
    else if (!pf.ops.empty()) {
        std::vector<FilterOp> fo;  // slots of the probe pattern's own filter -> pair halves (x = subject, y = object)
        KB_TRY(compile_prog(ctx, pf, q.pv[pk], &fo));
        const bool typed = PS.typed(ctx->num_version) && fo.size() == 1 && fo[0].op == KB_F_CMP_NUM && fo[0].slot == 1u;
        if (typed) {
            P.pre_mode = 1; P.pre_cmp = fo[0].cmp; P.pre_val = fo[0].value;
        } else {
            P.pre_mode = 2; P.n_pre = (u32)fo.size();
            for (size_t i = 0; i < fo.size(); i++) P.pre_ops[i] = fo[i];
        }
    }
    ip->n_out = 2 + T;
    std::vector<FilterOp> fops;
    KB_TRY(compile_prog(ctx, postp, ip->out_slots, &fops));
    P.n_ops = (u32)fops.size();
    for (size_t i = 0; i < fops.size(); i++) P.ops[i] = fops[i];
    // table mode: the probe pattern's own subject table is the probe stream (keys ascending whatever the store / id order)
    const bool tab_mode = ctx->probe_table_mode && !ctx->ordered && ix.persistent[pk] && q.key_pos[pk] == 0 &&
                          (P.pre_mode != 1u || (PS.xkey && PS.xkey_version == ctx->num_version && ctx->numv_version == ctx->num_version));
    if (tab_mode) {
        // walk the slots that can hold a key (smallest to largest live subject), not the table's growth headroom nor the
        // slots an evicted past has left empty; the first slot stays 128-byte aligned for the bulk loads
        const u32 lo = ((compact_key(PS.xmin, PS.tab_cshift) - PS.xtab_min) / 32u) * 32u;
        const u32 hi = std::min<u32>(PS.xtab_range, compact_key(PS.xmax, PS.tab_cshift) - PS.xtab_min + 1u);
        P.ptab = static_cast<const u32*>(PS.xtab->p) + lo;
        if (P.pre_mode == 1u) {  // FILTER(?o <cmp> c) on the value becomes a range of its ranks in the value order
            P.pkey = static_cast<const u16*>(PS.xkey->p) + lo;
            const u32 n_v = (u32)ctx->h_numv.size();
            P.key_shift = kb_nr::rank_shift(n_v);
            const kb_nr::Range16 r = kb_nr::range16(kb_nr::cmp_range(P.pre_cmp, ctx->h_numv.data(), n_v, P.pre_val), P.key_shift);
            P.key_lo = r.lo;
            P.key_hi = r.hi;
        }
        P.ptab_min = PS.xtab_min + lo;
        P.ptab_range = hi > lo ? hi - lo : 0u;
        P.ptab_cshift = PS.tab_cshift;
        P.shard_rank = ctx->shard_rank;
        P.n_tiles = (u32)(((u64)P.ptab_range + PROBEF_TILE - 1) / PROBEF_TILE);
    } else {
        for (auto& ch : PS.chunks) {  // one chunk per store segment: an RSP window of slides is walked in ONE launch
            if (ch.n == 0) continue;
            ProbeISeg& g = P.seg[P.n_seg++];
            g.pairs = reinterpret_cast<const uint2*>(ch.pairs.ptr);
            g.ynum = P.pre_mode == 1u ? static_cast<const double*>(ch.ynum->p) : nullptr;
            g.n = (u32)ch.n;
            g.tile0 = P.n_tiles;
            P.n_tiles += (u32)((ch.n + PROBEF_TILE - 1) / PROBEF_TILE);
        }
    }
    P.key_is_y = q.key_pos[pk] == 2 ? 1u : 0u;
    P.n = (u32)PS.n;
    P.T = T;
    P.cap = (u32)PS.n;
    P.nt = numtab(ctx);
    P.cb = ctx->fast_cb;
    P.host_total = ctx->d_fast;
    ip->all_slots = q.all_slots;
    ip->probe_rows = PS.n;
    if (agg) {  // GROUP BY folded into the kernel when the join binds the group variable (and the aggregated one, if any)
        int gsel = -1, asel = -1;
        for (u32 c = 0; c < ip->n_out; c++) {
            if (ip->out_slots[c] == agg->group_slot) gsel = (int)c;
            if (agg->has_agg && ip->out_slots[c] == agg->agg_slot) asel = (int)c;
        }
        const bool needs_value = agg->has_agg && agg->kind != KB_AGG_COUNT;
        if (gsel >= 0 && (!needs_value || asel >= 0)) {
            ip->agg = true;
            ip->has_agg = agg->has_agg;
            ip->agg_kind = agg->has_agg ? agg->kind : (u32)KB_AGG_COUNT;
            ip->agg_slot = agg->agg_slot;
            ip->group_slot = agg->group_slot;
            P.gsel = (u32)gsel;
            P.asel = asel >= 0 ? (u32)asel : 0u;
            P.akind = ip->agg_kind;
        }
    }
    ip->ok = true;
    return KB_OK;
}

kb_status resolve_index_plan(kb_ctx* ctx, u32 join_slot, const kb_pattern* pats, u32 K, const kb_filter_op* filter, u32 n_ops, const AggSpec* agg,
                             IndexPlan* plan) {
    StarQuery q;
    KB_TRY(star_query(ctx, join_slot, pats, K, filter, n_ops, &q));
    return resolve_index_plan(ctx, q, index_slices(ctx, q), agg, plan);
}

// R1: the whole join is one launch of probe_index_kernel
static kb_status index_join_one_kernel(kb_ctx* ctx, const StarQuery& q, const IndexSlices& ix, AggSpec* agg, std::unique_ptr<kb_rel>* out,
                                       Route* route) {
    *route = Route::answered;
    if (ix.empty) return empty_rel(ctx, q.all_slots, out);
    IndexPlan ip;
    KB_TRY(resolve_index_plan(ctx, q, ix, agg, &ip));
    if (!ip.ok) {
        *route = Route::declined;
        return KB_OK;
    }
    ProbeIParams& P = ip.P;
    if (ip.agg) {
        // GROUP BY folded into the probe kernel: no joined row is written. One try with a 4096-slot table; more groups than that (or
        // a group / aggregate variable the join does not bind) leave agg->applied false: the caller groups separately
        const kb_agg a1{agg->kind, agg->agg_slot};
        const u32 n_aggs = agg->has_agg ? 1u : 0u;
        GroupParams G = group_params(ctx, 1, &a1, n_aggs);
        GroupTable tab;
        KB_TRY(group_table_create(ctx, 1u << 12, true, &G, &tab));
        KB_TRY(compact_setup(ctx, P.n_tiles, ctx->fast_cb, &P.c));
        P.c.ordered = 0;  // the rows are folded into groups: no output order to keep
        timer_begin(ctx, F_PROBE);
        launch_probe_index(P, &G, ctx->n_sms, ctx->st);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        ctx->stats.rows_probed += ip.probe_rows;
        ctx->stats.index_joins++;
        auto g = std::make_unique<kb_groups>(1, &a1, n_aggs);
        bool overflowed;
        KB_TRY(group_table_collect(ctx, tab, g.get(), &overflowed));
        if (!overflowed) {
            agg->n_rows = *reinterpret_cast<volatile u32*>(ctx->h_fast);
            agg->groups = std::move(g);
            agg->applied = true;
            return KB_OK;
        }
        // fall through: join without the fused GROUP BY (the control block was left clean by the kernel)
    }
    auto res = std::make_unique<kb_rel>();
    res->slots = ip.out_slots;
    KB_TRY(alloc_strided_cols(ctx, ip.probe_rows, ip.n_out, &res->cols));
    KB_TRY(launch_index_rows(ctx, P, res->cols));
    ctx->stats.rows_probed += ip.probe_rows;
    ctx->stats.index_joins++;
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    timers_flush(ctx);
    ctx->stats.d2h_bytes += sizeof(u32);
    res->n = *reinterpret_cast<volatile u32*>(ctx->h_fast);
    *out = select_cols(*res, q.all_slots);
    return KB_OK;
}

// R2: build sides are inserted from their slices (pushed-down FILTER evaluated in the build kernel), the probe side IS its slice
// (zero copy). A duplicate key asks for a retry: the (predicate, position) is then cached as multi-valued, which this route declines
static kb_status index_join_built(kb_ctx* ctx, const StarQuery& q, const IndexSlices& ix, std::unique_ptr<kb_rel>* out, Route* route) {
    *route = Route::declined;
    if (!ix.usable) return KB_OK;
    const u32 K = q.K, pk = (u32)ix.probe_k, T = K - 1;
    const u64 rng = ix.kmax >= ix.kmin ? (u64)ix.kmax - ix.kmin + 1 : 0;
    for (u32 k = 0; k < K; k++) {
        if (k == pk || ix.persistent[k]) continue;
        if (rng == 0 || rng > std::max<u64>(8 * ix.sl[k]->n, 1ull << 16) || rng > (1ull << 31)) return KB_OK;
        if (build_keys(ctx, q, k) == Keys::multi) return KB_OK;
    }
    for (u32 k = 0; k < K; k++) if (!ix.sl[k]->single()) return KB_OK;  // the build kernel reads one contiguous slice per pattern
    const u32 range = (u32)rng;
    const u32 off = ctrl_alloc(ctx, 16 + 2 * MAXT);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, (16 + 2 * MAXT) * sizeof(u32), ctx->st));
    std::vector<Buf> tabs;
    DirectTab dt[MAXT];
    std::vector<u32> tab_k;
    std::vector<u32> out_slots = q.pv[pk];
    std::vector<OutCol> ocs{OutCol{OUT_PROBE, 0, 0}, OutCol{OUT_PROBE, 1, 0}};
    FilterProg postp = q.post;  // filters of patterns that are not built (probe side, persistent tables) run on the joined row
    const bool pre_filter = !q.pushdown[pk].ops.empty() && q.pushdown[pk].ops.size() <= 8;
    if (!pre_filter) and_into(&postp, q.pushdown[pk]);
    for (u32 k = 0; k < K; k++) if (k != pk && !ix.persistent[k]) { Buf b; KB_TRY(alloc_buf(ctx, (size_t)range * sizeof(u32), &b)); tabs.push_back(b); }
    const u32 n_build = (u32)tabs.size();
    if (n_build) timer_begin(ctx, F_BUILD, (int)n_build);
    if (n_build > 1) {
        KB_CUDA(ctx, cudaEventRecord(ctx->ev_fork, ctx->st));
        KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st2, ctx->ev_fork, 0));
    }
    u32 t = 0, bi = 0;
    for (u32 k = 0; k < K; k++) {
        if (k == pk) continue;
        const bool y = q.key_pos[k] == 2;
        if (ix.persistent[k]) {
            dt[t] = persistent_tab(*ix.sl[k], y);
            and_into(&postp, q.pushdown[k]);
        } else {
            cudaStream_t bs = (n_build > 1 && (bi & 1)) ? ctx->st2 : ctx->st;
            u32* tab = static_cast<u32*>(tabs[bi]->p);
            KB_CUDA(ctx, cudaMemsetAsync(tab, 0xFF, (size_t)range * sizeof(u32), bs));
            BuildPairsParams B{};
            B.kv = reinterpret_cast<const uint2*>(ix.sl[k]->single()->pairs.ptr);
            B.n = (u32)ix.sl[k]->n;
            B.key_is_y = y ? 1u : 0u;
            B.pred = q.pats[k].p.value;
            B.table = tab; B.kmin = ix.kmin; B.range = range; B.cshift = ix.cshift;
            B.dup_flag = ctx->ctrl + off + 16 + t;
            B.count = ctx->ctrl + off + 16 + MAXT + t;
            B.trusted = build_keys(ctx, q, k, y ? ix.sl[k]->y_unique : ix.sl[k]->x_unique) == Keys::single ? 1u : 0u;
            B.nt = numtab(ctx);
            std::vector<FilterOp> fo;  // the pattern's own filter, over the positions of (s, P, o)
            KB_TRY(compile_prog(ctx, q.pushdown[k], q.pv[k], &fo, &q.psrc[k]));
            B.n_ops = (u32)fo.size();
            for (size_t i = 0; i < fo.size(); i++) B.ops[i] = fo[i];
            launch_build_direct_pairs_filtered(B, ctx->n_sms, bs);
            dt[t] = DirectTab{};
            dt[t].tab = tab; dt[t].kmin = ix.kmin; dt[t].range = range; dt[t].cshift = ix.cshift;
            ctx->stats.rows_built += ix.sl[k]->n;
            bi++;
        }
        out_slots.push_back(q.pv[k][y ? 0 : 1]);
        ocs.push_back(OutCol{OUT_TABVAL, t, 0});
        tab_k.push_back(k);
        t++;
    }
    if (n_build > 1) {
        KB_CUDA(ctx, cudaEventRecord(ctx->ev_join, ctx->st2));
        KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, ctx->ev_join, 0));
    }
    if (n_build) timer_end(ctx);
    const PredSlice& PS = *ix.sl[pk];
    auto res = std::make_unique<kb_rel>();
    res->slots = out_slots;
    std::vector<FilterOp> fops;
    KB_TRY(compile_prog(ctx, postp, out_slots, &fops));
    ProbeFParams P{};
    if (pre_filter) {  // slots of the probe pattern's own filter -> pair halves (x = subject, y = object)
        std::vector<FilterOp> fo;
        KB_TRY(compile_prog(ctx, q.pushdown[pk], q.pv[pk], &fo));
        P.n_pre = (u32)fo.size();
        for (size_t i = 0; i < fo.size(); i++) P.pre_ops[i] = fo[i];
        if (PS.typed(ctx->num_version)) P.pre_num = static_cast<const double*>(PS.single()->ynum->p);
    }
    KB_TRY(probe_fast(ctx, P, reinterpret_cast<const uint2*>(PS.single()->pairs.ptr), PS.n, q.key_pos[pk] == 2 ? 1u : 0u, dt, T, ocs, fops,
                      ctx->ctrl + off, nullptr, res.get()));
    ctx->stats.index_joins++;
    KB_TRY(ctrl_read(ctx));
    for (u32 q2 = 0; q2 < T; q2++) if (ctx->h_ctrl[off + 16 + q2]) {
        *route = Route::retry;
        build_proved(ctx, q, tab_k[q2], true, true);
    }
    if (*route == Route::retry) return KB_OK;
    for (u32 q2 = 0; q2 < T; q2++) if (!ix.persistent[tab_k[q2]]) build_proved(ctx, q, tab_k[q2], false, true);
    res->n = ctx->h_ctrl[off + 1];
    *out = select_cols(*res, q.all_slots);
    *route = Route::answered;
    return KB_OK;
}

// R3: the build-side patterns insert straight into their direct tables while the store is scanned; only the probe-side pattern is
// materialised. Needs the key range before the scan (load-time statistics) and a probe side chosen without knowing the counts: the
// last pattern that carries no pushed-down filter (a filtered side is the smaller build side). A duplicate or out-of-range key asks
// for a retry without the fusion (the chained operator needs the build rows)
static kb_status fused_scan_join(kb_ctx* ctx, const StarQuery& q, std::unique_ptr<kb_rel>* out, Route* route) {
    *route = Route::declined;
    const u32 K = q.K;
    if (!q.all_pairs || K - 1 > (u32)MAXT || ctx->upload_stats_off >= 0 || ctx->n_triples == 0) return KB_OK;
    u32 kmn, kmx;
    KB_TRY(store_key_range(ctx, q, &kmn, &kmx));
    const u32 cshift = subject_cshift(ctx, q, false);
    if (kmx >= kmn) { kmn = compact_key(kmn, cshift); kmx = compact_key(kmx, cshift); }
    const u64 rng = kmx >= kmn ? (u64)kmx - kmn + 1 : 0;
    if (rng == 0 || rng > std::max<u64>(4 * ctx->n_triples, 1ull << 16) || rng > (1ull << 31) || !q.only_join_shared) return KB_OK;
    int probe_k = -1;
    for (u32 k = 0; k < K; k++) if (q.pushdown[k].ops.empty()) probe_k = (int)k;
    if (probe_k < 0) probe_k = (int)K - 1;
    for (u32 k = 0; k < K; k++)
        if ((int)k != probe_k && build_keys(ctx, q, k) == Keys::multi) return KB_OK;
    const u32 range = (u32)rng;
    const u32 off = ctrl_alloc(ctx, 8 + MAXT);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, (8 + MAXT) * sizeof(u32), ctx->st));
    std::vector<ScanTable> st(K);
    std::vector<Buf> tabs;
    std::vector<u32> tab_of(K, 0);
    DirectTab dt[MAXT];
    std::vector<u32> out_slots = q.pv[probe_k];
    std::vector<OutCol> ocs{OutCol{OUT_PROBE, 0, 0}, OutCol{OUT_PROBE, 1, 0}};
    timer_begin(ctx, F_BUILD, 0);
    u32 t = 0;
    for (u32 k = 0; k < K; k++) {
        if ((int)k == probe_k) continue;
        Buf b;
        KB_TRY(alloc_buf(ctx, (size_t)range * sizeof(u32), &b));
        tabs.push_back(b);
        st[k].tab = static_cast<u32*>(b->p);
        st[k].clear = true;  // cleared by the scan (scan_segments)
        st[k].kmin = kmn; st[k].range = range; st[k].cshift = cshift;
        st[k].key_is_o = q.key_pos[k] == 2 ? 1u : 0u;
        st[k].trusted = build_keys(ctx, q, k) == Keys::single ? 1u : 0u;
        st[k].dup_flag = ctx->ctrl + off + 8 + t;
        dt[t] = DirectTab{};
        dt[t].tab = st[k].tab; dt[t].kmin = kmn; dt[t].range = range; dt[t].cshift = cshift;
        out_slots.push_back(q.pv[k][q.key_pos[k] == 0 ? 1 : 0]);
        ocs.push_back(OutCol{OUT_TABVAL, t, 0});
        tab_of[k] = t;
        t++;
    }
    timer_end(ctx);
    std::vector<std::unique_ptr<kb_rel>> rels;
    KB_TRY(scan_segments(ctx, ctx->segs, q.pats, K, q.pushdown, ScanOut::Pairs, &rels, &st));
    ctx->stats.fused_scan_builds++;
    // duplicate keys: the scan stores without reading back, so a multi-valued key shows up as fewer occupied slots than
    // inserted rows. Tables of (predicate, position) pairs already verified for this store version are not re-counted.
    bool counted = false;
    const u32 offc = ctrl_alloc(ctx, MAXT);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + offc, 0, MAXT * sizeof(u32), ctx->st));
    for (u32 k = 0; k < K; k++) {
        if ((int)k == probe_k || st[k].trusted) continue;
        if (!counted) timer_begin(ctx, F_BUILD, 0);
        counted = true;
        ctx->stats.kernel_launches++;
        launch_count_nonempty(st[k].tab, range, ctx->ctrl + offc + tab_of[k], ctx->n_sms, ctx->st);
    }
    if (counted) timer_end(ctx);  // the counts are read together with the probe's result: no extra synchronisation
    auto check_dups = [&]() -> bool {
        bool dup = false;
        for (u32 k = 0; k < K; k++) {
            if ((int)k == probe_k) continue;
            const bool fewer = !st[k].trusted && ctx->h_ctrl[offc + tab_of[k]] != rels[k]->n;
            if (ctx->h_ctrl[off + 8 + tab_of[k]] || fewer) {
                dup = true;
                build_proved(ctx, q, k, true, true);
            }
        }
        return dup;
    };
    for (u32 k = 0; k < K; k++) if ((int)k != probe_k) ctx->stats.rows_built += rels[k]->n;
    *route = Route::answered;
    for (u32 k = 0; k < K; k++) if (rels[k]->n == 0) return empty_rel(ctx, q.all_slots, out);
    for (u32 k = 0; k < K; k++) if ((int)k != probe_k && ctx->h_ctrl[off + 8 + tab_of[k]]) {  // key outside the table range (cannot happen with store statistics)
        KB_TRY(ctrl_read(ctx));
        check_dups();
        *route = Route::retry;
        return KB_OK;
    }
    const kb_rel& PR = *rels[probe_k];
    auto res = std::make_unique<kb_rel>();
    res->slots = out_slots;
    std::vector<FilterOp> fops;
    KB_TRY(compile_prog(ctx, q.post, out_slots, &fops));
    const u32 off2 = ctrl_alloc(ctx, 8);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off2, 0, 8 * sizeof(u32), ctx->st));
    ProbeFParams P{};
    KB_TRY(probe_fast(ctx, P, reinterpret_cast<const uint2*>(PR.cols[0].ptr), PR.n, q.key_pos[probe_k] == 2 ? 1u : 0u, dt, t, ocs, fops,
                      ctx->ctrl + off2, nullptr, res.get()));
    KB_TRY(ctrl_read(ctx));
    if (check_dups()) { *route = Route::retry; return KB_OK; }
    for (u32 k = 0; k < K; k++) if ((int)k != probe_k) build_proved(ctx, q, k, false, true);
    res->n = ctx->h_ctrl[off2 + 1];
    *out = select_cols(*res, q.all_slots);
    return KB_OK;
}

// R5: natural joins of `cur` (null: the probe relation) with the relations `rest`, smallest build sides first; the post-filter rides on
// the last one
static kb_status chained_join(kb_ctx* ctx, const StarQuery& q, std::vector<std::unique_ptr<kb_rel>>& rels, u32 probe, std::unique_ptr<kb_rel> cur,
                              std::vector<u32> rest, std::unique_ptr<kb_rel>* out) {
    for (auto& r : rels) KB_TRY(unpair_rel(ctx, &r));
    if (!cur) cur = std::move(rels[probe]);
    std::sort(rest.begin(), rest.end(), [&](u32 a, u32 b) { return rels[a]->n < rels[b]->n; });
    for (size_t i = 0; i < rest.size(); i++) {
        std::unique_ptr<kb_rel> j;
        KB_TRY(hash_join_impl(ctx, *cur, *rels[rest[i]], (i + 1 == rest.size() && !q.post.ops.empty()) ? &q.post : nullptr, &j));
        cur = std::move(j);
    }
    *out = select_cols(*cur, q.all_slots);
    return KB_OK;
}

// R4: direct tables over the key range [kmin, kmin + range), built in batches of at most MAXT per probe launch; the first batch over
// pair relations takes the register-staged fast probe. A build side that meets a duplicate key hands what is left to R5
static kb_status batched_join(kb_ctx* ctx, const StarQuery& q, std::vector<std::unique_ptr<kb_rel>>& rels, u32 probe, const std::vector<u32>& builds,
                              u32 kmin, u32 range, std::unique_ptr<kb_rel>* out) {
    std::unique_ptr<kb_rel> cur;  // result of the batches done so far (columnar); null = still the scan output of `probe`
    bool dup_seen = false;
    size_t done = 0;
    while (done < builds.size() && !dup_seen) {
        const size_t nb = std::min<size_t>(MAXT, builds.size() - done);
        const bool last = done + nb == builds.size();
        const bool fast = q.all_pairs && !cur;  // first batch over pair relations -> register-staged fast probe
        const kb_rel& PR = cur ? *cur : *rels[probe];
        const u32 off = ctrl_alloc(ctx, 8 + MAXT);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, (8 + MAXT) * sizeof(u32), ctx->st));
        std::vector<Buf> tables(nb);
        DirectTab dt[MAXT];
        std::vector<u32> out_slots = PR.slots;
        std::vector<OutCol> ocs;
        for (u32 c = 0; c < (u32)PR.slots.size(); c++) ocs.push_back(OutCol{OUT_PROBE, c, 0});
        timer_begin(ctx, F_BUILD, (int)nb);
        for (size_t t = 0; t < nb; t++) KB_TRY(alloc_buf(ctx, (size_t)range * sizeof(u32), &tables[t]));  // stream-ordered on st
        if (nb > 1) {  // independent tables: odd ones are memset + built on the second stream, concurrently with the even ones
            KB_CUDA(ctx, cudaEventRecord(ctx->ev_fork, ctx->st));
            KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st2, ctx->ev_fork, 0));
        }
        for (size_t t = 0; t < nb; t++) {
            const u32 k = builds[done + t];
            const kb_rel& B = *rels[k];
            cudaStream_t bs = (nb > 1 && (t & 1)) ? ctx->st2 : ctx->st;
            u32* tab = static_cast<u32*>(tables[t]->p);
            KB_CUDA(ctx, cudaMemsetAsync(tab, 0xFF, (size_t)range * sizeof(u32), bs));
            DirectTab& D = dt[t];
            D = DirectTab{};
            D.tab = tab; D.kmin = kmin; D.range = range;
            const int kc = B.col_of(q.join_slot);
            if (B.pair) {
                out_slots.push_back(B.slots[kc == 0 ? 1 : 0]);
                ocs.push_back(OutCol{OUT_TABVAL, (u32)t, 0});
                const u32 trusted = build_keys(ctx, q, k) == Keys::single ? 1u : 0u;
                launch_build_direct_pairs(reinterpret_cast<const uint2*>(B.cols[0].ptr), kc == 1 ? 1u : 0u, (u32)B.n, tab, kmin, range, 0u,
                                          ctx->ctrl + off + 8 + (u32)t, trusted, ctx->n_sms, bs);
            } else {
                const u32* vals = nullptr;
                if (B.cols.size() == 1) { D.mode = 2; }
                else if (B.cols.size() == 2) {
                    const int vc = kc == 0 ? 1 : 0;
                    vals = B.cols[vc].ptr;
                    out_slots.push_back(B.slots[vc]);
                    ocs.push_back(OutCol{OUT_TABVAL, (u32)t, 0});
                } else {
                    D.mode = 1;
                    for (size_t c = 0; c < B.cols.size(); c++) if ((int)c != kc) {
                        D.pay[D.n_pay] = B.cols[c].ptr;
                        out_slots.push_back(B.slots[c]);
                        ocs.push_back(OutCol{OUT_TABPAY, (u32)t, D.n_pay});
                        D.n_pay++;
                    }
                }
                launch_build_direct(B.cols[kc].ptr, vals, (u32)B.n, tab, kmin, range, 0u, ctx->ctrl + off + 8 + (u32)t, ctx->n_sms, bs);
            }
            ctx->stats.rows_built += B.n;
        }
        if (nb > 1) {
            KB_CUDA(ctx, cudaEventRecord(ctx->ev_join, ctx->st2));
            KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, ctx->ev_join, 0));
        }
        timer_end(ctx);
        auto res = std::make_unique<kb_rel>();
        res->slots = out_slots;
        std::vector<FilterOp> fops;
        if (last) KB_TRY(compile_prog(ctx, q.post, out_slots, &fops));
        if (fast) {
            ProbeFParams P{};
            KB_TRY(probe_fast(ctx, P, reinterpret_cast<const uint2*>(PR.cols[0].ptr), PR.n, PR.col_of(q.join_slot) == 1 ? 1u : 0u, dt, (u32)nb, ocs, fops,
                              ctx->ctrl + off, ctx->ctrl + off + 8, res.get()));
        } else {
            ProbeDParams P{};  // columnar input: the previous batch's result, or a scan without pair output (not all_pairs)
            P.n_pcols = (u32)PR.cols.size();
            for (u32 c = 0; c < P.n_pcols; c++) P.pcol[c] = PR.cols[c].ptr;
            P.key_col = (u32)PR.col_of(q.join_slot);
            P.n = (u32)PR.n;
            P.n_tiles = (u32)((PR.n + PROBE_TILE - 1) / PROBE_TILE);
            P.T = (u32)nb;
            for (size_t t = 0; t < nb; t++) P.tab[t] = dt[t];
            KB_TRY(probe_setup(ctx, &P, PR.n, ocs, fops, ctx->ctrl + off, ctx->ctrl + off + 8, res.get()));
            timer_begin(ctx, F_PROBE);
            launch_probe_direct(P, ctx->n_sms, ctx->st);
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
            ctx->stats.rows_probed += PR.n;
        }
        KB_TRY(ctrl_read(ctx));
        for (size_t t = 0; t < nb; t++) if (ctx->h_ctrl[off + 8 + t]) {
            dup_seen = true;
            build_proved(ctx, q, builds[done + t], true, rels[builds[done + t]]->pair);
        }
        if (dup_seen) break;
        for (size_t t = 0; t < nb; t++) build_proved(ctx, q, builds[done + t], false, rels[builds[done + t]]->pair);
        res->n = ctx->h_ctrl[off + 1];
        cur = std::move(res);
        done += nb;
        if (cur->n == 0) return empty_rel(ctx, q.all_slots, out);
    }
    if (!dup_seen) {
        *out = select_cols(*cur, q.all_slots);
        return KB_OK;
    }
    // a build side has duplicate keys: join what is left with the chained (multimap) operator
    return chained_join(ctx, q, rels, probe, std::move(cur), std::vector<u32>(builds.begin() + done, builds.end()), out);
}

// R4 / R5: every pattern is scanned (or looked up in the index), then joined by direct tables (R4) or chained joins (R5)
static kb_status scan_join(kb_ctx* ctx, const StarQuery& q, std::unique_ptr<kb_rel>* out) {
    const u32 K = q.K;
    std::vector<std::unique_ptr<kb_rel>> rels;
    KB_TRY(q.all_pairs ? scan_segments(ctx, ctx->segs, q.pats, K, q.pushdown, ScanOut::Pairs, &rels) : scan_store(ctx, q.pats, K, q.pushdown, &rels));
    if (ctx->upload_stats_off >= 0) {  // one-shot host call: the copy stream computed the column ranges chunk by chunk
        const u32 o = (u32)ctx->upload_stats_off;
        for (auto& sg : ctx->segs) {
            for (int c = 0; c < 3; c++) { sg.cmin[c] = ctx->h_ctrl[o + c]; sg.cmax[c] = ctx->h_ctrl[o + 4 + c]; }
            sg.has_stats = true;
        }
        ctx->upload_stats_off = -1;
    }
    u32 kmin, kmax;
    KB_TRY(store_key_range(ctx, q, &kmin, &kmax));
    for (u32 k = 0; k < K; k++) if (rels[k]->n == 0) return empty_rel(ctx, q.all_slots, out);
    if (K == 1) {
        std::unique_ptr<kb_rel> r = std::move(rels[0]);
        KB_TRY(unpair_rel(ctx, &r));
        if (!q.post.ops.empty()) { std::unique_ptr<kb_rel> f; KB_TRY(filter_impl(ctx, *r, q.post, &f)); r = std::move(f); }
        *out = std::move(r);
        return KB_OK;
    }
    // probe side = largest relation (ties: first)
    u32 probe = 0;
    for (u32 k = 1; k < K; k++) if (rels[k]->n > rels[probe]->n) probe = k;
    std::vector<u32> builds;
    for (u32 k = 0; k < K; k++) if (k != probe) builds.push_back(k);
    // direct tables need: patterns that share only the join variable, a dense key range, and single-valued keys
    bool fused_ok = kmax >= kmin && q.only_join_shared;
    const u64 range64 = fused_ok ? (u64)kmax - kmin + 1 : 0;
    for (u32 k : builds) {
        if (range64 > std::max<u64>(8 * rels[k]->n, 1ull << 16) || range64 > (1ull << 31)) fused_ok = false;
        if (build_keys(ctx, q, k) == Keys::multi) fused_ok = false;
        if (q.pv[k].size() > 3) fused_ok = false;
    }
    if (fused_ok) return batched_join(ctx, q, rels, probe, builds, kmin, (u32)range64, out);
    return chained_join(ctx, q, rels, probe, nullptr, builds, out);
}

kb_status star_join_impl(kb_ctx* ctx, u32 join_slot, const kb_pattern* pats, u32 K, const kb_filter_op* filter, u32 n_ops,
                         std::unique_ptr<kb_rel>* out, AggSpec* agg) {
    StarQuery q;
    KB_TRY(star_query(ctx, join_slot, pats, K, filter, n_ops, &q));
    const IndexSlices ix = index_slices(ctx, q);  // R1 and R2 read it; neither changes what it describes
    Route r;
    do {  // R2's duplicate key: the pair is now cached as multi-valued — start again from the top, with the index allowed
        KB_TRY(index_join_one_kernel(ctx, q, ix, agg, out, &r));
        if (r == Route::declined) KB_TRY(index_join_built(ctx, q, ix, out, &r));
    } while (r == Route::retry);
    if (r == Route::answered) return KB_OK;
    KB_TRY(fused_scan_join(ctx, q, out, &r));
    if (r == Route::answered) return KB_OK;
    // declined, or a duplicate / out-of-range key in R3's tables (r == Route::retry): scan again, without the index and the fusion
    return scan_join(ctx, q, out);
}

kb_status bind_join_impl(kb_ctx* ctx, const kb_rel& L, const kb_pattern& pt, std::unique_ptr<kb_rel>* out) {
    const kb_rel* left = &L;
    const kb_pattern* pat = &pt;
    std::vector<u32> pv, psrc;
    pattern_vars(*pat, &pv, &psrc);
    const bool pair_shape = pv.size() == 2 && psrc[0] == 0 && psrc[1] == 2 && !pat->p.is_var;
    if (pair_shape && ctx->use_index && ctx->index_version == ctx->store_version && left->n > 0 && left->n < 0xFFFFFFF0ull && !left->pair &&
        left->cols.size() < KB_MAX_COLS) {
        const int cx = left->col_of(pv[0]), cy = left->col_of(pv[1]);
        auto it = ctx->index.find(pat->p.value);
        if ((cx >= 0) != (cy >= 0) && it != ctx->index.end() && it->second.n > 0) {
            const PredSlice& ps = it->second;
            const bool by_y = cy >= 0;  // the bound variable is the pattern's object: look up pos[P][y]
            const Buf& tab = by_y ? ps.ytab : ps.xtab;
            // the persistent tables of a subject-sharded store are keyed by the COMPACTED subject: a relation that went through a
            // shuffle holds exactly the keys this shard owns, so the compaction applies to its rows too
            bool usable = (bool)tab;
            if (usable && !by_y && ps.tab_cshift != 0u) {
                // compacted keys alias across shards: the lookup is only sound when every key of `left` belongs to this shard
                const u32 foff = ctrl_alloc(ctx, 4);
                KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + foff, 0, 4 * sizeof(u32), ctx->st));
                timer_begin(ctx, F_OTHER);
                launch_count_foreign(left->cols[cx].ptr, (u32)left->n, ctx->shard_rank, ctx->shard_world, ctx->ctrl + foff, ctx->n_sms, ctx->st);
                timer_end(ctx);
                KB_CUDA(ctx, cudaGetLastError());
                KB_TRY(ctrl_read(ctx));
                usable = ctx->h_ctrl[foff] == 0;
            }
            if (usable) {
                ProbeDParams P{};
                P.n_pcols = (u32)left->cols.size();
                for (u32 c = 0; c < P.n_pcols; c++) P.pcol[c] = left->cols[c].ptr;
                P.key_col = (u32)(by_y ? cy : cx);
                P.n = (u32)left->n;
                P.n_tiles = (u32)((left->n + PROBE_TILE - 1) / PROBE_TILE);
                P.T = 1;
                P.tab[0] = persistent_tab(ps, by_y);
                auto rel = std::make_unique<kb_rel>();
                rel->slots = left->slots;
                rel->slots.push_back(by_y ? pv[0] : pv[1]);
                std::vector<OutCol> ocs;
                for (u32 c = 0; c < P.n_pcols; c++) ocs.push_back(OutCol{OUT_PROBE, c, 0});
                ocs.push_back(OutCol{OUT_TABVAL, 0, 0});
                const u32 off = ctrl_alloc(ctx, 4);
                KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 4 * sizeof(u32), ctx->st));
                KB_TRY(probe_setup(ctx, &P, left->n, ocs, {}, ctx->ctrl + off, nullptr, rel.get()));
                timer_begin(ctx, F_PROBE);
                launch_probe_direct(P, ctx->n_sms, ctx->st);
                timer_end(ctx);
                KB_CUDA(ctx, cudaGetLastError());
                ctx->stats.rows_probed += left->n;
                ctx->stats.index_joins++;
                KB_TRY(ctrl_read(ctx));
                rel->n = ctx->h_ctrl[off + 1];
                *out = std::move(rel);
                return KB_OK;
            }
        }
    }
    std::vector<std::unique_ptr<kb_rel>> rels;
    std::vector<FilterProg> none;
    KB_TRY(scan_store(ctx, pat, 1, none, &rels));
    return hash_join_impl(ctx, *left, *rels[0], nullptr, out);
}

}  // namespace kb
