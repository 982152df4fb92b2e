// kb_device.cuh — sm_90a device helpers shared by all kernels: TMA bulk copies + mbarrier, the single-pass
// "decoupled look-back" tile prefix that gives every compaction kernel a deterministic, store-ordered output,
// hashing, and the FILTER evaluator (semantics: kolibrie/src/streamertail_optimizer/types.rs:110-186).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/kolibrie_b200.h"

namespace kb {

using u8 = uint8_t;
using u16 = uint16_t;
using u32 = uint32_t;
using u64 = uint64_t;

constexpr u32 EMPTY32 = 0xFFFFFFFFu;  // == KB_ID_NONE: reserved id, never a dictionary / quoted-triple id
constexpr u64 EMPTY64 = ~0ull;
constexpr int MAXP = KB_MAX_PATTERNS;

// the grid of a persistent tile kernel: as many CTAs as are resident on every SM at once, at most one per tile
static inline int grid_for(const void* kernel, int threads, size_t smem, int n_sms, u32 n_tiles) {
    int per_sm = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem);
    if (per_sm < 1) per_sm = 1;
    long long g = (long long)per_sm * n_sms;  // persistent: a whole number of resident CTAs per SM, on every SM
    if (g > (long long)n_tiles) g = n_tiles;
    if (g < 1) g = 1;
    return (int)g;
}

__host__ __device__ __forceinline__ u32 mix32(u32 x) {  // murmur3 finaliser; also the shard function (kb_shard_of)
    x ^= x >> 16; x *= 0x85ebca6bu; x ^= x >> 13; x *= 0xc2b2ae35u; x ^= x >> 16;
    return x;
}

// shard function and the per-shard key compaction (include/kolibrie_b200.h: kb_shard_of)
constexpr u32 SHARD_B = KB_SHARD_BLOCK_BITS;
__host__ __device__ __forceinline__ u32 shard_of(u32 key, u32 n) { return (key >> SHARD_B) % n; }
// cshift = log2(world) for a power-of-two world, 0 = no compaction. Monotone on the keys one shard owns.
__host__ __device__ __forceinline__ u32 compact_key(u32 key, u32 cshift) {
    return cshift ? ((((key >> SHARD_B) >> cshift) << SHARD_B) | (key & ((1u << SHARD_B) - 1u))) : key;
}

// ---------------------------------------------------------------------------------------------------------------
// mbarrier + TMA (cp.async.bulk, 1-D: no tensor map needed for flat u32 columns). SASS: UBLKCP / SYNCS.
__device__ __forceinline__ u32 smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(u64* bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(u64* bar, u32 bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(u64* bar, u32 parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "KB_WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra KB_WAIT_DONE;\n\t"
        "bra KB_WAIT_LOOP;\n\t"
        "KB_WAIT_DONE:\n\t"
        "}" ::"r"(smem_addr(bar)), "r"(parity)
        : "memory");
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes a multiple of 16; completion counted on `bar`
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, u32 bytes, u64* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// relaxed gpu-scope 64-bit accesses for the tile-state words
__device__ __forceinline__ u64 ld_relaxed(const u64* p) {
    u64 v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed(u64* p, u64 v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }

__device__ __forceinline__ u32 warp_sum(u32 v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Single-pass ordered prefix across tiles ("decoupled look-back"). One state word per (tile, counter):
//   [63:34] launch epoch (so the buffer is cleared only when the epoch wraps)  [33:32] status 1=A(ggregate) 2=P(refix)  [31:0] value.
// Tiles take tickets from an atomic counter, so a tile only ever waits on tiles that are already running.
// Called by ALL 32 lanes of one warp once counts[0..K) (shared memory) are final; writes the exclusive prefix of this tile
// to excl[0..K). base[k] (global, may be null) is added to tile 0: the running total of earlier launches (store segments).
constexpr u64 TS_A = 1ull << 32, TS_P = 2ull << 32;
constexpr int TS_EPOCH_BITS = 30;  // the epoch field: launches take epochs 1 .. 2^30 - 1 (next_epoch, kb_join.cu)
__device__ __forceinline__ void tile_prefix_warp(u64* __restrict__ state, u32 tile, u32 K, u64 epoch, const u32* counts, u32* excl,
                                                 const u32* base, int lane) {
    const u64 tag = epoch << 34;
    if (tile == 0) {
        if (lane < (int)K) {
            u32 b = base ? base[lane] : 0u;
            excl[lane] = b;
            st_relaxed(&state[lane], tag | TS_P | (u64)(b + counts[lane]));
        }
        __syncwarp();
        return;
    }
    if (lane < (int)K) st_relaxed(&state[(u64)tile * MAXP + lane], tag | TS_A | (u64)counts[lane]);
    for (u32 k = 0; k < K; k++) {
        u32 sum = 0;
        long long pred = (long long)tile - 1 - lane;
        for (;;) {
            u64 w;
            if (pred >= 0) {
                const u64* p = &state[(u64)pred * MAXP + k];
                w = ld_relaxed(p);
                while ((w >> 34) != epoch) { __nanosleep(32); w = ld_relaxed(p); }
            } else {
                w = tag | TS_P;  // virtual predecessor of tile 0
            }
            const bool is_p = ((w >> 32) & 3ull) == 2ull;
            const unsigned pm = __ballot_sync(0xffffffffu, is_p);
            const u32 v = (u32)w;
            if (pm) {
                const int first = __ffs(pm) - 1;  // nearest predecessor that already knows its full prefix
                sum += warp_sum(lane <= first ? v : 0u);
                break;
            }
            sum += warp_sum(v);
            pred -= 32;
        }
        if (lane == 0) {
            excl[k] = sum;
            st_relaxed(&state[(u64)tile * MAXP + k], tag | TS_P | (u64)(sum + counts[k]));
        }
    }
    __syncwarp();
}

// TWO-LEVEL ordered prefix (the one the kernels use). Tiles are grouped in blocks of 32 consecutive tickets.
//   level 1: state1[tile]  = this tile's count (epoch-tagged). A tile sums the counts of the earlier tiles of ITS block: it waits
//            only until those tiles have COUNTED (they run concurrently with it), never for anybody's look-back.
//   level 2: state2[block] = A(ggregate of the block) then P(refix through the block), published by the block's last tile.
//            A tile looks back over whole blocks; ~600 tiles in flight are < 20 blocks, i.e. always inside one 32-wide window.
// Cost per tile and counter: one publish, 32 + 32 word loads issued together, two memory round trips on the critical path,
// independent of how many tiles are in flight (the flat decoupled look-back above needs ~tiles_in_flight/32 dependent steps).
// mode 0 replaces all of this by one atomicAdd on a global cursor: same bytes, output order = tile completion order.
__device__ __forceinline__ u32 tile_prefix_2level(u64* __restrict__ state1, u64* __restrict__ state2, u32 tile, u32 n_tiles, u32 k, u64 epoch,
                                                  u32 count, const u32* totals_in, u32* totals_out, u32 ordered, int lane) {
    // ordered: totals_in[k] = rows written by earlier launches, totals_out[k] (a DIFFERENT word) receives the new total;
    // unordered: totals_out[k] is the atomic cursor and already holds the earlier launches' rows.
    if (!ordered) {
        u32 ex = 0;
        if (lane == 0) ex = atomicAdd(&totals_out[k], count);
        return __shfl_sync(0xffffffffu, ex, 0);
    }
    const u64 tag = epoch << 34;
    const u32 b = tile >> 5, i = tile & 31u;
    const u32 last_i = min(31u, n_tiles - 1u - (b << 5));
    if (lane == 0) st_relaxed(&state1[(u64)tile * MAXP + k], tag | (u64)count);
    const u64* p1 = &state1[(u64)((b << 5) + (u32)lane) * MAXP + k];
    long long pb = (long long)b - 1 - lane;
    const u32 base_in = totals_in[k];
    u64 w1 = ((u32)lane < i) ? ld_relaxed(p1) : tag;
    u64 w2 = (pb >= 0) ? ld_relaxed(&state2[(u64)pb * MAXP + k]) : (tag | TS_P | (u64)(pb == -1 ? base_in : 0u));
    while ((w1 >> 34) != epoch) w1 = ld_relaxed(p1);
    const u32 local = warp_sum(((u32)lane < i) ? (u32)w1 : 0u);
    if (i == last_i && lane == 0) st_relaxed(&state2[(u64)b * MAXP + k], tag | TS_A | (u64)(local + count));
    u32 sum = 0;
    for (;;) {
        if (pb >= 0) {
            const u64* p2 = &state2[(u64)pb * MAXP + k];
            while ((w2 >> 34) != epoch) w2 = ld_relaxed(p2);
        }
        const bool is_p = ((w2 >> 32) & 3ull) == 2ull;
        const unsigned pm = __ballot_sync(0xffffffffu, is_p);
        const u32 v = (u32)w2;
        if (pm) {
            const int first = __ffs(pm) - 1;
            sum += warp_sum(lane <= first ? v : 0u);
            break;
        }
        sum += warp_sum(v);
        pb -= 32;
        w2 = (pb >= 0) ? ld_relaxed(&state2[(u64)pb * MAXP + k]) : (tag | TS_P | (u64)(pb == -1 ? base_in : 0u));
    }
    const u32 ex = sum + local;
    if (lane == 0) {
        if (i == last_i) st_relaxed(&state2[(u64)b * MAXP + k], tag | TS_P | (u64)(ex + count));
        if (tile == n_tiles - 1u) totals_out[k] = ex + count;
    }
    return ex;
}

// One counter, WIDE window: every lane inspects LBQ consecutive predecessors per step, so a step covers 32*LBQ tiles and "prefix
// known" (P) status propagates through the in-flight tiles LBQ times faster than with a 32-tile window. With ~450-600 tiles in
// flight (3-4 CTAs on each of 132 SMs) a 256-tile window ends every look-back in one or two memory round trips.
// Called by all 32 lanes of a warp; `count` is this tile's total for counter k; returns the exclusive prefix (valid in all lanes).
constexpr int LBQ = 8;
__device__ __forceinline__ u32 tile_prefix_wide(u64* __restrict__ state, u32 tile, u32 k, u64 epoch, u32 count, const u32* base, int lane) {
    const u64 tag = epoch << 34;
    if (tile == 0) {
        const u32 b = base ? base[k] : 0u;
        if (lane == 0) st_relaxed(&state[k], tag | TS_P | (u64)(b + count));
        return b;
    }
    if (lane == 0) st_relaxed(&state[(u64)tile * MAXP + k], tag | TS_A | (u64)count);
    u32 sum = 0;
    long long pred0 = (long long)tile - 1 - (long long)lane * LBQ;  // this lane covers pred0, pred0-1, ..., pred0-LBQ+1 (nearest first)
    for (;;) {
        u64 w[LBQ];
#pragma unroll
        for (int q = 0; q < LBQ; q++) w[q] = (pred0 - q >= 0) ? ld_relaxed(&state[(u64)(pred0 - q) * MAXP + k]) : (tag | TS_P);
        u32 lane_sum = 0;
        bool lane_p = false;
#pragma unroll
        for (int q = 0; q < LBQ; q++) {
            if (!lane_p) {
                while ((w[q] >> 34) != epoch) w[q] = ld_relaxed(&state[(u64)(pred0 - q) * MAXP + k]);
                lane_sum += (u32)w[q];
                lane_p = ((w[q] >> 32) & 3ull) == 2ull;
            }
        }
        const unsigned pm = __ballot_sync(0xffffffffu, lane_p);
        if (pm) {
            const int first = __ffs(pm) - 1;
            sum += warp_sum(lane <= first ? lane_sum : 0u);
            break;
        }
        sum += warp_sum(lane_sum);
        pred0 -= 32 * LBQ;
    }
    if (lane == 0) st_relaxed(&state[(u64)tile * MAXP + k], tag | TS_P | (u64)(sum + count));
    return sum;
}

// Same protocol for K counters at once (compile-time K): the K state words of a predecessor tile are read with K independent
// loads, so the look-back costs one memory round trip per window instead of K.
template <int K>
__device__ __forceinline__ void tile_prefix_warp_k(u64* __restrict__ state, u32 tile, u64 epoch, const u32* counts, u32* excl, const u32* base,
                                                   int lane) {
    const u64 tag = epoch << 34;
    if (tile == 0) {
        if (lane < K) {
            u32 b = base ? base[lane] : 0u;
            excl[lane] = b;
            st_relaxed(&state[lane], tag | TS_P | (u64)(b + counts[lane]));
        }
        __syncwarp();
        return;
    }
    if (lane < K) st_relaxed(&state[(u64)tile * MAXP + lane], tag | TS_A | (u64)counts[lane]);
    u32 sum[K];
    bool done[K];
#pragma unroll
    for (int k = 0; k < K; k++) { sum[k] = 0; done[k] = false; }
    long long pred = (long long)tile - 1 - lane;
    for (;;) {
        u64 w[K];
        const u64* p = &state[(u64)(pred >= 0 ? pred : 0) * MAXP];
#pragma unroll
        for (int k = 0; k < K; k++) w[k] = (pred >= 0) ? ld_relaxed(p + k) : (tag | TS_P);
        bool all = true;
#pragma unroll
        for (int k = 0; k < K; k++) {
            if (done[k]) continue;
            while ((w[k] >> 34) != epoch) { __nanosleep(20); w[k] = ld_relaxed(p + k); }
            const bool is_p = ((w[k] >> 32) & 3ull) == 2ull;
            const unsigned pm = __ballot_sync(0xffffffffu, is_p);
            const u32 v = (u32)w[k];
            if (pm) {
                const int first = __ffs(pm) - 1;
                sum[k] += warp_sum(lane <= first ? v : 0u);
                done[k] = true;
            } else {
                sum[k] += warp_sum(v);
                all = false;
            }
        }
        if (all) break;
        pred -= 32;
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < K; k++) {
            excl[k] = sum[k];
            st_relaxed(&state[(u64)tile * MAXP + k], tag | TS_P | (u64)(sum[k] + counts[k]));
        }
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------------------------------------------
// FILTER evaluation on the device. vals[slot] = id bound to the (remapped) slot.
struct FilterOp {  // same layout as kb_filter_op
    u32 op, slot, cmp, id;
    double value;
};
static_assert(sizeof(FilterOp) == sizeof(kb_filter_op), "layout");

struct NumTab {
    const double* num_or0;
    const u8* is_num;
    u32 n_ids;
    const int* i32_val;  // legacy executor: the term parsed as i32 (kb_dict_legacy_i32_load); null when not loaded
    const u8* is_i32;
    u32 n_i32;
};
__device__ __forceinline__ double num_of(const NumTab& nt, u32 id) { return id < nt.n_ids ? __ldg(nt.num_or0 + id) : 0.0; }
__device__ __forceinline__ bool isnum_of(const NumTab& nt, u32 id) { return id < nt.n_ids ? __ldg(nt.is_num + id) != 0 : false; }

// Seed of an aggregate accumulator: the identity of its fold, so that a slot no row (or only some rows) reached gives what folding
// the group's rows from its first value gives (execute_query.rs:1198-1201). MIN / MAX: a quiet NaN — fmin / fmax and
// atomic_min_f64 / atomic_max_f64 replace it by any non-NaN value, and a group whose values are all NaN stays NaN (f64::min(NaN, NaN)).
// SUM / AVG: -0.0, the only identity of IEEE addition (+0.0 + -0.0 = +0.0 would turn an all-(-0.0) group positive).
__device__ __forceinline__ double agg_identity(u32 kind) {
    return (kind == KB_AGG_MIN || kind == KB_AGG_MAX) ? __longlong_as_double(0x7FF8000000000000ll) : -0.0;
}

__device__ __forceinline__ bool cmp_num(u32 cmp, double a, double b) {
    switch (cmp) {  // types.rs:133-148 — only the four ordering operators reach the numeric path
        case KB_CMP_GT: return a > b;
        case KB_CMP_GE: return a >= b;
        case KB_CMP_LT: return a < b;
        case KB_CMP_LE: return a <= b;
        default: return false;
    }
}

static __device__ __noinline__ bool eval_filter_general(const FilterOp* ops, u32 n_ops, const u32* vals, const NumTab& nt) {
    double st[12];
    u32 okm = 0;  // bit i: st[i] valid
    int sp = 0;
    for (u32 i = 0; i < n_ops; i++) {
        const FilterOp op = ops[i];
        switch (op.op) {
            // a row that leaves the variable unbound (KB_ID_NONE, written by kb_bind, kb_natural_join or a ragged InMemoryBuffer) fails
            // every comparison, != included (types.rs:128, :143-145): its NOT is true
            case KB_F_CMP_NUM: st[sp] = (vals[op.slot] != EMPTY32 && cmp_num(op.cmp, num_of(nt, vals[op.slot]), op.value)) ? 1.0 : 0.0; okm |= 1u << sp; sp++; break;
            case KB_F_EQ_ID: st[sp] = (op.id != EMPTY32 && vals[op.slot] == op.id) ? 1.0 : 0.0; okm |= 1u << sp; sp++; break;
            case KB_F_NE_ID: st[sp] = (vals[op.slot] != EMPTY32 && (op.id == EMPTY32 || vals[op.slot] != op.id)) ? 1.0 : 0.0; okm |= 1u << sp; sp++; break;
            case KB_F_AND: sp--; st[sp - 1] = (st[sp - 1] != 0.0 && st[sp] != 0.0) ? 1.0 : 0.0; break;
            case KB_F_OR: sp--; st[sp - 1] = (st[sp - 1] != 0.0 || st[sp] != 0.0) ? 1.0 : 0.0; break;
            case KB_F_NOT: st[sp - 1] = (st[sp - 1] == 0.0) ? 1.0 : 0.0; break;
            case KB_F_PUSH_VAR: {
                u32 id = vals[op.slot];
                st[sp] = num_of(nt, id);
                if (id != EMPTY32 && isnum_of(nt, id)) okm |= 1u << sp; else okm &= ~(1u << sp);  // unbound: the resolver's `?` (types.rs:161)
                sp++;
            } break;
            case KB_F_PUSH_CONST: st[sp] = op.value; okm |= 1u << sp; sp++; break;
            case KB_F_ADD: case KB_F_SUB: case KB_F_MUL: case KB_F_DIV: {
                sp--;
                bool v = ((okm >> (sp - 1)) & 1u) && ((okm >> sp) & 1u);
                double a = st[sp - 1], b = st[sp], r;
                if (op.op == KB_F_ADD) r = a + b;
                else if (op.op == KB_F_SUB) r = a - b;
                else if (op.op == KB_F_MUL) r = a * b;
                else { v = v && b != 0.0; r = v ? a / b : 0.0; }
                st[sp - 1] = r;
                if (v) okm |= 1u << (sp - 1); else okm &= ~(1u << (sp - 1));
            } break;
            case KB_F_TRUTHY: st[sp - 1] = (((okm >> (sp - 1)) & 1u) && st[sp - 1] != 0.0) ? 1.0 : 0.0; okm |= 1u << (sp - 1); break;
            case KB_F_IS_TRIPLE: st[sp] = (vals[op.slot] != EMPTY32 && (vals[op.slot] & 0x80000000u)) ? 1.0 : 0.0; okm |= 1u << sp; sp++; break;  // types.rs:172-176
            case KB_F_CMP_LEGACY: {  // sparql_database.rs:1420-1620: i32 comparison when both sides are integers, else string equality
                const u32 id = vals[op.slot];
                const u32 cmp = op.cmp & 0xFFu;
                const bool nested = (op.cmp & KB_LEGACY_NESTED_F64) != 0u;
                const bool both_int = !nested && (op.cmp & KB_LEGACY_CONST_IS_I32) && nt.is_i32 != nullptr && id < nt.n_i32 && __ldg(nt.is_i32 + id) != 0;
                bool r;
                if (nested && (op.cmp & KB_LEGACY_CONST_IS_I32) && isnum_of(nt, id)) {
                    const double a = num_of(nt, id), b = op.value;
                    r = cmp == KB_CMP_EQ ? a == b : cmp == KB_CMP_NE ? a != b : cmp == KB_CMP_GT ? a > b : cmp == KB_CMP_GE ? a >= b : cmp == KB_CMP_LT ? a < b : cmp == KB_CMP_LE ? a <= b : false;
                } else if (both_int) {
                    const int a = __ldg(nt.i32_val + id), b = (int)op.value;
                    r = cmp == KB_CMP_EQ ? a == b : cmp == KB_CMP_NE ? a != b : cmp == KB_CMP_GT ? a > b : cmp == KB_CMP_GE ? a >= b : cmp == KB_CMP_LT ? a < b : cmp == KB_CMP_LE ? a <= b : false;
                } else {
                    const bool same = op.id != EMPTY32 && id == op.id;  // byte-wise equal strings <=> the same dictionary id
                    r = cmp == KB_CMP_EQ ? same : cmp == KB_CMP_NE ? !same : false;
                }
                st[sp] = r ? 1.0 : 0.0; okm |= 1u << sp; sp++;
            } break;
            default: return false;
        }
        if (sp > 11) return false;
    }
    return sp == 1 && st[0] != 0.0;
}

__device__ __forceinline__ bool eval_filter(const FilterOp* ops, u32 n_ops, const u32* vals, const NumTab& nt) {
    if (n_ops == 0) return true;
    if (n_ops == 1 && ops[0].op == KB_F_CMP_NUM)  // FILTER(?x > c): the common case, no stack machine; unbound is false
        return vals[ops[0].slot] != EMPTY32 && cmp_num(ops[0].cmp, num_of(nt, vals[ops[0].slot]), ops[0].value);
    return eval_filter_general(ops, n_ops, vals, nt);
}

}  // namespace kb
