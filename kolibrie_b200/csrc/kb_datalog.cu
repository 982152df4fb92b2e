// kb_datalog.cu — Datalog on the device: semi-naive / naive materialisation (kb_datalog_fixpoint, kb_datalog_fixpoint_seed),
// backward-chaining queries (kb_datalog_query; demand patterns and the answer pass in kb_backward.cu) and delete-and-rederive
// maintenance (kb_datalog_maintain). The file owns the Datalog kernels (known-fact sets, derive and its radix-partitioned variant, the
// maintenance kernels), their launch formats, and the host driver that launches them.
// Replaces Reasoner::infer_with_strategy (datalog/src/reasoning/materialisation/infer_generic.rs:27-53) driving
// SemiNaiveStrategy (semi_naive.rs:17-85) or NaiveStrategy (my_naive.rs:18-69), whose join is
// perform_hash_join_for_rules (shared/src/join_algorithm.rs:499-677).
//
// Layout: one (s,o) column pair per predicate that occurs in a rule, append-only, exactly like the reference's
// `all_facts: Vec<Triple>` with its delta suffix (semi_naive.rs:57-59) but partitioned by predicate once instead of
// re-filtered by predicate for every premise of every rule of every round (join_algorithm.rs:528-534).
// known_facts (infer_generic.rs:30) is a device hash set of 64-bit (s,o) keys per head predicate; a derived fact is new iff its insert
// wins. Round structure is the reference's: every rule of a round sees the same snapshot; new facts become visible (and become the
// next delta) only after the round (infer_generic.rs:42-48) — so round counts and per-round fact counts match the oracle.
//
// kb_datalog_maintain keeps a closed store closed across a window slide by delete-and-rederive (DRed) over the same per-predicate
// relations and known-fact sets, kept in the context between calls, plus a base multiplicity table per predicate (see maintain_impl).
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>

#include "kb_internal.hpp"

using namespace kb;

namespace kb {

// =====================================================================================================================================
// Device side. The launch formats below and everything behind them are private to this file; what kb_backward.cu reads too (set64_insert,
// set64_find, bc_demanded, emit_pair) is in kb_kernels.cuh.

// ---- known-fact sets: 64-bit (s,o) keys of one predicate
static __global__ void __launch_bounds__(256) set64_insert_kernel(u64* set, u32 set_slots, const u32* s, const u32* o, u32 n, u32* overflow) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        if (set64_insert(set, set_slots, s[i], o[i]) == 2u) *overflow = 1u;
}
static void launch_set64_insert(u64* set, u32 set_slots, const u32* s, const u32* o, u32 n, u32* overflow, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    int grid = grid_1d(n, n_sms);
    set64_insert_kernel<<<grid, 256, 0, st>>>(set, set_slots, s, o, n, overflow);
}

// ---- derive
// instantiate rule heads from binding columns, apply rule filters (rules.rs:133-165), insert into the head predicate's known-fact set
// and append the facts that were new (infer_generic.rs:42-48)
struct HeadTerm { u32 is_var, value; };  // value = binding column index or constant id
struct RuleFilterDev { u32 lhs_col, cmp, rhs_is_var, rhs_col; double rhs_value; };
struct DeriveParams {
    const u32* bcol[KB_MAX_COLS];
    u32 n;
    HeadTerm head_s, head_o;  // the head predicate is a constant: one known-fact set per predicate, keyed by (s << 32) | o
    RuleFilterDev filt[KB_MAX_RULE_FILTERS];
    u32 n_filt;
    NumTab nt;
    u64* set;       // open addressing, EMPTY64 = free; a fact is new iff its atomicCAS wins
    u32 set_slots;  // power of two
    u32 *out_s, *out_o;
    u32 out_cap;
    u32 budget;                   // stop inserting once this many facts were appended (keeps the set's load bounded): overflow = 2
    u32* out_count;               // appended so far (atomic cursor)
    unsigned long long* n_deriv;  // candidates that passed the filters
    u32* overflow;                // 1: set or output full (error); 2: budget reached, the host grows the set and runs the launch again
    // kb_datalog_maintain (delete-and-rederive): a candidate takes part in the dedup only if it is a member of gate_set (when non-null)
    // and has no positive count in the veto table (when non-null). Gated launches never take the partitioned path.
    const u64* gate_set;
    u32 gate_slots;
    const u64* veto_keys;
    const u32* veto_cnt;
    u32 veto_slots;
    // kb_datalog_query: a candidate takes part in the dedup only if it matches one of the head predicate's n_demand demand patterns
    // (x = subject, y = object, KB_ID_NONE = any; null: every fact is demanded). Applied on both dedup routes.
    const uint2* demand;
    u32 n_demand;
};
// RADIX-PARTITIONED candidate dedup (the same work as launch_derive for large candidate sets). The known-fact set is an open-addressing
// table far larger than L2 (config 4: 8 GB), so a direct probe per candidate is one random DRAM line per candidate. Here the
// candidates are first partitioned by the HIGH bits of their home slot (tile sorted by partition in shared memory, one range
// reservation per tile and partition, coalesced runs), so that partition p only touches slice p of the table; the probe pass then walks
// the partitions in order, every CTA on (nearly) the same slice, which is sized to stay resident in L2.
struct DerivePartParams {
    DeriveParams d;            // candidates, head, filters, set, outputs, counters (as for launch_derive)
    u32 slice_bits;            // log2(slots per slice); partition = home slot >> slice_bits
    u32 n_parts;               // set_slots >> slice_bits, <= 1024
    u64* buckets;              // [n_parts][bucket_cap] candidate keys (s << 32 | o)
    u32 bucket_cap;
    u32* cursors;              // [n_parts] keys in each bucket (zeroed)
    u32* tile_start;           // [n_parts + 1] first probe tile of each partition (written by the launch)
    u32* tickets;              // [2] zeroed: tile counters of the two passes
};

// set64_insert that returns the key's slot (EMPTY32: table full); *claimed = this call took a free slot for the key
static __device__ __forceinline__ u32 set64_insert_slot(u64* set, u32 n_slots, u32 s, u32 o, bool* claimed) {
    const u64 key = ((u64)s << 32) | (u64)o;
    const u32 mask = n_slots - 1u;
    u32 slot = mix32(mix32(s) * 0x9E3779B1u ^ mix32(o + 0x632BE5ABu)) & mask;
    *claimed = false;
    for (u32 probes = 0; probes < n_slots; probes++) {
        const u64 cur = *reinterpret_cast<volatile u64*>(&set[slot]);
        if (cur == key) return slot;
        if (cur == EMPTY64) {
            const u64 old = atomicCAS(reinterpret_cast<unsigned long long*>(&set[slot]), (unsigned long long)EMPTY64, (unsigned long long)key);
            if (old == EMPTY64) { *claimed = true; return slot; }
            if (old == key) return slot;
        }
        slot = (slot + 1u) & mask;
    }
    return EMPTY32;
}
// the acceptance test in front of the dedup: demanded (kb_datalog_query), member of the gate set and no positive count in the veto table
// (kb_datalog_maintain)
static __device__ __forceinline__ bool derive_gate_pass(const DeriveParams& P, u32 s, u32 o) {
    if (P.demand && !bc_demanded(P.demand, P.n_demand, s, o)) return false;
    if (P.gate_set && set64_find(P.gate_set, P.gate_slots, s, o) == EMPTY32) return false;
    if (P.veto_keys) {
        const u32 slot = set64_find(P.veto_keys, P.veto_slots, s, o);
        if (slot != EMPTY32 && P.veto_cnt[slot] > 0u) return false;
    }
    return true;
}

static __device__ __forceinline__ bool rule_filters_pass(const DeriveParams& P, u32 i) {
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

template <bool GATED>
static __global__ void __launch_bounds__(256) derive_kernel(const __grid_constant__ DeriveParams P) {
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
            if (GATED && !derive_gate_pass(P, s, o)) pass = false;
        }
        if (pass) {
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
static __device__ __forceinline__ u32 set64_home(u32 n_slots, u32 s, u32 o) { return mix32(mix32(s) * 0x9E3779B1u ^ mix32(o + 0x632BE5ABu)) & (n_slots - 1u); }

// insert + append of ONE candidate outside any warp-cooperative section (bucket overflow path of the partition pass)
static __device__ __noinline__ void derive_one(const DeriveParams& P, u32 s, u32 o) {
    if (*reinterpret_cast<volatile u32*>(P.out_count) >= P.budget) { *P.overflow = 2u; return; }
    const u32 r = set64_insert(P.set, P.set_slots, s, o);
    if (r == 2u) *P.overflow = 2u;
    if (r == 1u) {
        const u32 at = atomicAdd(P.out_count, 1u);
        if (at < P.out_cap) { P.out_s[at] = s; P.out_o[at] = o; }
        else *P.overflow = 1u;
    }
}

static __global__ void __launch_bounds__(DPART_THREADS) derive_partition_kernel(const __grid_constant__ DerivePartParams Q) {
    extern __shared__ __align__(128) u64 sh_keys[];  // [DPART_TILE] keys sorted by partition, then u16 partition ids
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
                if (P.demand && !bc_demanded(P.demand, P.n_demand, s, o)) pass = false;
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
static __global__ void __launch_bounds__(1024) derive_tile_starts_kernel(const __grid_constant__ DerivePartParams Q) {
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

static __global__ void __launch_bounds__(256) derive_probe_kernel(const __grid_constant__ DerivePartParams Q) {
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

static void launch_derive_partitioned(const DerivePartParams& p, int n_sms, cudaStream_t st) {
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

static void launch_derive(const DeriveParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    int grid = grid_1d(p.n, n_sms);
    if (p.gate_set || p.veto_keys || p.demand) derive_kernel<true><<<grid, 256, 0, st>>>(p);
    else derive_kernel<false><<<grid, 256, 0, st>>>(p);
}

// *found = 1 when (s,o) is a member of the 64-bit set (a one-thread probe: kb_datalog_query's ground query)
static __global__ void bc_probe_kernel(const u64* set, u32 set_slots, u32 s, u32 o, u32* found) {
    *found = set64_find(set, set_slots, s, o) != EMPTY32 ? 1u : 0u;
}
static void launch_bc_probe(const u64* set, u32 set_slots, u32 s, u32 o, u32* found, cudaStream_t st) {
    bc_probe_kernel<<<1, 1, 0, st>>>(set, set_slots, s, o, found);
}

// ---- kb_datalog_maintain: base multiplicities, selection by set membership, erasure
// An erased key of a 64-bit (s,o) set: lookups walk past it, inserts never reuse it (s = KB_ID_NONE is never a fact). The set is rebuilt
// from its relation when it fills up, which drops the tombstones.
constexpr u64 TOMB64 = 0xFFFFFFFFFFFFFFFEull;
// base multiplicity of a predicate's facts: a 64-bit (s,o) key table and a parallel u32 count per slot (a key whose count is 0 is not a
// base fact; it keeps its slot until the table is rehashed)
struct BaseCountParams {
    u64* keys;
    u32* cnt;
    u32 slots;  // power of two
    const u32 *s, *o;
    u32 n;
    int delta;  // +1: the rows join the base (a count that leaves 0 emits the fact), -1: they leave it (a count that reaches 0 emits it)
    u32 *out_s, *out_o;  // nullable: no emission (the facts that crossed zero are then only counted)
    u32* out_count;      // facts that crossed zero
    u32* claimed;        // keys that took a free slot of the table
    u32* overflow;       // 1: key table full
};
static __global__ void __launch_bounds__(256) base_count_kernel(const __grid_constant__ BaseCountParams P) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (P.n + 31u) & ~31u;
    u32 n_edges = 0, n_claimed = 0;  // (counted here when nothing is emitted)
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        bool edge = false;  // this row moved the count across zero
        u32 s = 0, o = 0;
        if (i < P.n) {
            s = P.s[i];
            o = P.o[i];
            if (P.delta > 0) {
                bool claimed = false;
                const u32 slot = set64_insert_slot(P.keys, P.slots, s, o, &claimed);
                if (slot == EMPTY32) *P.overflow = 1u;
                else edge = atomicAdd(&P.cnt[slot], 1u) == 0u;
                n_claimed += claimed ? 1u : 0u;
            } else {
                const u32 slot = set64_find(P.keys, P.slots, s, o);
                if (slot != EMPTY32) edge = atomicSub(&P.cnt[slot], 1u) == 1u;
            }
        }
        if (P.out_s) emit_pair(edge, s, o, P.out_s, P.out_o, P.out_count);
        else n_edges += edge ? 1u : 0u;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        n_edges += __shfl_xor_sync(0xffffffffu, n_edges, d);
        n_claimed += __shfl_xor_sync(0xffffffffu, n_claimed, d);
    }
    if ((threadIdx.x & 31) == 0) {
        if (n_edges) atomicAdd(P.out_count, n_edges);
        if (n_claimed) atomicAdd(P.claimed, n_claimed);
    }
}
static void launch_base_count(const BaseCountParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    const int grid = grid_1d(p.n, n_sms);
    base_count_kernel<<<grid, 256, 0, st>>>(p);
}

// live entries (count > 0) of one count table into an empty larger one; *n_live += entries moved
static __global__ void __launch_bounds__(256) base_count_rehash_kernel(const u64* okeys, const u32* ocnt, u32 oslots, u64* nkeys, u32* ncnt, u32 nslots,
                                                                u32* n_live, u32* overflow) {
    const u32 stride = gridDim.x * blockDim.x;
    u32 moved = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < oslots; i += stride) {
        const u64 k = okeys[i];
        const u32 c = ocnt[i];
        if (k == EMPTY64 || c == 0u) continue;
        bool claimed = false;
        const u32 slot = set64_insert_slot(nkeys, nslots, (u32)(k >> 32), (u32)k, &claimed);
        if (slot == EMPTY32) { *overflow = 1u; continue; }
        ncnt[slot] = c;  // keys are distinct: one writer per slot
        moved++;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) moved += __shfl_xor_sync(0xffffffffu, moved, d);
    if ((threadIdx.x & 31) == 0 && moved) atomicAdd(n_live, moved);
}
static void launch_base_count_rehash(const u64* okeys, const u32* ocnt, u32 oslots, u64* nkeys, u32* ncnt, u32 nslots, u32* n_live, u32* overflow, int n_sms,
                              cudaStream_t st) {
    if (oslots == 0) return;
    const int grid = grid_1d(oslots, n_sms);
    base_count_rehash_kernel<<<grid, 256, 0, st>>>(okeys, ocnt, oslots, nkeys, ncnt, nslots, n_live, overflow);
}

// rows (s,o) whose presence in a 64-bit set equals keep_present go to out (warp-aggregated compaction, order not kept). With `cnt` the
// set is a count table and a key is present only with a positive count.
struct PairSelectParams {
    const u32 *s, *o;
    u32 n;
    const u64* keys;
    const u32* cnt;
    u32 slots;
    u32 keep_present;
    u32 *out_s, *out_o;
    u32* out_count;
};
static __global__ void __launch_bounds__(256) pair_select_kernel(const __grid_constant__ PairSelectParams P) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 n_round = (P.n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += stride) {
        bool take = false;
        u32 s = 0, o = 0;
        if (i < P.n) {
            s = P.s[i];
            o = P.o[i];
            const u32 slot = set64_find(P.keys, P.slots, s, o);
            const bool present = slot != EMPTY32 && (!P.cnt || P.cnt[slot] > 0u);
            take = present == (P.keep_present != 0u);
        }
        emit_pair(take, s, o, P.out_s, P.out_o, P.out_count);
    }
}
static void launch_pair_select(const PairSelectParams& p, int n_sms, cudaStream_t st) {
    if (p.n == 0) return;
    const int grid = grid_1d(p.n, n_sms);
    pair_select_kernel<<<grid, 256, 0, st>>>(p);
}

// the keys (s,o) of the rows become TOMB64 in the set (keys that are not there are ignored)
static __global__ void __launch_bounds__(256) set64_erase_kernel(u64* set, u32 set_slots, const u32* s, const u32* o, u32 n) {
    const u32 stride = gridDim.x * blockDim.x;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u32 slot = set64_find(set, set_slots, s[i], o[i]);
        if (slot != EMPTY32) set[slot] = TOMB64;
    }
}
static void launch_set64_erase(u64* set, u32 set_slots, const u32* s, const u32* o, u32 n, int n_sms, cudaStream_t st) {
    if (n == 0) return;
    const int grid = grid_1d(n, n_sms);
    set64_erase_kernel<<<grid, 256, 0, st>>>(set, set_slots, s, o, n);
}

}  // namespace kb

// =====================================================================================================================================
// Host side: the driver
namespace {

struct PredRel {
    u32 pred = 0;
    Col s, o;
    u64 n = 0, cap = 0;
    u64 base_n = 0;       // facts present before inference (with a seed: after the seed's new facts were accepted)
    u64 seed_from = 0;    // kb_datalog_fixpoint_seed: rows [seed_from, base_n) are the seed facts that were new
    u64 delta_start = 0;  // facts [delta_start, snapshot) were added by the previous round
    u64 snapshot = 0;
    bool is_head = false;
    Buf set;              // head predicates only: known (s,o) pairs of this predicate, 64-bit keys
    u32 set_slots = 0;
    u64 set_count = 0;
};

struct Premise {
    int s_var, o_var;  // variable slots (real or synthetic, quirk Q6)
    bool pred_const;
    u32 pred;
    bool s_is_const = false, o_is_const = false;  // enforced only by KB_SEMI_NAIVE_PARALLEL (matches_rule_pattern, rules.rs:9-72)
    u32 s_const = 0, o_const = 0;
};
struct RulePlan {
    std::vector<Premise> prem;
    u32 n_vars = 0;
    bool fires = false;  // it has premises and every premise predicate is a constant (a variable one never matches: join_algorithm.rs:515-521)
};

struct Pairs {  // a list of (s,o) facts of one predicate
    Col s, o;
    u64 n = 0;
};

struct Pending {  // facts derived in the current round, not yet visible to the joins
    u32 pred;
    Col s, o;
    u64 count;
};

// KOLIBRIE_TRACE=1: synchronise after every phase of the fixpoint and print where the wall-clock time went (stderr)
struct Trace {
    bool on = getenv("KOLIBRIE_TRACE") != nullptr;
    std::chrono::steady_clock::time_point t = std::chrono::steady_clock::now();
    void mark(kb_ctx* ctx, const char* what, unsigned long long rows = 0) {
        if (!on) return;
        cudaStreamSynchronize(ctx->st);
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[kb trace] %-28s %9.3f ms  rows=%llu\n", what, std::chrono::duration<double, std::milli>(now - t).count(), rows);
        t = std::chrono::steady_clock::now();
    }
};

struct Fix {
    kb_ctx* ctx;
    std::map<u32, PredRel> rels;
    std::vector<Pending> pend;
    Buf buckets;  // candidate buckets of the radix-partitioned dedup, kept across the derive calls of one fixpoint (a 3 GB allocation
                  // from the stream-ordered pool can cost milliseconds when the pool has to remap)
    const BcDemandDev* demand = nullptr;  // kb_datalog_query: a derived fact of a restricted predicate must match one of its demand patterns
    // kb_datalog_query, ground query whose predicate is a rule head: every derive launch of that predicate probes its known-fact set for
    // the queried fact, read back with the launch's own counts
    struct Probe { u32 pred = 0, s = 0, o = 0; bool found = false; };
    Probe* probe = nullptr;
};

// What a seeded call leaves in the context for the next one: the store split by predicate and a known-fact set per rule predicate. While
// the store is the one that call left (store_version) and the rules are the same, the next seed costs what its delta costs — no scan
// of the store, no set rebuilt. KOLIBRIE_FIX_STATE=0: every seeded call starts from the store (A/B switch).
struct FixState {
    std::string sig;  // the rules, byte for byte
    u64 version = 0;  // ctx->store_version the state belongs to
    std::map<u32, PredRel> rels;
};

// base multiplicity of one predicate's facts: how many live base segments hold each (s,o) (kb_datalog_maintain)
struct BaseCount {
    Buf keys, cnt;     // 64-bit (s,o) keys, u32 count per slot
    u32 slots = 0;
    u64 occupied = 0;  // keys that hold a slot (a key whose count fell to 0 keeps its slot until the next rehash)
    u64 live = 0;      // keys with a positive count: the distinct base facts of the predicate
};

// The "closed" token: kb_datalog_fixpoint (hash-join strategies, on a store without inferred segments) or kb_datalog_maintain returned
// OK, so the store holds closure(B) \ B as its KB_TAG_INFERRED segments, for these rules, at these store / numeric-table versions.
// kb_datalog_maintain also leaves its working state here: the per-predicate relations of B ∪ I with their known-fact sets and the base
// multiplicities, so that the next slide reads nothing but its own delta. KOLIBRIE_FIX_STATE=0: that state is rebuilt from the store.
struct Closed {
    std::string sig;
    u64 store_version = 0, num_version = 0;
    bool numeric = false;  // a rule filter compares numbers: the closure depends on the numeric side table (num_version counts)
    bool has_state = false;
    std::map<u32, PredRel> rels;
    std::map<u32, BaseCount> base;
};

std::string rules_signature(const kb_rule* rules, u32 n_rules) {
    std::string s;
    auto put = [&](const void* p, size_t n) { s.append(static_cast<const char*>(p), n); };
    auto pat = [&](const kb_pattern& x) {
        const u32 w[6] = {x.s.is_var, x.s.value, x.p.is_var, x.p.value, x.o.is_var, x.o.value};
        put(w, sizeof w);
    };
    for (u32 r = 0; r < n_rules; r++) {
        const kb_rule& k = rules[r];
        const u32 h[3] = {k.n_premise, k.n_conclusion, k.n_filters};
        put(h, sizeof h);
        for (u32 i = 0; i < k.n_premise; i++) pat(k.premise[i]);
        for (u32 i = 0; i < k.n_conclusion; i++) pat(k.conclusion[i]);
        for (u32 i = 0; i < k.n_filters; i++) {
            const kb_rule_filter& f = k.filters[i];
            const u32 w[4] = {f.lhs_slot, f.cmp, f.rhs_is_var, f.rhs_slot};
            put(w, sizeof w);
            put(&f.rhs_value, sizeof f.rhs_value);
        }
    }
    return s;
}

// whether the closure reads the numeric side table: a rule filter that takes the numeric branch of evaluate_filters (rules.rs:148-160) —
// a constant right-hand side, or a variable no premise binds. Rules without one have the same closure whatever kb_dict_numeric_load holds.
bool rules_read_numbers(const kb_rule* rules, u32 n_rules) {
    for (u32 r = 0; r < n_rules; r++) {
        const kb_rule& k = rules[r];
        for (u32 f = 0; f < k.n_filters; f++) {
            const kb_rule_filter& fl = k.filters[f];
            if (fl.cmp == 0) continue;
            if (!fl.rhs_is_var) return true;
            bool bound = false;
            for (u32 i = 0; i < k.n_premise; i++) {
                const kb_pattern& p = k.premise[i];
                if ((p.s.is_var && p.s.value == fl.rhs_slot) || (p.p.is_var && p.p.value == fl.rhs_slot) || (p.o.is_var && p.o.value == fl.rhs_slot)) bound = true;
            }
            if (!bound) return true;
        }
    }
    return false;
}

bool state_disabled() { return getenv("KOLIBRIE_FIX_STATE") && getenv("KOLIBRIE_FIX_STATE")[0] == '0'; }  // (read per call: a test flips it)

kb_status grow_rel(kb_ctx* ctx, PredRel& r, u64 need) {
    if (need <= r.cap) return KB_OK;
    u64 cap = std::max<u64>(need, r.cap * 2);
    cap = std::max<u64>(cap, 1024);
    Col ns, no;
    KB_TRY(alloc_col(ctx, cap, &ns));
    KB_TRY(alloc_col(ctx, cap, &no));
    if (r.n) {
        KB_CUDA(ctx, cudaMemcpyAsync(ns.ptr, r.s.ptr, r.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(no.ptr, r.o.ptr, r.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    }
    r.s = ns; r.o = no; r.cap = cap;
    return KB_OK;
}

// append n rows (s,o) to a predicate relation
kb_status append_rows(kb_ctx* ctx, PredRel& r, const u32* s, const u32* o, u64 n) {
    if (!n) return KB_OK;
    KB_TRY(grow_rel(ctx, r, r.n + n));
    KB_CUDA(ctx, cudaMemcpyAsync(r.s.ptr + r.n, s, n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(r.o.ptr + r.n, o, n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    r.n += n;
    return KB_OK;
}

// (re)build the known-fact set of predicate `r` so that it can take the facts the next launch is EXPECTED to add at load <= 0.5.
// `extra` counts candidates, most of which are usually known already (cfg4: 1.25e9 candidates for 2.9e8 new facts), so the
// expectation is capped at half the set's size (and at least 2^20 facts); derive_kernel enforces the real bound (budget) and the launch is repeated on a
// larger table when the cap was too optimistic. A rebuild re-inserts every known fact, so every (re)build allocates twice the need.
kb_status ensure_set(Fix& fx, PredRel& r, u64 extra, bool must_grow = false, bool exact_expectation = false) {
    kb_ctx* ctx = fx.ctx;
    const u64 expect = exact_expectation ? extra : std::min<u64>(extra, std::max<u64>(r.set_count / 2, 1u << 20));
    const u64 need = exact_expectation ? r.set_count + expect : (r.set_count + expect) * 2;  // (a known final size: load <= 1/2 is enough)
    if (r.set && need <= r.set_slots && !must_grow) return KB_OK;
    static const u64 slack = getenv("KOLIBRIE_SET_SLACK") ? std::max(1, atoi(getenv("KOLIBRIE_SET_SLACK"))) : 2;
    static const u64 tight = getenv("KOLIBRIE_SET_TIGHT") ? (u64)atoi(getenv("KOLIBRIE_SET_TIGHT")) : 0;  // experiment: known final size at load <= 2/3
    u64 slots = 1024;
    if (exact_expectation && tight) { while (slots * 2 < need * 3) slots <<= 1; }
    else while (slots < need * slack) slots <<= 1;
    if (must_grow) slots = std::max<u64>(slots, (u64)r.set_slots * 2);
    if (slots > (1ull << 31)) slots = 1ull << 31;
    if (slots < need || (must_grow && r.set && slots <= r.set_slots))
        return fail(ctx, KB_E_LIMIT, "known-fact set of predicate %u would need more than 2^31 slots", r.pred);
    Buf nb;
    KB_TRY(alloc_buf(ctx, slots * sizeof(u64), &nb));
    KB_CUDA(ctx, cudaMemsetAsync(nb->p, 0xFF, slots * sizeof(u64), ctx->st));
    const u32 off = ctrl_alloc(ctx, 4);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 4 * sizeof(u32), ctx->st));
    u64 count = 0;
    timer_begin(ctx, F_BUILD);
    launch_set64_insert(static_cast<u64*>(nb->p), (u32)slots, r.s.ptr, r.o.ptr, (u32)r.n, ctx->ctrl + off, ctx->n_sms, ctx->st);
    count += r.n;
    for (auto& pd : fx.pend) {  // a rebuild in the middle of a round must keep this round's facts
        if (pd.pred != r.pred) continue;
        launch_set64_insert(static_cast<u64*>(nb->p), (u32)slots, pd.s.ptr, pd.o.ptr, (u32)pd.count, ctx->ctrl + off, ctx->n_sms, ctx->st);
        count += pd.count;
    }
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    r.set = nb;
    r.set_slots = (u32)slots;
    r.set_count = count;
    return KB_OK;
}

// a relation view over rows [start, start+n) of a predicate's columns; the probe kernels TMA-load their inputs, which needs
// 16-byte aligned column starts, so a misaligned suffix (the delta) is copied
kb_status make_view(kb_ctx* ctx, const PredRel& r, u64 start, u64 n, u32 s_slot, u32 o_slot, std::unique_ptr<kb_rel>* out) {
    auto v = std::make_unique<kb_rel>();
    v->slots = {s_slot, o_slot};
    v->n = n;
    const Col* src[2] = {&r.s, &r.o};
    for (int c = 0; c < 2; c++) {
        Col col;
        if ((start & 3ull) == 0) {
            col.buf = src[c]->buf;
            col.ptr = src[c]->ptr + start;
        } else {
            KB_TRY(alloc_col(ctx, n, &col));
            if (n) KB_CUDA(ctx, cudaMemcpyAsync(col.ptr, src[c]->ptr + start, n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        }
        v->cols.push_back(col);
    }
    *out = std::move(v);
    return KB_OK;
}

// KB_SEMI_NAIVE_PARALLEL: keep only the rows whose subject / object equal the premise's constants (the synthetic columns then
// carry a single value and simply ride along)
kb_status enforce_constants(kb_ctx* ctx, const Premise& pr, std::unique_ptr<kb_rel>* v) {
    if (!pr.s_is_const && !pr.o_is_const) return KB_OK;
    FilterProg f;
    auto eq = [&](u32 slot, u32 id) { kb_filter_op op{}; op.op = KB_F_EQ_ID; op.slot = slot; op.id = id; f.ops.push_back(op); };
    if (pr.s_is_const) eq((u32)pr.s_var, pr.s_const);
    if (pr.o_is_const) eq((u32)pr.o_var, pr.o_const);
    if (pr.s_is_const && pr.o_is_const) { kb_filter_op a{}; a.op = KB_F_AND; f.ops.push_back(a); }
    std::unique_ptr<kb_rel> out;
    KB_TRY(filter_impl(ctx, **v, f, &out));
    *v = std::move(out);
    return KB_OK;
}

// compile the rules (host): variable slots, synthetic variables for constants in s/o (quirk Q6), safety checks; every predicate a rule
// mentions gets an entry in `rels` (is_head: it occurs in a conclusion)
kb_status compile_rules(kb_ctx* ctx, const kb_rule* rules, u32 n_rules, std::vector<RulePlan>* plans_out, std::map<u32, PredRel>* rels) {
    std::vector<RulePlan>& plans = *plans_out;
    plans.assign(n_rules, RulePlan{});
    for (u32 r = 0; r < n_rules; r++) {
        const kb_rule& rule = rules[r];
        if (rule.n_premise > KB_MAX_PREMISES || rule.n_conclusion > KB_MAX_CONCLUSIONS || rule.n_filters > KB_MAX_RULE_FILTERS)
            return fail(ctx, KB_E_LIMIT, "rule %u exceeds the premise/conclusion/filter limits", r);
        u32 mx = 0;
        auto upd = [&](const kb_term& t) { if (t.is_var) mx = std::max(mx, t.value + 1); };
        for (u32 i = 0; i < rule.n_premise; i++) { upd(rule.premise[i].s); upd(rule.premise[i].p); upd(rule.premise[i].o); }
        for (u32 i = 0; i < rule.n_conclusion; i++) { upd(rule.conclusion[i].s); upd(rule.conclusion[i].p); upd(rule.conclusion[i].o); }
        u32 next = mx;
        std::map<std::pair<u32, u32>, u32> synth;  // (position, constant) -> synthetic slot: "__const_subj_{c}" / "__const_obj_{c}"
        auto syn = [&](u32 pos, u32 c) {
            auto it = synth.find({pos, c});
            if (it != synth.end()) return it->second;
            synth[{pos, c}] = next;
            return next++;
        };
        std::set<u32> bound;
        for (u32 i = 0; i < rule.n_premise; i++) {
            const kb_pattern& p = rule.premise[i];
            Premise pr;
            pr.s_var = (int)(p.s.is_var ? p.s.value : syn(0, p.s.value));
            pr.o_var = (int)(p.o.is_var ? p.o.value : syn(2, p.o.value));
            pr.pred_const = !p.p.is_var;
            pr.pred = p.p.value;
            pr.s_is_const = !p.s.is_var; pr.s_const = p.s.value;
            pr.o_is_const = !p.o.is_var; pr.o_const = p.o.value;
            if (pr.s_var == pr.o_var)
                return fail(ctx, KB_E_UNSUPPORTED, "rule %u premise %u repeats one variable in subject and object", r, i);
            if (pr.pred_const) { (*rels)[pr.pred].pred = pr.pred; bound.insert((u32)pr.s_var); bound.insert((u32)pr.o_var); }
            plans[r].prem.push_back(pr);
        }
        plans[r].n_vars = next;
        plans[r].fires = rule.n_premise > 0 && std::all_of(plans[r].prem.begin(), plans[r].prem.end(), [](const Premise& p) { return p.pred_const; });
        if (next > KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "rule %u uses more than %d variables", r, KB_MAX_COLS);
        for (u32 c = 0; c < rule.n_conclusion; c++) {
            const kb_pattern& h = rule.conclusion[c];
            if (h.p.is_var) return fail(ctx, KB_E_UNSUPPORTED, "rule %u: variable predicate in a conclusion", r);
            const kb_term* ts[2] = {&h.s, &h.o};
            for (auto* t : ts) if (t->is_var && !bound.count(t->value))
                return fail(ctx, KB_E_UNSUPPORTED, "rule %u: head variable (slot %u) is not bound by the premises (quirk Q8: the reference invents ml_output_placeholder terms / id 0)", r, t->value);
            (*rels)[h.p.value].pred = h.p.value;
            (*rels)[h.p.value].is_head = true;
        }
        for (u32 f = 0; f < rule.n_filters; f++) {
            if (rule.filters[f].cmp > KB_CMP_NE) return fail(ctx, KB_E_INVALID, "rule %u filter %u: bad comparison", r, f);
        }
    }
    return KB_OK;
}

// kb_datalog_maintain's acceptance test in front of the dedup (launch_derive, gated): the candidate must be a member of `must` and must
// have no positive count in the `veto` table
struct Gate {
    const u64* must = nullptr;
    u32 must_slots = 0;
    const BaseCount* veto = nullptr;
};

// ---- one head of one rule over the joined bindings `cur`: filters + instantiate + dedup against the known facts of `fx` + append to
// fx's pending facts (`rule_p` == nullptr: no rule filters — the seed facts of kb_datalog_fixpoint_seed take the same way in)
kb_status derive_head(Fix& fx, const kb_rel* cur, const kb_pattern& h, const kb_rule* rule_p, bool strict, const Gate* gate, Trace& tr,
                      u64* derivations) {
    kb_ctx* ctx = fx.ctx;
    DeriveParams D{};
    for (size_t k = 0; k < cur->cols.size(); k++) D.bcol[k] = cur->cols[k].ptr;
    D.n = (u32)cur->n;
    auto term = [&](const kb_term& t) {
        HeadTerm ht;
        ht.is_var = t.is_var;
        ht.value = t.is_var ? (u32)cur->col_of(t.value) : t.value;
        return ht;
    };
    D.head_s = term(h.s);
    D.head_o = term(h.o);
    D.n_filt = 0;
    for (u32 f = 0; f < (strict || !rule_p ? 0u : rule_p->n_filters); f++) {  // the parallel variant never evaluates the rule filters
        const kb_rule_filter& rf = rule_p->filters[f];
        const int lc = cur->col_of(rf.lhs_slot);
        if (lc < 0 || rf.cmp == 0) continue;  // unbound lhs: the reference skips the filter (rules.rs:139)
        RuleFilterDev d;
        d.lhs_col = (u32)lc;
        d.cmp = rf.cmp;
        d.rhs_value = rf.rhs_value;
        d.rhs_is_var = 0; d.rhs_col = 0;
        if (rf.rhs_is_var) {
            const int rc = cur->col_of(rf.rhs_slot);
            if (rc >= 0) { d.rhs_is_var = 1; d.rhs_col = (u32)rc; }
            // rhs names an unbound variable: the reference falls to the numeric branch with value.parse() (rules.rs:148-151)
        }
        D.filt[D.n_filt++] = d;
    }
    D.nt = numtab(ctx);
    if (gate) {
        D.gate_set = gate->must;
        D.gate_slots = gate->must_slots;
        if (gate->veto) {
            D.veto_keys = static_cast<const u64*>(gate->veto->keys->p);
            D.veto_cnt = static_cast<const u32*>(gate->veto->cnt->p);
            D.veto_slots = gate->veto->slots;
        }
    }
    if (fx.demand) {
        auto it = fx.demand->of.find(h.p.value);
        if (it != fx.demand->of.end()) { D.demand = it->second.first; D.n_demand = it->second.second; }
    }
    PredRel& hr = fx.rels[h.p.value];
    KB_TRY(ensure_set(fx, hr, cur->n));
    tr.mark(ctx, "  ensure_set", hr.set_slots);
    Pending pd;
    pd.pred = h.p.value;
    pd.count = 0;
    KB_TRY(alloc_col(ctx, cur->n, &pd.s));
    KB_TRY(alloc_col(ctx, cur->n, &pd.o));
    const u32 coff = ctrl_alloc(ctx, 8);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + coff, 0, 8 * sizeof(u32), ctx->st));
    D.out_s = pd.s.ptr; D.out_o = pd.o.ptr;
    D.out_cap = (u32)cur->n;
    D.out_count = ctx->ctrl + coff;
    D.overflow = ctx->ctrl + coff + 1;
    D.n_deriv = reinterpret_cast<unsigned long long*>(ctx->ctrl + coff + 4);
    const bool probe = fx.probe && fx.probe->pred == h.p.value;
    const u32 poff = probe ? ctrl_alloc(ctx, 1) : 0u;
    const u64 count_before = hr.set_count;
    for (;;) {
        D.set = static_cast<u64*>(hr.set->p);
        D.set_slots = hr.set_slots;
        // the set may fill up to 3/4 before it has to grow (expected: 1/2)
        D.budget = (u32)std::min<u64>((u64)hr.set_slots / 4 * 3 - count_before, 0xFFFFFFFFull);
        // Large candidate sets against a table far beyond L2: radix-partition the candidates by the high bits of their
        // home slot and probe partition by partition (each slice stays L2-resident) instead of one random DRAM line per
        // candidate. Partitions: ~32 MB slices, at least ~1 M candidates each (so that the CTAs of the probe pass sit on
        // one or two slices at a time), at most 1024. (A gated launch always takes the direct path.)
        u64 n_parts = 0;
        {
            const u64 set_bytes = (u64)hr.set_slots * sizeof(u64);
            u64 want = std::min<u64>(set_bytes / ctx->derive_slice_bytes, std::min<u64>(cur->n / ctx->derive_min_part_rows, 1024));
            while (want >= 2 && n_parts * 2 <= want) n_parts = n_parts ? n_parts * 2 : 2;  // power of two
            if (ctx->derive_part == 0 || gate) n_parts = 0;
        }
        if (n_parts >= 2) {
            DerivePartParams Q{};
            Q.d = D;
            Q.n_parts = (u32)n_parts;
            u32 set_bits = 0;
            while ((1ull << set_bits) < hr.set_slots) set_bits++;
            u32 part_bits = 0;
            while ((1ull << part_bits) < n_parts) part_bits++;
            Q.slice_bits = set_bits - part_bits;
            Q.bucket_cap = (u32)std::min<u64>(cur->n / n_parts + cur->n / n_parts / 8 + ctx->derive_bucket_slack, 0xFFFFFFF0ull);
            Buf ctl;
            const size_t bucket_bytes = n_parts * (u64)Q.bucket_cap * sizeof(u64);
            if (!fx.buckets || fx.buckets->bytes < bucket_bytes) {
                fx.buckets.reset();
                KB_TRY(alloc_buf(ctx, bucket_bytes + bucket_bytes / 4, &fx.buckets));
            }
            Buf buckets = fx.buckets;
            KB_TRY(alloc_buf(ctx, (2 * n_parts + 8) * sizeof(u32), &ctl));
            KB_CUDA(ctx, cudaMemsetAsync(ctl->p, 0, (2 * n_parts + 8) * sizeof(u32), ctx->st));
            Q.buckets = static_cast<u64*>(buckets->p);
            Q.cursors = static_cast<u32*>(ctl->p);
            Q.tile_start = Q.cursors + n_parts;
            Q.tickets = Q.tile_start + n_parts + 1 + ((n_parts + 1) & 1u);
            tr.mark(ctx, "    derive: buckets allocated", n_parts);
            timer_begin(ctx, F_OTHER, 3);
            launch_derive_partitioned(Q, ctx->n_sms, ctx->st);
            timer_end(ctx);
            ctx->stats.rows_built += cur->n;  // (counted as table traffic: partitioned candidates)
        } else {
            timer_begin(ctx, F_OTHER);
            launch_derive(D, ctx->n_sms, ctx->st);
            timer_end(ctx);
        }
        if (probe) launch_bc_probe(D.set, D.set_slots, fx.probe->s, fx.probe->o, ctx->ctrl + poff, ctx->st);
        KB_CUDA(ctx, cudaGetLastError());
        // counts are read immediately: the control arena may be recycled by later joins of this round
        KB_TRY(ctrl_read(ctx));
        pd.count = ctx->h_ctrl[coff];
        if (ctx->h_ctrl[coff + 1] == 1u) return fail(ctx, KB_E_LIMIT, "known-fact set overflow");
        if (ctx->h_ctrl[coff + 1] == 0u) break;
        // budget reached: rebuild the set larger WITH the facts appended so far, then repeat the launch (facts already
        // inserted are found present and are not appended twice; the derivation count is the last, complete pass's)
        fx.pend.push_back(pd);
        const kb_status gs = ensure_set(fx, hr, cur->n, true);
        fx.pend.pop_back();
        if (gs != KB_OK) return gs;
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + coff + 1, 0, sizeof(u32), ctx->st));
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + coff + 4, 0, 2 * sizeof(u32), ctx->st));
    }
    if (probe && ctx->h_ctrl[poff]) fx.probe->found = true;
    unsigned long long nd;
    memcpy(&nd, ctx->h_ctrl + coff + 4, sizeof nd);
    *derivations += nd;
    hr.set_count = count_before;
    hr.set_count += pd.count;
    if (pd.count) fx.pend.push_back(pd);
    tr.mark(ctx, "  derive", pd.count);
    return KB_OK;
}

// end of a round: the pending facts become visible (appended to their relations); returns how many there were
kb_status flush_pending(Fix& fx, u64* appended) {
    *appended = 0;
    for (auto& pd : fx.pend) {
        KB_TRY(append_rows(fx.ctx, fx.rels[pd.pred], pd.s.ptr, pd.o.ptr, pd.count));
        *appended += pd.count;
    }
    fx.pend.clear();
    return KB_OK;
}

kb_status check_strategy(kb_ctx* ctx, u32 strategy) {
    if (strategy != KB_SEMI_NAIVE && strategy != KB_NAIVE && strategy != KB_SEMI_NAIVE_PARALLEL && strategy != KB_SEMI_NAIVE_OLD_DELTA)
        return fail(ctx, KB_E_INVALID, "unknown strategy %u", strategy);
    return KB_OK;
}

// the rows of an (s,p,o) relation (slots 0,1,2) whose predicate is p
kb_status rows_of_predicate(kb_ctx* ctx, const kb_rel& spo, u32 p, std::unique_ptr<kb_rel>* out) {
    FilterProg f;
    kb_filter_op op{};
    op.op = KB_F_EQ_ID; op.slot = 1; op.id = p;
    f.ops.push_back(op);
    return filter_impl(ctx, spo, f, out);
}

// seed facts take the way of rule-less derived heads: the ones the known facts lack become visible now as the first delta, all else is
// old. The seeds: `seeds` (predicate, relation with s and o in slots 0 and 2), then the rows of `spo` (nullable; slots 0,1,2 = s,p,o)
// of each predicate of fx.rels, split off one predicate at a time so that only one predicate's rows are held at once. *accepted = the
// facts that were new (seed facts are no derivations).
kb_status accept_seeds(Fix& fx, const std::vector<std::pair<u32, const kb_rel*>>& seeds, const kb_rel* spo, Trace& tr, u64* accepted) {
    for (auto& kv : fx.rels) kv.second.snapshot = kv.second.seed_from = kv.second.n;
    u64 derivations = 0;
    auto seed = [&](u32 p, const kb_rel* rel) -> kb_status {
        if (rel->n == 0) return KB_OK;
        kb_pattern h{};
        h.s = kb_term{1, 0}; h.p = kb_term{0, p}; h.o = kb_term{1, 2};
        return derive_head(fx, rel, h, nullptr, false, nullptr, tr, &derivations);
    };
    for (auto& sd : seeds) KB_TRY(seed(sd.first, sd.second));
    if (spo && spo->n)
        for (auto& kv : fx.rels) {
            std::unique_ptr<kb_rel> sub;
            KB_TRY(rows_of_predicate(fx.ctx, *spo, kv.first, &sub));
            KB_TRY(seed(kv.first, sub.get()));
        }
    for (auto& kv : fx.rels) kv.second.delta_start = kv.second.snapshot;
    KB_TRY(flush_pending(fx, accepted));
    for (auto& kv : fx.rels) kv.second.base_n = kv.second.n;
    return KB_OK;
}

// joins premise `pr` over rows [0, visible) of its relation into the bindings `cur` (null: they become the premise's rows); strict:
// the premise's constants are enforced
kb_status join_premise(kb_ctx* ctx, std::unique_ptr<kb_rel>& cur, const Premise& pr, const PredRel& r, u64 visible, bool strict, Trace& tr) {
    if (cur && visible == 0) { cur->n = 0; return KB_OK; }
    std::unique_ptr<kb_rel> all, joined;
    KB_TRY(make_view(ctx, r, 0, visible, (u32)pr.s_var, (u32)pr.o_var, &all));
    if (strict) KB_TRY(enforce_constants(ctx, pr, &all));
    if (!cur) { cur = std::move(all); return KB_OK; }
    tr.mark(ctx, "  views");
    KB_TRY(hash_join_impl(ctx, *cur, *all, nullptr, &joined));
    cur = std::move(joined);
    tr.mark(ctx, "  join", cur->n);
    return KB_OK;
}

// rows [from, to) of a predicate relation
Pairs rows_of(const PredRel& r, u64 from, u64 to) {
    Pairs p;
    p.s = Col{r.s.buf, r.s.ptr + from};
    p.o = Col{r.o.buf, r.o.ptr + from};
    p.n = to - from;
    return p;
}

// (s,p,o) relation of per-predicate fact lists
kb_status assemble(kb_ctx* ctx, const std::vector<std::pair<u32, Pairs>>& parts, std::unique_ptr<kb_rel>* out) {
    u64 total = 0;
    for (auto& pp : parts) total += pp.second.n;
    if (total >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "result exceeds 2^32 - 16 rows");
    auto res = std::make_unique<kb_rel>();
    res->slots = {0, 1, 2};
    res->n = total;
    Col cs, cp, co;
    KB_TRY(alloc_col(ctx, total, &cs));
    KB_TRY(alloc_col(ctx, total, &cp));
    KB_TRY(alloc_col(ctx, total, &co));
    u64 off = 0;
    for (auto& pp : parts) {
        const u64 cnt = pp.second.n;
        if (!cnt) continue;
        KB_CUDA(ctx, cudaMemcpyAsync(cs.ptr + off, pp.second.s.ptr, cnt * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(co.ptr + off, pp.second.o.ptr, cnt * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        launch_fill_u32(cp.ptr + off, pp.first, cnt, ctx->st);
        off += cnt;
    }
    res->cols = {cs, cp, co};
    *out = std::move(res);
    return KB_OK;
}

// the rows of the segments `segs` split by predicate: out[p] = (s, o) of every predicate of `preds` (one fused scan per MAXP predicates;
// none when the segments hold no row)
kb_status split_segments(kb_ctx* ctx, const std::vector<Segment>& segs, const std::vector<u32>& preds, std::map<u32, Pairs>* out) {
    u64 n = 0;
    for (auto& sg : segs) n += sg.n;
    for (u32 p : preds) (*out)[p] = Pairs{};
    if (n == 0 || preds.empty()) return KB_OK;
    for (size_t b = 0; b < preds.size(); b += MAXP) {
        const u32 k = (u32)std::min<size_t>(MAXP, preds.size() - b);
        std::vector<std::unique_ptr<kb_rel>> res;
        KB_TRY(scan_predicates(ctx, segs, preds.data() + b, k, ScanOut::Cols, &res));
        for (u32 i = 0; i < k; i++) {
            Pairs& p = (*out)[preds[b + i]];
            p.s = res[i]->cols[0];
            p.o = res[i]->cols[1];
            p.n = res[i]->n;
        }
    }
    return KB_OK;
}

// the store split by predicate: every relation of fx.rels gets its predicate's facts, MAXP predicates at a time. demand
// (kb_datalog_query): a restricted predicate keeps only the facts that match one of its demand patterns.
kb_status split_store(Fix& fx) {
    kb_ctx* ctx = fx.ctx;
    std::vector<u32> preds;
    for (auto& kv : fx.rels) preds.push_back(kv.first);
    for (size_t b = 0; b < preds.size(); b += MAXP) {
        const std::vector<u32> batch(preds.begin() + b, preds.begin() + std::min<size_t>(b + MAXP, preds.size()));
        std::map<u32, Pairs> split;
        // the predicate relations are append-only buffers with the capacity of a whole-store scan output: take the scan, not the
        // (exactly sized) index slices
        KB_TRY(split_segments(ctx, ctx->segs, batch, &split));
        // a restricted predicate's rows are selected into new columns of the scanned row count, which is then their capacity; the
        // selections of a batch are read back together
        std::map<u32, u32> selected;  // predicate -> control word of its selected row count
        for (u32 p : batch) {
            PredRel& r = fx.rels[p];
            r.s = split[p].s;
            r.o = split[p].o;
            r.n = split[p].n;
            r.cap = ctx->n_triples;
            if (!fx.demand) continue;
            auto it = fx.demand->of.find(p);
            if (it == fx.demand->of.end()) continue;
            selected[p] = ctrl_alloc(ctx, 1);
            Col ns, no;
            KB_TRY(bc_demand_select(ctx, it->second.first, it->second.second, r.s, r.o, r.n, &ns, &no, selected[p]));
            r.s = ns;
            r.o = no;
            r.cap = r.n;
        }
        if (!selected.empty()) KB_TRY(ctrl_read(ctx));
        for (u32 p : batch) {
            PredRel& r = fx.rels[p];
            if (selected.count(p)) r.n = ctx->h_ctrl[selected[p]];
            r.base_n = r.n;
            if (r.n * 4 < r.cap) {  // shrink: the scan allocates for the worst case (grow_rel from no capacity copies the rows over)
                r.cap = 0;
                KB_TRY(grow_rel(ctx, r, std::max<u64>(r.n * 2, 1024)));
            }
        }
    }
    return KB_OK;
}

// kb_datalog_query's rounds: premise constants enforced at every arity, no rule filters (derive_head's strict mode), at most max_rounds
// rounds, and a ground query stops at the end of the first round in which a derive launch found the queried fact in its known-fact set
// (fx.probe)
struct QueryMode {
    u32 max_rounds = 0;
    u32 rounds = 0;                  // rounds run
    bool fixpoint = false, stopped_early = false;
};

// ---- rounds: from the current delta of every relation ([delta_start, n)) to the fixpoint (qm: a query's rounds)
kb_status run_rounds(Fix& fx, const kb_rule* rules, u32 n_rules, const std::vector<RulePlan>& plans, u32 strategy, kb_fixpoint_stats& st,
                     Trace& tr, QueryMode* qm = nullptr) {
    kb_ctx* ctx = fx.ctx;
    const bool old_delta = strategy == KB_SEMI_NAIVE_OLD_DELTA;
    const bool strict = strategy == KB_SEMI_NAIVE_PARALLEL || qm;
    for (u32 round = 0;; round++) {
        if (qm) {
            if (round >= qm->max_rounds) break;
            qm->rounds++;
        }
        for (auto& kv : fx.rels) kv.second.snapshot = kv.second.n;
        fx.pend.clear();
        for (u32 r = 0; r < n_rules; r++) {
            const kb_rule& rule = rules[r];
            const RulePlan& pl = plans[r];
            const u32 np = (u32)pl.prem.size();
            if (!pl.fires) continue;
            if (strategy == KB_SEMI_NAIVE_PARALLEL && np != 1 && np != 2) continue;  // semi_naive_parallel.rs:149: other arities are skipped
            const u32 n_start = strategy == KB_NAIVE ? 1 : np;
            for (u32 i = 0; i < n_start; i++) {
                // premise i over the delta (semi-naive) or over all facts (naive), then the others over all facts
                std::unique_ptr<kb_rel> cur;
                {
                    const PredRel& pr = fx.rels[pl.prem[i].pred];
                    const u64 a = strategy == KB_NAIVE ? 0 : pr.delta_start;
                    const u64 n = pr.snapshot - a;
                    if (n == 0) continue;
                    KB_TRY(make_view(ctx, pr, a, n, (u32)pl.prem[i].s_var, (u32)pl.prem[i].o_var, &cur));
                    if (strict) KB_TRY(enforce_constants(ctx, pl.prem[i], &cur));
                }
                for (u32 j = 0; j < np && cur->n; j++) {
                    if (j == i) continue;
                    const PredRel& pr = fx.rels[pl.prem[j].pred];
                    // KB_SEMI_NAIVE_OLD_DELTA: a premise before the delta premise sees only the facts older than its delta
                    KB_TRY(join_premise(ctx, cur, pl.prem[j], pr, old_delta && j < i ? pr.delta_start : pr.snapshot, strict, tr));
                }
                if (cur->n == 0) continue;
                // heads: filters + instantiate + dedup against known facts + append
                for (u32 c = 0; c < rule.n_conclusion; c++) {
                    KB_TRY(derive_head(fx, cur.get(), rule.conclusion[c], &rule, strict, nullptr, tr, &st.derivations));
                }
            }
        }
        // ---- end of round: the facts that were new become visible (infer_generic.rs:42-48)
        for (auto& kv : fx.rels) kv.second.delta_start = kv.second.snapshot;
        u64 round_new = 0;
        KB_TRY(flush_pending(fx, &round_new));
        tr.mark(ctx, "round end: append", round_new);
        const bool found = qm && fx.probe && fx.probe->found;
        if (round_new == 0 && !found) {
            if (qm) qm->fixpoint = true;
            break;
        }
        if (round_new) {
            if (st.rounds < 64) st.round_new[st.rounds] = round_new;
            st.rounds++;
            st.inferred += round_new;
        }
        if (found) {
            qm->stopped_early = true;
            break;
        }
        if (round > 100000) return fail(ctx, KB_E_LIMIT, "fixpoint did not converge");
    }
    return KB_OK;
}

}  // namespace

// `seed` == nullptr: kb_datalog_fixpoint (every fact of the store is the first delta). With a seed (kb_datalog_fixpoint_seed): the store
// is taken as closed under the rules already, the seed facts the store does not hold yet are accepted into it and form the first delta.
static kb_status fixpoint_impl(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy, bool seeded, const kb_rel* seed,
                               kb_rel** inferred, uint64_t* n_seed_new, kb_fixpoint_stats* stats) {
    KB_ENTER(ctx);
    if ((n_rules && !rules) || !inferred) return fail(ctx, KB_E_INVALID, "NULL argument");
    KB_TRY(check_strategy(ctx, strategy));
    if (seeded && !seed) return fail(ctx, KB_E_INVALID, "NULL seed");
    if (seed && (seed->pair || seed->cols.size() != 3 || seed->col_of(0) != 0 || seed->col_of(1) != 1 || seed->col_of(2) != 2))
        return fail(ctx, KB_E_INVALID, "the seed must be a 3-column relation with slots 0,1,2 = s,p,o");
    if (seed && seed->n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "seed too large");
    const bool strict = strategy == KB_SEMI_NAIVE_PARALLEL;
    kb_fixpoint_stats st{};
    ScopedEvent ev0, ev1;
    cudaEventRecord(ev0, ctx->st);

    // ---- compile the rules (host): variable slots, synthetic variables for constants in s/o (quirk Q6), safety checks
    std::vector<RulePlan> plans;
    Fix fx;
    Trace tr;
    fx.ctx = ctx;
    KB_TRY(compile_rules(ctx, rules, n_rules, &plans, &fx.rels));
    // a seed fact may belong to any predicate of the rules: each of them needs its known-fact set (to tell the new seed facts from the old)
    if (seed) for (auto& kv : fx.rels) kv.second.is_head = true;
    // the closed token (kb_datalog_maintain's precondition) is recorded again only by an unseeded hash-join fixpoint over a store that has
    // no inferred segment yet: then the inferred segment it appends is exactly closure(B) \ B
    bool had_inferred = false;
    for (auto& sg : ctx->segs) if (sg.tag == KB_TAG_INFERRED) had_inferred = true;
    ctx->closed.reset();

    // ---- a seeded call may find the state its predecessor left (FixState): then nothing below reads the store
    const bool state_off = state_disabled();
    const std::string sig = seed && !state_off ? rules_signature(rules, n_rules) : std::string();
    bool reused = false;
    if (seed && !state_off && ctx->fix_state) {
        FixState* fs = static_cast<FixState*>(ctx->fix_state.get());
        if (fs->version == ctx->store_version && fs->sig == sig) {
            fx.rels = std::move(fs->rels);
            reused = true;
        }
    }
    ctx->fix_state.reset();  // taken, stale, or about to be (an unseeded run appends to the store)

    // ---- split the store by predicate
    if (!reused) KB_TRY(split_store(fx));
    tr.mark(ctx, "split store by predicate");
    if (!reused) for (auto& kv : fx.rels) if (kv.second.is_head) {
        kv.second.set_count = kv.second.n;
        // A window that re-materialises the same rules every firing (simple_r2r.rs:103-128) ends with about as many facts as last time:
        // the set is built for that size at once (config 4: otherwise a 2^28 -> 2^30 rebuild lands in the middle of round 0)
        u64 expect = 1024;
        auto hint = ctx->fix_hint.find(kv.first);
        if (hint != ctx->fix_hint.end() && hint->second > kv.second.n) expect = std::min<u64>(hint->second - kv.second.n, 0x7FFFFFFFull);
        KB_TRY(ensure_set(fx, kv.second, expect, false, /*exact_expectation=*/expect > 1024));
    }
    tr.mark(ctx, "initial known-fact sets");

    // ---- seed: the facts the store does not hold yet
    u64 seed_new = 0;
    if (seed) {
        KB_TRY(accept_seeds(fx, {}, seed, tr, &seed_new));
        tr.mark(ctx, "seed accepted", seed_new);
    }

    // ---- rounds
    KB_TRY(run_rounds(fx, rules, n_rules, plans, strategy, st, tr));

    // ---- result: inferred facts as (s,p,o) columns; also appended to the store (infer_generic.rs:46 index_manager.insert). With a seed:
    // the accepted seed facts first, then the inferred ones, predicate by predicate.
    const u64 total = seed_new + st.inferred;
    if (total >= 0xFFFFFFF0ull || ctx->n_triples + total >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "the closure exceeds 2^32 - 16 triples");
    std::vector<std::pair<u32, Pairs>> parts;
    if (seed) for (auto& kv : fx.rels) parts.push_back({kv.first, rows_of(kv.second, kv.second.seed_from, kv.second.base_n)});
    for (auto& kv : fx.rels) parts.push_back({kv.first, rows_of(kv.second, kv.second.base_n, kv.second.n)});
    std::unique_ptr<kb_rel> res;
    KB_TRY(assemble(ctx, parts, &res));
    for (auto& kv : fx.rels) if (kv.second.is_head) ctx->fix_hint[kv.first] = kv.second.n;
    if (total) {
        Segment sg;
        sg.tag = KB_TAG_INFERRED;
        sg.n = total;
        sg.s = res->cols[0]; sg.p = res->cols[1]; sg.o = res->cols[2];
        KB_TRY(store_add_device_segment(ctx, sg, /*keep_index=*/false));  // (no statistics pass over the closure)
    }
    tr.mark(ctx, "result assembly", total);
    cudaEventRecord(ev1, ctx->st);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    timers_flush(ctx);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev0, ev1);
    st.device_ms = ms;
    if (seed && !state_off) {  // the next seeded call continues from here
        auto fs = std::make_shared<FixState>();
        fs->sig = sig;
        fs->version = ctx->store_version;
        fs->rels = std::move(fx.rels);
        ctx->fix_state = fs;
    }
    if (!seed && !strict && !had_inferred) {
        auto cl = std::make_shared<Closed>();
        cl->sig = rules_signature(rules, n_rules);
        cl->store_version = ctx->store_version;
        cl->num_version = ctx->num_version;
        cl->numeric = rules_read_numbers(rules, n_rules);
        ctx->closed = cl;
    }
    if (stats) *stats = st;
    if (n_seed_new) *n_seed_new = seed_new;
    ctx->stats.rows_out = st.inferred;
    *inferred = res.release();
    return KB_OK;
}

extern "C" kb_status kb_datalog_fixpoint(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy, kb_rel** inferred,
                                         kb_fixpoint_stats* stats) {
    return fixpoint_impl(ctx, rules, n_rules, strategy, false, nullptr, inferred, nullptr, stats);
}

// Incremental materialisation: what Reasoner::add_abox_triple + infer_new_facts_semi_naive (reasoning.rs, semi_naive.rs:89) reach by
// starting over, reached from the delta alone. Used per window slide (simple_r2r.rs:95-128 adds the slide's triples and materialises
// again) and by the sharded fixpoint (kolibrie_b200/dist.py: facts derived on another rank arrive as seeds).
extern "C" kb_status kb_datalog_fixpoint_seed(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy, const kb_rel* seed,
                                              kb_rel** out, uint64_t* n_seed_new, kb_fixpoint_stats* stats) {
    // (the seed facts are stored with KB_TAG_INFERRED: base and inferred facts can no longer be told apart, so the closed token goes)
    return fixpoint_impl(ctx, rules, n_rules, strategy, true, seed, out, n_seed_new, stats);
}

// Reasoner::backward_chaining (backward_chaining.rs:165-259): the distinct bindings of the query's variables over T^max_depth, the facts
// with a proof of height <= max_depth, computed by at most max_depth semi-naive rounds over the demanded facts (kb_backward.cu). Reads
// the store and leaves it, its index and every state kept for the forward calls as they were.
extern "C" kb_status kb_datalog_query(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, const kb_pattern* query, uint32_t max_depth,
                                      kb_rel** out, kb_bc_stats* stats) {
    KB_ENTER(ctx);
    if ((n_rules && !rules) || !query || !out) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (max_depth > KB_BC_DEPTH_LIMIT) return fail(ctx, KB_E_LIMIT, "max_depth %u exceeds %u", max_depth, KB_BC_DEPTH_LIMIT);
    auto term_ok = [&](const kb_term& t, const char* what, u32 r) -> kb_status {
        if (t.is_var == KB_TERM_QUOTED) return fail(ctx, KB_E_UNSUPPORTED, "%s %u: a quoted-triple term (quoted-triple unification is not supported)", what, r);
        if (t.is_var > 1) return fail(ctx, KB_E_INVALID, "%s %u: bad term kind %u", what, r, t.is_var);
        if (!t.is_var && t.value == KB_ID_NONE) return fail(ctx, KB_E_INVALID, "%s %u: KB_ID_NONE is reserved", what, r);
        return KB_OK;
    };
    for (const kb_term* t : {&query->s, &query->p, &query->o}) KB_TRY(term_ok(*t, "query", 0));
    for (u32 r = 0; r < n_rules; r++) {
        const kb_rule& rule = rules[r];
        if (rule.n_premise == 0) return fail(ctx, KB_E_UNSUPPORTED, "rule %u has no premise", r);
        for (u32 i = 0; i < rule.n_premise; i++) {
            for (const kb_term* t : {&rule.premise[i].s, &rule.premise[i].p, &rule.premise[i].o}) KB_TRY(term_ok(*t, "rule", r));
            // the forward rounds never match a variable predicate, SLD resolution would match every fact: refused rather than answered differently
            if (rule.premise[i].p.is_var) return fail(ctx, KB_E_UNSUPPORTED, "rule %u premise %u: variable predicate", r, i);
        }
        for (u32 c = 0; c < rule.n_conclusion; c++)
            for (const kb_term* t : {&rule.conclusion[c].s, &rule.conclusion[c].p, &rule.conclusion[c].o}) KB_TRY(term_ok(*t, "rule", r));
    }
    {  // the shapes the forward driver refuses (unsafe head, variable head predicate, one variable as subject and object of a premise)
        std::vector<RulePlan> pl;
        std::map<u32, PredRel> scratch;
        KB_TRY(compile_rules(ctx, rules, n_rules, &pl, &scratch));
    }
    ScopedEvent ev0, ev1;
    cudaEventRecord(ev0, ctx->st);
    kb_bc_stats bs{};

    // ---- demand (host): the relevant rules and, per predicate, the patterns its useful facts match
    BcDemand dem;
    bc_demand_compile(rules, n_rules, *query, &dem);
    std::vector<kb_rule> relevant;
    for (u32 r = 0; r < n_rules; r++) if (dem.relevant[r]) relevant.push_back(rules[r]);
    Fix fx;
    Trace tr;
    fx.ctx = ctx;
    std::vector<RulePlan> plans;
    KB_TRY(compile_rules(ctx, relevant.data(), (u32)relevant.size(), &plans, &fx.rels));
    if (!query->p.is_var) fx.rels[query->p.value].pred = query->p.value;
    std::vector<u32> preds;
    for (auto& kv : fx.rels) preds.push_back(kv.first);
    BcDemandDev dd;
    KB_TRY(bc_demand_upload(ctx, dem, preds, &dd));
    fx.demand = &dd;

    // ---- the demanded facts of every predicate the relevant rules and the query mention, and the known-fact sets of the heads
    KB_TRY(split_store(fx));
    for (auto& kv : fx.rels) {
        bs.base_facts += kv.second.n;
        if (!kv.second.is_head) continue;
        kv.second.set_count = kv.second.n;
        KB_TRY(ensure_set(fx, kv.second, 1024));
    }
    tr.mark(ctx, "query: demanded facts", bs.base_facts);

    // ---- rounds
    QueryMode qm;
    qm.max_rounds = max_depth;
    Fix::Probe probe;
    if (!query->s.is_var && !query->p.is_var && !query->o.is_var && fx.rels[query->p.value].is_head) {
        probe.pred = query->p.value;
        probe.s = query->s.value;
        probe.o = query->o.value;
        fx.probe = &probe;
    }
    kb_fixpoint_stats st{};
    KB_TRY(run_rounds(fx, relevant.data(), (u32)relevant.size(), plans, KB_SEMI_NAIVE, st, tr, &qm));

    // ---- answers: the query's predicate relation; a variable predicate reads every store segment and every derived fact
    std::vector<BcSource> src;
    auto rel_source = [&](const PredRel& r, u64 from) {
        BcSource b;
        b.in[0] = r.s.ptr + from;
        b.cval[1] = r.pred;
        b.in[2] = r.o.ptr + from;
        b.n = r.n - from;
        if (b.n) src.push_back(b);
    };
    if (!query->p.is_var) rel_source(fx.rels[query->p.value], 0);
    else {
        for (auto& sg : ctx->segs) {
            if (sg.ready) KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, sg.ready, 0));
            BcSource b;
            b.in[0] = sg.s.ptr; b.in[1] = sg.p.ptr; b.in[2] = sg.o.ptr;
            b.n = sg.n;
            if (b.n) src.push_back(b);
        }
        for (auto& kv : fx.rels) rel_source(kv.second, kv.second.base_n);
    }
    std::unique_ptr<kb_rel> res;
    KB_TRY(bc_answer(ctx, *query, src, &res));
    tr.mark(ctx, "query: answers", res->n);
    cudaEventRecord(ev1, ctx->st);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    timers_flush(ctx);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev0, ev1);
    bs.rounds = qm.rounds;
    bs.reached_fixpoint = qm.fixpoint;
    bs.stopped_early = qm.stopped_early;
    bs.relevant_rules = (u32)relevant.size();
    bs.demand_patterns = dem.n_patterns;
    bs.restricted_predicates = (u32)dd.of.size();
    bs.derived = st.inferred;
    bs.derivations = st.derivations;
    bs.answers = res->n;
    bs.device_ms = ms;
    if (stats) *stats = bs;
    ctx->stats.rows_out = res->n;
    *out = res.release();
    return KB_OK;
}

// =====================================================================================================================================
// kb_datalog_maintain: delete-and-rederive (DRed) of the inferred segment across a window slide
namespace {

u64 slots_for(u64 n) {
    u64 s = 1024;
    while (s < 2 * n) s <<= 1;
    return s;
}

kb_status base_alloc(kb_ctx* ctx, BaseCount& b, u64 slots) {
    if (slots > (1ull << 31)) return fail(ctx, KB_E_LIMIT, "base count table would need more than 2^31 slots");
    BaseCount nb;
    nb.slots = (u32)slots;
    KB_TRY(alloc_buf(ctx, slots * sizeof(u64), &nb.keys));
    KB_TRY(alloc_buf(ctx, slots * sizeof(u32), &nb.cnt));
    KB_CUDA(ctx, cudaMemsetAsync(nb.keys->p, 0xFF, slots * sizeof(u64), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(nb.cnt->p, 0, slots * sizeof(u32), ctx->st));
    b = nb;
    return KB_OK;
}

// n rows join (delta +1) or leave (delta -1) the base; *edge (nullable) receives the facts whose count crossed zero: the facts that were
// not base facts before (+1), the facts that are no base facts any more (-1). Every such fact comes out once.
kb_status base_update(kb_ctx* ctx, BaseCount& b, const u32* s, const u32* o, u64 n, int delta, Pairs* edge) {
    if (edge) *edge = Pairs{};
    // +1 may claim up to n slots. When that could take the table past 3/4, the LIVE keys move to a fresh table sized for them and the
    // rows (the keys whose count fell to 0 are dropped): the table follows the live facts, not the rows a long-running window has seen
    // (the reference's firing protocol re-adds the whole window every firing, n ~ the window, most keys already there)
    if (delta > 0 && (b.occupied + n) * 4 > (u64)b.slots * 3) {
        BaseCount nb;
        KB_TRY(base_alloc(ctx, nb, slots_for(b.live + n)));
        const u32 off = ctrl_alloc(ctx, 2);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 2 * sizeof(u32), ctx->st));
        launch_base_count_rehash(static_cast<const u64*>(b.keys->p), static_cast<const u32*>(b.cnt->p), b.slots, static_cast<u64*>(nb.keys->p),
                                 static_cast<u32*>(nb.cnt->p), nb.slots, ctx->ctrl + off, ctx->ctrl + off + 1, ctx->n_sms, ctx->st);
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        if (ctx->h_ctrl[off + 1]) return fail(ctx, KB_E_LIMIT, "base count table overflow");
        if (ctx->h_ctrl[off] != b.live) return fail(ctx, KB_E_INVALID, "base count table: %u live keys moved, %llu expected", ctx->h_ctrl[off], (unsigned long long)b.live);
        nb.occupied = nb.live = b.live;
        b = nb;
    }
    if (n == 0) return KB_OK;
    BaseCountParams P{};
    P.keys = static_cast<u64*>(b.keys->p);
    P.cnt = static_cast<u32*>(b.cnt->p);
    P.slots = b.slots;
    P.s = s; P.o = o;
    P.n = (u32)n;
    P.delta = delta;
    if (edge) {
        KB_TRY(alloc_col(ctx, n, &edge->s));
        KB_TRY(alloc_col(ctx, n, &edge->o));
        P.out_s = edge->s.ptr; P.out_o = edge->o.ptr;
    }
    const u32 off = ctrl_alloc(ctx, 4);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 4 * sizeof(u32), ctx->st));
    P.out_count = ctx->ctrl + off;
    P.overflow = ctx->ctrl + off + 1;
    P.claimed = ctx->ctrl + off + 2;
    timer_begin(ctx, F_BUILD);
    launch_base_count(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    if (ctx->h_ctrl[off + 1]) return fail(ctx, KB_E_LIMIT, "base count table overflow");
    const u64 crossed = ctx->h_ctrl[off];
    b.occupied += ctx->h_ctrl[off + 2];
    if (delta > 0) b.live += crossed;
    else b.live -= std::min<u64>(crossed, b.live);
    if (edge) edge->n = crossed;
    return KB_OK;
}

// the rows (s,o) whose membership in a set (keys/cnt/slots: a count table, cnt == nullptr: a plain 64-bit set; keys == nullptr: the
// empty set) equals `keep_present`
kb_status select_pairs(kb_ctx* ctx, const u32* s, const u32* o, u64 n, const u64* keys, const u32* cnt, u32 slots, bool keep_present, Pairs* out) {
    *out = Pairs{};
    KB_TRY(alloc_col(ctx, n, &out->s));
    KB_TRY(alloc_col(ctx, n, &out->o));
    if (n == 0) return KB_OK;
    if (!keys) {
        if (keep_present) return KB_OK;
        KB_CUDA(ctx, cudaMemcpyAsync(out->s.ptr, s, n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(out->o.ptr, o, n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
        out->n = n;
        return KB_OK;
    }
    PairSelectParams P{};
    P.s = s; P.o = o;
    P.n = (u32)n;
    P.keys = keys; P.cnt = cnt; P.slots = slots;
    P.keep_present = keep_present ? 1u : 0u;
    P.out_s = out->s.ptr; P.out_o = out->o.ptr;
    const u32 off = ctrl_alloc(ctx, 1);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, sizeof(u32), ctx->st));
    P.out_count = ctx->ctrl + off;
    timer_begin(ctx, F_FILTER);
    launch_pair_select(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    out->n = ctx->h_ctrl[off];
    return KB_OK;
}
const u64* set_of(const PredRel& r) { return r.set ? static_cast<const u64*>(r.set->p) : nullptr; }

// the facts of a head predicate as bindings of the head's variables (a constant of the head binds nothing: every fact derived from
// these bindings is checked against the facts themselves by the gate); nullptr when the head has no variable
std::unique_ptr<kb_rel> head_view(const PredRel& D, const kb_pattern& h) {
    auto v = std::make_unique<kb_rel>();
    v->n = D.n;
    if (h.s.is_var) { v->slots.push_back(h.s.value); v->cols.push_back(D.s); }
    if (h.o.is_var && !(h.s.is_var && h.o.value == h.s.value)) { v->slots.push_back(h.o.value); v->cols.push_back(D.o); }
    if (v->slots.empty()) return nullptr;
    return v;
}

}  // namespace

static kb_status maintain_impl(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy, const uint64_t* evict_tags, uint32_t n_evict,
                               const kb_rel* add, uint64_t add_tag, kb_rel** inferred_removed, kb_rel** inferred_added, kb_maintain_stats* stats) {
    // ---- validation: nothing changes before all of it passed
    if ((n_rules && !rules) || (n_evict && !evict_tags)) return fail(ctx, KB_E_INVALID, "NULL argument");
    KB_TRY(check_strategy(ctx, strategy));
    if (strategy == KB_SEMI_NAIVE_PARALLEL) return fail(ctx, KB_E_UNSUPPORTED, "kb_datalog_maintain: KB_SEMI_NAIVE_PARALLEL has its own closure; not maintained");
    if (add && (add->pair || add->cols.size() != 3 || add->col_of(0) != 0 || add->col_of(1) != 1 || add->col_of(2) != 2))
        return fail(ctx, KB_E_INVALID, "`add` must be a 3-column relation with slots 0,1,2 = s,p,o");
    if (add && add->n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "`add` too large");
    if (add && add_tag == KB_TAG_INFERRED) return fail(ctx, KB_E_INVALID, "KB_TAG_INFERRED is not a tag `add` can take");
    std::set<u64> evict(evict_tags, evict_tags + n_evict);
    if (evict.count(KB_TAG_INFERRED)) return fail(ctx, KB_E_INVALID, "KB_TAG_INFERRED cannot be evicted by kb_datalog_maintain");
    std::vector<RulePlan> plans;
    Fix fx;
    fx.ctx = ctx;
    KB_TRY(compile_rules(ctx, rules, n_rules, &plans, &fx.rels));
    std::map<u32, bool> head;  // predicates that occur in a conclusion (the only ones with inferred facts)
    for (auto& kv : fx.rels) { head[kv.first] = kv.second.is_head; kv.second.is_head = true; }
    const std::string sig = rules_signature(rules, n_rules);
    auto cl = std::static_pointer_cast<Closed>(ctx->closed);
    if (!cl || cl->sig != sig || cl->store_version != ctx->store_version || (cl->numeric && cl->num_version != ctx->num_version))
        return fail(ctx, KB_E_INVALID, "store not closed under these rules: run kb_datalog_fixpoint");
    for (u64 t : evict) {
        bool found = false;
        for (auto& sg : ctx->segs) if (sg.tag == t) found = true;
        if (!found) return fail(ctx, KB_E_NOT_FOUND, "no segment with tag %llu", (unsigned long long)t);
    }
    kb_maintain_stats ms{};
    ScopedEvent ev0, ev1;
    cudaEventRecord(ev0, ctx->st);
    Trace tr;
    std::unique_ptr<kb_rel> out_removed, out_added;
    if (evict.empty() && !add) {  // nothing moves
        KB_TRY(assemble(ctx, {}, &out_removed));
        KB_TRY(assemble(ctx, {}, &out_added));
        if (stats) *stats = ms;
        if (inferred_removed) *inferred_removed = out_removed.release();
        if (inferred_added) *inferred_added = out_added.release();
        return KB_OK;
    }
    std::vector<u32> preds;
    for (auto& kv : fx.rels) preds.push_back(kv.first);

    // ---- the kept state (the relations of B ∪ I, their known-fact sets, the base multiplicities) or the same rebuilt from the store.
    // From here until the store is rewritten the store does not change: a failure drops the state (the next call rebuilds it) and keeps
    // the token, since the store is still closed.
    const bool state_off = state_disabled();
    std::map<u32, BaseCount> base;
    if (cl->has_state && !state_off) {
        fx.rels = std::move(cl->rels);
        base = std::move(cl->base);
    }
    const bool reused = cl->has_state && !state_off;
    cl->has_state = false;
    cl->rels.clear();
    cl->base.clear();
    std::vector<Segment> base_segs, inferred_segs, evicted_segs;
    for (auto& sg : ctx->segs) {
        (sg.tag == KB_TAG_INFERRED ? inferred_segs : base_segs).push_back(sg);
        if (evict.count(sg.tag)) evicted_segs.push_back(sg);
    }
    if (!reused) {
        std::map<u32, Pairs> bsplit, isplit;
        KB_TRY(split_segments(ctx, base_segs, preds, &bsplit));
        KB_TRY(split_segments(ctx, inferred_segs, preds, &isplit));
        for (u32 p : preds) {
            PredRel& r = fx.rels[p];
            const Pairs &b = bsplit[p], &i = isplit[p];
            KB_TRY(grow_rel(ctx, r, std::max<u64>((b.n + i.n) * 2, 1024)));
            KB_TRY(append_rows(ctx, r, b.s.ptr, b.o.ptr, b.n));
            KB_TRY(append_rows(ctx, r, i.s.ptr, i.o.ptr, i.n));
            r.set_count = r.n;
            KB_TRY(ensure_set(fx, r, 1024));
            KB_TRY(base_alloc(ctx, base[p], slots_for(b.n + 1024)));
            KB_TRY(base_update(ctx, base[p], b.s.ptr, b.o.ptr, b.n, +1, nullptr));
        }
    }
    tr.mark(ctx, "maintain: state", reused);

    // ---- 1. base difference from set membership: the rows of `add` join the base, then the rows of the evicted segments leave it.
    // D0 = facts whose count reached 0 (B \ B'), `fresh` = facts of `add` whose count left 0 (B' \ B). A fact that another live segment
    // or `add` still holds keeps a positive count and does not move.
    std::map<u32, Pairs> evicted, d0, fresh;
    std::map<u32, std::unique_ptr<kb_rel>> add_of;
    KB_TRY(split_segments(ctx, evicted_segs, preds, &evicted));
    for (u32 p : preds) {
        if (add && add->n) {
            KB_TRY(rows_of_predicate(ctx, *add, p, &add_of[p]));
            const kb_rel& a = *add_of[p];
            KB_TRY(base_update(ctx, base[p], a.cols[a.col_of(0)].ptr, a.cols[a.col_of(2)].ptr, a.n, +1, &fresh[p]));
        }
        KB_TRY(base_update(ctx, base[p], evicted[p].s.ptr, evicted[p].o.ptr, evicted[p].n, -1, &d0[p]));
        ms.base_added += fresh[p].n;
        ms.base_removed += d0[p].n;
    }
    // facts of `add` that were inferred: they leave I (they are base facts now), read before the known-fact sets change
    std::vector<std::pair<u32, Pairs>> removed_parts, added_parts;
    for (u32 p : preds) {
        if (!head[p] || fresh[p].n == 0) continue;
        Pairs moved;
        const PredRel& r = fx.rels[p];
        KB_TRY(select_pairs(ctx, fresh[p].s.ptr, fresh[p].o.ptr, fresh[p].n, set_of(r), nullptr, r.set_slots, true, &moved));
        removed_parts.push_back({p, moved});
    }
    tr.mark(ctx, "maintain: base difference", ms.base_removed);
    if (tr.on) {  // (what a long-running window holds in base count tables: bounded by the live facts)
        u64 slots = 0;
        for (auto& kv : base) slots += kv.second.slots;
        tr.mark(ctx, "maintain: base count slots", slots);
    }

    // ---- 2. over-delete, semi-naive from D0: the delta of one premise joined against the OLD facts (B ∪ I) of the others; a head that is
    // known, is no fact of B', and was not marked yet joins the next delta. `del` holds D0 ∪ OD per predicate (list + set).
    Fix del;
    del.ctx = ctx;
    std::map<u32, u64> d0n;
    for (u32 p : preds) {
        PredRel& r = del.rels[p];
        r.pred = p;
        r.is_head = true;
        KB_TRY(append_rows(ctx, r, d0[p].s.ptr, d0[p].o.ptr, d0[p].n));
        d0n[p] = r.n;
        r.set_count = r.n;
        KB_TRY(ensure_set(del, r, 1024));
    }
    u64 derivations = 0;
    for (;;) {
        for (auto& kv : del.rels) kv.second.snapshot = kv.second.n;
        del.pend.clear();
        for (u32 r = 0; r < n_rules; r++) {
            const kb_rule& rule = rules[r];
            const RulePlan& pl = plans[r];
            const u32 np = (u32)pl.prem.size();
            if (!pl.fires) continue;
            for (u32 i = 0; i < np; i++) {
                const PredRel& dr = del.rels[pl.prem[i].pred];
                const u64 n = dr.snapshot - dr.delta_start;
                if (n == 0) continue;
                std::unique_ptr<kb_rel> cur;
                KB_TRY(make_view(ctx, dr, dr.delta_start, n, (u32)pl.prem[i].s_var, (u32)pl.prem[i].o_var, &cur));
                for (u32 j = 0; j < np && cur->n; j++) {
                    if (j == i) continue;
                    const PredRel& pr = fx.rels[pl.prem[j].pred];
                    KB_TRY(join_premise(ctx, cur, pl.prem[j], pr, pr.n, false, tr));
                }
                if (cur->n == 0) continue;
                for (u32 c = 0; c < rule.n_conclusion; c++) {
                    const PredRel& known = fx.rels[rule.conclusion[c].p.value];
                    Gate g;
                    g.must = set_of(known);
                    g.must_slots = known.set_slots;
                    g.veto = &base[rule.conclusion[c].p.value];
                    KB_TRY(derive_head(del, cur.get(), rule.conclusion[c], &rule, false, &g, tr, &derivations));
                }
            }
        }
        for (auto& kv : del.rels) kv.second.delta_start = kv.second.snapshot;
        u64 marked = 0;
        KB_TRY(flush_pending(del, &marked));
        if (marked == 0) break;
        ms.overdeleted += marked;
        ms.overdelete_rounds++;
        if (ms.overdelete_rounds > 100000) return fail(ctx, KB_E_LIMIT, "over-deletion did not converge");
    }
    tr.mark(ctx, "maintain: over-delete", ms.overdeleted);

    // ---- 3. remove D0 ∪ OD: the relations are compacted (mark-and-compact against the deletion set), the known-fact sets get
    // tombstones (they go when the set is next rebuilt from its relation)
    for (u32 p : preds) {
        const PredRel& dr = del.rels[p];
        if (dr.n == 0) continue;
        PredRel& r = fx.rels[p];
        Pairs keep;
        KB_TRY(select_pairs(ctx, r.s.ptr, r.o.ptr, r.n, set_of(dr), nullptr, dr.set_slots, false, &keep));
        r.s = keep.s; r.o = keep.o; r.n = keep.n; r.cap = keep.n;  // (the next append reallocates)
        launch_set64_erase(static_cast<u64*>(r.set->p), r.set_slots, dr.s.ptr, dr.o.ptr, (u32)dr.n, ctx->n_sms, ctx->st);
        KB_CUDA(ctx, cudaGetLastError());
    }
    tr.mark(ctx, "maintain: remove");

    // ---- 4. rederive: the removed facts of a head, used as an extra first premise that binds the head's variables, joined against the
    // remaining facts; a derived head that is one of the removed facts (gate) is still derivable
    Fix red;
    red.ctx = ctx;
    for (u32 p : preds) { red.rels[p].pred = p; red.rels[p].is_head = true; }
    for (u32 r = 0; r < n_rules; r++) {
        const kb_rule& rule = rules[r];
        const RulePlan& pl = plans[r];
        const u32 np = (u32)pl.prem.size();
        if (!pl.fires) continue;
        for (u32 c = 0; c < rule.n_conclusion; c++) {
            const kb_pattern& h = rule.conclusion[c];
            const PredRel& dr = del.rels[h.p.value];
            if (dr.n == 0) continue;
            std::unique_ptr<kb_rel> cur = head_view(dr, h);
            std::vector<bool> used(np, false);
            for (u32 step = 0; step < np && (!cur || cur->n); step++) {
                u32 j = np;  // next premise: the first one that shares a variable with the bindings so far (no cartesian products)
                for (u32 k = 0; k < np && j == np; k++)
                    if (!used[k] && cur && (cur->col_of((u32)pl.prem[k].s_var) >= 0 || cur->col_of((u32)pl.prem[k].o_var) >= 0)) j = k;
                for (u32 k = 0; k < np && j == np; k++) if (!used[k]) j = k;
                used[j] = true;
                const PredRel& pr = fx.rels[pl.prem[j].pred];
                KB_TRY(join_premise(ctx, cur, pl.prem[j], pr, pr.n, false, tr));
            }
            if (!cur || cur->n == 0) continue;
            Gate g;
            g.must = set_of(dr);
            g.must_slots = dr.set_slots;
            KB_TRY(derive_head(red, cur.get(), h, &rule, false, &g, tr, &derivations));
        }
    }
    {
        u64 n = 0;
        KB_TRY(flush_pending(red, &n));
        ms.rederived = n;
    }
    tr.mark(ctx, "maintain: rederive", ms.rederived);

    // ---- 5. insert: the seeds (rederived facts, then the facts of `add` the closure does not hold) take the seed path of
    // kb_datalog_fixpoint_seed, then semi-naive rounds (KB_NAIVE: the same closure, reached from the delta)
    {
        std::vector<std::unique_ptr<kb_rel>> views;
        std::vector<std::pair<u32, const kb_rel*>> seeds;
        for (u32 p : preds) {
            const PredRel& rr = red.rels[p];
            if (rr.n) {
                views.emplace_back();
                KB_TRY(make_view(ctx, rr, 0, rr.n, 0, 2, &views.back()));
                seeds.push_back({p, views.back().get()});
            }
            auto a = add_of.find(p);
            if (a != add_of.end()) seeds.push_back({p, a->second.get()});
        }
        u64 n = 0;
        KB_TRY(accept_seeds(fx, seeds, nullptr, tr, &n));
    }
    kb_fixpoint_stats ist{};
    KB_TRY(run_rounds(fx, rules, n_rules, plans, strategy == KB_SEMI_NAIVE_OLD_DELTA ? KB_SEMI_NAIVE_OLD_DELTA : KB_SEMI_NAIVE, ist, tr));
    ms.insert_rounds = ist.rounds;
    derivations += ist.derivations;
    ms.derivations = derivations;
    tr.mark(ctx, "maintain: insert", ist.inferred);

    // ---- the differences: I \ I' = over-deleted facts that did not come back (+ the inferred facts `add` made base facts, above);
    // I' \ I = removed base facts that are derivable now + the facts the rounds found that were never known
    for (u32 p : preds) {
        if (!head[p]) continue;
        const PredRel &r = fx.rels[p], &dr = del.rels[p];
        if (dr.n > d0n[p]) {
            Pairs gone;
            KB_TRY(select_pairs(ctx, dr.s.ptr + d0n[p], dr.o.ptr + d0n[p], dr.n - d0n[p], set_of(r), nullptr, r.set_slots, false, &gone));
            removed_parts.push_back({p, gone});
        }
        if (d0n[p]) {
            Pairs back;
            KB_TRY(select_pairs(ctx, dr.s.ptr, dr.o.ptr, d0n[p], set_of(r), nullptr, r.set_slots, true, &back));
            added_parts.push_back({p, back});
        }
        if (r.n > r.base_n) {
            Pairs fresh_inf;
            KB_TRY(select_pairs(ctx, r.s.ptr + r.base_n, r.o.ptr + r.base_n, r.n - r.base_n, set_of(dr), nullptr, dr.set_slots, false, &fresh_inf));
            added_parts.push_back({p, fresh_inf});
        }
    }
    KB_TRY(assemble(ctx, removed_parts, &out_removed));
    KB_TRY(assemble(ctx, added_parts, &out_added));
    ms.inferred_removed = out_removed->n;
    ms.inferred_added = out_added->n;

    // ---- 6. the new segments are built before the store changes: `add` as kb_store_append_device stores it, I' = the facts of the head
    // relations with no base count (when I did not change and is one segment, that segment stays)
    u32 n_inferred_segs = 0;
    u64 evicted_rows = 0;
    for (auto& sg : ctx->segs) {
        if (sg.tag == KB_TAG_INFERRED) n_inferred_segs++;
        if (evict.count(sg.tag)) evicted_rows += sg.n;
    }
    const bool rewrite = ms.inferred_removed || ms.inferred_added || n_inferred_segs > 1;
    Segment sa, si;
    if (add) {
        sa.tag = add_tag;
        sa.n = add->n;
        KB_TRY(alloc_col(ctx, sa.n, &sa.s));
        KB_TRY(alloc_col(ctx, sa.n, &sa.p));
        KB_TRY(alloc_col(ctx, sa.n, &sa.o));
        if (sa.n) {
            KB_CUDA(ctx, cudaMemcpyAsync(sa.s.ptr, add->cols[0].ptr, sa.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
            KB_CUDA(ctx, cudaMemcpyAsync(sa.p.ptr, add->cols[1].ptr, sa.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
            KB_CUDA(ctx, cudaMemcpyAsync(sa.o.ptr, add->cols[2].ptr, sa.n * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
            KB_TRY(segment_stats(ctx, &sa));
        }
    }
    if (rewrite) {
        std::vector<std::pair<u32, Pairs>> iparts;
        for (u32 p : preds) {
            if (!head[p]) continue;
            const PredRel& r = fx.rels[p];
            const BaseCount& b = base[p];
            Pairs inf;
            KB_TRY(select_pairs(ctx, r.s.ptr, r.o.ptr, r.n, static_cast<const u64*>(b.keys->p), static_cast<const u32*>(b.cnt->p), b.slots, false, &inf));
            iparts.push_back({p, inf});
        }
        std::unique_ptr<kb_rel> irel;
        KB_TRY(assemble(ctx, iparts, &irel));
        si.tag = KB_TAG_INFERRED;
        si.n = irel->n;
        si.s = irel->cols[0]; si.p = irel->cols[1]; si.o = irel->cols[2];
        if (si.n) KB_TRY(segment_stats(ctx, &si));
    }
    u64 live = ctx->n_triples - evicted_rows + (add ? add->n : 0);
    if (rewrite) {
        for (auto& sg : ctx->segs) if (sg.tag == KB_TAG_INFERRED) live -= sg.n;
        live += si.n;
    }
    if (live >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "store would exceed 2^32-16 triples");
    tr.mark(ctx, "maintain: segments built", si.n);

    // ---- rewrite the store, the index maintained in place (kb_store_evict / kb_store_append_device do the same). A failure from here on
    // leaves exactly the B' segments, no inferred segment, no kept state and no token: kb_datalog_fixpoint restores the precondition.
    auto drop_inferred = [&]() {
        store_evict_tag(ctx, KB_TAG_INFERRED, /*keep_index=*/false);
        ctx->closed.reset();
    };
    std::vector<u64> gone(evict.begin(), evict.end());
    if (rewrite) gone.push_back(KB_TAG_INFERRED);
    for (u64 t : gone) store_evict_tag(ctx, t, /*keep_index=*/true);
    if (add) {
        const kb_status rc = store_add_device_segment(ctx, sa);
        if (rc != KB_OK) { drop_inferred(); return rc; }
    }
    if (rewrite && si.n) {
        const kb_status rc = store_add_device_segment(ctx, si);
        if (rc != KB_OK) { drop_inferred(); return rc; }
    }
    ctx->fix_state.reset();
    cudaEventRecord(ev1, ctx->st);
    {
        const cudaError_t e = cudaStreamSynchronize(ctx->st);
        if (e != cudaSuccess) { drop_inferred(); return fail(ctx, KB_E_CUDA, "kb_datalog_maintain: %s", cudaGetErrorString(e)); }
    }
    timers_flush(ctx);
    float ms_dev = 0.f;
    cudaEventElapsedTime(&ms_dev, ev0, ev1);
    ms.device_ms = ms_dev;
    cl->store_version = ctx->store_version;
    cl->num_version = ctx->num_version;
    if (!state_off) {
        for (auto& kv : fx.rels) { kv.second.base_n = kv.second.seed_from = kv.second.delta_start = kv.second.snapshot = kv.second.n; }
        cl->rels = std::move(fx.rels);
        cl->base = std::move(base);
        cl->has_state = true;
    }
    tr.mark(ctx, "maintain: store rewritten");
    if (stats) *stats = ms;
    ctx->stats.rows_out = ms.inferred_added;
    if (inferred_removed) *inferred_removed = out_removed.release();
    if (inferred_added) *inferred_added = out_added.release();
    return KB_OK;
}

// Delete-and-rederive across a window slide (rsp_engine.rs:94-109 + simple_r2r.rs:103-128 without the closure from scratch)
extern "C" kb_status kb_datalog_maintain(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy, const uint64_t* evict_tags,
                                         uint32_t n_evict, const kb_rel* add, uint64_t add_tag, kb_rel** inferred_removed, kb_rel** inferred_added,
                                         kb_maintain_stats* stats) {
    KB_ENTER(ctx);
    if (inferred_removed) *inferred_removed = nullptr;
    if (inferred_added) *inferred_added = nullptr;
    return maintain_impl(ctx, rules, n_rules, strategy, evict_tags, n_evict, add, add_tag, inferred_removed, inferred_added, stats);
}
