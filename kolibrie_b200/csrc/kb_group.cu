// kb_group.cu — GROUP BY (execute_query.rs:1150-1227): the device group table, the kernels that fill, merge and compact it, and the
// entry points kb_group_aggregate, kb_star_join_aggregate, kb_groups_* and kb_groups_merge. The fused GROUP BY of the one-kernel
// index join (kb_join.cu) and the prepared grouped plans (kb_plan.cu) build, read and share their tables through the functions here.
#include <algorithm>

#include "kb_group.cuh"
#include "kb_internal.hpp"

namespace kb {

__global__ void group_init_kernel(const GroupParams P) {
    const u32 stride = gridDim.x * blockDim.x;
    if (P.overflow != nullptr && blockIdx.x == 0 && threadIdx.x == 0) *P.overflow = 0u;  // wherever the table keeps it (GroupTable)
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

// Two levels of pre-aggregation keep a GROUP BY with a handful of groups from serialising on a handful of addresses:
// (1) a warp folds its 32 rows per distinct group (__match_any_sync), (2) leaders accumulate into a 64-entry shared-memory
// table of the CTA, flushed to the global table once per CTA. Rows whose group does not fit the CTA table go straight to global.
constexpr int GROUP_SMEM = 64;

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
    const int grid = grid_1d(n, n_sms, 256, 4);
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
        int grid = grid_1d(p.n, n_sms, 1024);
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
    int grid = grid_1d(p.n, n_sms);
    group_kernel<<<grid, 256, 0, st>>>(p);
}

// ---- the table on the host side
GroupParams group_params(const kb_ctx* ctx, u32 n_group, const kb_agg* aggs, u32 n_aggs) {
    GroupParams P{};
    P.n_gcols = n_group;
    P.n_aggs = n_aggs;
    for (u32 a = 0; a < n_aggs; a++) P.akind[a] = aggs[a].kind;
    P.nt = numtab(ctx);
    return P;
}

kb_status check_group_spec(kb_ctx* ctx, const uint32_t* group_slots, u32 n_group, const kb_agg* aggs, u32 n_aggs) {
    if ((n_group && !group_slots) || (n_aggs && !aggs)) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_group == 0 || n_group > 4) return fail(ctx, KB_E_LIMIT, "GROUP BY takes 1..4 variables");
    if (n_aggs > 8) return fail(ctx, KB_E_LIMIT, "at most 8 aggregates");
    for (u32 a = 0; a < n_aggs; a++) if (aggs[a].kind > KB_AGG_AVG) return fail(ctx, KB_E_INVALID, "unknown aggregate kind %u", aggs[a].kind);
    return KB_OK;
}

void GroupTable::point(GroupParams* P, char* base) const {
    P->n_slots = (u32)slots;
    P->gval = (double*)(base + o_val);
    P->gcnt = (unsigned long long*)(base + o_cnt);
    P->gkeys = (u32*)(base + o_keys);
    P->gstate = (u32*)(base + o_state);
    P->overflow = ctrl ? ctrl : (u32*)(base + bytes);
}

kb_status group_table_create(kb_ctx* ctx, u64 slots, bool in_ctrl, GroupParams* P, GroupTable* t) {
    t->slots = slots;
    t->o_val = 0;
    t->o_cnt = t->o_val + slots * 8 * sizeof(double);
    t->o_keys = t->o_cnt + slots * sizeof(unsigned long long);
    t->o_state = t->o_keys + slots * 4 * sizeof(u32);
    t->bytes = t->o_state + slots * sizeof(u32);
    if (in_ctrl) {
        t->ctrl_off = ctrl_alloc(ctx, 4);
        t->ctrl = ctx->ctrl + t->ctrl_off;
    }
    KB_TRY(alloc_buf(ctx, t->bytes + (in_ctrl ? 0 : 16), &t->buf));
    t->point(P, static_cast<char*>(t->buf->p));
    launch_group_init(*P, ctx->st);  // (also zeroes the overflow word)
    return KB_OK;
}

kb_status group_table_collect(kb_ctx* ctx, const GroupTable& t, kb_groups* g, bool* overflowed) {
    KB_TRY(ctrl_read(ctx));
    *overflowed = ctx->h_ctrl[t.ctrl_off] != 0;
    if (*overflowed) return KB_OK;
    std::vector<char> big;  // tables past 32 MB (hundreds of thousands of groups) are not worth pinning
    void* dst = nullptr;
    if (t.bytes <= (32u << 20)) {
        if (ctx->pinned_bytes < t.bytes) {
            if (ctx->pinned) cudaFreeHost(ctx->pinned);
            ctx->pinned = nullptr; ctx->pinned_bytes = 0;
            KB_CUDA(ctx, cudaMallocHost(&ctx->pinned, t.bytes));
            ctx->pinned_bytes = t.bytes;
        }
        dst = ctx->pinned;
    } else {
        big.resize(t.bytes);
        dst = big.data();
    }
    KB_CUDA(ctx, cudaMemcpyAsync(dst, t.buf->p, t.bytes, cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += t.bytes;
    const char* hb = static_cast<const char*>(dst);
    const double* hval = (const double*)(hb + t.o_val);
    const unsigned long long* hcnt = (const unsigned long long*)(hb + t.o_cnt);
    const u32* hkeys = (const u32*)(hb + t.o_keys);
    const u32* hstate = (const u32*)(hb + t.o_state);
    for (u64 i = 0; i < t.slots; i++) if (hstate[i] == 2u) g->add(hkeys + i * 4, hcnt[i], hval + i * 8);
    return KB_OK;
}

static size_t group_peer_stride(const GroupTable& t) { return round256(t.bytes + 16); }
u64 group_peer_scratch_bytes(const GroupTable& t, u32 ring) { return 256 + (u64)ring * group_peer_stride(t); }
char* group_peer_table(char* scratch, const GroupTable& t, u32 ring_slot) { return scratch + 256 + (size_t)ring_slot * group_peer_stride(t); }

PeerTables group_peer_tables(const GroupTable& t, const std::vector<char*>& scratch, u32 rank, u32 ring_slot) {
    PeerTables T{};
    T.world = (u32)scratch.size(); T.rank = rank;
    T.n_slots = (u32)t.slots;
    T.o_val = (u32)t.o_val; T.o_cnt = (u32)t.o_cnt; T.o_keys = (u32)t.o_keys; T.o_state = (u32)t.o_state;
    T.o_overflow = (u32)t.bytes;
    for (u32 r = 0; r < T.world; r++) {
        T.flags[r] = reinterpret_cast<u32*>(scratch[r]);
        T.table[r] = group_peer_table(scratch[r], t, ring_slot);
    }
    return T;
}

}  // namespace kb

using namespace kb;

kb_groups::kb_groups(kb::u32 n_group, const kb_agg* aggs, kb::u32 n_aggs) : keys(n_group), vals(n_aggs), raw(n_aggs) {
    for (kb::u32 a = 0; a < n_aggs; a++) kinds.push_back(aggs[a].kind);
}

void kb_groups::add(const kb::u32* key, uint64_t count, const double* acc) {
    for (size_t c = 0; c < keys.size(); c++) keys[c].push_back(key[c]);
    counts.push_back(count);
    for (size_t a = 0; a < vals.size(); a++) {
        double v = acc[a];
        raw[a].push_back(v);
        if (kinds[a] == KB_AGG_AVG) v = v / (double)count;  // execute_query.rs:1216
        if (kinds[a] == KB_AGG_COUNT) v = (double)count;
        vals[a].push_back(v);
    }
}

extern "C" {

kb_status kb_group_aggregate(kb_ctx* ctx, const kb_rel* in, const uint32_t* group_slots, uint32_t n_group, const kb_agg* aggs, uint32_t n_aggs, kb_groups** out) {
    KB_ENTER(ctx);
    if (!in || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    KB_TRY(kb::check_group_spec(ctx, group_slots, n_group, aggs, n_aggs));
    if (in->n >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "relation too large");
    kb::GroupParams P = kb::group_params(ctx, n_group, aggs, n_aggs);
    for (u32 c = 0; c < n_group; c++) {
        int ci = in->col_of(group_slots[c]);
        if (ci < 0) return kb::fail(ctx, KB_E_INVALID, "GROUP BY slot %u is not a column", group_slots[c]);
        P.gcol[c] = in->cols[ci].ptr;
    }
    for (u32 a = 0; a < n_aggs; a++) {
        if (aggs[a].kind == KB_AGG_COUNT) continue;
        int ci = in->col_of(aggs[a].slot);
        if (ci < 0) return kb::fail(ctx, KB_E_INVALID, "aggregate slot %u is not a column", aggs[a].slot);
        P.acol[a] = in->cols[ci].ptr;
    }
    P.n = (u32)in->n;
    auto g = std::make_unique<kb_groups>(n_group, aggs, n_aggs);
    if (in->n == 0) { *out = g.release(); return KB_OK; }
    u64 slots = 1u << 12;  // small first try: the table is downloaded whole; overflow -> 16x larger and rerun
    for (;;) {
        kb::GroupTable tab;
        KB_TRY(kb::group_table_create(ctx, slots, true, &P, &tab));
        kb::timer_begin(ctx, kb::F_GROUP, 2);
        kb::launch_group(P, ctx->n_sms, ctx->st);
        kb::timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        bool overflowed;
        KB_TRY(kb::group_table_collect(ctx, tab, g.get(), &overflowed));
        if (!overflowed) break;
        if (slots >= 2 * in->n && slots >= (1u << 20)) return kb::fail(ctx, KB_E_LIMIT, "group table overflow");
        slots = std::min<u64>(slots * 16, 1ull << 30);
    }
    *out = g.release();
    return KB_OK;
}
kb_status kb_groups_info(const kb_groups* g, uint64_t* n_groups, uint32_t* n_group_cols, uint32_t* n_aggs) {
    if (!g) return KB_E_INVALID;
    if (n_groups) *n_groups = g->counts.size();
    if (n_group_cols) *n_group_cols = (uint32_t)g->keys.size();
    if (n_aggs) *n_aggs = (uint32_t)g->vals.size();
    return KB_OK;
}
kb_status kb_groups_keys(const kb_groups* g, uint32_t col, const uint32_t** keys) {
    if (!g || !keys || col >= g->keys.size()) return KB_E_INVALID;
    *keys = g->keys[col].data();
    return KB_OK;
}
kb_status kb_groups_values(const kb_groups* g, uint32_t agg, const double** values) {
    if (!g || !values || agg >= g->vals.size()) return KB_E_INVALID;
    *values = g->vals[agg].data();
    return KB_OK;
}
kb_status kb_groups_counts(const kb_groups* g, const uint64_t** counts) {
    if (!g || !counts) return KB_E_INVALID;
    *counts = g->counts.data();
    return KB_OK;
}
void kb_groups_free(kb_groups* g) { delete g; }

// ---- partial GROUP BY results across ranks (SURVEY.md 8e): pack on every rank, gather, merge on the device
namespace {
struct GroupsHeader {
    uint64_t magic, n_groups;
    uint32_t n_group_cols, n_aggs;
    uint32_t kinds[8];
};
static_assert(sizeof(GroupsHeader) == 56, "layout");
constexpr uint64_t GROUPS_MAGIC = 0x4B4247524F555031ull;  // "KBGROUP1"
}  // namespace

kb_status kb_groups_pack(const kb_groups* g, void* dst, uint64_t capacity_bytes, uint64_t* bytes) {
    if (!g || !bytes) return KB_E_INVALID;
    const uint64_t n = g->counts.size();
    const uint64_t need = sizeof(GroupsHeader) + n * sizeof(kb::GroupRecord);
    *bytes = need;
    if (!dst) return KB_OK;  // size query
    if (capacity_bytes < need) return KB_E_LIMIT;
    if (g->keys.size() > 4 || g->vals.size() > 8 || g->raw.size() != g->vals.size() || g->kinds.size() != g->vals.size()) return KB_E_INVALID;
    GroupsHeader h{};
    h.magic = GROUPS_MAGIC;
    h.n_groups = n;
    h.n_group_cols = (uint32_t)g->keys.size();
    h.n_aggs = (uint32_t)g->vals.size();
    for (size_t a = 0; a < g->kinds.size(); a++) h.kinds[a] = g->kinds[a];
    memcpy(dst, &h, sizeof h);
    auto* rec = reinterpret_cast<kb::GroupRecord*>(static_cast<char*>(dst) + sizeof h);
    for (uint64_t i = 0; i < n; i++) {
        kb::GroupRecord r{};
        for (size_t c = 0; c < g->keys.size(); c++) r.keys[c] = g->keys[c][i];
        r.count = g->counts[i];
        for (size_t a = 0; a < g->raw.size(); a++) r.raw[a] = g->raw[a][i];
        memcpy(rec + i, &r, sizeof r);
    }
    return KB_OK;
}

kb_status kb_groups_merge(kb_ctx* ctx, const void* const* parts, const uint64_t* part_bytes, uint32_t n_parts, kb_groups** out) {
    KB_ENTER(ctx);
    if (!parts || !part_bytes || !out || n_parts == 0) return kb::fail(ctx, KB_E_INVALID, "NULL or empty argument");
    GroupsHeader h0{};
    uint64_t total = 0;
    for (u32 i = 0; i < n_parts; i++) {
        if (!parts[i] || part_bytes[i] < sizeof(GroupsHeader)) return kb::fail(ctx, KB_E_INVALID, "partial %u is truncated", i);
        GroupsHeader h;
        memcpy(&h, parts[i], sizeof h);
        if (h.magic != GROUPS_MAGIC) return kb::fail(ctx, KB_E_INVALID, "partial %u is not a kb_groups_pack buffer", i);
        if (part_bytes[i] < sizeof h + h.n_groups * sizeof(kb::GroupRecord)) return kb::fail(ctx, KB_E_INVALID, "partial %u is truncated", i);
        if (i == 0) h0 = h;
        else if (h.n_group_cols != h0.n_group_cols || h.n_aggs != h0.n_aggs || memcmp(h.kinds, h0.kinds, sizeof h.kinds) != 0)
            return kb::fail(ctx, KB_E_INVALID, "partial %u was produced by a different GROUP BY (columns / aggregates differ)", i);
        total += h.n_groups;
    }
    if (h0.n_group_cols == 0 || h0.n_group_cols > 4 || h0.n_aggs > 8) return kb::fail(ctx, KB_E_INVALID, "bad header");
    if (total >= (1ull << 30)) return kb::fail(ctx, KB_E_LIMIT, "too many partial groups");
    std::vector<kb_agg> aggs(h0.n_aggs);
    for (u32 a = 0; a < h0.n_aggs; a++) { aggs[a].kind = h0.kinds[a]; aggs[a].slot = 0; }
    auto g = std::make_unique<kb_groups>(h0.n_group_cols, aggs.data(), h0.n_aggs);
    if (total == 0) {
        *out = g.release();
        return KB_OK;
    }
    // partial records -> device, merged by find-or-insert into a group table sized for the worst case (every partial group distinct)
    kb::Buf recs;
    KB_TRY(kb::alloc_buf(ctx, total * sizeof(kb::GroupRecord), &recs));
    uint64_t at = 0;
    for (u32 i = 0; i < n_parts; i++) {
        GroupsHeader h;
        memcpy(&h, parts[i], sizeof h);
        if (h.n_groups == 0) continue;
        KB_CUDA(ctx, cudaMemcpyAsync(static_cast<kb::GroupRecord*>(recs->p) + at, static_cast<const char*>(parts[i]) + sizeof h, h.n_groups * sizeof(kb::GroupRecord),
                                     cudaMemcpyHostToDevice, ctx->st));
        at += h.n_groups;
    }
    ctx->stats.h2d_bytes += total * sizeof(kb::GroupRecord);
    kb::GroupParams P = kb::group_params(ctx, h0.n_group_cols, aggs.data(), h0.n_aggs);
    kb::GroupTable tab;
    KB_TRY(kb::group_table_create(ctx, kb::pow2_at_least(std::max<u64>(2 * total, 1024)), true, &P, &tab));
    kb::timer_begin(ctx, kb::F_GROUP);
    kb::launch_group_merge(P, static_cast<const kb::GroupRecord*>(recs->p), (u32)total, ctx->n_sms, ctx->st);
    kb::timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    bool overflowed;
    KB_TRY(kb::group_table_collect(ctx, tab, g.get(), &overflowed));
    if (overflowed) return kb::fail(ctx, KB_E_LIMIT, "group table overflow while merging partials");
    *out = g.release();
    return KB_OK;
}

kb_status kb_star_join_aggregate(kb_ctx* ctx, uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter, uint32_t n_ops,
                                 const uint32_t* group_slots, uint32_t n_group, const kb_agg* aggs, uint32_t n_aggs, kb_groups** out, uint64_t* n_rows) {
    KB_ENTER(ctx);
    if (!pats || !out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    KB_TRY(kb::check_group_spec(ctx, group_slots, n_group, aggs, n_aggs));
    const bool fusable = n_group == 1 && n_aggs <= 1;
    kb::AggSpec spec(group_slots[0], n_aggs ? aggs : nullptr);
    std::unique_ptr<kb_rel> rel;
    KB_TRY(kb::star_join_impl(ctx, join_slot, pats, n_pats, filter, n_ops, &rel, fusable ? &spec : nullptr));
    if (spec.applied) {
        if (n_rows) *n_rows = spec.n_rows;
        *out = spec.groups.release();
        return KB_OK;
    }
    if (n_rows) *n_rows = rel->n;
    return kb_group_aggregate(ctx, rel.get(), group_slots, n_group, aggs, n_aggs, out);
}

}  // extern "C"
