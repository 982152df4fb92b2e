// kb_group.cuh — the device side of the GROUP BY hash table that the group kernels (kb_group.cu) and the index probe's fused GROUP BY
// (probe_index_kernel, kb_join.cu) both insert into.
#pragma once
#include "kb_kernels.cuh"

namespace kb {

static __device__ void atomic_min_f64(double* addr, double v) {
    unsigned long long* a = reinterpret_cast<unsigned long long*>(addr);
    unsigned long long old = *a;
    while (v < __longlong_as_double((long long)old) || __longlong_as_double((long long)old) != __longlong_as_double((long long)old)) {
        const unsigned long long assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)__double_as_longlong(v));
        if (old == assumed) break;
    }
}
static __device__ void atomic_max_f64(double* addr, double v) {
    unsigned long long* a = reinterpret_cast<unsigned long long*>(addr);
    unsigned long long old = *a;
    while (v > __longlong_as_double((long long)old) || __longlong_as_double((long long)old) != __longlong_as_double((long long)old)) {
        const unsigned long long assumed = old;
        old = atomicCAS(a, assumed, (unsigned long long)__double_as_longlong(v));
        if (old == assumed) break;
    }
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

static __device__ void group_update_global(const GroupParams& P, const u32* k, unsigned long long cnt, const double* val) {
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

}  // namespace kb
