// kb_tagtab.cuh — the open-addressing table of the batch encodes (kb_dict_encode's strings, kb_bind TRIPLE's quoted triples): one u64
// per slot, (hash tag in the high 32 bits) | payload in the low 32, all ones when empty, linear probing from h & mask. The table holds
// no keys: a tag match is confirmed by the caller's `eq(payload)`, which compares the key the payload names (an id of the persistent
// index, a position of the batch) with the probed one. Each caller keeps its own hash; only the high 32 bits of it are stored.
#pragma once
#include "kb_device.cuh"

namespace kb {

constexpr u64 TAG_EMPTY = 0xFFFFFFFFFFFFFFFFull;
__host__ __device__ __forceinline__ u64 tag_entry(u64 h, u32 payload) { return (h & 0xFFFFFFFF00000000ull) | payload; }

// the payload of the entry whose key equals the probed one, else EMPTY32 (a read-only probe of a table no one writes concurrently)
template <class Eq>
__device__ __forceinline__ u32 tag_find(const u64* tab, u64 mask, u64 h, Eq eq) {
    for (u64 slot = h & mask, probes = 0; probes <= mask; probes++, slot = (slot + 1) & mask) {
        const u64 e = tab[slot];
        if (e == TAG_EMPTY) break;
        if ((e >> 32) != (h >> 32)) continue;
        if (eq((u32)e)) return (u32)e;
    }
    return EMPTY32;
}

// the key enters the table with payload `pos`: a CAS claims an empty slot, and on a slot that holds an equal key atomicMin keeps the
// smaller payload (same tag: the minimum is over the payload; whatever payload a concurrent writer leaves names the same key). *slot is
// the key's slot; false when the table is full.
template <class Eq>
__device__ __forceinline__ bool tag_claim_min(u64* tab, u64 mask, u64 h, u32 pos, Eq eq, u32* slot_out) {
    for (u64 slot = h & mask, probes = 0; probes <= mask; probes++, slot = (slot + 1) & mask) {
        u64 e = *reinterpret_cast<volatile u64*>(&tab[slot]);
        if (e == TAG_EMPTY) {
            e = atomicCAS(reinterpret_cast<unsigned long long*>(&tab[slot]), TAG_EMPTY, tag_entry(h, pos));
            if (e == TAG_EMPTY) { *slot_out = (u32)slot; return true; }
        }
        if ((e >> 32) != (h >> 32)) continue;
        if (eq((u32)e)) {
            atomicMin(reinterpret_cast<unsigned long long*>(&tab[slot]), tag_entry(h, pos));
            *slot_out = (u32)slot;
            return true;
        }
    }
    return false;
}

}  // namespace kb
