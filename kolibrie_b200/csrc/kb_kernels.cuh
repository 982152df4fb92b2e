// kb_kernels.cuh — what more than one file shares on the device side: the compaction state every compacting launch hands
// tile_prefix_2level, the direct-table layout that kb_join.cu's probes read and both kb_join.cu and kb_store.cu build, the index
// probe's launch format (a prepared plan, kb_plan.cu, holds and launches one), the GROUP BY declarations (kb_group.cu), the key sets and
// demand patterns of Datalog, backward chaining, repairs and the store, the quoted-triple and dictionary views, and the launchers of
// kb_kernels.cu. A kernel with one calling file keeps its launch format and launcher in that file.
#pragma once
#include "kb_device.cuh"

namespace kb {

static inline u64 umin64(u64 a, u64 b) { return a < b ? a : b; }
// grid-stride utility kernels are capped at a few CTAs per SM of an H100; the persistent kernels size their grids from the device's count
constexpr u64 H100_SMS = 132;

// what a compacting launch hands tile_prefix_2level (kb_device.cuh): the look-back state, the order mode, the launch's epoch, and the
// control words {ticket, total, zero} (set by compact_setup, kb_join.cu)
struct Compact {
    u64* tile_state;   // level 1: [n_tiles][MAXP]
    u64* block_state;  // level 2: [ceil(n_tiles/32)][MAXP]
    u32 ordered;       // 1: output in input order (two-level prefix)  0: tile completion order (atomic cursor)
    u64 epoch;
    u32* ticket;
    u32* total;            // result row count; must be zero at launch
    const u32* zero_word;  // a word that stays zero (ordered mode reads its base from here)
};

// ---------------------------------------------------------------------------------------------------------------
// Direct tables: dense dictionary ids make the identity a perfect hash: table[key - kmin] = payload (u32, EMPTY32 = none).
// The build from an interleaved (subject, object) pair relation; key_is_y selects which half is the key, the other is the payload
// trusted=1: the (predicate, key position) is known single-valued for this store version -> plain stores, no read-modify-write
void launch_build_direct_pairs(const uint2* kv, u32 key_is_y, u32 n, u32* table, u32 kmin, u32 range, u32 cshift, u32* dup_flag, u32 trusted,
                               int n_sms, cudaStream_t st);

constexpr int MAXT = 4;  // direct tables one probe reads

constexpr u32 CODE_MAX = 255;  // objects a subject table may hold to be coded in one byte per slot (code 0xFF: no object)
struct DirectTab {
    const u32* tab;
    u32 kmin, range;  // in compacted key space when cshift != 0
    u32 cshift;
    u32 mode;  // 0: payload is a value column  1: payload is a build-row index (gather pay[])  2: existence only
    u32 n_pay;
    const u32* pay[2];
    // non-null: the table's one-byte codes (PredSlice::xcode), which probe_index_kernel reads instead of tab: code[slot] indexes dict
    // (n_dict <= CODE_MAX object ids), 0xFF where tab holds EMPTY32. The other kernels read tab.
    const u8* code;
    const u32* dict;
    u32 n_dict;
};

// K_probe (INDEX): the star join over the store index when every non-probe pattern has a persistent per-predicate table. The probe
// rows are one predicate slice (x = subject, y = object) and, when the pattern carries FILTER(?y <cmp> c), the slice's typed literal
// column; both are TMA-staged into shared memory by the same mbarrier, so the FILTER is resolved BEFORE any table lookup is issued.
// Output layout is fixed: column 0 = x, 1 = y, 2+t = value found in table t. The launch owns a 4-word control block
// {ticket, total, zero, done} that the last CTA to finish resets to zero after publishing the row count to pinned host memory: a
// query is ONE device operation (no memset before, no copy after).
constexpr int PROBEI_MAXSEG = 16;  // chunks of the probe slice one launch can walk (one per store segment: an RSP window of slides)
struct ProbeISeg {
    const uint2* pairs;
    const double* ynum;  // typed literal column of the chunk (non-null iff pre_mode == 1)
    u32 n, tile0;        // rows; first tile of this chunk in the launch's tile numbering
};
struct ProbeIParams {
    ProbeISeg seg[PROBEI_MAXSEG];
    u32 n_seg;
    // table mode (ptab != nullptr): the probe stream is the probe pattern's own persistent table, slot by slot (keys ascending), and
    // pkey the rank of the numeric value of the slot's other half in the value order of the numeric side table (pre_mode == 1: the
    // FILTER is `rank in [key_lo, key_hi)`, kb_numrank.cuh); keys are rebuilt from the slot number (ptab_min + slot, then the inverse
    // of the shard compaction)
    const u32* ptab;
    const u16* pkey;
    u32 key_lo, key_hi, key_shift;  // stored ranks [key_lo, key_hi] pass; key_shift != 0: the two ends are decided on the value
    u32 ptab_min, ptab_range, ptab_cshift, shard_rank;
    u32 key_is_y, n, n_tiles, T;  // n = rows over all chunks
    DirectTab tab[MAXT];
    u32* out[2 + MAXT];
    u32 cap;
    u32 pre_mode;  // 0: none, 1: cmp_num(pre_cmp, ynum[row], pre_val), 2: pre_ops over (x, y)
    u32 pre_cmp;
    double pre_val;
    FilterOp pre_ops[8];
    u32 n_pre;
    FilterOp ops[KB_MAX_FILTER_OPS];  // conjuncts that need a looked-up value: evaluated over the output row
    u32 n_ops;
    NumTab nt;
    Compact c;  // {ticket, total, zero} = cb[0..2]
    u32 gsel, asel, akind;  // fused GROUP BY (launch_probe_index with `agg`): output column of the key / of the aggregated value, kb_agg kind
    u32* cb;          // device control block: [0] ticket, [1] total, [2] always 0, [3] CTAs done
    u32* host_total;  // mapped pinned host word
};
struct GroupParams;
// agg == nullptr: the joined rows are written to p.out; else they are folded into the group table *agg (GROUP BY column p.gsel)
void launch_probe_index(const ProbeIParams& p, const GroupParams* agg, int n_sms, cudaStream_t st);

// in-place exclusive prefix sum of a[0..n) (n >= 1); scratch holds ceil(n / 2048) + 1 words
void launch_exclusive_scan_u32(u32* a, u32 n, u32* scratch, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------------------
// K_group: hash aggregate (execute_query.rs:1150-1227)
struct GroupParams {
    const u32* gcol[4];
    u32 n_gcols;
    const u32* acol[8];  // null for COUNT
    u32 akind[8];
    u32 n_aggs;
    u32 n;
    NumTab nt;
    // global group table
    u32 n_slots;   // power of two
    u32* gkeys;    // [n_slots][4] (EMPTY32 in [.,0] lane = free is tracked by gstate)
    u32* gstate;   // [n_slots] 0 free, 1 being written, 2 ready
    double* gval;  // [n_slots][8]
    unsigned long long* gcnt;  // [n_slots]
    u32* overflow;
};
void launch_group(const GroupParams& p, int n_sms, cudaStream_t st);
void launch_group_init(const GroupParams& p, cudaStream_t st);
// one partial group of a GROUP BY evaluated elsewhere (another rank): its key, its row count and the raw accumulators (AVG: the sum)
struct GroupRecord {
    u32 keys[4];
    unsigned long long count;
    double raw[8];
};
static_assert(sizeof(GroupRecord) == 88, "layout");
// folds n partial groups into the global table of p: counts add, SUM/AVG accumulators add, MIN/MAX fold (execute_query.rs:1150-1227
// applied to the union of the partials' rows)
void launch_group_merge(const GroupParams& p, const GroupRecord* recs, u32 n, int n_sms, cudaStream_t st);
// Cross-rank GROUP BY without a host round trip (one process per GPU, partial tables in peer-mapped memory):
//   launch_peer_barrier: rank `rank` stores `epoch` into slot [rank] of every peer's flag array (system-scope release) and waits until
//                        every slot of its OWN flag array has reached `epoch` (acquire): all ranks' earlier kernels are then visible
//   launch_group_merge_peers: folds the `world` partial group tables (layout of GroupTable: val | cnt | keys | state, then the overflow
//                        word) — read straight from the peers' memory over NVLink — into the local table of p
struct PeerTables {
    const char* table[64];   // device-visible address of rank r's partial table
    u32* flags[64];          // device-visible address of rank r's flag array [64]
    u32 world, rank;
    u32 n_slots;             // slots per partial table
    u32 o_val, o_cnt, o_keys, o_state, o_overflow;  // byte offsets inside a partial table
};
// the occupied slots of p's table as a dense GroupRecord list: out[0 .. *count), header[0] = count, header[1] = the table's overflow
// word. `out` / `header` may be mapped pinned host memory: a prepared query then needs no device-to-host copy of the sparse table
void launch_group_compact(const GroupParams& p, GroupRecord* out, u32* header, u32 cap, cudaStream_t st);
void launch_peer_barrier(const PeerTables& t, u32 epoch, cudaStream_t st);
void launch_group_merge_peers(const GroupParams& p, const PeerTables& t, int n_sms, cudaStream_t st);

// ---- key sets (device side): the Datalog launches (kb_datalog.cu), the answer pass of kb_backward.cu, the store (kb_store.cu) and
// kb_repairs.cu read them
// 96-bit (s,p,o) keys in 16-byte slots {s,p,o,state}
__device__ __forceinline__ u32 set_hash(u32 s, u32 p, u32 o) { return mix32(mix32(s) * 0x9E3779B1u ^ mix32(o + 0x632BE5ABu) ^ (p * 0x85EBCA77u)); }

// returns 1 if (s,p,o) was inserted now, 0 if it was already there, 2 on overflow; *at = the key's slot (1 and 0)
__device__ __forceinline__ u32 set_insert_at(uint4* set, u32 n_slots, u32 s, u32 p, u32 o, u32* at) {
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
            *at = slot;
            return 1u;
        }
        while (st == 1u) st = *reinterpret_cast<volatile u32*>(st_ptr);
        __threadfence();
        const volatile u32* w = reinterpret_cast<const volatile u32*>(&set[slot]);
        if (w[0] == s && w[1] == p && w[2] == o) { *at = slot; return 0u; }
        slot = (slot + 1u) & mask;
    }
    return 2u;
}
__device__ __forceinline__ u32 set_insert(uint4* set, u32 n_slots, u32 s, u32 p, u32 o) {
    u32 at;
    return set_insert_at(set, n_slots, s, p, o, &at);
}
// slot of (s,p,o) in a 96-bit set, EMPTY32 when absent (the set is not written by the same launch)
__device__ __forceinline__ u32 set_find(const uint4* set, u32 n_slots, u32 s, u32 p, u32 o) {
    const u32 mask = n_slots - 1u;
    u32 slot = set_hash(s, p, o) & mask;
    for (u32 probes = 0; probes < n_slots; probes++) {
        const uint4 w = set[slot];
        if (w.w == 0u) return EMPTY32;
        if (w.x == s && w.y == p && w.z == o) return slot;
        slot = (slot + 1u) & mask;
    }
    return EMPTY32;
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

// slot of (s,o) in a 64-bit set, EMPTY32 when absent (the set is not written by the same launch)
__device__ __forceinline__ u32 set64_find(const u64* set, u32 n_slots, u32 s, u32 o) {
    const u64 key = ((u64)s << 32) | (u64)o;
    const u32 mask = n_slots - 1u;
    u32 slot = mix32(mix32(s) * 0x9E3779B1u ^ mix32(o + 0x632BE5ABu)) & mask;
    for (u32 probes = 0; probes < n_slots; probes++) {
        const u64 cur = set[slot];
        if (cur == key) return slot;
        if (cur == EMPTY64) return EMPTY32;
        slot = (slot + 1u) & mask;
    }
    return EMPTY32;
}

// ---- demand patterns and compaction, shared by kb_datalog.cu and kb_backward.cu
// whether (s,o) matches one of n demand patterns (x = subject, y = object, KB_ID_NONE = any)
__device__ __forceinline__ bool bc_demanded(const uint2* dem, u32 n, u32 s, u32 o) {
    for (u32 k = 0; k < n; k++) {
        const uint2 d = dem[k];
        if ((d.x == 0xFFFFFFFFu || d.x == s) && (d.y == 0xFFFFFFFFu || d.y == o)) return true;
    }
    return false;
}
// warp-aggregated append of (s,o) for the lanes that `take` it, at *out_count (every lane of the warp calls it)
__device__ __forceinline__ void emit_pair(bool take, u32 s, u32 o, u32* out_s, u32* out_o, u32* out_count) {
    const int lane = threadIdx.x & 31;
    const unsigned b = __ballot_sync(0xffffffffu, take);
    if (!b) return;
    u32 basepos = 0;
    if (lane == __ffs(b) - 1) basepos = atomicAdd(out_count, (u32)__popc(b));
    basepos = __shfl_sync(0xffffffffu, basepos, __ffs(b) - 1);
    if (take) {
        const u32 r = basepos + (u32)__popc(b & ((1u << lane) - 1u));
        out_s[r] = s;
        out_o[r] = o;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// The quoted-triple table (kb_quoted.cu): entry id & 0x7FFFFFFF -> (s, p, o); an empty slot holds EMPTY32 in all three columns.
// n == 0: no table.
struct QuotedTab {
    const u32 *s, *p, *o;
    u32 n;
};
// The device dictionary (kb_dict.cu): string of id i = bytes[off[i] .. off[i + 1]) for i < ids. ids == 0: no dictionary (null pointers).
struct DictTab {
    const unsigned long long* off;
    const unsigned char* bytes;
    u32 ids;
};
// a BIND write pass (kb_bind.cu, kb_quoted.cu): *n_unbound += the rows of the warp left unbound (every lane of the warp calls it)
__device__ __forceinline__ void bind_count_unbound(bool unbound, unsigned long long* n_unbound) {
    const unsigned b = __ballot_sync(0xffffffffu, unbound);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_unbound, (unsigned long long)__popc(b));
}

// ---------------------------------------------------------------------------------------------------------------
// small utilities
void launch_fill_u32(u32* p, u32 v, u64 n, cudaStream_t st);
void launch_col_minmax(const u32* col, u32 n, u32* out_min, u32* out_max, int n_sms, cudaStream_t st);

}  // namespace kb
