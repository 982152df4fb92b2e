// kb_kernels.cuh — parameter blocks and launch wrappers of the shared sm_90a kernels (definitions in kb_kernels.cu), and the device
// functions more than one file's kernels read (the key sets, demand patterns, emit_pair). Kernels with a single owner keep their launch
// formats in that file: the Datalog ones in kb_datalog.cu, the backward-chaining ones in kb_backward.cu.
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
// K_build
// DIRECT: dense dictionary ids make the identity a perfect hash: table[key - kmin] = payload (u32, EMPTY32 = none).
void launch_build_direct(const u32* keys, const u32* vals /*null: row index*/, u32 n, u32* table, u32 kmin, u32 range, u32 cshift,
                         u32* dup_flag, int n_sms, cudaStream_t st);
// same from an interleaved (subject, object) pair relation; key_is_y selects which half is the key, the other is the payload
// trusted=1: the (predicate, key position) is known single-valued for this store version -> plain stores, no read-modify-write
void launch_build_direct_pairs(const uint2* kv, u32 key_is_y, u32 n, u32* table, u32 kmin, u32 range, u32 cshift, u32* dup_flag, u32 trusted,
                               int n_sms, cudaStream_t st);
// CHAINED multimap: open-addressing slots {key tag, head row} + next[] chains. Insert cost is O(1) whatever the key
// multiplicity (1:N joins and heavy hitters of the Datalog joins).
struct ChainTab {
    u64* slots;   // lo 32: key tag (EMPTY32 free), hi 32: head row index (EMPTY32 = end)
    u32 n_slots;  // power of two
    u32* next;    // [n_build]
    u32 n_keys;   // 1..4 key columns; tag = key itself when n_keys==1 else a 32-bit mix of all
    const u32* bkey[4];
};
void launch_build_chained(const ChainTab& t, u32 n, int n_sms, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------------------
// K_probe (direct, fused multiway): one probe stream against T<=4 direct tables + FILTER + ordered compaction.
// Replaces execute_star_join_with_ids (engine.rs:587-691) / bind-join chains (engine.rs:840-885) on unique keys.
constexpr int PROBE_THREADS = 256;
constexpr int PROBE_ITEMS = 4;
constexpr int PROBE_TILE = PROBE_THREADS * PROBE_ITEMS;  // 1024 rows
constexpr int MAXT = 4;

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
void launch_probe_direct(const ProbeDParams& p, int n_sms, cudaStream_t st);

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
void launch_probe_fast(const ProbeFParams& p, int n_sms, cudaStream_t st);

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
void launch_build_direct_pairs_filtered(const BuildPairsParams& p, int n_sms, cudaStream_t st);
// distinct values of a column other than EMPTY32 into a small open-addressing set (EMPTY32 = free). ctrl = {overflow, count}, both 0
// at launch: the overflow word is set when the set fills up or when a value past the first `limit` arrives, and ends the pass
void launch_distinct(const u32* col, u32 n, u32* set, u32 set_slots, u32 limit, u32* ctrl, int n_sms, cudaStream_t st);
// code[i] = index of tab[i] in dict (ascending, every value of tab but EMPTY32, n_dict <= CODE_MAX), 0xFF where tab[i] is EMPTY32, for
// i < range; tab and code start 16-byte aligned and may be read / written up to the next multiple of 4 slots
void launch_tab_code(const u32* tab, u32 range, const u32* dict, u32 n_dict, u8* code, int n_sms, cudaStream_t st);

// ---- window-slide maintenance of the store index: ONE pass profiles a new segment (column ranges, foreign subjects, its distinct
// predicates with their row counts), ONE pass splits it into the predicate slices' new chunks — pairs, id ranges, typed literal
// column, in-place inserts into the persistent tables — and ONE pass clears an evicted segment's keys from all of its slices' tables.
constexpr u32 SEGP_SLOTS = 32;  // open-addressing slots for a segment's distinct predicates (more than that: the batched scan path)
// control words of segment_profile: [0..2] min s/p/o, [3] unused, [4 .. 4+SLOTS) predicate slots (all 0xFF at launch);
// then (all 0 at launch) [P_MAX .. +3) max s/p/o, P_FOREIGN, P_OVERFLOW, [P_COUNT .. +SLOTS) rows per slot
constexpr u32 SEGP_MIN = 0, SEGP_SLOT = 4, SEGP_MAX = 4 + SEGP_SLOTS, SEGP_FOREIGN = SEGP_MAX + 3, SEGP_OVERFLOW = SEGP_MAX + 4, SEGP_COUNT = SEGP_MAX + 8,
              SEGP_WORDS = SEGP_COUNT + SEGP_SLOTS;
void launch_segment_profile(const u32* s, const u32* p, const u32* o, u32 n, u32 rank, u32 world, u32* ctrl, int n_sms, cudaStream_t st);

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
void launch_segment_split(const SplitParams& p, int n_sms, cudaStream_t st);

constexpr u32 CLEAR_MAX = 16;
struct ClearEntry {
    const uint2* pairs; u32 n;
    u32* xtab; u32 xtab_min, xtab_range, cshift;
    u32* ytab; u32 ytab_min, ytab_range;
};
struct ClearParams { ClearEntry e[CLEAR_MAX]; u32 k; };
void launch_clear_chunks(const ClearParams& p, int n_sms, cudaStream_t st);
// min/max of both halves of a pair relation: out[0..3] = min x, min y, max x, max y
// typed literal column of a predicate slice: out[i] = num_or0[kv[i].y]; *n_numeric += rows whose object is numeric
void launch_pair_numcol(const uint2* kv, u32 n, NumTab nt, double* out, u32* n_numeric, int n_sms, cudaStream_t st);
// the ranks of those values in the value order numv[0 .. n_numv) (kb_numrank.cuh), laid out like the subject-keyed direct table:
// out[compact(subject) - kmin] = rank_of(num_of(object))
void launch_pair_ranktab(const uint2* kv, u32 n, NumTab nt, const double* numv, u32 n_numv, u16* out, u32 kmin, u32 range, u32 cshift, int n_sms,
                         cudaStream_t st);
// the value order of the numeric side table: keys[i] = order-preserving u64 of fold(num_or0[i]) for i < n, of 0.0 for i == n and for NaN
void launch_numorder_keys(const double* num_or0, u32 n, unsigned long long* keys, int n_sms, cudaStream_t st);
// the inverse, over the sorted distinct keys
void launch_numorder_values(const unsigned long long* keys, u32 n, double* out, int n_sms, cudaStream_t st);
void launch_pair_minmax(const uint2* kv, u32 n, u32* out4, int n_sms, cudaStream_t st);
// number of occupied (non-EMPTY32) slots of a direct table: equals the number of inserted rows iff the keys were single-valued
void launch_count_nonempty(const u32* table, u32 n, u32* out_count, int n_sms, cudaStream_t st);
// number of keys that do NOT belong to shard `rank` of `world` (kb_shard_of): 0 for a correctly sharded column
void launch_count_foreign(const u32* col, u32 n, u32 rank, u32 world, u32* out, int n_sms, cudaStream_t st);
void launch_col_minmax(const u32* col, u32 n, u32* out_min, u32* out_max, int n_sms, cudaStream_t st);

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
void launch_probe_chained(const ProbeCParams& p, int n_sms, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------------------
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
void launch_csr_count(const u32* keys, u32 n, u32 kmin, u32* counts, int n_sms, cudaStream_t st);
// in-place exclusive prefix sum of a[0..n) (n >= 1); scratch holds ceil(n / 2048) + 1 words
void launch_exclusive_scan_u32(u32* a, u32 n, u32* scratch, cudaStream_t st);
void launch_csr_fill(const u32* keys, u32 n, u32 kmin, u32* cursor, const u32* const* pay_in, u32* const* pay_out, u32 n_pay, int n_sms, cudaStream_t st);
void launch_csr_total(const u32* pkeys, u32 n, const CsrTab& tab, unsigned long long* total, int n_sms, cudaStream_t st);
// the same directory built from an interleaved (subject, object) slice of the store index: key = one half, payload = the other half
void launch_csr_count_pairs(const uint2* kv, u32 key_is_y, u32 n, u32 kmin, u32* counts, int n_sms, cudaStream_t st);
void launch_csr_fill_pairs(const uint2* kv, u32 key_is_y, u32 n, u32 kmin, u32* cursor, u32* val_out, int n_sms, cudaStream_t st);
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
void launch_probe_grouped(const ProbeGParams& p, int n_sms, cudaStream_t st);

// cartesian product (engine.rs:1054-1071) — small inputs only
void launch_cartesian(const u32* const* lcols, u32 nl, u32 n_lcols, const u32* const* rcols, u32 nr, u32 n_rcols, u32* const* out,
                      cudaStream_t st);

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
// the store's batch insert into a 96-bit set (kb_store.cu)
void launch_set_insert(uint4* set, u32 set_slots, const u32* s, const u32* p /*null: p_const*/, u32 p_const, const u32* o, u32 n, u32* overflow,
                       int n_sms, cudaStream_t st);

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

// fused partition + transfer of the multi-GPU join-key shuffle: a tile of rows is sorted by destination rank d = shard_of(key, n_parts)
// in shared memory, one range per (tile, destination) is reserved with an atomicAdd on *cursor_ptrs[d] — the destination's own cursor
// in peer memory (push mode, base = 0) or a local cursor behind a precomputed base[d] — and the runs are streamed into d's receive
// buffer (peer memory over NVLink) as 128-byte-aligned warp stores
struct ShuffleParams {
    const u32* key;
    u32 n, n_parts, n_cols;
    const u32* in[KB_MAX_COLS];
    u32* const* peer_cols;     // device array [n_parts * n_cols]
    u32* const* cursor_ptrs;   // device array [n_parts]: word the range of destination d is reserved on
    const u32* base;           // device array [n_parts]
    u32 capacity;
    u32* overflow;
    u32* ticket;               // zeroed tile counter
    u32 tile, n_tiles, stride, pow2_mask;  // set by the launcher
};
void launch_shuffle_scatter(const ShuffleParams& p, int n_sms, cudaStream_t st);

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
// Relation-to-Stream operators (kb_r2s_eval; Relation2StreamOperator::eval, r2s.rs:37-58). A set of rows is an open-addressing table
// of u32 row indices (EMPTY32 = free slot) keyed by a 64-bit mix of the row's columns in the operator's slot order; a hash hit is
// confirmed by comparing every column.
struct R2sRows {
    const u32* col[KB_MAX_COLS];  // columns in the operator's slot order
    u32 n;
    u32* tab;                     // table over the rows (unused when n == 0)
    u32 mask;                     // table slots - 1
};
struct R2sParams {
    R2sRows cur;      // the response: its table is built, then remapped to the new state's columns
    R2sRows last;     // the previous state (read only)
    u32 n_cols;
    u32 probe_last;   // ISTREAM: flag the response rows whose tuple `last` does not hold
    u32* rep;         // [cur.n] 1 where row i is its tuple's representative (first occurrence); then its exclusive prefix
    u32* slot_of;     // [cur.n] table slot of row i's tuple
    u32* emit;        // ISTREAM: [cur.n] emitted response rows; DSTREAM: [last.n] rows of `last` that are gone (flags, then prefix)
    u32* counts;      // [2] zeroed: representatives, emitted rows
    u32 n_rep, n_emit;  // write passes: the totals of the two flag arrays
    u32* out_state[KB_MAX_COLS];
    u32* out_emit[KB_MAX_COLS];
};
// build: every response row goes into cur's table (atomicCAS on a free slot, atomicMin on a slot holding an equal row: the slot ends
// up holding the tuple's first occurrence, whatever the thread order)
void launch_r2s_build(const R2sParams& p, int n_sms, cudaStream_t st);
// mark: rep, slot_of and, with probe_last, emit (+ counts)
void launch_r2s_mark(const R2sParams& p, int n_sms, cudaStream_t st);
// DSTREAM mark: emit[j] = row j of `last` has no equal row in the response (+ counts[1]); runs before the remap
void launch_r2s_gone_mark(const R2sParams& p, int n_sms, cudaStream_t st);
// write, after the exclusive scans: the representatives into out_state (and cur's table remapped to them), with probe_last the
// emitted rows into out_emit
void launch_r2s_write(const R2sParams& p, int n_sms, cudaStream_t st);
// DSTREAM write: the gone rows of `last` into out_emit, in `last` order
void launch_r2s_gone_write(const R2sParams& p, int n_sms, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------------------
// small utilities
void launch_fill_u32(u32* p, u32 v, u64 n, cudaStream_t st);
// partition rows by mix32(key) % n_parts (multi-GPU shuffle): count then scatter
void launch_part_count(const u32* key, u32 n, u32 n_parts, u32* counts, int n_sms, cudaStream_t st);
void launch_part_scatter(const u32* key, u32 n, u32 n_parts, u32* cursors, const u32* const* in_cols, u32* const* out_cols, u32 n_cols,
                         int n_sms, cudaStream_t st);
// mark rows of a segment that equal any triple of a (small) delete set held in a 96-bit set; then compaction is a scan with flags
void launch_delete_mark(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots, u32* p_out /*p with EMPTY32 where deleted*/,
                        int n_sms, cudaStream_t st);
// kb_store_insert / kb_store_remove (kb_store.cu). The batch's keys go into a set laid out as launch_set_insert's (set_slots a power of
// two, zeroed); slot_of[i] = the slot of triple i, first[slot] (set to EMPTY32 before) = the smallest batch index holding that key;
// *overflow = 1 when the set is full
void launch_batch_set(uint4* set, u32 set_slots, const u32* s, const u32* p, const u32* o, u32 n, u32* first, u32* slot_of, u32* overflow,
                      int n_sms, cudaStream_t st);
// one stored segment against the batch set: found[slot] = 1 for every key the segment holds, *hits += its triples that match a key
void launch_batch_mark(const u32* s, const u32* p, const u32* o, u32 n, const uint4* set, u32 set_slots, u32* found, u32* hits, int n_sms,
                       cudaStream_t st);
// flag[i] = 1 iff triple i is the first of its key in the batch and found[its slot] equals want_found; *count += the flags set.
// flag8 is what the caller reads back, flag32 what an exclusive scan turns into output positions
void launch_batch_flags(u32 n, const u32* slot_of, const u32* first, const u32* found, bool want_found, u8* flag8, u32* flag32, u32* count, int n_sms,
                        cudaStream_t st);
// out[pos[i]] = triple i for every flagged i (batch order is kept: pos is the exclusive scan of the flags)
void launch_batch_gather(const u32* s, const u32* p, const u32* o, u32 n, const u8* flag8, const u32* pos, u32* out_s, u32* out_p, u32* out_o, int n_sms,
                         cudaStream_t st);
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
void launch_template_fill(const TemplateFillParams& P, int n_sms, cudaStream_t st);

}  // namespace kb
