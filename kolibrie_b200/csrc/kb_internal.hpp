// kb_internal.hpp — host-side state behind the C ABI (context, device buffers, relations, store segments).
#pragma once
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "kb_kernels.cuh"

namespace kb {

struct Life {  // shared by a context and every buffer it handed out: relations may outlive their context (bindings' GC order)
    bool alive = true;
    // Large buffers are recycled here instead of going back to the stream-ordered pool: a freed 267 MB result buffer that the pool has
    // to re-map for the next query costs several times the query itself, a closure's multi-GB join outputs more. Everything is allocated and released on the context's one stream, so a recycled buffer is
    // ordered behind its previous user exactly like a pool allocation would be.
    struct Cached { void* p; size_t bytes; };
    std::vector<Cached> cache;
    size_t cached_bytes = 0;
    bool cache_off = false;  // KOLIBRIE_BUF_CACHE=0
    // Sized for the working set of the largest workload (a config-4 closure releases tens of GB of buffers when it ends and asks for
    // the same sizes in the same order the next time; its 8 GB known-fact set must stay cached, or a later closure waits for the pool
    // to re-map it). The bound is 3/8 of the device's memory (30 GB on an 80 GB H100), set by kb_ctx_create: parked buffers are
    // invisible to other contexts of the process, so the rest stays free for them. When the cache is full the OLDEST entries go back
    // to the pool.
    static constexpr size_t MIN_BYTES = 1u << 20, MAX_ENTRIES = 256;
    size_t max_bytes = 30ull << 30;
};
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    cudaStream_t st = nullptr;
    std::shared_ptr<Life> life;
    ~DevBuf() {
        if (!p) return;
        if (life && life->alive) {
            if (!life->cache_off && bytes >= Life::MIN_BYTES && bytes <= life->max_bytes / 2) {
                while (!life->cache.empty() && (life->cache.size() >= Life::MAX_ENTRIES || life->cached_bytes + bytes > life->max_bytes)) {
                    cudaFreeAsync(life->cache.front().p, st);  // (entries are in release order: the front is the oldest)
                    life->cached_bytes -= life->cache.front().bytes;
                    life->cache.erase(life->cache.begin());
                }
                life->cache.push_back({p, bytes});
                life->cached_bytes += bytes;
                return;
            }
            cudaFreeAsync(p, st);  // stream-ordered: kernels still queued on st may be using it
        } else cudaFree(p);         // the context (and its stream) is gone
    }
};
using Buf = std::shared_ptr<DevBuf>;

struct Col {
    Buf buf;            // owner (may be shared by views / projections)
    u32* ptr = nullptr;  // 16-byte aligned, readable up to the next multiple of 256 B past the last row
};

// a timing event that is destroyed on every return path
struct ScopedEvent {
    cudaEvent_t e = nullptr;
    ScopedEvent() { cudaEventCreate(&e); }
    ~ScopedEvent() { if (e) cudaEventDestroy(e); }
    ScopedEvent(const ScopedEvent&) = delete;
    ScopedEvent& operator=(const ScopedEvent&) = delete;
    operator cudaEvent_t() const { return e; }
};

// device time between marks on a stream (an info struct's phase_ms): N marks bound N - 1 phases; ms(k) after a sync
template <int N>
struct PhaseTimer {
    ScopedEvent e[N];
    int at = 0;
    void mark(cudaStream_t st) { cudaEventRecord(e[at++], st); }
    double ms(int k) const {
        float v = 0.f;
        cudaEventElapsedTime(&v, e[k], e[k + 1]);
        return v;
    }
};

enum Family { F_SCAN = 0, F_BUILD, F_PROBE, F_FILTER, F_GROUP, F_OTHER, F_COUNT };

struct PendingTimer {
    cudaEvent_t a, b;
    int fam;
};

// A persistent tag-indexed table (kb_tagtab.cuh) over keys 0, 1, ... of a growing set: keys [0, indexed) are in it.
struct TagIndex {
    Buf tab;
    u64 slots = 0;
    u32 indexed = 0;
};

// the grid of a 1-D grid-stride kernel over n items
inline int grid_1d(u64 n, int n_sms, int threads = 256, int per_sm = 8) {
    const u64 want = (n + threads - 1) / threads, cap = (u64)n_sms * per_sm;
    return (int)(want < 1 ? 1 : want < cap ? want : cap);
}
inline u32 bits_of(u64 x) { return x ? 64u - (u32)__builtin_clzll(x) : 0u; }

}  // namespace kb

struct kb_rel {
    std::vector<kb::u32> slots;
    std::vector<kb::Col> cols;
    kb::u64 n = 0;
    bool pair = false;  // internal only: slots = {subject var, object var}, cols[0] = interleaved uint2 (s,o) rows
    int col_of(kb::u32 slot) const {
        for (size_t i = 0; i < slots.size(); i++) if (slots[i] == slot) return (int)i;
        return -1;
    }
};

struct kb_strings {
    kb::Buf off;    // u32 [n + 1] (exclusive prefix of the lengths)
    kb::Buf bytes;
    kb::u64 n = 0, total = 0;
};

struct kb_groups {  // (kb_group.cu)
    kb_groups(kb::u32 n_group, const kb_agg* aggs, kb::u32 n_aggs);  // no group yet: n_group key columns, the kinds of `aggs`
    // appends one group: its key, its row count and the accumulators as the device left them
    void add(const kb::u32* key, uint64_t count, const double* acc);
    std::vector<std::vector<kb::u32>> keys;
    std::vector<std::vector<double>> vals;
    std::vector<uint64_t> counts;
    std::vector<kb::u32> kinds;            // kb_agg_kind of every aggregate
    std::vector<std::vector<double>> raw;  // the accumulators as the device left them (AVG: the SUM, before the division): what a
                                           // cross-rank merge combines (kb_groups_pack / kb_groups_merge)
};

namespace kb {
struct Segment {
    u64 tag = 0;
    u64 id = 0;  // unique within the context, given when the segment joins the store: the index chunks built from it carry it
    Col s, p, o;
    u64 n = 0;
    cudaEvent_t ready = nullptr;  // set while a chunked upload is in flight: the scan waits on it
    u32 cmin[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};  // per-column id range (s,p,o), computed when the segment is loaded
    u32 cmax[3] = {0, 0, 0};
    bool has_stats = false;
    u32 stats_world = 0;   // sharding the statistics were checked against
    bool sharded_ok = true;  // every subject belongs to this context's shard (checked when kb_set_sharding is in effect)
    // distinct predicates of the segment with their row counts, from the same pass as the ranges (empty + preds_overflow when it
    // carries more than SEGP_SLOTS of them): what the index maintenance of a window slide allocates its chunks from
    std::vector<std::pair<u32, u32>> pred_rows;
    bool has_preds = false, preds_overflow = false;
};
}  // namespace kb

namespace kb {
struct SliceChunk {  // the rows of ONE store segment that carry the predicate: interleaved (subject, object)
    u64 tag = 0;           // the segment's tag (kb_store_append): evicting the segment drops the chunk
    u64 seg = 0;           // the segment's id: a set-semantic write that compacts or merges the segment replaces the chunk
    Col pairs;
    u64 n = 0;
    Buf ynum;              // typed literal column: f64 value of every object (num_or0), kept when the chunk has numeric objects
    u64 ynum_version = 0;  // numeric side table version it was built from
    u32 xmin = 0xFFFFFFFFu, xmax = 0, ymin = 0xFFFFFFFFu, ymax = 0;  // id ranges of the chunk (an eviction re-derives the slice's from the survivors)
};
struct PredSlice {  // one predicate's (subject, object) rows of the store — the device analogue of pos[P] (index_manager.rs:18-26) — as one
                    // chunk per store segment, so that an RSP window slide (append one segment, evict another) maintains the index
                    // instead of dropping it (rsp_engine.rs:94-104; simple_r2r.rs:95-142)
    std::vector<SliceChunk> chunks;
    u64 n = 0;  // rows over all chunks
    u32 xmin = 0xFFFFFFFFu, xmax = 0, ymin = 0xFFFFFFFFu, ymax = 0;  // id range of subjects (x) and objects (y) over the live chunks
    // persistent direct tables kept while the column is unique and dense: xtab[subject - xtab_min] = object (what the reference's
    // spo[s][P] lookup answers, index_manager.rs:18-26) and ytab[object - ytab_min] = subject (pos[P][o]). *_range is the table's
    // CAPACITY in slots: it is allocated with headroom above the largest key (dictionary ids grow), appended chunks are inserted in
    // place, evicted chunks are cleared in place, and the table is rebuilt only when a key falls outside it.
    Buf xtab, ytab;
    u32 xtab_min = 0, xtab_range = 0, ytab_min = 0, ytab_range = 0, tab_cshift = 0;
    bool x_unique = false, y_unique = false;  // no subject (object) occurs twice -> builds keyed on it need no duplicate detection
                                              // (functional / inverse-functional predicate in this store)
    bool x_tried = false, y_tried = false;    // a table for the column was attempted (false: never dense enough)
    // key-grouped directories for the columns that are NOT unique (multi-valued predicates, objects shared by many subjects): the
    // slice sorted by that column — a counting sort, the ids being dense — as off[key - min .. ] + the other half in key order. What the
    // reference's spo[s][P] -> {o} and pos[P][o] -> {s} sets are (index_manager.rs:18-26, 253-340): a bound subject / object is a range
    // of val, not a scan. Built by kb_store_build_index for single-chunk slices; dropped when the predicate's slice is appended to.
    Buf xkey;                // value ranks in TABLE order: xkey[compact(subject) - xtab_min] = rank of num_or0[object] in the context's value
    u64 xkey_version = 0;    // order (kb_numrank.cuh; built with xtab by kb_store_build_index when the slice has numeric objects; the
                             // table-mode probe filters on it sequentially, 4 bytes a slot)
    // one-byte codes in TABLE order when the subject table holds at most CODE_MAX distinct objects: xcode[slot] = index of xtab[slot]
    // in xdict (the objects, ascending), 0xFF where xtab holds EMPTY32. Built by kb_store_build_index only and dropped by every store
    // mutation (bump_version): xtab stays what the maintenance writes and every other reader reads; the index probe reads xcode.
    Buf xcode, xdict;
    u32 n_xdict = 0;
    Buf xoff, xval, yoff, yval;
    u32 xcsr_min = 0, xcsr_range = 0, ycsr_min = 0, ycsr_range = 0;
    const SliceChunk* single() const { return chunks.size() == 1 ? &chunks[0] : nullptr; }
    bool typed(u64 num_version) const {
        for (auto& c : chunks) if (!c.ynum || c.ynum_version != num_version) return false;
        return !chunks.empty();
    }
};
}  // namespace kb

struct kb_ctx {
    int device = 0;
    int n_sms = 132;
    cudaStream_t st = nullptr;
    cudaStream_t st_copy = nullptr;
    cudaEvent_t ev_copy = nullptr;
    std::string err;
    std::shared_ptr<kb::Life> life = std::make_shared<kb::Life>();
    // the store: written only by kb_store.cu (store_replace, store_add_device_segment, store_evict_tag), like store_version, the two
    // hint sets and the index below
    std::vector<kb::Segment> segs;
    kb::u64 n_triples = 0;
    kb::u64 seg_ids = 0;  // the last Segment::id given
    kb::Buf num, isnum;
    kb::Buf i32val, isi32;  // kb_dict_legacy_i32_load: the legacy executor's integer view of the terms
    kb::u32 n_i32 = 0;
    // the device dictionary: written only by kb_dict.cu (kb_dict_strings_load, dict_encode_device), and released by kb_ctx_destroy
    kb::Buf dict_off, dict_bytes;  // u64 offsets [dict_ids + 1] + UTF-8 bytes
    kb::u32 dict_ids = 0;
    kb::TagIndex dict_index;       // kb_dict_encode: string -> id (payload: the id), built lazily
    // the quoted-triple table: written only by kb_quoted.cu (kb_quoted_load, quoted_encode)
    kb::Buf quoted_s, quoted_p, quoted_o;  // indexed by id & 0x7FFFFFFF (EMPTY32: no entry)
    kb::u32 quoted_slots = 0;
    kb::u32 quoted_cap = 0;        // slots the three buffers hold (TRIPLE grows them with headroom; slots past quoted_slots are EMPTY32)
    kb::TagIndex quoted_rev;       // TRIPLE: (s, p, o) -> table index (payload: the index), built lazily, dropped by kb_quoted_load
    kb::u32 n_ids = 0;
    kb::u64 num_version = 1;  // bumped by kb_dict_numeric_load: typed literal columns of the index are tied to it
    // value order of the numeric side table (kb_numrank.cuh: sorted distinct non-NaN values, -0.0 folded, 0.0 included), on the device
    // and on the host (a FILTER constant becomes a rank range there); built with the index's rank columns, valid while numv_version ==
    // num_version
    kb::Buf numv;
    std::vector<double> h_numv;
    kb::u64 numv_version = 0;
    // tile-state buffer of the look-back prefix (words carry the launch epoch; cleared only when it wraps: compact_setup, kb_join.cu)
    kb::Buf tile_state, block_state;
    size_t tile_state_tiles = 0;
    // 0 (default): compaction in tile-completion order (one atomic per tile; row order of results is unspecified, as in the
    // reference whose row order is hash-iteration order). 1 (KOLIBRIE_ORDERED=1, and always for the legacy FFI symbol): store order.
    kb::u32 ordered = 0;
    kb::u64 epoch = 1;
    // control arena: small device words (tickets, totals, flags) zeroed at the start of every API call, mirrored in pinned memory
    kb::u32* ctrl = nullptr;
    kb::u32* h_ctrl = nullptr;
    kb::u32 ctrl_used = 0;
    bool ctrl_dirty = true;  // words handed out since the arena was last zeroed (a call that hands out none skips the memset)
    // control block of the one-kernel index join: device words {ticket, total, 0, done} that the kernel itself leaves zeroed, and the
    // pinned host word the kernel publishes the row count to
    kb::u32* fast_cb = nullptr;
    kb::u32* h_fast = nullptr;
    kb::u32* d_fast = nullptr;  // device address of h_fast
    static constexpr kb::u32 CTRL_WORDS = 8192;
    // pinned staging for uploads / downloads
    void* pinned = nullptr;
    size_t pinned_bytes = 0;
    // timing
    bool timing = false;
    std::vector<kb::PendingTimer> timers;
    std::vector<cudaEvent_t> ev_pool;
    kb_stats stats{};
    // knowledge cached across calls: (predicate, key position) pairs whose direct build met duplicate keys
    std::map<kb::u32, kb::u64> fix_hint;  // head predicate -> facts it held when the last fixpoint ended (sizes the next run's known-fact sets)
    std::shared_ptr<void> fix_state;      // kb_datalog_fixpoint_seed: the per-predicate relations and known-fact sets of the last seeded
                                          // call (kb_datalog.cu: FixState), valid while store_version is the one it was left at
    std::shared_ptr<void> closed;         // kb_datalog_fixpoint / kb_datalog_maintain: the store is closed under the rules (kb_datalog.cu:
                                          // Closed), valid while store_version / num_version are the ones recorded; kb_datalog_maintain's kept state
    std::set<std::pair<kb::u32, kb::u32>> multi_valued;
    std::set<std::pair<kb::u32, kb::u32>> single_valued;  // verified duplicate-free by an earlier direct build on this store version
    cudaStream_t st2 = nullptr;                            // second compute stream: independent direct builds run concurrently
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    kb::u64 store_version = 0;
    std::map<kb::u32, kb::PredSlice> index;  // kb_store_build_index: predicate -> slice; valid while index_version == store_version
    kb::u64 index_version = ~0ull;
    bool csr_join = true;                // KOLIBRIE_CSR_JOIN=0: 1:N joins always use the chained table (A/B switch)
    // Datalog candidate dedup: radix-partitioned above these sizes (KOLIBRIE_DERIVE_PART=0: never; =1 with KOLIBRIE_DERIVE_SLICE /
    // KOLIBRIE_DERIVE_MIN_ROWS: tests force it on small inputs)
    int derive_part = 1;
    kb::u64 derive_slice_bytes = 32ull << 20;
    kb::u64 derive_min_part_rows = 1ull << 20;
    kb::u64 derive_bucket_slack = 8192;  // KOLIBRIE_DERIVE_SLACK: rows a bucket holds beyond 9/8 of its fair share
    bool fast_index_kernel = true;       // KOLIBRIE_INDEX_KERNEL=0: index joins go through the generic probe kernel (A/B switch)
    bool use_index = true;               // KOLIBRIE_USE_INDEX=0 / kb_set_use_index: force the scanning path
    bool probe_table_mode = true;        // KOLIBRIE_PROBE_TABLE=0: the index probe always streams the slice (A/B switch)
    bool index_maintain = true;          // KOLIBRIE_INDEX_MAINTAIN=0: append / evict drop the index instead of maintaining it (A/B switch)
    kb::u32 shard_rank = 0, shard_world = 1;  // kb_set_sharding: the store is shard `rank` of `world`, sharded by subject
    int upload_stats_off = -1;  // chunked upload in flight: control words where the copy stream accumulates the column ranges
    kb_bgp_plan_info bgp_last{};  // kb_bgp_last_plan
};

namespace kb {

kb_status fail(kb_ctx* ctx, kb_status code, const char* fmt, ...);
struct DeviceGuard {  // the calling thread's current device is restored on return
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};
inline size_t round256(size_t b) { return (b + 255) & ~(size_t)255; }
#define KB_CUDA(ctx, call)                                                                                             \
    do {                                                                                                               \
        cudaError_t _e = (call);                                                                                       \
        if (_e != cudaSuccess) return kb::fail((ctx), KB_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)
#define KB_TRY(expr)                     \
    do {                                 \
        kb_status _s = (expr);           \
        if (_s != KB_OK) return _s;      \
    } while (0)
// the preamble of an entry point that takes a context: the context's device is current until it returns, its control arena is zeroed
#define KB_ENTER(ctx)                      \
    if (!(ctx)) return KB_E_INVALID;       \
    kb::DeviceGuard _guard((ctx)->device); \
    KB_TRY(kb::begin_call(ctx))

kb_status alloc_buf(kb_ctx* ctx, size_t bytes, Buf* out);
// one CUB device call: size query, scratch, call
template <class F>
kb_status cub_run(kb_ctx* ctx, F f) {
    size_t t = 0;
    KB_CUDA(ctx, f(nullptr, t));
    Buf b;
    KB_TRY(alloc_buf(ctx, t > 16 ? t : 16, &b));
    KB_CUDA(ctx, f(b->p, t));
    return KB_OK;
}
kb_status alloc_col(kb_ctx* ctx, u64 rows, Col* out);
kb_status begin_call(kb_ctx* ctx);                      // zero the control arena
u32 ctrl_alloc(kb_ctx* ctx, u32 words);                 // returns word offset into ctx->ctrl
kb_status ctrl_read(kb_ctx* ctx);                       // D2H of the used part of the arena + stream sync
kb_status ensure_tile_state(kb_ctx* ctx, u64 tiles);  // (compact_setup calls it; kb_star_join_prepare, so that a submit allocates nothing)
NumTab numtab(const kb_ctx* ctx);
// ctx->numv / h_numv for the current num_version (a device sort of the side table; one read-back). *ok = false: no value order (the
// table holds 2^31 ids or more), the index keeps no rank columns
kb_status ensure_num_order(kb_ctx* ctx, bool* ok);
void timer_begin(kb_ctx* ctx, int fam, int n_kernels = 1);
void timer_end(kb_ctx* ctx);
void timers_flush(kb_ctx* ctx);  // after a stream sync

// internal operators (device-resident, return relations whose row counts are known on the host)
struct FilterProg {
    std::vector<kb_filter_op> ops;
};
kb_status validate_filter(kb_ctx* ctx, const kb_filter_op* ops, u32 n);
// split a postfix program into its top-level AND conjuncts
bool split_conjuncts(const kb_filter_op* ops, u32 n, std::vector<FilterProg>* out);
std::set<u32> filter_slots(const FilterProg& f);
// a program over the variables `slots` as device ops: variable slots[i] is read from column i of the kernel's row, or from position
// (*pos)[i] (0 s, 1 p, 2 o) of a pattern's triple
kb_status compile_prog(kb_ctx* ctx, const FilterProg& f, const std::vector<u32>& slots, std::vector<FilterOp>* ops,
                       const std::vector<u32>* pos = nullptr);

struct ScanTable {  // scan+build fusion: pattern k inserts its matches into this direct table instead of emitting rows
    u32* tab = nullptr;
    u32 kmin = 0, range = 0;  // compacted key space when cshift != 0
    u32 cshift = 0;
    u32 key_is_o = 0, trusted = 0;
    u32* dup_flag = nullptr;
    bool clear = false;  // the table has not been set to 0xFF yet: scan_segments clears it (inside the scan kernel when it can)
};
// The triple scan (kb_scan.cu). What a scan emits per pattern: its variables as columns (s,p,o order); a 2-variable (?s P ?o)-shaped
// pattern as one interleaved (s,o) pair relation (internal fast path; other shapes still get columns); or the row positions of its
// matches.
enum class ScanOut { Cols, Pairs, RowIndex };
// One fused scan of `segs` (the store, ctx->segs, or segments a caller selected or built) for 1..MAXP patterns. tables: per pattern,
// a direct table that takes its matches instead of an output relation.
kb_status scan_segments(kb_ctx* ctx, const std::vector<Segment>& segs, const kb_pattern* pats, u32 n_pats, const std::vector<FilterProg>& pushdown,
                        ScanOut mode, std::vector<std::unique_ptr<kb_rel>>* out, const std::vector<ScanTable>* tables = nullptr);
// The patterns over the store, as columns: with a valid index (and ctx->use_index) the patterns it answers are looked up, and one fused
// scan of ctx->segs handles the rest.
kb_status scan_store(kb_ctx* ctx, const kb_pattern* pats, u32 n_pats, const std::vector<FilterProg>& pushdown, std::vector<std::unique_ptr<kb_rel>>* out);
// (?0 P ?1) for each of the k <= MAXP predicates `preds`, in one fused scan of `segs` without pushdown
kb_status scan_predicates(kb_ctx* ctx, const std::vector<Segment>& segs, const u32* preds, u32 k, ScanOut mode,
                          std::vector<std::unique_ptr<kb_rel>>* out);
// fused GROUP BY of a star join (kb_star_join_aggregate): in = group / aggregate spec; out = groups when the one-kernel index path took it
struct AggSpec {
    AggSpec() = default;
    AggSpec(u32 group, const kb_agg* a) : group_slot(group), has_agg(a != nullptr), kind(a ? a->kind : 0u), agg_slot(a ? a->slot : 0u) {}
    u32 group_slot = 0;
    bool has_agg = false;
    u32 kind = 0, agg_slot = 0;
    bool applied = false;  // false on return: the caller joins and groups in two steps
    u64 n_rows = 0;        // joined rows (when applied)
    std::unique_ptr<kb_groups> groups;
};
// What the one-kernel index path resolves a star join into (kb_star_join_prepare keeps it; kb_plan_submit only launches): the kernel
// parameters minus everything that belongs to one launch (output buffers, control block, epoch).
struct IndexPlan {
    bool ok = false;
    ProbeIParams P{};
    std::vector<u32> out_slots;  // variable of kernel output column c
    std::vector<u32> all_slots;  // column order of the relation handed to the caller
    u32 n_out = 0;
    u64 probe_rows = 0;          // rows of the probe slice = capacity a result buffer needs
    bool agg = false;            // GROUP BY folded into the kernel (P.gsel / P.asel / P.akind are set)
    bool has_agg = false;
    u32 agg_kind = 0, agg_slot = 0, group_slot = 0;
    const char* why = nullptr;   // not ok: what the one-kernel index path needs that the query lacks
};
// errors only for an invalid query; a query the one-kernel index path does not take leaves plan->ok false. agg: the GROUP BY is folded
// into the plan (plan->agg) when the join binds its variables
kb_status resolve_index_plan(kb_ctx* ctx, u32 join_slot, const kb_pattern* pats, u32 n_pats, const kb_filter_op* filter, u32 n_ops,
                             const AggSpec* agg, IndexPlan* plan);
// n_cols columns of `rows` rows in one allocation
kb_status alloc_strided_cols(kb_ctx* ctx, u64 rows, u32 n_cols, std::vector<Col>* cols);
// the compaction block of one launch over n_tiles tiles: the tile state (allocated whether or not the output is ordered), the order
// mode, a fresh epoch and the control words ctrl = {ticket, total, zero} (null: the launch brings its own, as the scan does)
kb_status compact_setup(kb_ctx* ctx, u64 n_tiles, u32* ctrl, Compact* c);
// the row-writing launch of the one-kernel index join into n_out columns of probe_rows rows
kb_status launch_index_rows(kb_ctx* ctx, ProbeIParams& P, const std::vector<Col>& cols);
// GROUP BY (kb_group.cu). The spec every entry point takes: group slots and aggregates present, 1..4 variables and at most 8
// aggregates (KB_E_LIMIT), of known kinds (KB_E_INVALID). Each entry point adds its own restrictions.
kb_status check_group_spec(kb_ctx* ctx, const uint32_t* group_slots, u32 n_group, const kb_agg* aggs, u32 n_aggs);
// the GroupParams of n_group key columns and these aggregates, without input columns and table
GroupParams group_params(const kb_ctx* ctx, u32 n_group, const kb_agg* aggs, u32 n_aggs);
// the device hash table: one buffer [val | cnt | keys | state], and the overflow word, which is either a control-arena word (the
// synchronous calls read it with the arena) or the 16 bytes behind the table (prepared plans: the word travels with the table)
struct GroupTable {
    Buf buf;
    u64 slots = 0;
    size_t o_val = 0, o_cnt = 0, o_keys = 0, o_state = 0, bytes = 0;
    u32* ctrl = nullptr;  // the control-arena word (ctrl_off), or null: the word is behind the table
    u32 ctrl_off = 0;
    // point P at a table of this layout that starts at `base` (this table's buffer, or a rank's copy in peer scratch)
    void point(GroupParams* P, char* base) const;
};
// allocates a table of `slots` slots, points P at it and runs the init kernel (which zeroes the overflow word); in_ctrl: the word
// is a control-arena word, else it is behind the table
kb_status group_table_create(kb_ctx* ctx, u64 slots, bool in_ctrl, GroupParams* P, GroupTable* t);
// after a launch into a table whose word is in the control arena: reads the arena back, and unless *overflowed downloads the table
// and appends its groups to g
kb_status group_table_collect(kb_ctx* ctx, const GroupTable& t, kb_groups* g, bool* overflowed);
// a grouped plan's partial tables in peer scratch: 64 flag words (256 bytes), then per ring slot one table laid out like t with its
// overflow word behind it
u64 group_peer_scratch_bytes(const GroupTable& t, u32 ring);
char* group_peer_table(char* scratch, const GroupTable& t, u32 ring_slot);
// what the peer merge of ring slot `ring_slot` reads: every rank's flags and partial table
PeerTables group_peer_tables(const GroupTable& t, const std::vector<char*>& scratch, u32 rank, u32 ring_slot);
kb_status segment_stats(kb_ctx* ctx, Segment* sg);
// KB_ID_NONE is reserved: the direct tables use it as their empty slot, so a stored triple holding it would drop out of a join.
// cmax: a new segment's largest id per column (its profile pass, or a segment file's header) -> KB_E_INVALID naming the position
kb_status refuse_reserved_id(kb_ctx* ctx, const u32 cmax[3]);
// Changes to the store (kb_store.cu). Each one bumps store_version, which voids what is keyed to it (prepared plans, the seeded
// fixpoint's state, the closed token), and clears the hint sets.
// the store becomes `segs`; the index is dropped
void store_replace(kb_ctx* ctx, std::vector<Segment> segs);
// a segment whose columns are already in HBM joins the store. keep_index: its statistics are computed (if it has none) and the index is
// maintained when it describes the store (else dropped); false: the segment joins as it is and the index is dropped
kb_status store_add_device_segment(kb_ctx* ctx, Segment& sg, bool keep_index = true);
// the segments tagged `tag` leave the store; keep_index: the index is maintained when it describes the store (else dropped).
// Returns whether a segment carried the tag.
bool store_evict_tag(kb_ctx* ctx, u64 tag, bool keep_index);
kb_status unpair_rel(kb_ctx* ctx, std::unique_ptr<kb_rel>* r);
kb_status filter_impl(kb_ctx* ctx, const kb_rel& in, const FilterProg& f, std::unique_ptr<kb_rel>* out);
kb_status hash_join_impl(kb_ctx* ctx, const kb_rel& L, const kb_rel& R, const FilterProg* post, std::unique_ptr<kb_rel>* out);
// agg != nullptr (kb_star_join_aggregate): agg->applied when the GROUP BY was folded into the join, else *out is the joined relation
kb_status star_join_impl(kb_ctx* ctx, u32 join_slot, const kb_pattern* pats, u32 n_pats, const kb_filter_op* filter, u32 n_ops,
                         std::unique_ptr<kb_rel>* out, AggSpec* agg = nullptr);
// kb_bind_join behind the entry point (the pattern is checked by the caller)
kb_status bind_join_impl(kb_ctx* ctx, const kb_rel& left, const kb_pattern& pat, std::unique_ptr<kb_rel>* out);
// the device dictionary and the quoted-triple table as the kernels read them (null / n = 0 while empty)
DictTab dicttab(const kb_ctx* ctx);
QuotedTab quotedtab(const kb_ctx* ctx);
// How decode_ids renders an id: Unknown as kb_rel_decode does (a term the tables do not hold is "unknown"); Empty as decode_any(..)
// .unwrap_or_default() does (such a term is ""); Plain as Dictionary::decode(..).unwrap_or("") does (a quoted id is not walked: it is ""
// like any id past the dictionary).
enum class Decode { Unknown, Empty, Plain };
// The text of n ids (kb_dict.cu) rendered by `mode`, followed by n_empty more "": *off = u32 offsets [n + n_empty + 1], *bytes the text,
// *total (nullable) its bytes. One control-arena read. A quoted id without a table (Unknown / Empty) is KB_E_UNSUPPORTED, a walk past
// KB_QUOTED_MAX_DEPTH or more than 2^32-1 bytes KB_E_LIMIT; `what` names the ids.
// from (nullable): the dictionary to read instead of ctx's (another context's on the same device, whose last writes are done).
kb_status decode_ids(kb_ctx* ctx, const u32* ids, u32 n, u32 n_empty, Decode mode, const char* what, Buf* off, Buf* bytes, u64* total,
                     const DictTab* from = nullptr);
// A context's device dictionary as kb_dict.cu keeps it. dict_copy: dst's dictionary becomes a copy of src's strings (device to device on
// dst's stream; src's last writes are done; the string -> id index is rebuilt by dst's next encode), and *prev receives the one dst held;
// dict_restore puts that back when a later step of the caller fails. Refused (KB_E_OOM, KB_E_CUDA) with dst unchanged.
struct DictState {
    Buf off, bytes;
    u32 ids = 0;
    TagIndex index;
};
kb_status dict_copy(kb_ctx* dst, const kb_ctx* src, DictState* prev);
void dict_restore(kb_ctx* dst, DictState&& prev);
// dst's quoted-triple table becomes a copy of src's (kb_quoted.cu; device to device, src's last writes are done; dst's reverse index is
// rebuilt by its next TRIPLE). Refused (KB_E_OOM, KB_E_CUDA) with dst's table unchanged.
kb_status quoted_copy(kb_ctx* dst, const kb_ctx* src);
// ensure the persistent index holds keys [0, n_keys) and stays below load 1/2 with `extra` more (kb_api.cu): rebuilt larger (1024 slots
// at least, 1.5x headroom) when too small, then insert(first, n, tab, mask, overflow word) launches the insert of the keys it lacks
// (one kernel). KB_E_LIMIT names `what` when the insert overflows.
template <class Insert>
kb_status tag_index_ensure(kb_ctx* ctx, TagIndex* ix, u32 n_keys, u64 extra, const char* what, Insert insert);
// a batch table for n keys (kb_tagtab.cuh): a power of two >= 2n, 1024 slots at least, every slot empty
kb_status tag_batch_table(kb_ctx* ctx, u64 n, Buf* tab, u64* slots);
// TRIPLE of kb_bind: QuotedTripleStore::encode of n rows (kb_quoted.cu). col[k] (null: the constant cval[k]) are the components; a new
// triple gets id next_qt_id + rank of its first row and joins the table. out[i] = the id, or old[i] (null: EMPTY32) where a component is
// unbound; *n_unbound += rows left EMPTY32.
kb_status quoted_encode(kb_ctx* ctx, const u32* const* col, const u32* cval, u32 n, u32 next_qt_id, const u32* old, u32* out,
                        unsigned long long* n_unbound, kb_bind_info* info);
// Dense ranks of d >= 1 values (kb_order.cu), given by an order key per value (nkey, numeric) or by their rendered strings (str_off[d + 1]
// u32 offsets into bytes, compared byte by byte, a proper prefix first): afterwards rank_of[v] is the rank of value v, *n_values the
// number of distinct values and *rounds the refinement rounds taken (7 bytes of string a round).
kb_status rank_values(kb_ctx* ctx, u32 d, const unsigned long long* nkey, const u32* str_off, const u8* bytes, u32* rank_of, u32* n_values, u32* rounds);
// n rows of three id columns in device memory; ready (nullable): an event the rows wait for (a segment's chunked upload)
struct ColSpan {
    const u32 *s = nullptr, *p = nullptr, *o = nullptr;
    u64 n = 0;
    cudaEvent_t ready = nullptr;
};
// the live segments of a store as spans, and their rows
std::vector<ColSpan> store_spans(const kb_ctx* ctx, u64* n_raw);
// The distinct triples of the spans' rows in ascending (s, p, o) order, the reference's BTreeSet<Triple> order (kb_serialize.cu):
// *S their subjects, *PO their (p << 32 | o), *n how many. The spans hold 0 < n_raw < 2^32 - 16 rows (the caller checks); the buffers
// hold n_raw entries. One control-arena read; launches count in the `other` family. The spans are not changed.
kb_status store_distinct(kb_ctx* ctx, const std::vector<ColSpan>& spans, Buf* S, Buf* PO, u32* n);
// Pair relations (kb_qbuilder.cu). distinct_pairs: the distinct (key << 32 | carried) pairs of the rows (cols[k].first, cols[k].second)
// over rows[k] rows each, sorted: *out, *n_out of them. pair_rel: n sorted distinct pairs as a two-column relation over (key slot, carried
// slot). pair_join_count: *cnt = sum over the nl left pairs of the nr right pairs with the same key (both sorted), the exact size of
// their join. split_sorted: rows [lo, lo + n) of a store_distinct result (S, PO) as three columns.
kb_status distinct_pairs(kb_ctx* ctx, const std::vector<std::pair<const u32*, const u32*>>& cols, const std::vector<u64>& rows, Buf* out, u32* n_out);
kb_status pair_rel(kb_ctx* ctx, const Buf& pairs, u32 n, u32 key_slot, u32 car_slot, std::unique_ptr<kb_rel>* out);
kb_status pair_join_count(kb_ctx* ctx, const Buf& lp, u32 nl, const Buf& rp, u32 nr, u64* cnt);
kb_status split_sorted(kb_ctx* ctx, const Buf& S, const Buf& PO, u64 lo, u64 n, u32* s, u32* p, u32* o);
// kb_dict_encode's body over a batch already in device memory (kb_dict.cu)
kb_status dict_encode_device(kb_ctx* ctx, const u64* d_off, const unsigned char* d_bytes, u64 n_terms, u64 total, u32* d_out_ids, u32* n_new,
                             Buf* first_pos);
// kb_dict_numeric_derive behind the entry point (kb_numeric.cu)
kb_status numeric_derive(kb_ctx* ctx, uint32_t tables, uint32_t first_id, kb_numeric_info* info);
void pattern_vars(const kb_pattern& pt, std::vector<u32>* slots, std::vector<u32>* src);
kb_status empty_rel(kb_ctx* ctx, const std::vector<u32>& slots, std::unique_ptr<kb_rel>* out);  // zero rows over `slots`
std::unique_ptr<kb_rel> select_cols(const kb_rel& in, const std::vector<u32>& slots);          // reorder / select columns (zero-copy)
// FILTER: a conjunct over one pattern's variables goes to the first pattern that binds them all, every other conjunct to `post`
kb_status split_filter(kb_ctx* ctx, const kb_filter_op* filter, u32 n_ops, const std::vector<std::vector<u32>>& pv,
                       const std::vector<u32>& all_slots, std::vector<FilterProg>* pushdown, FilterProg* post);
// kb_bgp_execute's component route (kb_bgp.cu): pv / all_slots as kb_bgp_execute derived them; *out has the columns of all_slots.
// Fills ctx->bgp_last.
kb_status bgp_components(kb_ctx* ctx, const kb_pattern* pats, u32 n_pats, const kb_filter_op* filter, u32 n_ops,
                         const std::vector<std::vector<u32>>& pv, const std::vector<u32>& all_slots, std::unique_ptr<kb_rel>* out);
u32 pow2_at_least(u64 x);
kb_status check_pattern(kb_ctx* ctx, const kb_pattern& pt);

// Backward-chaining queries (kb_backward.cu). Demand patterns of a query: per predicate, (x = subject, y = object) with KB_ID_NONE for
// "any"; a predicate whose list is {(any, any)} is demanded in full, one without a list not at all.
constexpr u32 BC_MAX_DEMAND = 64;  // patterns per predicate on the host, and in the device table of one call
struct BcDemand {
    std::vector<bool> relevant;  // per rule: a conclusion unifies with a demand pattern
    std::map<u32, std::vector<uint2>> pats;
    u32 n_patterns = 0;
};
// the query's demand patterns: the query's own, then for every rule head that unifies with a demand pattern each premise, with its own
// constants and the head variables the demand binds, until no new pattern appears (rules as kb_datalog_query has checked them)
void bc_demand_compile(const kb_rule* rules, u32 n_rules, const kb_pattern& q, BcDemand* d);
struct BcDemandDev {
    Buf tab;                                              // the device table
    std::map<u32, std::pair<const uint2*, u32>> of;       // restricted predicates of `preds`: their patterns in tab (the others: every fact)
};
kb_status bc_demand_upload(kb_ctx* ctx, const BcDemand& d, const std::vector<u32>& preds, BcDemandDev* out);
// launches the selection of the rows of (s, o) [0, n) that match one of the n_dem patterns into new columns of n rows (*out_s, *out_o);
// their count is control-arena word `count_word` after the caller's next ctrl_read
kb_status bc_demand_select(kb_ctx* ctx, const uint2* dem, u32 n_dem, const Col& s, const Col& o, u64 n, Col* out_s, Col* out_o, u32 count_word);
struct BcSource {  // n rows of (s, p, o); in[k] null: every row holds cval[k]
    const u32* in[3] = {nullptr, nullptr, nullptr};
    u32 cval[3] = {0, 0, 0};
    u64 n = 0;
};
struct BcExclude {  // facts left out of an answer: those of the 96-bit fact set `set` whose slot has a non-zero byte in `flag`
    const uint4* set = nullptr;
    u32 slots = 0;
    const u8* flag = nullptr;
};
// the distinct bindings of the query's variables over the facts of `src` that match it (and that `excl`, when given, does not exclude):
// one column per distinct variable in s, p, o first-appearance order; a ground query gives no column and 0 or 1 rows
kb_status bc_answer(kb_ctx* ctx, const kb_pattern& q, const std::vector<BcSource>& src, std::unique_ptr<kb_rel>* out,
                    const BcExclude* excl = nullptr);
// kb_bgp_execute without the entry preamble, for calls that run a BGP inside their own (kb_datalog_query_repairs)
kb_status bgp_execute_impl(kb_ctx* ctx, const kb_pattern* pats, u32 n_pats, const kb_filter_op* filter, u32 n_ops, const u32* project,
                           u32 n_project, std::unique_ptr<kb_rel>* out);

template <class Insert>
kb_status tag_index_ensure(kb_ctx* ctx, TagIndex* ix, u32 n_keys, u64 extra, const char* what, Insert insert) {
    const u64 need = ((u64)n_keys + extra) * 2 + 64;
    if (!ix->tab || ix->slots < need) {
        u64 slots = 1024;
        while (slots < need + need / 2) slots <<= 1;  // headroom: the next batches insert in place
        ix->tab.reset();
        KB_TRY(alloc_buf(ctx, slots * sizeof(u64), &ix->tab));
        KB_CUDA(ctx, cudaMemsetAsync(ix->tab->p, 0xFF, slots * sizeof(u64), ctx->st));
        ix->slots = slots;
        ix->indexed = 0;
    }
    if (ix->indexed < n_keys) {
        const u32 c = ctrl_alloc(ctx, 1);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, sizeof(u32), ctx->st));
        insert(ix->indexed, n_keys - ix->indexed, static_cast<u64*>(ix->tab->p), ix->slots - 1, ctx->ctrl + c);
        ctx->stats.kernel_launches++;
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        if (ctx->h_ctrl[c]) return fail(ctx, KB_E_LIMIT, "%s overflow", what);
        ix->indexed = n_keys;
    }
    return KB_OK;
}

}  // namespace kb
