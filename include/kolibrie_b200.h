/*
 * kolibrie_b200.h — C ABI of libkolibrie_b200.so: the H100-native (sm_90a) replacement for the
 * data-parallel hot path of Kolibrie (dictionary-encoded triple scan + filter, multi-way hash join,
 * GROUP BY aggregate, Datalog semi-naive fixpoint).
 *
 * Plain C, no C++/torch types. All ids are the reference's u32 dictionary term ids
 * (shared/src/dictionary.rs:32-48; quoted-triple ids carry bit 31, shared/src/quoted_triple_store.rs:17-55).
 * Variables exist only on the host: a "slot" is a small integer the caller assigns to each variable name.
 *
 * Threading: a kb_ctx is NOT re-entrant (one call in flight at a time, any thread) — the reference holds
 * `&mut SparqlDatabase` (kolibrie/src/streamertail_optimizer/execution/engine.rs:54) or the R2R mutex
 * (kolibrie/src/rsp_engine.rs:92) around every call. Distinct contexts may run concurrently.
 *
 * Ownership: inputs are borrowed for the duration of the call only (the reference passes slices,
 * kolibrie/src/cuda/cuda_join.rs:41-46). Outputs (kb_rel / kb_groups) are library-owned until *_free.
 *
 * Errors: every call returns kb_status; message via kb_last_error(). KB_E_UNSUPPORTED means "shape not
 * handled on the device — run the reference CPU path" (the `#[cfg(not(feature = "cuda"))]` fallback at
 * kolibrie/src/execute_query.rs:598-602). There is no CPU fallback inside this library.
 */
#ifndef KOLIBRIE_B200_H
#define KOLIBRIE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KB_API __attribute__((visibility("default")))

typedef int32_t kb_status;
#define KB_OK 0
#define KB_E_INVALID (-1)     /* bad argument */
#define KB_E_CUDA (-2)        /* CUDA runtime error (message has the cudaError string) */
#define KB_E_OOM (-3)         /* device or host allocation failed */
#define KB_E_UNSUPPORTED (-4) /* shape not supported on the device: caller falls back to its CPU path */
#define KB_E_NOT_FOUND (-5)
#define KB_E_LIMIT (-6)       /* a documented limit was exceeded (rows >= 2^32, > KB_MAX_* ...) */

/* Reserved id. The reference reserves the same value as RuleIndex WILDCARD (shared/src/rule_index.rs:16);
 * it is never a dictionary id (< 0x8000_0000) and is used here as "no such term" / empty hash slot. */
#define KB_ID_NONE 0xFFFFFFFFu

#define KB_MAX_PATTERNS 8   /* patterns fused in one scan / one star join (kb_bgp_execute takes up to KB_BGP_MAX_PATTERNS) */
#define KB_MAX_COLS 16      /* columns (variables) per relation */
#define KB_MAX_FILTER_OPS 32
#define KB_MAX_PREMISES 6
#define KB_MAX_CONCLUSIONS 4
#define KB_MAX_RULE_FILTERS 4

typedef struct kb_ctx kb_ctx;
typedef struct kb_rel kb_rel;       /* device-resident columnar bag of binding rows (reference `Bindings`, shared/src/terms.rs:23) */
typedef struct kb_groups kb_groups; /* host-resident GROUP BY result */

/* Term of a triple pattern — reference `Term::{Variable,Constant}` (shared/src/terms.rs:14-21).
 * `Term::QuotedTriple` is KB_TERM_QUOTED, which only kb_scan_quoted accepts; every other entry point refuses is_var > 1 (KB_E_INVALID). */
typedef struct kb_term {
    uint32_t is_var; /* 1: `value` is a variable slot; 0: `value` is a constant term id; KB_TERM_QUOTED: see kb_quoted_pattern */
    uint32_t value;
} kb_term;
#define KB_TERM_QUOTED 2u

/* reference `TriplePattern = (Term, Term, Term)` (shared/src/terms.rs:22) */
typedef struct kb_pattern {
    kb_term s, p, o;
} kb_pattern;

/* An RDF-star pattern (engine.rs:1111-1188). In `outer`, a subject (object) whose is_var is KB_TERM_QUOTED is the term
 * `<< inner_s >>` (`<< inner_o >>`); the inner pattern of a position that is not quoted is ignored. Inside an inner pattern a
 * KB_TERM_QUOTED term stands for "any quoted-triple id" — all the reference checks for a nested term (engine.rs:1100-1105).
 * A quoted predicate in `outer` -> KB_E_UNSUPPORTED. */
typedef struct kb_quoted_pattern {
    kb_pattern outer, inner_s, inner_o;
} kb_quoted_pattern;

/* ---- FILTER programs: postfix encoding of `FilterExpression` (shared/src/query.rs:15-22) with the
 *      semantics of `Condition::evaluate_with_ids` (kolibrie/src/streamertail_optimizer/types.rs:110-186) ---- */
enum kb_filter_opcode {
    KB_F_CMP_NUM = 1, /* push ( num_or0[row[slot]] <cmp> value )          types.rs:133-148: parse::<f64>().unwrap_or(0.0) */
    KB_F_EQ_ID = 2,   /* push ( row[slot] == id ); id==KB_ID_NONE -> false types.rs:131  (literal not in dictionary) */
    KB_F_NE_ID = 3,   /* push ( row[slot] != id ); id==KB_ID_NONE -> true  types.rs:132 */
    KB_F_AND = 4,
    KB_F_OR = 5,
    KB_F_NOT = 6,
    KB_F_PUSH_VAR = 7,   /* arithmetic operand: numeric value of row[slot]; invalid if the term is not numeric (types.rs:163-167) */
    KB_F_PUSH_CONST = 8, /* arithmetic operand: `value` */
    KB_F_ADD = 9,
    KB_F_SUB = 10,
    KB_F_MUL = 11,
    KB_F_DIV = 12,      /* divisor == 0.0 -> whole expression invalid (shared/src/query.rs:47-53) */
    KB_F_TRUTHY = 13,   /* pop number, push ( valid && v != 0.0 )            types.rs:168 */
    KB_F_IS_TRIPLE = 14, /* push ( row[slot] has bit 31 )                      types.rs:170-183 */
    /* the LEGACY executor's comparison (SparqlDatabase::apply_filters_simd, kolibrie/src/sparql_database.rs:1381-1669; the path
     * execute_query takes, execute_query.rs:311): when the bound term AND the constant both parse as i32 the comparison is an integer
     * one (all six operators); otherwise it is a byte-wise string comparison where only = and != can hold. Fields: `cmp` = kb_cmp,
     * OR-ed with KB_LEGACY_CONST_IS_I32 when the constant parses as i32, `value` = that integer, `id` = dictionary id of the constant
     * string (KB_ID_NONE when the dictionary does not hold it: no term equals it). Needs kb_dict_legacy_i32_load. */
    KB_F_CMP_LEGACY = 15
};
#define KB_LEGACY_CONST_IS_I32 0x100u  /* the constant parses as a number (i32; f64 in nested mode) */
/* a comparison NESTED inside AND / OR / NOT is evaluated by evaluate_filter_expression instead (sparql_database.rs:1784-1836): both sides
 * parsed as f64 (`value` = the constant), all six operators when both are numbers, string = / != otherwise */
#define KB_LEGACY_NESTED_F64 0x200u
enum kb_cmp { KB_CMP_GT = 1, KB_CMP_GE = 2, KB_CMP_LT = 3, KB_CMP_LE = 4, KB_CMP_EQ = 5, KB_CMP_NE = 6 };

typedef struct kb_filter_op {
    uint32_t op;   /* kb_filter_opcode */
    uint32_t slot; /* variable slot (operand ops) */
    uint32_t cmp;  /* kb_cmp for KB_F_CMP_NUM */
    uint32_t id;   /* term id for KB_F_EQ_ID / KB_F_NE_ID */
    double value;  /* constant for KB_F_CMP_NUM / KB_F_PUSH_CONST */
} kb_filter_op;

/* ---- aggregates: `group_and_aggregate_results` (kolibrie/src/execute_query.rs:1150-1227) ---- */
enum kb_agg_kind { KB_AGG_COUNT = 0, KB_AGG_SUM = 1, KB_AGG_MIN = 2, KB_AGG_MAX = 3, KB_AGG_AVG = 4 };
typedef struct kb_agg {
    uint32_t kind; /* kb_agg_kind; COUNT ignores slot (rows per group — advertised README.md:415, not parsed by the reference) */
    uint32_t slot; /* variable aggregated: value = num_or0[row[slot]] (non-numeric -> 0.0, execute_query.rs:1171-1175,1184) */
} kb_agg;

/* ---- Datalog: `Rule{premise,filters,conclusion}` (shared/src/rule.rs:14-25) ---- */
typedef struct kb_rule_filter { /* `FilterCondition{variable,operator,value}` with `evaluate_filters` semantics (datalog/src/reasoning/rules.rs:133-165) */
    uint32_t lhs_slot;
    uint32_t cmp;        /* kb_cmp; 0 = operator the reference ignores (e.g. "OR:>"): no-op */
    uint32_t rhs_is_var; /* 1: compare ids of two bound variables (only = and != have an effect, rules.rs:141-146) */
    uint32_t rhs_slot;
    double rhs_value;    /* rhs_is_var==0: value.parse::<f64>().unwrap_or(0.0); = / != use f64::EPSILON (rules.rs:157-158) */
} kb_rule_filter;

typedef struct kb_rule {
    const kb_pattern* premise;
    uint32_t n_premise;
    const kb_rule_filter* filters;
    uint32_t n_filters;
    const kb_pattern* conclusion;
    uint32_t n_conclusion;
} kb_rule;

enum kb_strategy {
    KB_SEMI_NAIVE = 0, /* datalog/src/reasoning/materialisation/semi_naive.rs:53-91 */
    KB_NAIVE = 1,      /* datalog/src/reasoning/materialisation/my_naive.rs:10-71 */
    /* datalog/src/reasoning/materialisation/semi_naive_parallel.rs:11-176: semi-naive rounds over rules with 1 or 2 premises only
     * (others are skipped, :149), rule filters are NOT evaluated, premises are matched with matches_rule_pattern (rules.rs:9-72):
     * constants in subject/object positions ARE enforced (unlike the hash-join strategies, quirk Q6). */
    KB_SEMI_NAIVE_PARALLEL = 2,
    /* KB_SEMI_NAIVE with the textbook delta scheme: the premises BEFORE the delta premise read only the facts older than the delta
     * (OLD), the ones after it all facts — every derivation that uses a delta fact is produced exactly once, where semi_naive.rs:22-44
     * (delta of premise i against ALL facts of every other premise) produces a derivation with m delta facts m times. Same inferred
     * facts, same rounds, same new facts per round; `derivations` is smaller (config-4 shape: 0.79e9 instead of 1.25e9 candidates). */
    KB_SEMI_NAIVE_OLD_DELTA = 3
};

typedef struct kb_fixpoint_stats {
    uint32_t rounds;            /* infer_round calls that produced facts (infer_generic.rs:33-50) */
    uint64_t inferred;          /* facts appended to the store */
    uint64_t derivations;       /* candidate head instances before dedup */
    uint64_t round_new[64];     /* new facts per round (first 64 rounds) */
    double device_ms;           /* CUDA-event time of the whole fixpoint */
} kb_fixpoint_stats;

/* per-call device timings (CUDA events on the library's stream); enabled by kb_set_timing(ctx,1) */
typedef struct kb_stats {
    double scan_ms, build_ms, probe_ms, filter_ms, group_ms, other_ms, total_ms;
    uint64_t scan_launches, build_launches, probe_launches, filter_launches, group_launches, other_launches;
    uint64_t rows_scanned;   /* triples read by scan kernels */
    uint64_t rows_built;     /* rows inserted in hash tables */
    uint64_t rows_probed;    /* probe-side rows */
    uint64_t rows_out;       /* rows of the last result */
    uint64_t h2d_bytes, d2h_bytes;
    uint64_t kernel_launches; /* launches of this library's own kernels (memsets and copies not counted) */
    uint64_t fused_scan_builds; /* star joins whose build sides were inserted into their tables by the scan kernel itself */
    uint64_t index_joins;       /* star joins answered from the predicate-partitioned index (no store scan) */
} kb_stats;

/* ------------------------------------------------------------------ context */
KB_API const char* kb_version(void);
KB_API kb_status kb_ctx_create(int device, kb_ctx** out);
KB_API void kb_ctx_destroy(kb_ctx* ctx);
KB_API const char* kb_last_error(const kb_ctx* ctx); /* ctx may be NULL: last error of a failed kb_ctx_create */
KB_API kb_status kb_set_timing(kb_ctx* ctx, int enabled);
KB_API kb_status kb_get_stats(kb_ctx* ctx, kb_stats* out, int reset);
KB_API kb_status kb_synchronize(kb_ctx* ctx);

/* ------------------------------------------------------------------ triple store (device cache of `SparqlDatabase.triples`,
 * kolibrie/src/sparql_database.rs:50; segments = RSP window slides, kolibrie/src/rsp_engine.rs:94-104) */
KB_API kb_status kb_store_load(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n);
/* same, columns already in device memory of ctx's device (copied device-to-device) */
KB_API kb_status kb_store_load_device(kb_ctx* ctx, const uint32_t* d_s, const uint32_t* d_p, const uint32_t* d_o, uint64_t n);
KB_API kb_status kb_store_append(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t segment_tag);
/* kb_store_append for a slide whose columns are already in device memory of ctx's device (the receive side of kb_shuffle_push, a
 * producer kernel): copied device-to-device into a new segment; the store index is maintained exactly as for kb_store_append */
KB_API kb_status kb_store_append_device(kb_ctx* ctx, const uint32_t* d_s, const uint32_t* d_p, const uint32_t* d_o, uint64_t n, uint64_t segment_tag);
KB_API kb_status kb_store_evict(kb_ctx* ctx, uint64_t segment_tag);
/* set-difference by value (SparqlDatabase::delete_triple, sparql_database.rs:229-242) */
KB_API kb_status kb_store_delete(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n);
KB_API kb_status kb_store_clear(kb_ctx* ctx);
/* SparqlDatabase::build_all_indexes (kolibrie/src/sparql_database.rs:3364-3394) on the device: partitions the store by predicate into
 * interleaved (subject, object) slices — what the reference's pos/pso indexes give an index scan of `?s P ?o` (engine.rs:1364-1378).
 * Joins over such patterns then read 8 bytes per MATCHING triple instead of scanning 12 bytes per triple of the store. Dropped by
 * any store mutation (load/append/evict/delete/inferred facts); skipped (KB_OK, n_predicates = 0) above 4096 distinct predicates. */
KB_API kb_status kb_store_build_index(kb_ctx* ctx, uint32_t* n_predicates, double* build_ms);
KB_API kb_status kb_set_use_index(kb_ctx* ctx, int enabled);
KB_API kb_status kb_store_size(kb_ctx* ctx, uint64_t* n_triples, uint32_t* n_segments);
/* id -> f64 side table computed by the host with Rust `str::parse::<f64>` acceptance:
 * num_or0[id] = parse().unwrap_or(0.0); is_num[id] = parse().is_ok(). ids >= n_ids read as (0.0, not numeric). */
KB_API kb_status kb_dict_numeric_load(kb_ctx* ctx, const double* num_or0, const uint8_t* is_num, uint32_t n_ids);

/* id -> i32 side table of the legacy executor's filter (KB_F_CMP_LEGACY): val[id] = the term parsed with Rust `str::parse::<i32>`,
 * is_i32[id] = whether it parses. ids >= n_ids are not integers. */
KB_API kb_status kb_dict_legacy_i32_load(kb_ctx* ctx, const int32_t* val, const uint8_t* is_i32, uint32_t n_ids);

/* The same side tables DERIVED ON THE DEVICE from the device dictionary's strings (kb_dict_strings_load, kb_dict_encode, kb_bind's CONCAT
 * and isTRIPLE), so a host never parses the dictionary or uploads a table:
 *   KB_NUMERIC_F64: num_or0 / is_num exactly as kb_dict_numeric_load takes them: Rust `str::parse::<f64>()` — optional sign, then
 *                   inf / infinity / nan in any case, or digits[.digits] / .digits / digits. with an optional e|E[+-]digits, nothing else;
 *                   the nearest double, ties to even, for input of any length; "-0" is -0.0 and "-nan" has its sign bit set;
 *   KB_NUMERIC_I32: val / is_i32 exactly as kb_dict_legacy_i32_load takes them: `str::parse::<i32>()`, [+-]?[0-9]+ within range.
 * n_ids = the ids the device dictionary holds. For each table in `tables`, ids [first_id, n_ids) are parsed; entries below first_id stay as
 * they were (a load or an earlier derive); afterwards the table covers exactly n_ids ids. first_id = KB_NUMERIC_APPEND: from the first
 * id the table does not hold yet (per table). Refused with KB_E_INVALID, tables unchanged: tables 0 or with unknown bits; first_id
 * greater than the ids a selected table holds (a hole); first_id greater than n_ids. The tables grow with headroom, so an append per
 * window firing does not reallocate each time. KB_NUMERIC_F64 voids what kb_dict_numeric_load voids: num_version (prepared plans go
 * stale, typed index columns are rebuilt) and hence the closed-store token only when a rule filter compares numbers; KB_NUMERIC_I32
 * voids nothing, like kb_dict_legacy_i32_load. No host-to-device bytes; launches and device time count in kb_stats' `other` family.
 * info (may be NULL): n_ids; n_derived = ids parsed (n_ids - the smallest first id); n_numeric / n_i32 = how many of them parse;
 * n_slow = how many took the exact slow path (the 128-bit Eisel–Lemire step could not decide them). */
#define KB_NUMERIC_F64 1u             /* the numeric side table of kb_dict_numeric_load */
#define KB_NUMERIC_I32 2u             /* the legacy view of kb_dict_legacy_i32_load */
#define KB_NUMERIC_APPEND 0xFFFFFFFFu /* first_id: from the first id the table does not hold yet */
typedef struct kb_numeric_info { uint32_t n_ids, n_derived, n_numeric, n_i32, n_slow; } kb_numeric_info;
KB_API kb_status kb_dict_numeric_derive(kb_ctx* ctx, uint32_t tables, uint32_t first_id, kb_numeric_info* info /* nullable */);
/* Entries [first, first + n) of the side tables: each non-NULL pointer receives its table's entries (num_or0 / is_num: the f64 table;
 * val / is_i32: the i32 table). first + n past the entries a requested table holds -> KB_E_INVALID. */
KB_API kb_status kb_dict_numeric_download(kb_ctx* ctx, uint32_t first, uint32_t n, double* num_or0, uint8_t* is_num, int32_t* val, uint8_t* is_i32);

/* Dictionary strings on the device + result decode: the id -> string step that ends ExecutionEngine::execute
 * (kolibrie/src/streamertail_optimizer/execution/engine.rs:27-51) and Dictionary::decode (shared/src/dictionary.rs:50-52).
 * String i is bytes[offsets[i] .. offsets[i+1]) (UTF-8, no terminator). */
KB_API kb_status kb_dict_strings_load(kb_ctx* ctx, const uint64_t* offsets /* [n_ids + 1] */, const uint8_t* bytes, uint32_t n_ids);
typedef struct kb_strings kb_strings; /* device-resident decoded column: offsets [n+1] + bytes */
/* Decodes column `col` of `r`: row i becomes the string of its id; an id the dictionary does not hold becomes "unknown" (engine.rs:44).
 * Quoted-triple ids (bit 31, shared/src/quoted_triple_store.rs:28-55): without a quoted-triple table (kb_quoted_load) -> KB_E_UNSUPPORTED.
 * With one, a quoted id renders as Dictionary::decode_term renders it (shared/src/dictionary.rs:60-72): `<< s p o >>`, components decoded
 * the same way, recursively. When decode_term gives None at any depth (an id neither table holds), the whole term is "unknown"
 * (engine.rs:42-43). A walk that reaches a quoted id more than KB_QUOTED_MAX_DEPTH levels deep (the top-level id is level 1) before it
 * meets such an id -> KB_E_LIMIT: the table comes from the caller and a cycle in it would otherwise never end. At most 2^32-1 bytes per
 * call. Launches and device time count in kb_stats' `other` family. */
#define KB_QUOTED_MAX_DEPTH 16
KB_API kb_status kb_rel_decode(kb_ctx* ctx, const kb_rel* r, uint32_t col, kb_strings** out);
/* Dictionary::encode (shared/src/dictionary.rs:32-48) for a BATCH of terms — the load-time encode of sparql_database.rs:1000-1013 — on
 * the device: term i = bytes[offsets[i] .. offsets[i+1]) (host memory, offsets[0] = 0). A term the device dictionary already holds
 * (kb_dict_strings_load, earlier kb_dict_encode calls) gets its id; every other distinct string gets the next id in FIRST-SEEN order
 * over the batch — exactly the ids n_terms sequential Dictionary::encode calls hand out — and is appended to the device dictionary
 * (kb_rel_decode sees it). out_ids[n_terms]; *n_new = number of new strings; new_first_pos (may be NULL, room for n_terms entries):
 * new_first_pos[k] = index in the batch of the term that introduced id (ids before the call) + k, so the host dictionary can add the
 * same strings without a lookup of its own. Limits: < 2^32-16 terms and bytes per call (split larger loads); ids stay below bit 31. */
KB_API kb_status kb_dict_encode(kb_ctx* ctx, const uint64_t* offsets /* [n_terms + 1] */, const uint8_t* bytes, uint64_t n_terms, uint32_t* out_ids,
                                uint32_t* n_new, uint64_t* new_first_pos);
/* ids and bytes the device dictionary holds */
KB_API kb_status kb_dict_strings_info(kb_ctx* ctx, uint32_t* n_ids, uint64_t* n_bytes);
KB_API kb_status kb_strings_info(const kb_strings* s, uint64_t* n_strings, uint64_t* total_bytes);
KB_API kb_status kb_strings_download(kb_ctx* ctx, const kb_strings* s, uint64_t* offsets /* [n + 1] */, uint8_t* bytes /* total_bytes */);
KB_API void kb_strings_free(kb_ctx* ctx, kb_strings* s);

/* Quoted-triple table on the device: QuotedTripleStore::id_to_components (shared/src/quoted_triple_store.rs:28-55), entry i =
 * (ids[i] -> (s[i], p[i], o[i])). It REPLACES the context's table; n = 0 clears it. The table is indexed by id & 0x7FFFFFFF (the
 * reference hands ids out sequentially from 0x80000000); ids never given are empty slots. A component may itself be a quoted id
 * (nesting). Checked before anything changes — a refused call leaves the previous table in place:
 *   an id without bit 31, an id or a component equal to KB_ID_NONE, a repeated id -> KB_E_INVALID;
 *   an index id & 0x7FFFFFFF >= KB_QUOTED_MAX_SLOTS -> KB_E_LIMIT (the table takes 12 bytes per slot up to the largest index).
 * Like the dictionary tables, the quoted table is not tied to the store version: store mutations and index builds keep it. */
#define KB_QUOTED_MAX_SLOTS (1u << 28)
KB_API kb_status kb_quoted_load(kb_ctx* ctx, const uint32_t* ids, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n);
/* Entries of the quoted-triple table with ids [first_id, first_id + n) (first_id has bit 31): s[k], p[k], o[k] of id first_id + k, all
 * three KB_ID_NONE for an id the table does not hold. Together with kb_dict_strings_download, what a host QuotedTripleStore and Dictionary
 * take from kb_bind's kb_bind_info tails to stay equal to the device's. */
KB_API kb_status kb_quoted_download(kb_ctx* ctx, uint32_t first_id, uint32_t n, uint32_t* s, uint32_t* p, uint32_t* o);
/* Strings of the device dictionary with ids [first, first + n): offsets[k] .. offsets[k+1] of `bytes` is the string of id first + k,
 * offsets[0] = 0 (offsets: n + 1 entries). bytes may be NULL (offsets only: offsets[n] is the size `bytes` needs). first + n must not
 * pass the ids the device dictionary holds (KB_E_INVALID). */
KB_API kb_status kb_dict_strings_download(kb_ctx* ctx, uint32_t first, uint32_t n, uint64_t* offsets, uint8_t* bytes);

/* ------------------------------------------------------------------ BIND: `PhysicalOperator::Bind` with the built-in functions of
 * ExecutionEngine::execute_with_ids (kolibrie/src/streamertail_optimizer/execution/engine.rs:144-277) over the rows of `in`, in the order
 * they lie. *out = `in` with the output column: appended when out_slot is not a column of `in`, else that column replaced (the other
 * columns are shared with `in`, which is left as it was).
 *   Unbound (engine.rs:218-273): where the reference inserts nothing into a row, the output column holds KB_ID_NONE —
 *     or, when out_slot was already a column of `in`, that row's old value (row.insert overwrites, a skipped insert keeps it). An
 *     argument column holding KB_ID_NONE (an earlier BIND left it unbound) is a missing variable. info.n_unbound = rows whose output
 *     value is KB_ID_NONE after the call.
 *   KB_BIND_SUBJECT / _PREDICATE / _OBJECT (engine.rs:218-239): one variable argument; the output is that component of the quoted-triple
 *     table entry of the argument's id. Unbound when the id is not a quoted id (bit 31), the table does not hold it (a hole, past the end,
 *     no table) or the argument is missing.
 *   KB_BIND_IS_TRIPLE (engine.rs:260-273): one variable argument; the output is the dictionary id of "true" (quoted id) or "false".
 *     Unbound when the argument is missing. The two strings are encoded only when a row needs them, in the order of the first row that
 *     needs each (the reference calls Dictionary::encode inside its row loop); a string already held keeps its id.
 *   KB_BIND_TRIPLE (engine.rs:240-259): three arguments, each a variable or a constant id. The reference encodes a constant with
 *     Dictionary::encode inside the row loop, so constants exist only when `in` has a row: the caller encodes them (in argument order,
 *     only for a non-empty `in`) and passes their ids. When the three values are bound, QuotedTripleStore::encode(s, p, o)
 *     (shared/src/quoted_triple_store.rs:45-56): a triple the table holds keeps its id (the smallest, should the table hold it twice);
 *     every other distinct (s, p, o) gets next_qt_id + the rank of its first row among the first rows of the new triples — the ids the
 *     sequential loop hands out. The new entries join the table (kb_scan_quoted and kb_rel_decode see them). Unbound when any argument
 *     is missing.
 *   KB_BIND_CONCAT (engine.rs:148-182): zero or more arguments. A variable contributes Dictionary::decode(id).unwrap_or("") (dictionary.rs:49-51) — decode,
 *     not decode_term: a quoted id, an id the dictionary does not hold and a missing variable contribute "" — and a constant contributes
 *     its bytes as given (the caller passes `arg.trim_matches('"')`: a constant `"a"@en` is `a"@en`). Constant k of the call (is_var 0,
 *     value k) is const_bytes[const_offsets[k] .. const_offsets[k+1]). The concatenations are encoded as a batch with the ids the
 *     sequential Dictionary::encode loop gives (kb_dict_encode) and joined to the device dictionary. Every row is bound.
 * The reference's Bind checks `database.udfs` before SUBJECT..isTRIPLE (engine.rs:183): a caller with a user-defined function of the same name must not
 * call this. Refused before anything changes: an unknown function (the reference prints "not found" and binds nothing, engine.rs:274-276) or an argument count other than the above, a CONCAT constant index
 * past n_const, a variable argument that is not a column of `in` (KB_E_INVALID, as are next_qt_id without bit 31 or not above every id
 * the table holds, for TRIPLE); new quoted ids reaching KB_QUOTED_MAX_SLOTS, more than 2^32-16 concatenated bytes in one call, new
 * dictionary ids reaching bit 31, a relation of 2^32 rows or more (KB_E_LIMIT).
 * info: n_rows, n_unbound, the new dictionary ids [dict_first, dict_first + dict_new) and the new quoted ids [quoted_first,
 * quoted_first + quoted_new), each range in the order the reference creates them (kb_dict_strings_download / kb_quoted_download fetch
 * them). Launches and device time count in kb_stats' `other` family. */
enum kb_bind_function { KB_BIND_SUBJECT = 1, KB_BIND_PREDICATE = 2, KB_BIND_OBJECT = 3, KB_BIND_IS_TRIPLE = 4, KB_BIND_TRIPLE = 5, KB_BIND_CONCAT = 6 };
#define KB_BIND_MAX_ARGS 16
typedef struct kb_bind_spec {
    uint32_t function;              /* kb_bind_function */
    uint32_t n_args;
    const kb_term* args;            /* is_var 1: variable slot; 0: constant id (TRIPLE) or constant index (CONCAT) */
    uint32_t n_const;               /* CONCAT constants: const_offsets[n_const + 1] (const_offsets[0] = 0), const_bytes */
    const uint64_t* const_offsets;
    const uint8_t* const_bytes;
    uint32_t out_slot;
    uint32_t next_qt_id;            /* TRIPLE: QuotedTripleStore::next_qt_id */
} kb_bind_spec;
typedef struct kb_bind_info {
    uint64_t n_rows, n_unbound;
    uint32_t dict_first, dict_new;
    uint32_t quoted_first, quoted_new;
} kb_bind_info;
KB_API kb_status kb_bind(kb_ctx* ctx, const kb_rel* in, const kb_bind_spec* spec, kb_rel** out, kb_bind_info* info);

/* ------------------------------------------------------------------ relations */
KB_API kb_status kb_rel_info(const kb_rel* r, uint64_t* n_rows, uint32_t* n_cols, uint32_t* slots /* [KB_MAX_COLS] or NULL */);
KB_API kb_status kb_rel_download(kb_ctx* ctx, const kb_rel* r, uint32_t col, uint32_t* host_dst /* n_rows */);
KB_API kb_status kb_rel_device_col(const kb_rel* r, uint32_t col, const uint32_t** d_ptr);
/* `PhysicalOperator::InMemoryBuffer` / VALUES (operators/physical.rs:16-76; engine.rs:128-130) */
KB_API kb_status kb_rel_from_host(kb_ctx* ctx, const uint32_t* slots, uint32_t n_cols, const uint32_t* const* cols, uint64_t n_rows, kb_rel** out);
KB_API void kb_rel_free(kb_ctx* ctx, kb_rel* r);

/* ------------------------------------------------------------------ operators (mirror `PhysicalOperator`, operators/physical.rs:16-76) */
/* TableScan/IndexScan (engine.rs:510-584, 1192-1245): ONE fused pass over the store evaluates n_pats patterns.
 * out[k] has one column per distinct variable of pattern k in s,p,o order. A repeated variable inside one
 * pattern is enforced as equality (SURVEY quirk Q4: the reference's index scans do not — documented divergence).
 * pushdown[k] (nullable) is a filter program over pattern k's own variables applied while scanning. */
KB_API kb_status kb_scan(kb_ctx* ctx, const kb_pattern* pats, uint32_t n_pats,
                         const kb_filter_op* const* pushdown, const uint32_t* pushdown_len, kb_rel** out);
/* Filter (engine.rs:73-85). A KB_ID_NONE cell is a variable the row leaves unbound (kb_bind, kb_natural_join, a ragged InMemoryBuffer):
 * as in types.rs:126-183, KB_F_CMP_NUM, KB_F_EQ_ID, KB_F_NE_ID and KB_F_IS_TRIPLE over it are false, KB_F_PUSH_VAR pushes an invalid
 * operand (so the arithmetic and its KB_F_TRUTHY are false), and KB_F_NOT inverts each of these. */
KB_API kb_status kb_filter(kb_ctx* ctx, const kb_rel* in, const kb_filter_op* prog, uint32_t n_ops, kb_rel** out);
/* Projection — bag semantics, duplicates kept (engine.rs:86-106); zero-copy */
KB_API kb_status kb_project(kb_ctx* ctx, const kb_rel* in, const uint32_t* slots, uint32_t n_slots, kb_rel** out);
/* OptimizedHashJoin / HashJoin / merge join / NestedLoopJoin (engine.rs:710-837, 970-1039): natural join on the
 * common slots; no common slot -> cartesian product (engine.rs:1054-1071, limited to 2^28 output rows). */
KB_API kb_status kb_hash_join(kb_ctx* ctx, const kb_rel* left, const kb_rel* right, kb_rel** out);
/* The join of SPARQL mappings over rows that may leave variables unbound: natural_join (rsp_engine.rs:684-718), which the RSP engine's
 * emit step uses to join the latest results of several windows and the static data (rsp_engine.rs:647-681), on ids. The dictionary is
 * shared by every window and the static store (rsp_engine.rs:215-243), so the reference's string equality is id equality. A cell holding
 * KB_ID_NONE means "this row does not bind this variable" (what kb_bind leaves unbound).
 *   Columns. The union of both slot sets: `left`'s slots in order, then the slots of `right` that `left` lacks.
 *   Rows. A (left, right) row pair is emitted iff every shared slot bound in BOTH rows holds equal ids. The merged cell holds the right
 *     value when it is bound, else the left one (`merged.insert` overwrites, rsp_engine.rs:708-711; where both are bound they are equal),
 *     so a slot unbound on both sides stays KB_ID_NONE.
 *   A bag: every compatible pair once, so duplicates multiply. Row order is unspecified. Either side empty -> 0 rows (:688-690).
 *   No shared slot -> the cartesian product, limited to 2^28 rows as in kb_hash_join.
 * Routes. A check pass reads the shared columns of both sides (launch and time in kb_stats' `other` family).
 *   - No shared column holds KB_ID_NONE: exactly kb_hash_join (its launches, its limits: at most 4 shared slots).
 *   - Otherwise U = the shared slots holding KB_ID_NONE on at least one side. Each side is partitioned by its rows' bound-masks over U
 *     (two more `other` launches), and every pair of non-empty mask groups (mL, mR) is joined as kb_hash_join joins, on the key (shared
 *     slots outside U) ∪ (U ∩ mL ∩ mR) — an empty key is the cartesian product of the two groups, limited to 2^28 rows per pair. The
 *     output is then written from the pairs' row indices (one coalesce launch per non-empty pair, timed together in `other`).
 * Refused before any output exists (*out untouched): |U| > 4 (more than 256 mask pairs), a join key of more than 4 slots, more than
 * KB_MAX_COLS output columns, a relation of 2^32 rows or more, an output of 2^32 rows or more (KB_E_LIMIT). */
KB_API kb_status kb_natural_join(kb_ctx* ctx, const kb_rel* left, const kb_rel* right, kb_rel** out);
/* BindJoin of a relation with ONE store pattern (engine.rs:840-885): natural join of `left` with the pattern's matches. With a valid store
 * index, the pattern (?x P ?y) and exactly one of its variables bound by `left` through a unique dense column of the predicate, it is
 * one probe kernel against the index's persistent table (the reference's spo[x][P] / pos[P][y] lookups); otherwise scan + hash join. */
KB_API kb_status kb_bind_join(kb_ctx* ctx, const kb_rel* left, const kb_pattern* pattern, kb_rel** out);
/* Quoted-triple scan: the bag resolve_quoted_triple_scan returns (engine.rs:1111-1188). Every table entry that match_term accepts
 * (engine.rs:1088-1107; constants by id, a variable binds on first use and must be equal afterwards, within and across both inner
 * patterns) fills the quoted position(s) of `outer`; with subject AND object quoted, ONE entry must satisfy both inner patterns and fills
 * both positions (engine.rs:1135-1163). The outer pattern is then matched with the bindings merged; rows whose shared variables conflict
 * are dropped. Columns: one per distinct variable, in order of first appearance when the pattern is read s, p, o with each quoted term
 * inlined as its own s, p, o. Row order is unspecified (the reference's is HashMap order). No table loaded, or no entry matching ->
 * 0 rows. `outer` must quote its subject or its object (otherwise KB_E_INVALID: use kb_scan).
 * Work: ONE streaming pass over the table (the match kernel, counted in kb_stats' `scan` family) yields (entry id, inner variables);
 * the outer pattern with a fresh variable in the quoted position(s) is then bind-joined to it exactly as kb_bind_join does — with a
 * valid index, (q P ?o) and a unique, dense subject column of quoted ids, that is one probe launch — and the fresh variable projected away. */
KB_API kb_status kb_scan_quoted(kb_ctx* ctx, const kb_quoted_pattern* qp, kb_rel** out);
/* StarJoin (engine.rs:587-691) and bind-join chains on one variable (engine.rs:840-885): fused scan + build + probe.
 * Every pattern must contain join_slot. `filter` (nullable) is applied to the joined rows (engine.rs:73-85);
 * conjuncts that touch one pattern only are pushed into the scan. Result caps of the reference (quirk Q1) are NOT applied. */
KB_API kb_status kb_star_join(kb_ctx* ctx, uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats,
                              const kb_filter_op* filter, uint32_t n_filter_ops, kb_rel** out);
/* Whole BGP: the bag of rows of the patterns' natural join, with one column per distinct variable in order of first appearance
 * over the patterns; then FILTER (conjuncts over one pattern's variables are applied while that pattern is read, the rest to the
 * joined rows), then projection (NULL = all variables). Row order is unspecified. Two routes:
 *   star        at most KB_MAX_PATTERNS patterns and one variable shared by every pattern: kb_star_join (optimizer.rs:84-152).
 *   components  every other BGP of 1..KB_BGP_MAX_PATTERNS patterns. The patterns are scanned (fused groups of KB_MAX_PATTERNS; index
 *               lookups with a valid index); an empty pattern ends the call with an empty result. They are split into connected
 *               components over shared variables (a pattern without variables is a component of its own). A component of three
 *               or more patterns is first reduced on the device: every variable held by two or more of its patterns keeps a bitmap
 *               over the store's id range of the values all of them hold, and each round drops the rows that a bitmap rejects
 *               (ids beyond the bitmap, such as quoted ids, are kept) until no relation shrinks, at most one round per pattern.
 *               Inside a component only patterns that share a variable are joined: along the GYO join tree when the component is
 *               acyclic, starting at its smallest relation and adding the smallest tree neighbour; otherwise adding the smallest
 *               relation that shares a variable with the rows so far. The components are then cross-joined, smallest first.
 * Limits: more than KB_BGP_MAX_PATTERNS patterns or more than KB_MAX_COLS variables -> KB_E_LIMIT; a cartesian product of more
 * than 2^28 rows, which only a cross join between components forms -> KB_E_LIMIT. kb_bgp_last_plan describes the call. The
 * reduction's launches and device time count in kb_stats' `filter` family. */
#define KB_BGP_MAX_PATTERNS 16
KB_API kb_status kb_bgp_execute(kb_ctx* ctx, const kb_pattern* pats, uint32_t n_pats,
                                const kb_filter_op* filter, uint32_t n_filter_ops,
                                const uint32_t* project_slots, uint32_t n_project, kb_rel** out);
/* What the context's last successful kb_bgp_execute did. Arrays are indexed by pattern (k < n_patterns), by component
 * (c < n_components) or by join step. Star route: n_components = 1 and only route / n_patterns / rows_unprojected are set. */
enum kb_bgp_route { KB_BGP_NONE = 0, KB_BGP_STAR = 1, KB_BGP_COMPONENTS = 2 };
typedef struct kb_bgp_plan_info {
    uint32_t route;                                   /* kb_bgp_route */
    uint32_t n_patterns, n_components;
    uint32_t component[KB_BGP_MAX_PATTERNS];          /* component of pattern k (components in the order of their first pattern) */
    uint32_t acyclic[KB_BGP_MAX_PATTERNS];            /* per component: 1 when GYO reduces it (its joins follow the join tree) */
    uint32_t reduce_rounds[KB_BGP_MAX_PATTERNS];      /* per component: domain-reduction rounds run (0: not reduced) */
    uint64_t rows_scanned[KB_BGP_MAX_PATTERNS];       /* rows of pattern k after its scan */
    uint64_t rows_reduced[KB_BGP_MAX_PATTERNS];       /* rows of pattern k after the reduction (= rows_scanned when not reduced) */
    uint32_t join_order[KB_BGP_MAX_PATTERNS];         /* patterns in the order they were joined, component by component (not set
                                                         when a pattern's relation is empty: the call returns before any join) */
    uint64_t component_rows[KB_BGP_MAX_PATTERNS];     /* per component: rows of its join */
    uint64_t component_max_rows[KB_BGP_MAX_PATTERNS]; /* per component: the largest relation among its joins' outputs */
    uint32_t cross_order[KB_BGP_MAX_PATTERNS];        /* components in the order they were cross-joined */
    uint64_t reduce_bytes;                            /* the reduction's modelled HBM bytes: 4 per column and row read, 4 per column and row written */
    uint64_t reduce_bit_ops;                          /* the reduction's bitmap operations: one probe (filtering rounds) and one atomicOr per row and reduced variable */
    uint64_t max_intermediate;                        /* the largest join output of the call, cross joins included */
    uint64_t rows_unprojected;                        /* rows before projection */
} kb_bgp_plan_info;
KB_API kb_status kb_bgp_last_plan(kb_ctx* ctx, kb_bgp_plan_info* out);
/* GROUP BY + aggregates (execute_query.rs:1150-1227) */
KB_API kb_status kb_group_aggregate(kb_ctx* ctx, const kb_rel* in, const uint32_t* group_slots, uint32_t n_group,
                                    const kb_agg* aggs, uint32_t n_aggs, kb_groups** out);
KB_API kb_status kb_groups_info(const kb_groups* g, uint64_t* n_groups, uint32_t* n_group_cols, uint32_t* n_aggs);
KB_API kb_status kb_groups_keys(const kb_groups* g, uint32_t col, const uint32_t** keys);   /* host pointer, n_groups */
KB_API kb_status kb_groups_values(const kb_groups* g, uint32_t agg, const double** values); /* host pointer, n_groups */
KB_API kb_status kb_groups_counts(const kb_groups* g, const uint64_t** counts);            /* rows per group */
KB_API void kb_groups_free(kb_groups* g);
/* Cross-rank GROUP BY (one process per GPU, store sharded by subject): every rank aggregates its shard, serialises the partial result
 * with kb_groups_pack (dst == NULL: *bytes = size needed), the host layer gathers the buffers (NCCL / any all-gather), and
 * kb_groups_merge folds them on the device: counts and SUM/AVG accumulators add, MIN/MAX fold, AVG = total sum / total count —
 * the aggregate of execute_query.rs:1150-1227 over the union of the shards' rows. */
KB_API kb_status kb_groups_pack(const kb_groups* g, void* dst, uint64_t capacity_bytes, uint64_t* bytes);
KB_API kb_status kb_groups_merge(kb_ctx* ctx, const void* const* parts, const uint64_t* part_bytes, uint32_t n_parts, kb_groups** out);
/* StarJoin + GROUP BY in one call (the aggregate of execute_query.rs:1150-1227 over the rows of engine.rs:587-691). With the store
 * index valid, one GROUP BY variable and at most one aggregate, the grouping is folded into the probe kernel and no joined row is
 * ever written; every other shape = kb_star_join followed by kb_group_aggregate. *n_rows (nullable) receives the joined row count. */
KB_API kb_status kb_star_join_aggregate(kb_ctx* ctx, uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter,
                                        uint32_t n_filter_ops, const uint32_t* group_slots, uint32_t n_group, const kb_agg* aggs, uint32_t n_aggs,
                                        kb_groups** out, uint64_t* n_rows);

/* ------------------------------------------------------------------ prepared star joins: resolve once, launch many times.
 * The reference optimises a query into a PhysicalOperator once and executes it per call (engine.rs:54); here the per-call work of the
 * synchronous operators — pattern/filter marshalling, cudaMallocAsync of the result, the stream synchronisation after the launch — is
 * what limits a 0.1 ms query, so a plan keeps the resolved launch and a ring of `ring` pre-allocated result buffers:
 *   kb_plan_submit   ONE kernel launch (asynchronous; no allocation, no host synchronisation), returns a ticket
 *   kb_plan_collect  waits for exactly that launch; *n_rows = joined rows; *rows (nullable) = a VIEW of the ring slot (kb_rel_free it;
 *                    its columns stay valid until `ring` further submits reuse the slot); *groups (nullable) = the GROUP BY result of
 *                    a grouped plan (kb_groups_free it).
 * Only queries that take the one-kernel index path can be prepared (kb_store_build_index done; every pattern (?s P ?o) whose key
 * column has a persistent table): anything else -> KB_E_UNSUPPORTED, use the synchronous operators. n_group = 0: rows are produced;
 * n_group = 1 and n_aggs <= 1: GROUP BY folded into the kernel as in kb_star_join_aggregate (fixed 4096-group table; more groups ->
 * KB_E_LIMIT from kb_plan_collect). A plan is bound to the store / index / numeric-table version it was prepared on: after any
 * mutation kb_plan_submit returns KB_E_INVALID ("stale plan"). Submitting while the ring slot's previous ticket is uncollected ->
 * KB_E_LIMIT. Row order and bag of rows are those of kb_star_join. */
typedef struct kb_plan kb_plan;
KB_API kb_status kb_star_join_prepare(kb_ctx* ctx, uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter,
                                      uint32_t n_filter_ops, const uint32_t* group_slots, uint32_t n_group, const kb_agg* aggs, uint32_t n_aggs,
                                      uint32_t ring, kb_plan** out);
KB_API kb_status kb_plan_submit(kb_ctx* ctx, kb_plan* plan, uint64_t* ticket);
KB_API kb_status kb_plan_collect(kb_ctx* ctx, kb_plan* plan, uint64_t ticket, uint64_t* n_rows, kb_rel** rows, kb_groups** groups);
KB_API kb_status kb_plan_info(const kb_plan* plan, uint32_t* ring, uint64_t* capacity_rows, uint32_t* n_cols, uint32_t* slots /* [KB_MAX_COLS] or NULL */,
                              uint32_t* grouped);
KB_API void kb_plan_free(kb_ctx* ctx, kb_plan* plan);
/* Cross-rank GROUP BY inside the plan (one process per GPU, store sharded by subject): every rank allocates
 * kb_plan_peer_scratch_bytes(plan) bytes of ZEROED peer-mapped memory (torch symmetric memory, cudaIpc, VMM), exchanges the addresses and
 * attaches them before the first submit (ring >= 2, same plan on every rank). A submit then runs, on the library's stream and without
 * any host round trip: the fused join+group kernel (partial table into the own scratch) -> a device-side barrier over peer-memory
 * flags -> ONE merge kernel that reads all ranks' partial tables over NVLink and folds them; kb_plan_collect returns the GLOBAL groups
 * on every rank (*n_rows stays the rank's own joined rows). All ranks must submit the same number of queries. */
KB_API uint64_t kb_plan_peer_scratch_bytes(const kb_plan* plan);
KB_API kb_status kb_plan_attach_peers(kb_ctx* ctx, kb_plan* plan, uint32_t rank, uint32_t world, void* const* peer_scratch /* [world] */);

/* ------------------------------------------------------------------ Datalog (Reasoner::infer_with_strategy, infer_generic.rs:27-53)
 * Facts = the ctx store. Inferred facts are appended to the store (segment tag KB_TAG_INFERRED), exactly as the
 * reference inserts them into its index (infer_generic.rs:46), and returned as a 3-column relation (slots 0,1,2 = s,p,o).
 * Unsupported rule shapes (variable predicate in a premise, unbound head variable — SURVEY quirks Q6/Q8) -> KB_E_UNSUPPORTED. */
#define KB_TAG_INFERRED 0xFFFFFFFFFFFFFFF0ull
KB_API kb_status kb_datalog_fixpoint(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy,
                                     kb_rel** inferred, kb_fixpoint_stats* stats);
/* Incremental materialisation. The store is closed under `rules` already (an earlier kb_datalog_fixpoint[_seed] with the same rules, and
 * nothing deleted since); `seed` (3 columns, slots 0,1,2 = s,p,o; not yet in the store) are facts to ADD. The seed facts the store does
 * not hold yet are accepted and become the first delta; everything the store held is OLD, so the rounds join the delta alone against
 * the store instead of the store against itself — the closure Reasoner::add_abox_triple + infer_new_facts_semi_naive reach by
 * starting over (semi_naive.rs:89; per window slide: simple_r2r.rs:95-128). `*out` = the *n_seed_new accepted seed facts, then the
 * facts inferred from them (stats->inferred); both are appended to the store (tag KB_TAG_INFERRED). Duplicates inside the seed are
 * accepted once. Seed facts whose predicate no rule mentions are not looked at (load them with kb_store_append). The sharded
 * fixpoint (kolibrie_b200/dist.py) feeds the facts derived on other ranks through this call. */
KB_API kb_status kb_datalog_fixpoint_seed(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy, const kb_rel* seed,
                                          kb_rel** out, uint64_t* n_seed_new, kb_fixpoint_stats* stats);

/* Sliding-window maintenance of the closure by delete-and-rederive: what a window firing with rules reaches by evicting the previous
 * window, adding the current one and materialising from scratch (rsp_engine.rs:94-109, simple_r2r.rs:103-128), reached from the slide.
 *   B  = the distinct triples of every segment whose tag is not KB_TAG_INFERRED, I = the triples of the KB_TAG_INFERRED segments,
 *   B' = the segments left after the `evict_tags` segments are dropped, plus `add` (all taken as sets).
 * Precondition: I = closure(B) \ B under the same rules and closure semantics. The context records a "closed" token (store version,
 * numeric-table version, the rules byte for byte, a hash-join strategy) when kb_datalog_fixpoint (on a store without inferred segments,
 * strategy other than KB_SEMI_NAIVE_PARALLEL) or kb_datalog_maintain returns KB_OK; any other store mutation, other rules or
 * kb_datalog_fixpoint_seed (its seed facts are stored as KB_TAG_INFERRED) void it -> KB_E_INVALID ("store not closed under these
 * rules: run kb_datalog_fixpoint"). kb_dict_numeric_load voids it only when a rule filter compares numbers (a constant right-hand side,
 * or a variable no premise binds): other rules have the same closure whatever the numeric table holds.
 * Postcondition: the evicted segments are gone; `add` (nullable; 3 columns, slots 0,1,2 = s,p,o) is ONE new segment tagged add_tag,
 * stored as kb_store_append_device stores it; the KB_TAG_INFERRED segments are replaced by one segment holding closure(B') \ B', each
 * fact once (none when that set is empty; an unchanged single segment is kept). *inferred_removed = I \ I', *inferred_added = I' \ I
 * (nullable; 3 columns, every fact once). A base fact that is still derivable after it left the base moves into I'; a fact of `add` that
 * was inferred moves to the base; a fact that an evicted segment and a surviving segment (or `add`) both hold does not move.
 * KB_SEMI_NAIVE, KB_SEMI_NAIVE_OLD_DELTA and KB_NAIVE share one closure (hash-join premises, quirks Q6/Q7); KB_SEMI_NAIVE_PARALLEL ->
 * KB_E_UNSUPPORTED; rule shapes kb_datalog_fixpoint refuses are refused. n_evict = 0 and add = NULL: no-op, empty outputs.
 * Errors before anything changes (the store is untouched): unknown tag -> KB_E_NOT_FOUND; KB_TAG_INFERRED in evict_tags or as add_tag,
 * a bad `add`, a stale token -> KB_E_INVALID. A CUDA / out-of-memory error while the result is computed leaves the store as it was
 * (still closed); one while the store is rewritten leaves exactly the B' segments, no inferred segment and no token: run
 * kb_datalog_fixpoint to restore the precondition. A valid store index stays valid (maintained in place, as by kb_store_evict /
 * kb_store_append_device). The base counts (base_removed, base_added) cover the predicates the rules mention: the facts of other
 * predicates take no part in the closure. */
typedef struct kb_maintain_stats {
    uint64_t base_removed;      /* distinct facts that left the base set */
    uint64_t base_added;        /* distinct facts of `add` that were not base facts before the call */
    uint64_t overdeleted;       /* facts removed by the over-deletion phase, not counting the base_removed facts themselves */
    uint64_t rederived;         /* over-deleted or removed facts that the rederivation phase found still derivable */
    uint64_t inferred_removed;  /* rows of *inferred_removed */
    uint64_t inferred_added;    /* rows of *inferred_added */
    uint64_t derivations;       /* candidate head instances over all phases (compare kb_fixpoint_stats.derivations of a closure from scratch) */
    uint32_t overdelete_rounds, insert_rounds;
    double device_ms;
} kb_maintain_stats;
KB_API kb_status kb_datalog_maintain(kb_ctx* ctx, const kb_rule* rules, uint32_t n_rules, uint32_t strategy,
                                     const uint64_t* evict_tags, uint32_t n_evict,
                                     const kb_rel* add /* nullable; 3 columns, slots 0,1,2 = s,p,o */, uint64_t add_tag,
                                     kb_rel** inferred_removed /* nullable */, kb_rel** inferred_added /* nullable */,
                                     kb_maintain_stats* stats /* nullable */);

/* ------------------------------------------------------------------ Relation-to-Stream operators (Relation2StreamOperator,
 * kolibrie/src/rsp/r2s.rs:24-58), applied to every firing's result (rsp_engine.rs:349-360): the result stays in device memory and only
 * the rows that changed are emitted.
 * State. The operator holds `last`: the distinct rows of the previous ISTREAM/DSTREAM evaluation. It starts empty and lives in device
 *   memory owned by the operator. It holds ids only, so store mutations, index rebuilds and dictionary reloads do not affect it. It must
 *   be freed before its context is destroyed.
 * Rows. A row is the tuple of a response's columns, taken in the order of `slots` given at create time. `response` must have exactly
 *   that slot set, though its columns may come in any order; otherwise the call returns KB_E_INVALID and the state is unchanged.
 *   - Equality is equality of u32 ids. It equals the reference's equality of `Vec<(String,String)>` sorted by variable name, because the
 *     dictionary is a bijection.
 *   - `n_cols` is 1..KB_MAX_COLS.
 *   - A response with 0 rows is valid.
 *   - ISTREAM and DSTREAM emit their rows with the columns in the order of `slots`.
 * RSTREAM. `emitted` is a zero-copy view of `response`, as kb_project gives one. `last` is not touched, as in r2s.rs:39.
 * ISTREAM. `emitted` holds every row of `response` whose tuple is not in `last`.
 *   - It follows response order, and duplicates are kept: a bag row that is new is emitted once per occurrence (r2s.rs:41-44).
 *   - Then `last` becomes the distinct rows of `response`.
 * DSTREAM. `emitted` holds every row of `last` whose tuple is not in `response`, each row once.
 *   - Its order is the order of the row's first occurrence in the response that set `last`. The reference leaves this order unspecified
 *     (HashSet iteration, r2s.rs:50); pinning it makes the device deterministic.
 *   - Then `last` becomes the distinct rows of `response`.
 * Errors.
 *   - More than 2^32-1 response rows: KB_E_LIMIT.
 *   - A CUDA or out-of-memory error: `last` is exactly what it was before the call (the new state is built in fresh buffers and swapped
 *     in only on success).
 * kb_r2s_info: *last_rows = distinct rows held, *stream_op = the operator (either pointer may be NULL). */
enum kb_stream_op { KB_RSTREAM = 0, KB_ISTREAM = 1, KB_DSTREAM = 2 }; /* r2s.rs:15-17 */
typedef struct kb_r2s kb_r2s;
KB_API kb_status kb_r2s_create(kb_ctx* ctx, uint32_t stream_op, const uint32_t* slots, uint32_t n_cols, kb_r2s** out);
KB_API kb_status kb_r2s_eval(kb_ctx* ctx, kb_r2s* op, const kb_rel* response, kb_rel** emitted);
KB_API kb_status kb_r2s_info(const kb_r2s* op, uint64_t* last_rows, uint32_t* stream_op);
KB_API void kb_r2s_free(kb_ctx* ctx, kb_r2s* op);

/* ------------------------------------------------------------------ multi-GPU helpers (one process per GPU; the host layer
 * runs the NCCL all-to-all between kb_partition and kb_rel_from_device) */
/* Shard function (host and device agree): block-cyclic on the dictionary id, (key >> KB_SHARD_BLOCK_BITS) % n_shards. Dictionary ids
 * are dense (shared/src/dictionary.rs:32-48), so this balances like a hash AND keeps every shard's key domain dense: a shard's keys
 * compact to ((key >> B) / n) << B | (key & (2^B - 1)), which keeps the direct join tables as small on N GPUs as on one. */
#define KB_SHARD_BLOCK_BITS 10
KB_API uint32_t kb_shard_of(uint32_t key, uint32_t n_shards);
/* tell the context that its store holds shard `rank` of `world` (sharded by subject): enables the key compaction above */
KB_API kb_status kb_set_sharding(kb_ctx* ctx, uint32_t rank, uint32_t world);
/* split `in` by kb_shard_of(row[key_slot], n_parts) into n_parts contiguous ranges of ONE output relation;
 * part_offsets[n_parts+1] (host) receives the row offsets. */
KB_API kb_status kb_partition(kb_ctx* ctx, const kb_rel* in, uint32_t key_slot, uint32_t n_parts, kb_rel** out, uint64_t* part_offsets);
/* The same exchange FUSED with its transfer (SURVEY.md 8e "fused peer stores from the partition kernel"): every row is written straight
 * into the receive buffer of the rank that owns its key, over NVLink peer memory, instead of partition + all-to-all.
 * kb_partition_counts: rows of `r` per destination. The caller exchanges the counts (a world x world matrix of integers), derives
 * base[d] = first row of this rank's range in rank d's receive buffer, and passes peer_cols[d * n_cols + c] = device-visible address
 * of column c of rank d's receive buffer (peer-mapped memory, e.g. torch symmetric memory or cudaIpc). The call returns when this
 * rank's stores have been issued and fenced system-wide; a barrier across ranks must follow before the buffers are read. */
KB_API kb_status kb_partition_counts(kb_ctx* ctx, const kb_rel* r, uint32_t key_slot, uint32_t n_parts, uint64_t* counts /* [n_parts] */);
KB_API kb_status kb_shuffle_scatter(kb_ctx* ctx, const kb_rel* r, uint32_t key_slot, uint32_t n_parts, uint32_t* const* peer_cols /* [n_parts * n_cols] */,
                                    const uint64_t* base /* [n_parts] */, uint64_t capacity_rows);
/* The same without the count pass and without any count exchange: peer_cursors[d] = device-visible address of a u32 cursor that rank d
 * owns (peer-mapped, zeroed by d before the exchange, and a barrier across ranks before anybody pushes). A tile's rows for d are
 * appended where an atomicAdd on d's cursor reserves them, so after the barrier that follows the call every rank reads how many rows
 * it received from its OWN cursor. Rows of different senders interleave (a relation is a bag). */
KB_API kb_status kb_shuffle_push(kb_ctx* ctx, const kb_rel* r, uint32_t key_slot, uint32_t n_parts, uint32_t* const* peer_cols /* [n_parts * n_cols] */,
                                 uint32_t* const* peer_cursors /* [n_parts] */, uint64_t capacity_rows);
/* a relation over columns the CALLER owns (e.g. a shuffle's receive buffer): no copy. Every column must be 16-byte aligned, stay
 * allocated while the relation is in use and be readable up to the next multiple of 256 bytes past its last row (TMA tile loads). */
KB_API kb_status kb_rel_wrap_device(kb_ctx* ctx, const uint32_t* slots, uint32_t n_cols, uint32_t* const* d_cols, uint64_t n_rows, kb_rel** out);
KB_API kb_status kb_rel_from_device(kb_ctx* ctx, const uint32_t* slots, uint32_t n_cols, const uint32_t* const* d_cols, uint64_t n_rows, kb_rel** out);
KB_API kb_status kb_store_download(kb_ctx* ctx, uint32_t* s, uint32_t* p, uint32_t* o, uint64_t cap, uint64_t* n);

/* ------------------------------------------------------------------ on-disk columnar segments (the device store's layout on disk; the
 * reference persists SSTables of triples, kolibrie/src/disk_storage/sstable.rs:40-85). File = one 4096-byte header (triple count, tag,
 * id range and checksum of each column) + the s, p, o columns, each starting at a 4096-byte boundary.
 * kb_segment_write / kb_segment_info are host-only (no device needed). kb_segment_save writes the store segment(s) tagged `tag` (or
 * the whole store when whole_store != 0). kb_store_append_file streams a file into a NEW store segment tagged `tag` through two
 * pinned staging buffers (file reads overlap the host->device copies); the header's column ranges replace the load-time statistics
 * kernels; verify != 0 checks the column checksums while reading. The store index is maintained as for kb_store_append. */
KB_API kb_status kb_segment_write(const char* path, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t tag);
KB_API kb_status kb_segment_info(const char* path, uint64_t* n_triples, uint64_t* tag, uint32_t* cmin /* [3] or NULL */, uint32_t* cmax /* [3] or NULL */);
KB_API kb_status kb_segment_save(kb_ctx* ctx, uint64_t tag, int whole_store, const char* path);
KB_API kb_status kb_store_append_file(kb_ctx* ctx, const char* path, uint64_t tag, int verify);

/* ------------------------------------------------------------------ one-shot host-buffer entries (end-to-end measurement and the
 * reference's per-call GPU usage, sparql_database.rs:3193-3353): upload (chunked, overlapped with the scan), star-join, download.
 * The store of ctx is REPLACED by the uploaded triples (and is left empty when the call fails). Patterns and filter are validated
 * before the upload starts; on every return path the caller's input buffers are no longer read.
 * kb_star_join_host: result columns cols[0 .. *n_cols) are malloc'd by the callee and owned by the caller (free()); whatever cols[]
 * held on entry is ignored and entries past *n_cols are set to NULL. */
KB_API kb_status kb_star_join_host(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n,
                                   uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats,
                                   const kb_filter_op* filter, uint32_t n_filter_ops,
                                   uint32_t* n_cols, uint32_t* slots /* [KB_MAX_COLS] */, uint32_t** cols /* [KB_MAX_COLS] */, uint64_t* n_rows);
/* same, into CALLER-provided buffers (e.g. pinned memory): cols[c] must hold capacity_rows rows for every result column (one per
 * distinct variable of the patterns, at most KB_MAX_COLS); a result larger than capacity_rows -> KB_E_LIMIT with *n_rows = its size. */
KB_API kb_status kb_star_join_host_into(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n,
                                        uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats,
                                        const kb_filter_op* filter, uint32_t n_filter_ops,
                                        uint32_t* n_cols, uint32_t* slots /* [KB_MAX_COLS] */, uint32_t* const* cols /* [KB_MAX_COLS] */,
                                        uint64_t capacity_rows, uint64_t* n_rows);

#ifdef __cplusplus
}
#endif
#endif /* KOLIBRIE_B200_H */
