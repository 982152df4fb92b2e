//! Raw bindings of include/kolibrie_b200.h (one declaration per exported entry point; layouts checked by tests/test_abi.py on the C side).
#![allow(non_camel_case_types, dead_code)]
use std::os::raw::{c_char, c_double, c_int, c_void};

pub type kb_status = i32;
pub const KB_OK: kb_status = 0;
pub const KB_E_INVALID: kb_status = -1;
pub const KB_E_CUDA: kb_status = -2;
pub const KB_E_OOM: kb_status = -3;
pub const KB_E_UNSUPPORTED: kb_status = -4;
pub const KB_E_NOT_FOUND: kb_status = -5;
pub const KB_E_LIMIT: kb_status = -6;
pub const KB_ID_NONE: u32 = 0xFFFF_FFFF;
pub const KB_MAX_COLS: usize = 16;
pub const KB_TAG_INFERRED: u64 = 0xFFFF_FFFF_FFFF_FFF0;
pub const KB_TERM_QUOTED: u32 = 2;
pub const KB_QUOTED_MAX_DEPTH: u32 = 16;
pub const KB_QUOTED_MAX_SLOTS: u32 = 1 << 28;

#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbTerm { pub is_var: u32, pub value: u32 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbPattern { pub s: KbTerm, pub p: KbTerm, pub o: KbTerm }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbQuotedPattern { pub outer: KbPattern, pub inner_s: KbPattern, pub inner_o: KbPattern }
pub type kb_quoted_pattern = KbQuotedPattern;  // (the header's name, as the declaration below spells it)
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbFilterOp { pub op: u32, pub slot: u32, pub cmp: u32, pub id: u32, pub value: c_double }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbAgg { pub kind: u32, pub slot: u32 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbRuleFilter { pub lhs_slot: u32, pub cmp: u32, pub rhs_is_var: u32, pub rhs_slot: u32, pub rhs_value: c_double }
#[repr(C)] pub struct KbRule { pub premise: *const KbPattern, pub n_premise: u32, pub filters: *const KbRuleFilter, pub n_filters: u32,
                              pub conclusion: *const KbPattern, pub n_conclusion: u32 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbStats { pub scan_ms: c_double, pub build_ms: c_double, pub probe_ms: c_double, pub filter_ms: c_double,
    pub group_ms: c_double, pub other_ms: c_double, pub total_ms: c_double, pub scan_launches: u64, pub build_launches: u64, pub probe_launches: u64,
    pub filter_launches: u64, pub group_launches: u64, pub other_launches: u64, pub rows_scanned: u64, pub rows_built: u64, pub rows_probed: u64,
    pub rows_out: u64, pub h2d_bytes: u64, pub d2h_bytes: u64, pub kernel_launches: u64, pub fused_scan_builds: u64, pub index_joins: u64 }
#[repr(C)] pub struct KbFixpointStats { pub rounds: u32, pub inferred: u64, pub derivations: u64, pub round_new: [u64; 64], pub device_ms: c_double }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbMaintainStats { pub base_removed: u64, pub base_added: u64, pub overdeleted: u64, pub rederived: u64,
    pub inferred_removed: u64, pub inferred_added: u64, pub derivations: u64, pub overdelete_rounds: u32, pub insert_rounds: u32, pub device_ms: c_double }
pub type kb_maintain_stats = KbMaintainStats;  // (the header's name, as the declaration below spells it)
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbBcStats { pub rounds: u32, pub reached_fixpoint: u32, pub stopped_early: u32,
    pub relevant_rules: u32, pub demand_patterns: u32, pub restricted_predicates: u32, pub base_facts: u64, pub derived: u64, pub derivations: u64,
    pub answers: u64, pub device_ms: c_double }
pub type kb_bc_stats = KbBcStats;  // (the header's name, as the declaration below spells it)
pub const KB_BC_MAX_DEPTH: u32 = 10; pub const KB_BC_DEPTH_LIMIT: u32 = 64;
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbRepairStats { pub constraints: u32, pub subsets_probed: u32, pub matches: u64,
    pub conflicts: u64, pub minimal_conflicts: u64, pub conflicted_facts: u64, pub answers: u64, pub device_ms: c_double, pub match_ms: c_double,
    pub conflict_ms: c_double, pub answer_ms: c_double }
pub type kb_repair_stats = KbRepairStats;  // (the header's name, as the declaration below spells it)
#[repr(C)] #[derive(Clone, Copy, Debug)] pub struct KbBindSpec { pub function: u32, pub n_args: u32, pub args: *const KbTerm, pub n_const: u32,
    pub const_offsets: *const u64, pub const_bytes: *const u8, pub out_slot: u32, pub next_qt_id: u32 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbBindInfo { pub n_rows: u64, pub n_unbound: u64, pub dict_first: u32, pub dict_new: u32,
    pub quoted_first: u32, pub quoted_new: u32 }
pub type kb_bind_spec = KbBindSpec;  // (the header's names, as the declarations below spell them)
pub type kb_bind_info = KbBindInfo;
// kb_bind_function (engine.rs:144-277)
pub const KB_BIND_SUBJECT: u32 = 1; pub const KB_BIND_PREDICATE: u32 = 2; pub const KB_BIND_OBJECT: u32 = 3; pub const KB_BIND_IS_TRIPLE: u32 = 4;
pub const KB_BIND_TRIPLE: u32 = 5; pub const KB_BIND_CONCAT: u32 = 6;
pub const KB_BIND_MAX_ARGS: u32 = 16;
// kb_dict_numeric_derive: the side tables derived on the device from the device dictionary's strings
pub const KB_NUMERIC_F64: u32 = 1; pub const KB_NUMERIC_I32: u32 = 2; pub const KB_NUMERIC_APPEND: u32 = 0xFFFF_FFFF;
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbNumericInfo { pub n_ids: u32, pub n_derived: u32, pub n_numeric: u32, pub n_i32: u32, pub n_slow: u32 }
pub type kb_numeric_info = KbNumericInfo;  // (the header's name, as the declaration below spells it)
// kb_values (engine.rs:279-308) and kb_hash_join_keyed's merge policy
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbValuesInfo { pub dict_first: u32, pub dict_new: u32, pub rows_dropped: u64 }
pub type kb_values_info = KbValuesInfo;  // (the header's name, as the declaration below spells it)
pub const KB_MERGE_LEFT_FIRST: u32 = 0; pub const KB_MERGE_RIGHT_FIRST: u32 = 1;
// kb_bgp_execute: up to 16 patterns; kb_bgp_last_plan describes the last call (kb_bgp_route)
pub const KB_BGP_MAX_PATTERNS: usize = 16;
pub const KB_BGP_NONE: u32 = 0; pub const KB_BGP_STAR: u32 = 1; pub const KB_BGP_COMPONENTS: u32 = 2;
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbBgpPlanInfo { pub route: u32, pub n_patterns: u32, pub n_components: u32,
    pub component: [u32; KB_BGP_MAX_PATTERNS], pub acyclic: [u32; KB_BGP_MAX_PATTERNS], pub reduce_rounds: [u32; KB_BGP_MAX_PATTERNS],
    pub rows_scanned: [u64; KB_BGP_MAX_PATTERNS], pub rows_reduced: [u64; KB_BGP_MAX_PATTERNS], pub join_order: [u32; KB_BGP_MAX_PATTERNS],
    pub component_rows: [u64; KB_BGP_MAX_PATTERNS], pub component_max_rows: [u64; KB_BGP_MAX_PATTERNS], pub cross_order: [u32; KB_BGP_MAX_PATTERNS],
    pub reduce_bytes: u64, pub reduce_bit_ops: u64, pub max_intermediate: u64, pub rows_unprojected: u64 }
pub type kb_bgp_plan_info = KbBgpPlanInfo;  // (the header's name, as the declaration below spells it)
// kb_order_by: ORDER BY + LIMIT over a device relation (kb_order_route, kb_order_kind)
pub const KB_ORDER_VIEW: u32 = 0; pub const KB_ORDER_SORT: u32 = 1; pub const KB_ORDER_TOPK: u32 = 2;
pub const KB_ORDER_CONST: u32 = 0; pub const KB_ORDER_NUMERIC: u32 = 1; pub const KB_ORDER_STRING: u32 = 2;
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbOrderKey { pub slot: u32, pub descending: u32 }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbOrderInfo { pub n_rows_in: u64, pub n_rows_out: u64, pub route: u32,
    pub key_kind: [u32; KB_MAX_COLS], pub n_distinct: [u32; KB_MAX_COLS], pub string_rounds: [u32; KB_MAX_COLS] }
pub type kb_order_key = KbOrderKey;  // (the header's names, as the declaration below spells them)
pub type kb_order_info = KbOrderInfo;
// kb_serialize_begin / _next / _free: the store as N-Triples-star or Turtle-star text (kb_serialize_format)
pub const KB_SER_NTRIPLES: u32 = 0; pub const KB_SER_TURTLE: u32 = 1;
pub const KB_SER_STAGING_BYTES: u64 = 256 << 20;
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbSerializeInfo { pub n_triples: u64, pub total_bytes: u64, pub max_unit_bytes: u64,
    pub n_subject_groups: u64, pub n_terms: u32, pub rank_rounds: u32, pub phase_ms: [c_double; 4] }
pub type kb_serialize_info = KbSerializeInfo;  // (the header's name, as the declaration below spells it)
pub enum KbSerializer {}
pub type kb_serializer = KbSerializer;  // (the header's name, as the declarations below spell it)
// kb_store_gather_stats / kb_db_stats_counts / kb_db_stats_free: DatabaseStats::gather_stats_fast on the device store
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbDbStatsInfo { pub total_triples: u64, pub quoted_triple_count: u64, pub take: u64,
    pub step: u64, pub n_ids: [u64; 3], pub phase_ms: [c_double; 3] }
pub type kb_db_stats_info = KbDbStatsInfo;  // (the header's name, as the declaration below spells it)
pub enum KbDbStats {}
pub type kb_db_stats = KbDbStats;  // (the header's name, as the declarations below spell it)
// kb_qb_triples / kb_qb_terms: QueryBuilder triple queries on the device store
pub const KB_QB_ANY: u32 = 0; pub const KB_QB_EXACT: u32 = 1; pub const KB_QB_CONTAINS: u32 = 2; pub const KB_QB_STARTS: u32 = 3; pub const KB_QB_ENDS: u32 = 4;
pub const KB_QB_ON_SUBJECT: u32 = 1; pub const KB_QB_ON_PREDICATE: u32 = 2; pub const KB_QB_ON_OBJECT: u32 = 4;
pub const KB_QB_TERMS_EMPTY: u32 = 0; pub const KB_QB_TERMS_DROP: u32 = 1; pub const KB_QB_TERMS_DISTINCT: u32 = 2;
pub const KB_QB_PATTERN_MAX: u32 = 4096;
pub const KB_QB_NO_LIMIT: u64 = u64::MAX;
#[repr(C)] #[derive(Clone, Copy, Debug)] pub struct KbQbFilter { pub mode: u32, pub id: u32, pub pattern: *const u8, pub len: u64 }
impl Default for KbQbFilter { fn default() -> Self { Self { mode: KB_QB_ANY, id: 0, pattern: std::ptr::null(), len: 0 } } }
#[repr(C)] #[derive(Clone, Copy, Debug)] pub struct KbQbSpec { pub pos: [KbQbFilter; 3], pub join: u32, pub reserved: u32, pub offset: u64, pub limit: u64 }
impl Default for KbQbSpec { fn default() -> Self { Self { pos: [KbQbFilter::default(); 3], join: 0, reserved: 0, offset: 0, limit: KB_QB_NO_LIMIT } } }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbQbInfo { pub n_raw: u64, pub n_selected: u64, pub n_joined: u64, pub n_rows: u64,
    pub phase_ms: [c_double; 4] }
pub type kb_qb_spec = KbQbSpec;  // (the header's names, as the declarations below spell them)
pub type kb_qb_info = KbQbInfo;

// kb_store_union / kb_store_par_join: SparqlDatabase::union and par_join into a third context
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbUnionInfo { pub n_a: u64, pub n_b: u64, pub n_rows: u64, pub n_terms: u32, pub dict_first: u32,
    pub dict_new: u32, pub reserved: u32, pub phase_ms: [c_double; 5] }
#[repr(C)] #[derive(Clone, Copy, Debug, Default)] pub struct KbParJoinInfo { pub n_a: u64, pub n_b: u64, pub n_join: u64, pub n_semi: u64, pub n_rows: u64,
    pub phase_ms: [c_double; 4] }
pub type kb_union_info = KbUnionInfo;
pub type kb_par_join_info = KbParJoinInfo;

// kb_filter_opcode / kb_cmp / kb_agg_kind / kb_strategy
pub const KB_F_CMP_NUM: u32 = 1; pub const KB_F_EQ_ID: u32 = 2; pub const KB_F_NE_ID: u32 = 3; pub const KB_F_AND: u32 = 4; pub const KB_F_OR: u32 = 5;
pub const KB_F_NOT: u32 = 6; pub const KB_F_PUSH_VAR: u32 = 7; pub const KB_F_PUSH_CONST: u32 = 8; pub const KB_F_ADD: u32 = 9; pub const KB_F_SUB: u32 = 10;
pub const KB_F_MUL: u32 = 11; pub const KB_F_DIV: u32 = 12; pub const KB_F_TRUTHY: u32 = 13; pub const KB_F_IS_TRIPLE: u32 = 14;
pub const KB_CMP_GT: u32 = 1; pub const KB_CMP_GE: u32 = 2; pub const KB_CMP_LT: u32 = 3; pub const KB_CMP_LE: u32 = 4; pub const KB_CMP_EQ: u32 = 5; pub const KB_CMP_NE: u32 = 6;
pub const KB_AGG_COUNT: u32 = 0; pub const KB_AGG_SUM: u32 = 1; pub const KB_AGG_MIN: u32 = 2; pub const KB_AGG_MAX: u32 = 3; pub const KB_AGG_AVG: u32 = 4;
pub const KB_SEMI_NAIVE: u32 = 0; pub const KB_NAIVE: u32 = 1; pub const KB_SEMI_NAIVE_PARALLEL: u32 = 2; pub const KB_SEMI_NAIVE_OLD_DELTA: u32 = 3;

// kb_stream_op (r2s.rs:15-17)
pub const KB_RSTREAM: u32 = 0; pub const KB_ISTREAM: u32 = 1; pub const KB_DSTREAM: u32 = 2;

pub enum KbCtx {} pub enum KbRel {} pub enum KbGroups {} pub enum KbStrings {} pub enum KbPlan {} pub enum KbR2s {}
pub type kb_r2s = KbR2s;  // (the header's name, as the declarations below spell it)

extern "C" {
    pub fn kb_version() -> *const c_char;
    pub fn kb_ctx_create(device: c_int, out: *mut *mut KbCtx) -> kb_status;
    pub fn kb_ctx_destroy(ctx: *mut KbCtx);
    pub fn kb_last_error(ctx: *const KbCtx) -> *const c_char;
    pub fn kb_synchronize(ctx: *mut KbCtx) -> kb_status;
    // store
    pub fn kb_store_load(ctx: *mut KbCtx, s: *const u32, p: *const u32, o: *const u32, n: u64) -> kb_status;
    pub fn kb_store_append(ctx: *mut KbCtx, s: *const u32, p: *const u32, o: *const u32, n: u64, tag: u64) -> kb_status;
    pub fn kb_store_evict(ctx: *mut KbCtx, tag: u64) -> kb_status;
    pub fn kb_store_delete(ctx: *mut KbCtx, s: *const u32, p: *const u32, o: *const u32, n: u64) -> kb_status;
    pub fn kb_store_insert(ctx: *mut KbCtx, s: *const u32, p: *const u32, o: *const u32, n: u64, segment_tag: u64, inserted: *mut u8,
                           n_inserted: *mut u64) -> kb_status;
    pub fn kb_store_remove(ctx: *mut KbCtx, s: *const u32, p: *const u32, o: *const u32, n: u64, removed: *mut u8, n_removed: *mut u64) -> kb_status;
    pub fn kb_store_remove_template(ctx: *mut KbCtx, rel: *const KbRel, tmpl: *const KbPattern, n_tmpl: u32, n_removed: *mut u64) -> kb_status;
    pub fn kb_store_clear(ctx: *mut KbCtx) -> kb_status;
    pub fn kb_store_build_index(ctx: *mut KbCtx, n_predicates: *mut u32, build_ms: *mut c_double) -> kb_status;
    pub fn kb_store_size(ctx: *mut KbCtx, n_triples: *mut u64, n_segments: *mut u32) -> kb_status;
    pub fn kb_dict_numeric_load(ctx: *mut KbCtx, num_or0: *const c_double, is_num: *const u8, n_ids: u32) -> kb_status;
    pub fn kb_dict_strings_load(ctx: *mut KbCtx, offsets: *const u64, bytes: *const u8, n_ids: u32) -> kb_status;
    pub fn kb_dict_numeric_derive(ctx: *mut KbCtx, tables: u32, first_id: u32, info: *mut kb_numeric_info) -> kb_status;
    pub fn kb_dict_numeric_download(ctx: *mut KbCtx, first: u32, n: u32, num_or0: *mut c_double, is_num: *mut u8, val: *mut i32, is_i32: *mut u8) -> kb_status;
    pub fn kb_dict_encode(ctx: *mut KbCtx, offsets: *const u64, bytes: *const u8, n_terms: u64, out_ids: *mut u32, n_new: *mut u32, new_first_pos: *mut u64) -> kb_status;
    pub fn kb_dict_strings_info(ctx: *mut KbCtx, n_ids: *mut u32, n_bytes: *mut u64) -> kb_status;
    pub fn kb_store_append_device(ctx: *mut KbCtx, d_s: *const u32, d_p: *const u32, d_o: *const u32, n: u64, tag: u64) -> kb_status;
    // relations
    pub fn kb_rel_info(r: *const KbRel, n_rows: *mut u64, n_cols: *mut u32, slots: *mut u32) -> kb_status;
    pub fn kb_rel_download(ctx: *mut KbCtx, r: *const KbRel, col: u32, dst: *mut u32) -> kb_status;
    pub fn kb_rel_from_host(ctx: *mut KbCtx, slots: *const u32, n_cols: u32, cols: *const *const u32, n_rows: u64, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_rel_decode(ctx: *mut KbCtx, r: *const KbRel, col: u32, out: *mut *mut KbStrings) -> kb_status;
    pub fn kb_strings_info(s: *const KbStrings, n_strings: *mut u64, total_bytes: *mut u64) -> kb_status;
    pub fn kb_strings_download(ctx: *mut KbCtx, s: *const KbStrings, offsets: *mut u64, bytes: *mut u8) -> kb_status;
    pub fn kb_strings_free(ctx: *mut KbCtx, s: *mut KbStrings);
    // the quoted-triple table (QuotedTripleStore::id_to_components); n = 0 clears it
    pub fn kb_quoted_load(ctx: *mut KbCtx, ids: *const u32, s: *const u32, p: *const u32, o: *const u32, n: u64) -> kb_status;
    // the tails kb_bind adds: quoted-table entries and dictionary strings by id range
    pub fn kb_quoted_download(ctx: *mut KbCtx, first_id: u32, n: u32, s: *mut u32, p: *mut u32, o: *mut u32) -> kb_status;
    pub fn kb_dict_strings_download(ctx: *mut KbCtx, first: u32, n: u32, offsets: *mut u64, bytes: *mut u8) -> kb_status;
    pub fn kb_rel_free(ctx: *mut KbCtx, r: *mut KbRel);
    // the store as RDF text, in pieces of whole units (sparql_database.rs:301-382)
    pub fn kb_serialize_begin(ctx: *mut KbCtx, format: u32, prefix_offsets: *const u64, prefix_bytes: *const u8, n_prefixes: u32,
                              out: *mut *mut kb_serializer, info: *mut kb_serialize_info) -> kb_status;
    pub fn kb_serialize_next(ctx: *mut KbCtx, ser: *mut kb_serializer, host_dst: *mut u8, capacity: u64, bytes_written: *mut u64) -> kb_status;
    pub fn kb_serialize_free(ser: *mut kb_serializer);
    pub fn kb_store_gather_stats(ctx: *mut KbCtx, max_sample: u64, out: *mut *mut kb_db_stats, info: *mut kb_db_stats_info) -> kb_status;
    pub fn kb_db_stats_counts(st: *const kb_db_stats, position: u32, ids: *mut *const u32, counts: *mut *const u64, n: *mut u64) -> kb_status;
    pub fn kb_db_stats_free(st: *mut kb_db_stats);
    pub fn kb_qb_triples(ctx: *mut KbCtx, spec: *const kb_qb_spec, right: *const KbCtx, slots: *const u32, out: *mut *mut KbRel,
                         info: *mut kb_qb_info) -> kb_status;
    pub fn kb_qb_terms(ctx: *mut KbCtx, rows: *const KbRel, col: u32, mode: u32, out: *mut *mut KbStrings) -> kb_status;
    pub fn kb_store_union(dst: *mut KbCtx, a: *const KbCtx, b: *const KbCtx, info: *mut kb_union_info) -> kb_status;
    pub fn kb_store_par_join(dst: *mut KbCtx, a: *const KbCtx, b: *const KbCtx, predicate: u32, info: *mut kb_par_join_info) -> kb_status;
    // operators
    pub fn kb_scan(ctx: *mut KbCtx, pats: *const KbPattern, n: u32, pushdown: *const *const KbFilterOp, pushdown_len: *const u32, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_filter(ctx: *mut KbCtx, r: *const KbRel, prog: *const KbFilterOp, n: u32, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_project(ctx: *mut KbCtx, r: *const KbRel, slots: *const u32, n: u32, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_hash_join(ctx: *mut KbCtx, l: *const KbRel, r: *const KbRel, out: *mut *mut KbRel) -> kb_status;
    // natural_join of the RSP emit step: rows may leave shared variables unbound (KB_ID_NONE)
    pub fn kb_natural_join(ctx: *mut KbCtx, l: *const KbRel, r: *const KbRel, out: *mut *mut KbRel) -> kb_status;
    // the Streamertail hash joins over VALUES rows: pairs on key_slots (row 0's shared variables), the other shared slots by `merge`
    pub fn kb_hash_join_keyed(ctx: *mut KbCtx, l: *const KbRel, r: *const KbRel, key_slots: *const u32, n_key: u32, merge: u32,
                              out: *mut *mut KbRel) -> kb_status;
    pub fn kb_values(ctx: *mut KbCtx, slots: *const u32, n_vars: u32, n_rows: u64, undef: *const u8, offsets: *const u64, bytes: *const u8,
                     out: *mut *mut KbRel, info: *mut kb_values_info) -> kb_status;
    pub fn kb_bind_join(ctx: *mut KbCtx, l: *const KbRel, pattern: *const KbPattern, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_scan_quoted(ctx: *mut KbCtx, qp: *const kb_quoted_pattern, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_bind(ctx: *mut KbCtx, r: *const KbRel, spec: *const kb_bind_spec, out: *mut *mut KbRel, info: *mut kb_bind_info) -> kb_status;
    pub fn kb_star_join(ctx: *mut KbCtx, join_slot: u32, pats: *const KbPattern, n: u32, f: *const KbFilterOp, nf: u32, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_order_by(ctx: *mut KbCtx, r: *const KbRel, keys: *const kb_order_key, n_keys: u32, limit: u64, out: *mut *mut KbRel,
                       info: *mut kb_order_info) -> kb_status;
    pub fn kb_group_aggregate(ctx: *mut KbCtx, r: *const KbRel, group_slots: *const u32, n_group: u32, aggs: *const KbAgg, n_aggs: u32, out: *mut *mut KbGroups) -> kb_status;
    pub fn kb_star_join_aggregate(ctx: *mut KbCtx, join_slot: u32, pats: *const KbPattern, n: u32, f: *const KbFilterOp, nf: u32, group_slots: *const u32, n_group: u32,
                                  aggs: *const KbAgg, n_aggs: u32, out: *mut *mut KbGroups, n_rows: *mut u64) -> kb_status;
    pub fn kb_groups_info(g: *const KbGroups, n_groups: *mut u64, n_group_cols: *mut u32, n_aggs: *mut u32) -> kb_status;
    pub fn kb_groups_keys(g: *const KbGroups, col: u32, keys: *mut *const u32) -> kb_status;
    pub fn kb_groups_values(g: *const KbGroups, agg: u32, values: *mut *const c_double) -> kb_status;
    pub fn kb_groups_counts(g: *const KbGroups, counts: *mut *const u64) -> kb_status;
    pub fn kb_groups_free(g: *mut KbGroups);
    // prepared plans
    pub fn kb_star_join_prepare(ctx: *mut KbCtx, join_slot: u32, pats: *const KbPattern, n: u32, f: *const KbFilterOp, nf: u32, group_slots: *const u32, n_group: u32,
                                aggs: *const KbAgg, n_aggs: u32, ring: u32, out: *mut *mut KbPlan) -> kb_status;
    pub fn kb_plan_submit(ctx: *mut KbCtx, plan: *mut KbPlan, ticket: *mut u64) -> kb_status;
    pub fn kb_plan_collect(ctx: *mut KbCtx, plan: *mut KbPlan, ticket: u64, n_rows: *mut u64, rows: *mut *mut KbRel, groups: *mut *mut KbGroups) -> kb_status;
    pub fn kb_plan_free(ctx: *mut KbCtx, plan: *mut KbPlan);
    // Datalog
    pub fn kb_datalog_fixpoint(ctx: *mut KbCtx, rules: *const KbRule, n: u32, strategy: u32, out: *mut *mut KbRel, stats: *mut KbFixpointStats) -> kb_status;
    // incremental: the store is closed under the rules already, `seed` (s, p, o) are the triples added since
    pub fn kb_datalog_fixpoint_seed(ctx: *mut KbCtx, rules: *const KbRule, n: u32, strategy: u32, seed: *const KbRel, out: *mut *mut KbRel, n_seed_new: *mut u64,
                                    stats: *mut KbFixpointStats) -> kb_status;
    // delete-and-rederive across a window slide: the store is closed under the rules (the last fixpoint / maintain with the same rules)
    pub fn kb_datalog_maintain(ctx: *mut KbCtx, rules: *const KbRule, n: u32, strategy: u32, evict_tags: *const u64, n_evict: u32, add: *const KbRel,
                               add_tag: u64, inferred_removed: *mut *mut KbRel, inferred_added: *mut *mut KbRel, stats: *mut kb_maintain_stats) -> kb_status;
    // backward chaining: the distinct bindings of the query's variables over the facts with a proof of height <= max_depth; the store is only read
    pub fn kb_datalog_query(ctx: *mut KbCtx, rules: *const KbRule, n_rules: u32, query: *const KbPattern, max_depth: u32, out: *mut *mut KbRel,
                            stats: *mut kb_bc_stats) -> kb_status;
    pub fn kb_datalog_query_repairs(ctx: *mut KbCtx, constraints: *const KbRule, n_constraints: u32, query: *const KbPattern, out: *mut *mut KbRel,
                                    stats: *mut kb_repair_stats) -> kb_status;
    // Relation-to-Stream operators: the previous evaluation's distinct rows stay on the device, an evaluation emits the rows that changed
    pub fn kb_r2s_create(ctx: *mut KbCtx, stream_op: u32, slots: *const u32, n_cols: u32, out: *mut *mut kb_r2s) -> kb_status;
    pub fn kb_r2s_eval(ctx: *mut KbCtx, op: *mut kb_r2s, response: *const KbRel, emitted: *mut *mut KbRel) -> kb_status;
    pub fn kb_r2s_info(op: *const kb_r2s, last_rows: *mut u64, stream_op: *mut u32) -> kb_status;
    pub fn kb_r2s_free(ctx: *mut KbCtx, op: *mut kb_r2s);
    // multi-GPU helpers
    pub fn kb_shard_of(key: u32, n_shards: u32) -> u32;
    pub fn kb_set_sharding(ctx: *mut KbCtx, rank: u32, world: u32) -> kb_status;
    pub fn kb_shuffle_push(ctx: *mut KbCtx, r: *const KbRel, key_slot: u32, n_parts: u32, peer_cols: *const *mut u32, peer_cursors: *const *mut u32, capacity_rows: u64) -> kb_status;
    pub fn kb_rel_wrap_device(ctx: *mut KbCtx, slots: *const u32, n_cols: u32, d_cols: *const *mut u32, n_rows: u64, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_groups_pack(g: *const KbGroups, dst: *mut c_void, capacity_bytes: u64, bytes: *mut u64) -> kb_status;
    // the rest of the header (timing, device-resident loads, the legacy executor's i32 view, BGP execution, plan introspection and the
    // cross-rank GROUP BY attachment, the count-matrix shuffle, store download, on-disk segments, the one-shot host-buffer joins)
    pub fn kb_set_timing(ctx: *mut KbCtx, enabled: c_int) -> kb_status;
    pub fn kb_get_stats(ctx: *mut KbCtx, out: *mut KbStats, reset: c_int) -> kb_status;
    pub fn kb_store_load_device(ctx: *mut KbCtx, d_s: *const u32, d_p: *const u32, d_o: *const u32, n: u64) -> kb_status;
    pub fn kb_set_use_index(ctx: *mut KbCtx, enabled: c_int) -> kb_status;
    pub fn kb_dict_legacy_i32_load(ctx: *mut KbCtx, val: *const i32, is_i32: *const u8, n_ids: u32) -> kb_status;
    pub fn kb_rel_device_col(r: *const KbRel, col: u32, d_ptr: *mut *const u32) -> kb_status;
    pub fn kb_bgp_execute(ctx: *mut KbCtx, pats: *const KbPattern, n_pats: u32, filter: *const KbFilterOp, n_filter_ops: u32, project_slots: *const u32, n_project: u32,
                          out: *mut *mut KbRel) -> kb_status;
    pub fn kb_bgp_last_plan(ctx: *mut KbCtx, out: *mut kb_bgp_plan_info) -> kb_status;
    pub fn kb_plan_info(plan: *const KbPlan, ring: *mut u32, capacity_rows: *mut u64, n_cols: *mut u32, slots: *mut u32, grouped: *mut u32) -> kb_status;
    pub fn kb_plan_peer_scratch_bytes(plan: *const KbPlan) -> u64;
    pub fn kb_plan_attach_peers(ctx: *mut KbCtx, plan: *mut KbPlan, rank: u32, world: u32, peer_scratch: *const *mut c_void) -> kb_status;
    pub fn kb_partition(ctx: *mut KbCtx, r: *const KbRel, key_slot: u32, n_parts: u32, out: *mut *mut KbRel, part_offsets: *mut u64) -> kb_status;
    pub fn kb_partition_counts(ctx: *mut KbCtx, r: *const KbRel, key_slot: u32, n_parts: u32, counts: *mut u64) -> kb_status;
    pub fn kb_shuffle_scatter(ctx: *mut KbCtx, r: *const KbRel, key_slot: u32, n_parts: u32, peer_cols: *const *mut u32, base: *const u64, capacity_rows: u64) -> kb_status;
    pub fn kb_rel_from_device(ctx: *mut KbCtx, slots: *const u32, n_cols: u32, d_cols: *const *const u32, n_rows: u64, out: *mut *mut KbRel) -> kb_status;
    pub fn kb_store_download(ctx: *mut KbCtx, s: *mut u32, p: *mut u32, o: *mut u32, cap: u64, n: *mut u64) -> kb_status;
    pub fn kb_segment_write(path: *const c_char, s: *const u32, p: *const u32, o: *const u32, n: u64, tag: u64) -> kb_status;
    pub fn kb_segment_info(path: *const c_char, n_triples: *mut u64, tag: *mut u64, cmin: *mut u32, cmax: *mut u32) -> kb_status;
    pub fn kb_segment_save(ctx: *mut KbCtx, tag: u64, whole_store: c_int, path: *const c_char) -> kb_status;
    pub fn kb_store_append_file(ctx: *mut KbCtx, path: *const c_char, tag: u64, verify: c_int) -> kb_status;
    pub fn kb_star_join_host(ctx: *mut KbCtx, s: *const u32, p: *const u32, o: *const u32, n: u64, join_slot: u32, pats: *const KbPattern, n_pats: u32,
                             filter: *const KbFilterOp, n_filter_ops: u32, n_cols: *mut u32, slots: *mut u32, cols: *mut *mut u32, n_rows: *mut u64) -> kb_status;
    pub fn kb_star_join_host_into(ctx: *mut KbCtx, s: *const u32, p: *const u32, o: *const u32, n: u64, join_slot: u32, pats: *const KbPattern, n_pats: u32,
                                  filter: *const KbFilterOp, n_filter_ops: u32, n_cols: *mut u32, slots: *mut u32, cols: *const *mut u32, capacity_rows: u64,
                                  n_rows: *mut u64) -> kb_status;
    pub fn kb_groups_merge(ctx: *mut KbCtx, parts: *const *const c_void, part_bytes: *const u64, n_parts: u32, out: *mut *mut KbGroups) -> kb_status;
}
