"""ctypes binding of libkolibrie_b200.so (include/kolibrie_b200.h).

This is the Python stand-in for the Rust shim described in INTEGRATION.md: the reference is a Rust workspace and there is no
Rust toolchain in this image, so tests, bench.py and the multi-GPU plumbing drive the C ABI from Python. There is no CPU
fallback: if the library (or a GPU) is missing, every entry point raises.
"""
from __future__ import annotations

import atexit
import ctypes as C
import os
import weakref
from typing import List, Iterable, Optional, Sequence, Tuple, Union

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KOLIBRIE_B200_LIB") or os.path.join(_HERE, "libkolibrie_b200.so")  # override: A/B of build variants
LEGACY_LIB_PATH = os.path.join(_HERE, "libcudajoin.so")

KB_OK = 0
KB_E_INVALID, KB_E_CUDA, KB_E_OOM, KB_E_UNSUPPORTED, KB_E_NOT_FOUND, KB_E_LIMIT = -1, -2, -3, -4, -5, -6
KB_ID_NONE = 0xFFFFFFFF
KB_MAX_COLS = 16
KB_TAG_INFERRED = 0xFFFFFFFFFFFFFFF0
KB_TERM_QUOTED = 2  # kb_term.is_var of a `<< s p o >>` term (kb_scan_quoted)
KB_QUOTED_MAX_DEPTH = 16
NUMERIC_F64, NUMERIC_I32 = 1, 2  # kb_dict_numeric_derive's tables
NUMERIC_APPEND = 0xFFFFFFFF      # first_id: from the first id the table does not hold yet

# filter opcodes / comparisons / aggregates (mirror the header)
F_CMP_NUM, F_EQ_ID, F_NE_ID, F_AND, F_OR, F_NOT, F_PUSH_VAR, F_PUSH_CONST, F_ADD, F_SUB, F_MUL, F_DIV, F_TRUTHY, F_IS_TRIPLE, F_CMP_LEGACY = range(1, 16)
LEGACY_CONST_IS_I32 = 0x100
LEGACY_NESTED_F64 = 0x200
CMP_GT, CMP_GE, CMP_LT, CMP_LE, CMP_EQ, CMP_NE = range(1, 7)
AGG_COUNT, AGG_SUM, AGG_MIN, AGG_MAX, AGG_AVG = range(5)
SEMI_NAIVE, NAIVE, SEMI_NAIVE_PARALLEL = 0, 1, 2
SEMI_NAIVE_OLD_DELTA = 3  # textbook OLD/delta scheme: same facts, rounds and per-round counts, fewer candidates (include/kolibrie_b200.h)
RSTREAM, ISTREAM, DSTREAM = 0, 1, 2  # kb_stream_op (r2s.rs:15-17)
# kb_bind_function (engine.rs:144-277)
BIND_SUBJECT, BIND_PREDICATE, BIND_OBJECT, BIND_IS_TRIPLE, BIND_TRIPLE, BIND_CONCAT = range(1, 7)
KB_BIND_MAX_ARGS = 16


class KbTerm(C.Structure):
    _fields_ = [("is_var", C.c_uint32), ("value", C.c_uint32)]


class KbPattern(C.Structure):
    _fields_ = [("s", KbTerm), ("p", KbTerm), ("o", KbTerm)]


class KbQuotedPattern(C.Structure):
    """kb_quoted_pattern: `outer` with KB_TERM_QUOTED in its subject and/or object; those terms are `<< inner_s >>` / `<< inner_o >>`"""
    _fields_ = [("outer", KbPattern), ("inner_s", KbPattern), ("inner_o", KbPattern)]


class KbBindSpec(C.Structure):
    """kb_bind_spec: one BIND built-in over a relation"""
    _fields_ = [("function", C.c_uint32), ("n_args", C.c_uint32), ("args", C.POINTER(KbTerm)), ("n_const", C.c_uint32),
                ("const_offsets", C.POINTER(C.c_uint64)), ("const_bytes", C.POINTER(C.c_uint8)), ("out_slot", C.c_uint32), ("next_qt_id", C.c_uint32)]


class KbBindInfo(C.Structure):
    """kb_bind_info: rows, rows left unbound, and the new dictionary / quoted-triple ids (first, count)"""
    _fields_ = [("n_rows", C.c_uint64), ("n_unbound", C.c_uint64), ("dict_first", C.c_uint32), ("dict_new", C.c_uint32),
                ("quoted_first", C.c_uint32), ("quoted_new", C.c_uint32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class KbValuesInfo(C.Structure):
    """kb_values_info: the new dictionary ids (first, count) and the rows dropped for having no defined cell"""
    _fields_ = [("dict_first", C.c_uint32), ("dict_new", C.c_uint32), ("rows_dropped", C.c_uint64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


MERGE_LEFT_FIRST, MERGE_RIGHT_FIRST = 0, 1  # kb_merge_policy


class KbNumericInfo(C.Structure):
    """kb_numeric_info: ids of the device dictionary, ids parsed, how many of them are numbers / i32, how many took the slow path"""
    _fields_ = [("n_ids", C.c_uint32), ("n_derived", C.c_uint32), ("n_numeric", C.c_uint32), ("n_i32", C.c_uint32), ("n_slow", C.c_uint32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class KbFilterOp(C.Structure):
    _fields_ = [("op", C.c_uint32), ("slot", C.c_uint32), ("cmp", C.c_uint32), ("id", C.c_uint32), ("value", C.c_double)]


class KbAgg(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("slot", C.c_uint32)]


class KbRuleFilter(C.Structure):
    _fields_ = [("lhs_slot", C.c_uint32), ("cmp", C.c_uint32), ("rhs_is_var", C.c_uint32), ("rhs_slot", C.c_uint32), ("rhs_value", C.c_double)]


class KbRule(C.Structure):
    _fields_ = [
        ("premise", C.POINTER(KbPattern)), ("n_premise", C.c_uint32),
        ("filters", C.POINTER(KbRuleFilter)), ("n_filters", C.c_uint32),
        ("conclusion", C.POINTER(KbPattern)), ("n_conclusion", C.c_uint32),
    ]


class KbFixpointStats(C.Structure):
    _fields_ = [("rounds", C.c_uint32), ("inferred", C.c_uint64), ("derivations", C.c_uint64), ("round_new", C.c_uint64 * 64), ("device_ms", C.c_double)]


class KbMaintainStats(C.Structure):
    """kb_maintain_stats: what one kb_datalog_maintain call moved"""
    _fields_ = [(n, C.c_uint64) for n in ("base_removed", "base_added", "overdeleted", "rederived", "inferred_removed", "inferred_added", "derivations")] + [
        ("overdelete_rounds", C.c_uint32), ("insert_rounds", C.c_uint32), ("device_ms", C.c_double)]


BC_MAX_DEPTH = 10  # KB_BC_MAX_DEPTH: Reasoner::backward_chaining's MAX_DEPTH (backward_chaining.rs:197-198)


class KbBcStats(C.Structure):
    """kb_bc_stats: what one kb_datalog_query call ran and read"""
    _fields_ = [(n, C.c_uint32) for n in ("rounds", "reached_fixpoint", "stopped_early", "relevant_rules", "demand_patterns", "restricted_predicates")] + [
        (n, C.c_uint64) for n in ("base_facts", "derived", "derivations", "answers")] + [("device_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class KbRepairStats(C.Structure):
    """kb_repair_stats: what one kb_datalog_query_repairs call matched, found and answered"""
    _fields_ = [(n, C.c_uint32) for n in ("constraints", "subsets_probed")] + [
        (n, C.c_uint64) for n in ("matches", "conflicts", "minimal_conflicts", "conflicted_facts", "answers")] + [
        (n, C.c_double) for n in ("device_ms", "match_ms", "conflict_ms", "answer_ms")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


ORDER_VIEW, ORDER_SORT, ORDER_TOPK = 0, 1, 2          # kb_order_route
ORDER_CONST, ORDER_NUMERIC, ORDER_STRING = 0, 1, 2    # kb_order_kind


class KbOrderKey(C.Structure):
    _fields_ = [("slot", C.c_uint32), ("descending", C.c_uint32)]


class KbOrderInfo(C.Structure):
    """kb_order_info: rows in / out, the route, and per key its kind, distinct ids and string refinement rounds"""
    _fields_ = [("n_rows_in", C.c_uint64), ("n_rows_out", C.c_uint64), ("route", C.c_uint32), ("key_kind", C.c_uint32 * KB_MAX_COLS),
                ("n_distinct", C.c_uint32 * KB_MAX_COLS), ("string_rounds", C.c_uint32 * KB_MAX_COLS)]

    def as_dict(self, n_keys: int):
        """per-key arrays cut to the call's n_keys"""
        return {"n_rows_in": self.n_rows_in, "n_rows_out": self.n_rows_out, "route": self.route,
                **{n: list(getattr(self, n))[:n_keys] for n in ("key_kind", "n_distinct", "string_rounds")}}


SER_NTRIPLES, SER_TURTLE = 0, 1  # kb_serialize_format


class KbSerializeInfo(C.Structure):
    """kb_serialize_info: distinct triples, text bytes, the largest unit, Turtle subject groups, rendered terms, rank rounds, and the
    device time of kb_serialize_begin's phases (sort + dedup, render, ranks, unit lengths + scan)"""
    _fields_ = [("n_triples", C.c_uint64), ("total_bytes", C.c_uint64), ("max_unit_bytes", C.c_uint64), ("n_subject_groups", C.c_uint64),
                ("n_terms", C.c_uint32), ("rank_rounds", C.c_uint32), ("phase_ms", C.c_double * 4)]

    def as_dict(self):
        return {n: (list(getattr(self, n)) if n == "phase_ms" else int(getattr(self, n))) for n, _ in self._fields_}


class KbDbStatsInfo(C.Structure):
    """kb_db_stats_info: distinct triples T, quoted-triple entries, the sample (take rows every step-th), distinct ids per position
    (subject, predicate, object) and the device time of the phases (sort + dedup, gather, counts)"""
    _fields_ = [("total_triples", C.c_uint64), ("quoted_triple_count", C.c_uint64), ("take", C.c_uint64), ("step", C.c_uint64),
                ("n_ids", C.c_uint64 * 3), ("phase_ms", C.c_double * 3)]

    def as_dict(self):
        return {n: ([int(x) for x in getattr(self, n)] if n == "n_ids" else list(getattr(self, n)) if n == "phase_ms" else int(getattr(self, n)))
                for n, _ in self._fields_}


GATHER_STATS_FAST = 100000  # gather_stats_fast's sample size (database_stats.rs:50)

QB_ANY, QB_EXACT, QB_CONTAINS, QB_STARTS, QB_ENDS = 0, 1, 2, 3, 4  # kb_qb_mode
QB_ON_SUBJECT, QB_ON_PREDICATE, QB_ON_OBJECT = 1, 2, 4  # kb_qb_join
QB_TERMS_EMPTY, QB_TERMS_DROP, QB_TERMS_DISTINCT = 0, 1, 2  # kb_qb_terms_mode
QB_PATTERN_MAX = 4096
QB_NO_LIMIT = 0xFFFFFFFFFFFFFFFF


class KbQbFilter(C.Structure):
    """kb_qb_filter: one position's filter (mode, the id of KB_QB_EXACT, the pattern bytes of the text modes)"""
    _fields_ = [("mode", C.c_uint32), ("id", C.c_uint32), ("pattern", C.c_void_p), ("len", C.c_uint64)]


class KbQbSpec(C.Structure):
    """kb_qb_spec: subject / predicate / object filters, KB_QB_ON_* join bits, offset and limit (QB_NO_LIMIT: none)"""
    _fields_ = [("pos", KbQbFilter * 3), ("join", C.c_uint32), ("reserved", C.c_uint32), ("offset", C.c_uint64), ("limit", C.c_uint64)]


class KbQbInfo(C.Structure):
    """kb_qb_info: store rows read, distinct filtered triples, distinct joined triples, rows returned, and the device time of the phases
    (match, selection, sort + dedup, join)"""
    _fields_ = [("n_raw", C.c_uint64), ("n_selected", C.c_uint64), ("n_joined", C.c_uint64), ("n_rows", C.c_uint64), ("phase_ms", C.c_double * 4)]

    def as_dict(self):
        return {n: (list(getattr(self, n)) if n == "phase_ms" else int(getattr(self, n))) for n, _ in self._fields_}


class KbUnionInfo(C.Structure):
    """kb_union_info: distinct triples of a, of b and of the result, b's distinct ids, the first id and the number of the strings the
    union added, and the device time of the phases (the two sets, b's terms, dictionary, remap, union)"""
    _fields_ = [("n_a", C.c_uint64), ("n_b", C.c_uint64), ("n_rows", C.c_uint64), ("n_terms", C.c_uint32), ("dict_first", C.c_uint32),
                ("dict_new", C.c_uint32), ("reserved", C.c_uint32), ("phase_ms", C.c_double * 5)]

    def as_dict(self):
        return {n: (list(getattr(self, n)) if n == "phase_ms" else int(getattr(self, n))) for n, _ in self._fields_ if n != "reserved"}


class KbParJoinInfo(C.Structure):
    """kb_par_join_info: distinct triples of a and of b with the predicate, rows of the join and of the semi-join, distinct triples of
    the result, and the device time of the phases (selection, distinct pairs + counts, joins, sort + dedup)"""
    _fields_ = [("n_a", C.c_uint64), ("n_b", C.c_uint64), ("n_join", C.c_uint64), ("n_semi", C.c_uint64), ("n_rows", C.c_uint64),
                ("phase_ms", C.c_double * 4)]

    def as_dict(self):
        return {n: (list(getattr(self, n)) if n == "phase_ms" else int(getattr(self, n))) for n, _ in self._fields_}


KB_BGP_MAX_PATTERNS = 16
BGP_NONE, BGP_STAR, BGP_COMPONENTS = 0, 1, 2  # kb_bgp_route


class KbBgpPlanInfo(C.Structure):
    """kb_bgp_plan_info: what the last kb_bgp_execute did (route, components, reduction, join order, intermediate sizes)"""
    _M = KB_BGP_MAX_PATTERNS
    _fields_ = [("route", C.c_uint32), ("n_patterns", C.c_uint32), ("n_components", C.c_uint32), ("component", C.c_uint32 * _M),
                ("acyclic", C.c_uint32 * _M), ("reduce_rounds", C.c_uint32 * _M), ("rows_scanned", C.c_uint64 * _M), ("rows_reduced", C.c_uint64 * _M),
                ("join_order", C.c_uint32 * _M), ("component_rows", C.c_uint64 * _M), ("component_max_rows", C.c_uint64 * _M),
                ("cross_order", C.c_uint32 * _M), ("reduce_bytes", C.c_uint64), ("reduce_bit_ops", C.c_uint64), ("max_intermediate", C.c_uint64), ("rows_unprojected", C.c_uint64)]

    def as_dict(self):
        """arrays cut to the patterns / components / join steps the call had"""
        n, m = self.n_patterns, self.n_components
        cut = {"component": n, "rows_scanned": n, "rows_reduced": n, "join_order": n if self.route == BGP_COMPONENTS else 0, "acyclic": m,
               "reduce_rounds": m, "component_rows": m, "component_max_rows": m, "cross_order": m}
        out = {}
        for name, _ in self._fields_:
            v = getattr(self, name)
            out[name] = [int(x) for x in v[: cut[name]]] if name in cut else int(v)
        return out


class KbStats(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("scan_ms", "build_ms", "probe_ms", "filter_ms", "group_ms", "other_ms", "total_ms")] + [
        (n, C.c_uint64)
        for n in ("scan_launches", "build_launches", "probe_launches", "filter_launches", "group_launches", "other_launches",
                  "rows_scanned", "rows_built", "rows_probed", "rows_out", "h2d_bytes", "d2h_bytes", "kernel_launches", "fused_scan_builds", "index_joins")
    ]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


def V(slot: int) -> KbTerm:
    """variable term"""
    return KbTerm(1, slot)


def K(term_id: int) -> KbTerm:
    """constant term"""
    return KbTerm(0, term_id)


def pattern(s: KbTerm, p: KbTerm, o: KbTerm) -> KbPattern:
    return KbPattern(s, p, o)


def patterns(pats: Sequence[KbPattern]):
    arr = (KbPattern * max(len(pats), 1))()
    for i, p in enumerate(pats):
        arr[i] = p
    return arr


def fop(op, slot=0, cmp=0, id=0, value=0.0) -> KbFilterOp:
    return KbFilterOp(op, slot, cmp, id, value)


def filter_prog(ops: Optional[Sequence[KbFilterOp]]):
    ops = list(ops or [])
    arr = (KbFilterOp * max(len(ops), 1))()
    for i, o in enumerate(ops):
        arr[i] = o
    return arr, len(ops)


class KolibrieError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"kb_status {status}: {message}")
        self.status = status
        self.message = message


_lib = None
_LIVE_CONTEXTS = weakref.WeakSet()


@atexit.register
def _close_all():
    for ctx in list(_LIVE_CONTEXTS):
        try:
            ctx.close()
        except Exception:
            pass


def lib() -> C.CDLL:
    """Load the shared library; fail loudly when it is missing (no CPU fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
                          "kolibrie_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    P = C.POINTER
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32
    sig = {
        "kb_version": (C.c_char_p, []),
        "kb_ctx_create": (i32, [C.c_int, P(vp)]),
        "kb_ctx_destroy": (None, [vp]),
        "kb_last_error": (C.c_char_p, [vp]),
        "kb_set_timing": (i32, [vp, C.c_int]),
        "kb_get_stats": (i32, [vp, P(KbStats), C.c_int]),
        "kb_synchronize": (i32, [vp]),
        "kb_store_load": (i32, [vp, vp, vp, vp, u64]),
        "kb_store_load_device": (i32, [vp, vp, vp, vp, u64]),
        "kb_store_append_device": (i32, [vp, vp, vp, vp, u64, u64]),
        "kb_store_append": (i32, [vp, vp, vp, vp, u64, u64]),
        "kb_store_evict": (i32, [vp, u64]),
        "kb_store_delete": (i32, [vp, vp, vp, vp, u64]),
        "kb_store_insert": (i32, [vp, vp, vp, vp, u64, u64, vp, P(u64)]),
        "kb_store_remove": (i32, [vp, vp, vp, vp, u64, vp, P(u64)]),
        "kb_store_remove_template": (i32, [vp, vp, P(KbPattern), u32, P(u64)]),
        "kb_store_clear": (i32, [vp]),
        "kb_store_build_index": (i32, [vp, P(u32), P(C.c_double)]),
        "kb_set_use_index": (i32, [vp, C.c_int]),
        "kb_store_size": (i32, [vp, P(u64), P(u32)]),
        "kb_store_download": (i32, [vp, vp, vp, vp, u64, P(u64)]),
        "kb_dict_numeric_load": (i32, [vp, vp, vp, u32]),
        "kb_dict_strings_load": (i32, [vp, vp, vp, u32]),
        "kb_dict_encode": (i32, [vp, vp, vp, u64, vp, P(u32), vp]),
        "kb_dict_strings_info": (i32, [vp, P(u32), P(u64)]),
        "kb_dict_legacy_i32_load": (i32, [vp, vp, vp, u32]),
        "kb_dict_numeric_derive": (i32, [vp, u32, u32, P(KbNumericInfo)]),
        "kb_dict_numeric_download": (i32, [vp, u32, u32, vp, vp, vp, vp]),
        "kb_rel_decode": (i32, [vp, vp, u32, P(vp)]),
        "kb_strings_info": (i32, [vp, P(u64), P(u64)]),
        "kb_strings_download": (i32, [vp, vp, vp, vp]),
        "kb_strings_free": (None, [vp, vp]),
        "kb_quoted_load": (i32, [vp, vp, vp, vp, vp, u64]),
        "kb_quoted_download": (i32, [vp, u32, u32, vp, vp, vp]),
        "kb_dict_strings_download": (i32, [vp, u32, u32, vp, vp]),
        "kb_serialize_begin": (i32, [vp, u32, vp, vp, u32, P(vp), P(KbSerializeInfo)]),
        "kb_serialize_next": (i32, [vp, vp, vp, u64, P(u64)]),
        "kb_serialize_free": (None, [vp]),
        "kb_store_gather_stats": (i32, [vp, u64, P(vp), P(KbDbStatsInfo)]),
        "kb_db_stats_counts": (i32, [vp, u32, P(P(u32)), P(P(u64)), P(u64)]),
        "kb_db_stats_free": (None, [vp]),
        "kb_qb_triples": (i32, [vp, P(KbQbSpec), vp, P(u32), P(vp), P(KbQbInfo)]),
        "kb_qb_terms": (i32, [vp, vp, u32, u32, P(vp)]),
        "kb_store_union": (i32, [vp, vp, vp, P(KbUnionInfo)]),
        "kb_store_par_join": (i32, [vp, vp, vp, u32, P(KbParJoinInfo)]),
        "kb_bind": (i32, [vp, vp, P(KbBindSpec), P(vp), P(KbBindInfo)]),
        "kb_rel_info": (i32, [vp, P(u64), P(u32), P(u32)]),
        "kb_rel_download": (i32, [vp, vp, u32, vp]),
        "kb_rel_device_col": (i32, [vp, u32, P(vp)]),
        "kb_rel_from_host": (i32, [vp, P(u32), u32, P(vp), u64, P(vp)]),
        "kb_rel_from_device": (i32, [vp, P(u32), u32, P(vp), u64, P(vp)]),
        "kb_rel_free": (None, [vp, vp]),
        "kb_scan": (i32, [vp, P(KbPattern), u32, P(P(KbFilterOp)), P(u32), P(vp)]),
        "kb_filter": (i32, [vp, vp, P(KbFilterOp), u32, P(vp)]),
        "kb_project": (i32, [vp, vp, P(u32), u32, P(vp)]),
        "kb_hash_join": (i32, [vp, vp, vp, P(vp)]),
        "kb_natural_join": (i32, [vp, vp, vp, P(vp)]),
        "kb_hash_join_keyed": (i32, [vp, vp, vp, P(u32), u32, u32, P(vp)]),
        "kb_values": (i32, [vp, P(u32), u32, u64, vp, vp, vp, P(vp), P(KbValuesInfo)]),
        "kb_bind_join": (i32, [vp, vp, P(KbPattern), P(vp)]),
        "kb_scan_quoted": (i32, [vp, P(KbQuotedPattern), P(vp)]),
        "kb_star_join": (i32, [vp, u32, P(KbPattern), u32, P(KbFilterOp), u32, P(vp)]),
        "kb_bgp_execute": (i32, [vp, P(KbPattern), u32, P(KbFilterOp), u32, P(u32), u32, P(vp)]),
        "kb_bgp_last_plan": (i32, [vp, P(KbBgpPlanInfo)]),
        "kb_order_by": (i32, [vp, vp, P(KbOrderKey), u32, u64, P(vp), P(KbOrderInfo)]),
        "kb_group_aggregate": (i32, [vp, vp, P(u32), u32, P(KbAgg), u32, P(vp)]),
        "kb_groups_info": (i32, [vp, P(u64), P(u32), P(u32)]),
        "kb_groups_keys": (i32, [vp, u32, P(P(u32))]),
        "kb_groups_values": (i32, [vp, u32, P(P(C.c_double))]),
        "kb_groups_counts": (i32, [vp, P(P(u64))]),
        "kb_groups_free": (None, [vp]),
        "kb_groups_pack": (i32, [vp, vp, u64, P(u64)]),
        "kb_groups_merge": (i32, [vp, P(vp), P(u64), u32, P(vp)]),
        "kb_star_join_prepare": (i32, [vp, u32, P(KbPattern), u32, P(KbFilterOp), u32, P(u32), u32, P(KbAgg), u32, u32, P(vp)]),
        "kb_plan_submit": (i32, [vp, vp, P(u64)]),
        "kb_plan_collect": (i32, [vp, vp, u64, P(u64), P(vp), P(vp)]),
        "kb_plan_info": (i32, [vp, P(u32), P(u64), P(u32), P(u32), P(u32)]),
        "kb_plan_free": (None, [vp, vp]),
        "kb_plan_peer_scratch_bytes": (u64, [vp]),
        "kb_plan_attach_peers": (i32, [vp, vp, u32, u32, P(vp)]),
        "kb_star_join_aggregate": (i32, [vp, u32, P(KbPattern), u32, P(KbFilterOp), u32, P(u32), u32, P(KbAgg), u32, P(vp), P(u64)]),
        "kb_datalog_fixpoint": (i32, [vp, P(KbRule), u32, u32, P(vp), P(KbFixpointStats)]),
        "kb_datalog_fixpoint_seed": (i32, [vp, P(KbRule), u32, u32, vp, P(vp), P(u64), P(KbFixpointStats)]),
        "kb_datalog_maintain": (i32, [vp, P(KbRule), u32, u32, P(u64), u32, vp, u64, P(vp), P(vp), P(KbMaintainStats)]),
        "kb_datalog_query": (i32, [vp, P(KbRule), u32, P(KbPattern), u32, P(vp), P(KbBcStats)]),
        "kb_datalog_query_repairs": (i32, [vp, P(KbRule), u32, P(KbPattern), P(vp), P(KbRepairStats)]),
        "kb_r2s_create": (i32, [vp, u32, P(u32), u32, P(vp)]),
        "kb_r2s_eval": (i32, [vp, vp, vp, P(vp)]),
        "kb_r2s_info": (i32, [vp, P(u64), P(u32)]),
        "kb_r2s_free": (None, [vp, vp]),
        "kb_shard_of": (u32, [u32, u32]),
        "kb_set_sharding": (i32, [vp, u32, u32]),
        "kb_partition": (i32, [vp, vp, u32, u32, P(vp), P(u64)]),
        "kb_partition_counts": (i32, [vp, vp, u32, u32, P(u64)]),
        "kb_shuffle_scatter": (i32, [vp, vp, u32, u32, P(vp), P(u64), u64]),
        "kb_segment_write": (i32, [C.c_char_p, vp, vp, vp, u64, u64]),
        "kb_segment_info": (i32, [C.c_char_p, P(u64), P(u64), P(u32), P(u32)]),
        "kb_segment_save": (i32, [vp, u64, C.c_int, C.c_char_p]),
        "kb_store_append_file": (i32, [vp, C.c_char_p, u64, C.c_int]),
        "kb_shuffle_push": (i32, [vp, vp, u32, u32, P(vp), P(vp), u64]),
        "kb_rel_wrap_device": (i32, [vp, P(u32), u32, P(vp), u64, P(vp)]),
        "kb_star_join_host": (i32, [vp, vp, vp, vp, u64, u32, P(KbPattern), u32, P(KbFilterOp), u32, P(u32), P(u32), P(vp), P(u64)]),
        "kb_star_join_host_into": (i32, [vp, vp, vp, vp, u64, u32, P(KbPattern), u32, P(KbFilterOp), u32, P(u32), P(u32), P(vp), u64, P(u64)]),
        "perform_hash_join_cuda": (None, [vp, vp, vp, u32, u32, P(u32), P(P(u32)), P(u32)]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)  # AttributeError here = the library does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "kb_version", "kb_ctx_create", "kb_ctx_destroy", "kb_last_error", "kb_set_timing", "kb_get_stats", "kb_synchronize",
    "kb_store_load", "kb_store_load_device", "kb_store_append", "kb_store_append_device", "kb_store_evict", "kb_store_delete", "kb_store_insert", "kb_store_remove", "kb_store_remove_template", "kb_store_clear", "kb_store_build_index", "kb_set_use_index", "kb_store_size",
    "kb_store_download", "kb_dict_numeric_load", "kb_dict_legacy_i32_load", "kb_dict_numeric_derive", "kb_dict_numeric_download", "kb_dict_strings_load", "kb_dict_encode", "kb_dict_strings_info", "kb_rel_decode", "kb_strings_info", "kb_strings_download", "kb_strings_free", "kb_quoted_load", "kb_quoted_download", "kb_dict_strings_download", "kb_serialize_begin", "kb_serialize_next", "kb_serialize_free", "kb_store_gather_stats", "kb_db_stats_counts", "kb_db_stats_free", "kb_qb_triples", "kb_qb_terms", "kb_store_union", "kb_store_par_join", "kb_bind", "kb_rel_info", "kb_rel_download", "kb_rel_device_col", "kb_rel_from_host",
    "kb_rel_from_device", "kb_rel_free", "kb_scan", "kb_filter", "kb_project", "kb_hash_join", "kb_natural_join", "kb_hash_join_keyed", "kb_values", "kb_bind_join", "kb_scan_quoted", "kb_star_join", "kb_bgp_execute", "kb_bgp_last_plan",
    "kb_order_by", "kb_group_aggregate", "kb_groups_info", "kb_groups_keys", "kb_groups_values", "kb_groups_counts", "kb_groups_free", "kb_groups_pack", "kb_groups_merge", "kb_star_join_aggregate",
    "kb_star_join_prepare", "kb_plan_submit", "kb_plan_collect", "kb_plan_info", "kb_plan_free", "kb_plan_peer_scratch_bytes", "kb_plan_attach_peers",
    "kb_datalog_fixpoint", "kb_datalog_fixpoint_seed", "kb_datalog_maintain", "kb_datalog_query", "kb_datalog_query_repairs", "kb_r2s_create", "kb_r2s_eval", "kb_r2s_info", "kb_r2s_free", "kb_shard_of", "kb_set_sharding", "kb_partition", "kb_partition_counts", "kb_segment_write", "kb_segment_info", "kb_segment_save", "kb_store_append_file", "kb_shuffle_scatter", "kb_shuffle_push", "kb_rel_wrap_device", "kb_star_join_host", "kb_star_join_host_into", "perform_hash_join_cuda",
]


def _u32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.uint32)


def _ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


class Relation:
    """Device-resident columnar bag of binding rows (kb_rel)."""

    def __init__(self, ctx: "Context", handle):
        self.ctx = ctx
        self.h = C.c_void_p(handle) if not isinstance(handle, C.c_void_p) else handle
        ctx._rels.add(self)

    def info(self):
        n, nc = C.c_uint64(), C.c_uint32()
        slots = (C.c_uint32 * KB_MAX_COLS)()
        self.ctx._check(lib().kb_rel_info(self.h, C.byref(n), C.byref(nc), slots))
        return n.value, [slots[i] for i in range(nc.value)]

    @property
    def n_rows(self) -> int:
        return self.info()[0]

    @property
    def slots(self):
        return self.info()[1]

    def column(self, col: int) -> np.ndarray:
        n, _ = self.info()
        out = np.empty(n, dtype=np.uint32)
        self.ctx._check(lib().kb_rel_download(self.ctx.h, self.h, col, _ptr(out)))
        return out

    def decode(self, col: int):
        """kb_rel_decode: the column's ids as strings, decoded on the device. Returns (offsets uint64 [n+1], bytes uint8): string i
        is bytes[offsets[i]:offsets[i+1]] (UTF-8); ids the dictionary does not hold read "unknown" (engine.rs:44)."""
        h = C.c_void_p()
        self.ctx._check(lib().kb_rel_decode(self.ctx.h, self.h, col, C.byref(h)))
        try:
            n, total = C.c_uint64(), C.c_uint64()
            self.ctx._check(lib().kb_strings_info(h, C.byref(n), C.byref(total)))
            off = np.empty(n.value + 1, dtype=np.uint64)
            data = np.empty(total.value, dtype=np.uint8)
            self.ctx._check(lib().kb_strings_download(self.ctx.h, h, _ptr(off), _ptr(data)))
        finally:
            lib().kb_strings_free(self.ctx.h, h)
        return off, data

    def decode_strings(self, col: int) -> List[str]:
        off, data = self.decode(col)
        raw = data.tobytes()
        return [raw[int(off[i]):int(off[i + 1])].decode("utf-8") for i in range(len(off) - 1)]

    def device_ptr(self, col: int) -> int:
        p = C.c_void_p()
        self.ctx._check(lib().kb_rel_device_col(self.h, col, C.byref(p)))
        return p.value or 0

    def to_numpy(self, slot_order: Optional[Sequence[int]] = None) -> np.ndarray:
        """rows x cols uint32 array, columns ordered by `slot_order` (default: the relation's own order)"""
        n, slots = self.info()
        order = list(slot_order) if slot_order is not None else slots
        out = np.empty((n, len(order)), dtype=np.uint32)
        for j, s in enumerate(order):
            out[:, j] = self.column(slots.index(s))
        return out

    def free(self):
        if self.h:
            lib().kb_rel_free(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    """One device context = one GPU (multi-GPU = one process per GPU, see kolibrie_b200.dist)."""

    def __init__(self, device: int = 0):
        h = C.c_void_p()
        rc = lib().kb_ctx_create(device, C.byref(h))
        if rc != KB_OK:
            raise KolibrieError(rc, (lib().kb_last_error(None) or b"").decode())
        self.h = h
        self.device = device
        self._rels = weakref.WeakSet()
        self._plans = weakref.WeakSet()
        _LIVE_CONTEXTS.add(self)

    def close(self):
        if self.h:
            for pl in list(self._plans):
                pl.free()
            for r in list(self._rels):  # relations first, while their stream still exists
                r.free()
            lib().kb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != KB_OK:
            raise KolibrieError(rc, (lib().kb_last_error(self.h) or b"").decode())

    # ---- store
    def store_load(self, s, p, o):
        s, p, o = _u32(s), _u32(p), _u32(o)
        self._check(lib().kb_store_load(self.h, _ptr(s), _ptr(p), _ptr(o), len(s)))

    def store_load_device(self, d_s: int, d_p: int, d_o: int, n: int):
        self._check(lib().kb_store_load_device(self.h, C.c_void_p(d_s), C.c_void_p(d_p), C.c_void_p(d_o), n))

    def store_append(self, s, p, o, tag: int):
        s, p, o = _u32(s), _u32(p), _u32(o)
        self._check(lib().kb_store_append(self.h, _ptr(s), _ptr(p), _ptr(o), len(s), tag))

    def store_append_device(self, d_s: int, d_p: int, d_o: int, n: int, tag: int):
        """a slide whose columns are already in this device's memory (copied device-to-device; index maintained as store_append)"""
        self._check(lib().kb_store_append_device(self.h, C.c_void_p(d_s), C.c_void_p(d_p), C.c_void_p(d_o), n, tag))

    def store_evict(self, tag: int):
        self._check(lib().kb_store_evict(self.h, tag))

    def store_delete(self, s, p, o):
        s, p, o = _u32(s), _u32(p), _u32(o)
        self._check(lib().kb_store_delete(self.h, _ptr(s), _ptr(p), _ptr(o), len(s)))

    def store_insert(self, s, p, o, tag: int = 0) -> np.ndarray:
        """kb_store_insert: BTreeSet::insert of each triple in batch order. Returns inserted[i] (bool): triple i was in neither the
        store nor an earlier entry of the batch. The new triples go into a segment tagged `tag`."""
        s, p, o = _u32(s), _u32(p), _u32(o)
        flags = np.zeros(len(s), dtype=np.uint8)
        n = C.c_uint64()
        self._check(lib().kb_store_insert(self.h, _ptr(s), _ptr(p), _ptr(o), len(s), tag, _ptr(flags), C.byref(n)))
        return flags.astype(bool)

    def store_remove(self, s, p, o) -> np.ndarray:
        """kb_store_remove: BTreeSet::remove of each triple in batch order. Returns removed[i] (bool): triple i was in the store and
        no earlier entry of the batch removed it."""
        s, p, o = _u32(s), _u32(p), _u32(o)
        flags = np.zeros(len(s), dtype=np.uint8)
        n = C.c_uint64()
        self._check(lib().kb_store_remove(self.h, _ptr(s), _ptr(p), _ptr(o), len(s), _ptr(flags), C.byref(n)))
        return flags.astype(bool)

    def store_remove_template(self, rel: Relation, tmpl: Sequence[KbPattern]) -> int:
        """kb_store_remove_template: DELETE { tmpl } WHERE { ... } with the WHERE's bindings in `rel`. Returns the triples removed."""
        arr = patterns(tmpl)
        n = C.c_uint64()
        self._check(lib().kb_store_remove_template(self.h, rel.h, arr, len(tmpl), C.byref(n)))
        return n.value

    def store_clear(self):
        self._check(lib().kb_store_clear(self.h))

    def segment_save(self, path: str, tag: Optional[int] = None):
        """kb_segment_save: the segment(s) tagged `tag` — or the whole store when tag is None — as one columnar segment file"""
        self._check(lib().kb_segment_save(self.h, 0 if tag is None else tag, 1 if tag is None else 0, path.encode()))

    def store_append_file(self, path: str, tag: int, verify: bool = True):
        """kb_store_append_file: stream a columnar segment file into a new store segment"""
        self._check(lib().kb_store_append_file(self.h, path.encode(), tag, 1 if verify else 0))

    def build_index(self):
        """SparqlDatabase::build_all_indexes on the device: partition the store by predicate. Returns (n_predicates, build_ms)."""
        n, ms = C.c_uint32(), C.c_double()
        self._check(lib().kb_store_build_index(self.h, C.byref(n), C.byref(ms)))
        return n.value, ms.value

    def set_use_index(self, on: bool):
        self._check(lib().kb_set_use_index(self.h, 1 if on else 0))

    def store_size(self):
        n, ns = C.c_uint64(), C.c_uint32()
        self._check(lib().kb_store_size(self.h, C.byref(n), C.byref(ns)))
        return n.value, ns.value

    def store_download(self):
        n, _ = self.store_size()
        s, p, o = (np.empty(n, dtype=np.uint32) for _ in range(3))
        got = C.c_uint64()
        self._check(lib().kb_store_download(self.h, _ptr(s), _ptr(p), _ptr(o), n, C.byref(got)))
        return s, p, o

    def dict_numeric_load(self, num_or0, is_num):
        num = np.ascontiguousarray(num_or0, dtype=np.float64)
        isn = np.ascontiguousarray(is_num, dtype=np.uint8)
        assert len(num) == len(isn)
        self._check(lib().kb_dict_numeric_load(self.h, _ptr(num), _ptr(isn), len(num)))

    def dict_legacy_i32_load(self, val, is_i32):
        """kb_dict_legacy_i32_load: the i32 view of the terms the legacy executor's FILTER compares with (apply_filters_simd)"""
        v = np.ascontiguousarray(val, dtype=np.int32)
        f = np.ascontiguousarray(is_i32, dtype=np.uint8)
        assert len(v) == len(f)
        self._check(lib().kb_dict_legacy_i32_load(self.h, _ptr(v), _ptr(f), len(v)))

    def dict_numeric_derive(self, tables: int = NUMERIC_F64, first_id: int = 0) -> dict:
        """kb_dict_numeric_derive: the side tables of the ids [first_id, n_ids) the device dictionary holds, parsed from its strings on the
        device (NUMERIC_F64: the table of dict_numeric_load, NUMERIC_I32: that of dict_legacy_i32_load; first_id NUMERIC_APPEND: from the
        first id each table lacks). Returns kb_numeric_info as a dict."""
        info = KbNumericInfo()
        self._check(lib().kb_dict_numeric_derive(self.h, tables, first_id, C.byref(info)))
        return info.as_dict()

    def dict_numeric_download(self, first: int, n: int, f64: bool = True, i32: bool = False):
        """kb_dict_numeric_download: (num_or0 float64, is_num uint8) and/or (val int32, is_i32 uint8) of ids [first, first + n)"""
        num, isn = (np.empty(n, np.float64), np.empty(n, np.uint8)) if f64 else (None, None)
        val, isi = (np.empty(n, np.int32), np.empty(n, np.uint8)) if i32 else (None, None)
        p = lambda a: _ptr(a) if a is not None and len(a) else None
        self._check(lib().kb_dict_numeric_download(self.h, first, n, p(num), p(isn), p(val), p(isi)))
        return (num, isn, val, isi) if f64 and i32 else (num, isn) if f64 else (val, isi)

    def dict_strings_load(self, strings: Sequence[str]):
        """kb_dict_strings_load: string i = the term with dictionary id i (Dictionary::id_to_string, dictionary.rs:17-21)"""
        enc = [x.encode("utf-8") if isinstance(x, str) else bytes(x) for x in strings]
        off = np.zeros(len(enc) + 1, dtype=np.uint64)
        if enc:
            off[1:] = np.cumsum([len(b) for b in enc], dtype=np.uint64)
        data = np.frombuffer(b"".join(enc), dtype=np.uint8) if enc else np.empty(0, np.uint8)
        data = np.ascontiguousarray(data)
        self._check(lib().kb_dict_strings_load(self.h, _ptr(off), _ptr(data) if len(data) else None, len(enc)))

    def dict_encode(self, terms: Sequence[Union[str, bytes]]):
        """kb_dict_encode: Dictionary::encode of a batch of terms on the device. Returns (ids uint32[n], first_pos uint64[n_new]):
        first_pos[k] = index in `terms` of the term that introduced id (ids before the call) + k."""
        enc = [x.encode("utf-8") if isinstance(x, str) else bytes(x) for x in terms]
        n = len(enc)
        ids = np.empty(n, dtype=np.uint32)
        if n == 0:
            return ids, np.empty(0, np.uint64)
        off = np.zeros(n + 1, dtype=np.uint64)
        off[1:] = np.cumsum(np.fromiter((len(b) for b in enc), dtype=np.uint64, count=n), dtype=np.uint64)
        data = np.ascontiguousarray(np.frombuffer(b"".join(enc), dtype=np.uint8)) if off[-1] else np.empty(0, np.uint8)
        first = np.empty(n, dtype=np.uint64)
        n_new = C.c_uint32(0)
        self._check(lib().kb_dict_encode(self.h, _ptr(off), _ptr(data) if len(data) else None, n, _ptr(ids), C.byref(n_new), _ptr(first)))
        return ids, first[: n_new.value].copy()

    def dict_strings_info(self) -> Tuple[int, int]:
        n, b = C.c_uint32(0), C.c_uint64(0)
        self._check(lib().kb_dict_strings_info(self.h, C.byref(n), C.byref(b)))
        return int(n.value), int(b.value)

    def quoted_load(self, ids, s, p, o):
        """kb_quoted_load: the quoted-triple table (QuotedTripleStore::id_to_components) replaces the context's; empty arrays clear it"""
        ids, s, p, o = _u32(ids), _u32(s), _u32(p), _u32(o)
        assert len(ids) == len(s) == len(p) == len(o)
        self._check(lib().kb_quoted_load(self.h, _ptr(ids), _ptr(s), _ptr(p), _ptr(o), len(ids)))

    def quoted_download(self, first_id: int, n: int):
        """kb_quoted_download: (s, p, o) uint32 arrays of the table entries with ids [first_id, first_id + n) (KB_ID_NONE for a hole)"""
        s, p, o = (np.empty(n, dtype=np.uint32) for _ in range(3))
        self._check(lib().kb_quoted_download(self.h, first_id, n, _ptr(s), _ptr(p), _ptr(o)))
        return s, p, o

    def dict_strings_download(self, first: int, n: int) -> List[str]:
        """kb_dict_strings_download: the device dictionary's strings with ids [first, first + n)"""
        off = np.zeros(n + 1, dtype=np.uint64)
        self._check(lib().kb_dict_strings_download(self.h, first, n, _ptr(off), None))
        data = np.empty(max(int(off[-1]), 1), dtype=np.uint8)
        self._check(lib().kb_dict_strings_download(self.h, first, n, _ptr(off), _ptr(data)))
        raw = data.tobytes()
        return [raw[int(off[k]):int(off[k + 1])].decode("utf-8") for k in range(n)]

    def serialize(self, fmt: int, prefixes: Sequence[Tuple[str, str]] = (), capacity: int = 64 << 20, info: Optional[dict] = None):
        """kb_serialize_begin / _next: the store as N-Triples-star (SER_NTRIPLES) or Turtle-star (SER_TURTLE) text, yielded as bytes
        pieces of at most `capacity` bytes (whole units each; capacity must hold the largest unit). prefixes: (name, uri) pairs, in the
        order the Turtle header lists them. `info`, when given, receives kb_serialize_info as a dict before the first piece."""
        enc = [x.encode("utf-8") for pr in prefixes for x in pr]
        off = np.zeros(len(enc) + 1, dtype=np.uint64)
        if enc:
            off[1:] = np.cumsum([len(b) for b in enc], dtype=np.uint64)
        data = np.frombuffer(b"".join(enc), dtype=np.uint8) if off[-1] else np.empty(0, np.uint8)
        h, inf = C.c_void_p(), KbSerializeInfo()
        self._check(lib().kb_serialize_begin(self.h, fmt, _ptr(off), _ptr(data) if len(data) else None, len(prefixes), C.byref(h), C.byref(inf)))
        try:
            if info is not None:
                info.update(inf.as_dict())
            cap = min(capacity, inf.total_bytes)  # (a capacity below the largest unit is refused by the library)
            buf = np.empty(max(cap, 1), dtype=np.uint8)
            got = C.c_uint64()
            while True:
                self._check(lib().kb_serialize_next(self.h, h, _ptr(buf), cap, C.byref(got)))
                if got.value == 0:
                    return
                yield buf[: got.value].tobytes()
        finally:
            lib().kb_serialize_free(h)

    def store_gather_stats(self, max_sample: int = GATHER_STATS_FAST) -> dict:
        """kb_store_gather_stats: DatabaseStats::gather_stats_fast over the store's distinct triples, sampling at most max_sample of
        them (0: every triple). Returns kb_db_stats_info as a dict plus "subject", "predicate" and "object": (ids uint32, counts uint64),
        ids ascending, counts already multiplied by the sampling step."""
        h, inf = C.c_void_p(), KbDbStatsInfo()
        self._check(lib().kb_store_gather_stats(self.h, max_sample, C.byref(h), C.byref(inf)))
        try:
            out = inf.as_dict()
            for pos, name in enumerate(("subject", "predicate", "object")):
                ids, counts, n = C.POINTER(C.c_uint32)(), C.POINTER(C.c_uint64)(), C.c_uint64()
                self._check(lib().kb_db_stats_counts(h, pos, C.byref(ids), C.byref(counts), C.byref(n)))
                k = n.value
                out[name] = (np.ctypeslib.as_array(ids, (k,)).copy() if k else np.empty(0, np.uint32),
                             np.ctypeslib.as_array(counts, (k,)).copy() if k else np.empty(0, np.uint64))
            return out
        finally:
            lib().kb_db_stats_free(h)

    def qb_triples(self, filters: Sequence[Optional[Tuple[int, Union[int, bytes, str]]]] = (None, None, None), join: int = 0,
                   right: Optional["Context"] = None, offset: int = 0, limit: Optional[int] = None, slots: Sequence[int] = (0, 1, 2),
                   count_only: bool = False) -> Tuple[Optional[Relation], dict]:
        """kb_qb_triples: QueryBuilder's get_triples over the store. filters: per position None, (QB_EXACT, id) or (QB_CONTAINS /
        QB_STARTS / QB_ENDS, pattern as str or bytes); join: QB_ON_* bits against `right`'s whole store; rows [offset, offset + limit)
        of the (s, p, o) set order. Returns (relation with columns `slots` = s, p, o, or None when count_only; kb_qb_info as a dict)."""
        spec = KbQbSpec()
        keep = []
        for k, f in enumerate(filters):
            if f is None:
                continue
            mode, arg = f
            spec.pos[k].mode = mode
            if mode == QB_EXACT:
                spec.pos[k].id = int(arg)
            else:
                b = arg.encode("utf-8") if isinstance(arg, str) else bytes(arg)
                buf = C.create_string_buffer(b, max(len(b), 1))
                keep.append(buf)
                spec.pos[k].pattern = C.cast(buf, C.c_void_p)
                spec.pos[k].len = len(b)
        spec.join = join
        spec.offset = offset
        spec.limit = QB_NO_LIMIT if limit is None else limit
        sl = (C.c_uint32 * 3)(*slots)
        h, inf = C.c_void_p(), KbQbInfo()
        self._check(lib().kb_qb_triples(self.h, C.byref(spec), right.h if right is not None else None, sl, None if count_only else C.byref(h),
                                        C.byref(inf)))
        return (None if count_only else Relation(self, h)), inf.as_dict()

    def store_union(self, a: "Context", b: "Context") -> dict:
        """kb_store_union: this context's store, device dictionary and quoted-triple table become those of SparqlDatabase::union(a, b)
        (a and b are only read; both must be other contexts on this device). The index is dropped and the numeric side tables are left
        for dict_numeric_derive. Returns kb_union_info as a dict: the new strings are ids [dict_first, dict_first + dict_new)."""
        inf = KbUnionInfo()
        self._check(lib().kb_store_union(self.h, a.h, b.h, C.byref(inf)))
        return inf.as_dict()

    def store_par_join(self, a: "Context", b: "Context", predicate: int) -> dict:
        """kb_store_par_join: this context's store becomes SparqlDatabase::par_join(a, b, predicate) for a predicate id of a's
        dictionary, and its device dictionary and quoted-triple table copies of a's. Returns kb_par_join_info as a dict."""
        inf = KbParJoinInfo()
        self._check(lib().kb_store_par_join(self.h, a.h, b.h, predicate, C.byref(inf)))
        return inf.as_dict()

    def qb_terms(self, rel: Relation, col: int, mode: int) -> List[str]:
        """kb_qb_terms: column `col` of `rel` as Dictionary::decode(id).unwrap_or("") renders it: every row (QB_TERMS_EMPTY), the rows
        whose id decodes (QB_TERMS_DROP) or their distinct strings in byte order (QB_TERMS_DISTINCT)"""
        h = C.c_void_p()
        self._check(lib().kb_qb_terms(self.h, rel.h, col, mode, C.byref(h)))
        try:
            n, total = C.c_uint64(), C.c_uint64()
            self._check(lib().kb_strings_info(h, C.byref(n), C.byref(total)))
            off = np.empty(n.value + 1, dtype=np.uint64)
            data = np.empty(max(total.value, 1), dtype=np.uint8)
            self._check(lib().kb_strings_download(self.h, h, _ptr(off), _ptr(data)))
        finally:
            lib().kb_strings_free(self.h, h)
        raw = data.tobytes()
        return [raw[int(off[i]):int(off[i + 1])].decode("utf-8") for i in range(n.value)]

    # ---- operators
    def bind(self, rel: Relation, function: int, args: Sequence[KbTerm], out_slot: int, next_qt_id: int = 0,
             consts: Sequence[bytes] = ()) -> Tuple[Relation, dict]:
        """kb_bind: `rel` with the output column of one BIND built-in (appended, or replacing out_slot's column). args: V(slot) for a
        variable; for TRIPLE K(id) for a constant, for CONCAT K(k) for consts[k] (bytes). Returns (relation, kb_bind_info as a dict)."""
        terms = (KbTerm * max(len(args), 1))(*args)
        coff = np.zeros(len(consts) + 1, dtype=np.uint64)
        if consts:
            coff[1:] = np.cumsum([len(b) for b in consts], dtype=np.uint64)
        cdata = np.frombuffer(b"".join(consts) or b"\0", dtype=np.uint8).copy()
        spec = KbBindSpec(function, len(args), terms, len(consts), coff.ctypes.data_as(C.POINTER(C.c_uint64)),
                          cdata.ctypes.data_as(C.POINTER(C.c_uint8)), out_slot, next_qt_id)
        out, info = C.c_void_p(), KbBindInfo()
        self._check(lib().kb_bind(self.h, rel.h, C.byref(spec), C.byref(out), C.byref(info)))
        return Relation(self, out), info.as_dict()

    def scan_quoted(self, qp: KbQuotedPattern) -> Relation:
        """kb_scan_quoted: the bag of an RDF-star pattern (one match pass over the quoted-triple table, then a bind join)"""
        out = C.c_void_p()
        self._check(lib().kb_scan_quoted(self.h, C.byref(qp), C.byref(out)))
        return Relation(self, out)

    def scan(self, pats: Sequence[KbPattern], pushdown: Optional[Sequence[Optional[Sequence[KbFilterOp]]]] = None):
        arr = patterns(pats)
        k = len(pats)
        out = (C.c_void_p * k)()
        if pushdown:
            progs, keep = (C.POINTER(KbFilterOp) * k)(), []
            lens = (C.c_uint32 * k)()
            for i in range(k):
                a, n = filter_prog(pushdown[i] if i < len(pushdown) else None)
                keep.append(a)
                progs[i] = C.cast(a, C.POINTER(KbFilterOp))
                lens[i] = n
            self._check(lib().kb_scan(self.h, arr, k, progs, lens, out))
        else:
            self._check(lib().kb_scan(self.h, arr, k, None, None, out))
        return [Relation(self, out[i]) for i in range(k)]

    def filter(self, rel: Relation, ops: Sequence[KbFilterOp]) -> Relation:
        a, n = filter_prog(ops)
        out = C.c_void_p()
        self._check(lib().kb_filter(self.h, rel.h, a, n, C.byref(out)))
        return Relation(self, out)

    def project(self, rel: Relation, slots: Sequence[int]) -> Relation:
        a = (C.c_uint32 * max(len(slots), 1))(*slots)
        out = C.c_void_p()
        self._check(lib().kb_project(self.h, rel.h, a, len(slots), C.byref(out)))
        return Relation(self, out)

    def hash_join(self, left: Relation, right: Relation) -> Relation:
        out = C.c_void_p()
        self._check(lib().kb_hash_join(self.h, left.h, right.h, C.byref(out)))
        return Relation(self, out)

    def natural_join(self, left: Relation, right: Relation) -> Relation:
        """kb_natural_join: the join of mappings (rsp_engine.rs:684-718) — a KB_ID_NONE cell is an unbound variable, compatible with
        any value; the merged cell is the right value if bound, else the left one"""
        out = C.c_void_p()
        self._check(lib().kb_natural_join(self.h, left.h, right.h, C.byref(out)))
        return Relation(self, out)

    def hash_join_keyed(self, left: Relation, right: Relation, key_slots: Sequence[int], merge: int) -> Relation:
        """kb_hash_join_keyed: rows paired on key_slots only, every other shared slot coalesced MERGE_LEFT_FIRST or MERGE_RIGHT_FIRST;
        a key cell holding KB_ID_NONE raises KB_E_UNSUPPORTED"""
        keys = (C.c_uint32 * max(len(key_slots), 1))(*key_slots)
        out = C.c_void_p()
        self._check(lib().kb_hash_join_keyed(self.h, left.h, right.h, keys, len(key_slots), merge, C.byref(out)))
        return Relation(self, out)

    def values(self, slots: Sequence[int], rows: Sequence[Sequence[Optional[Union[str, bytes]]]]) -> Tuple[Relation, dict]:
        """kb_values: a VALUES block as a device relation. rows[r][v] is the term of header variable slots[v], None for UNDEF; a row
        shorter than the header is UNDEF in its missing cells. Returns (relation, kb_values_info as a dict)."""
        nv, nr = len(slots), len(rows)
        undef = np.ones(nr * nv, dtype=np.uint8)
        lens = np.zeros(nr * nv, dtype=np.uint64)
        parts = []
        for r, row in enumerate(rows):
            for v, t in enumerate(row[:nv]):
                if t is not None:
                    b = t.encode("utf-8") if isinstance(t, str) else bytes(t)
                    undef[r * nv + v] = 0
                    lens[r * nv + v] = len(b)
                    parts.append(b)
        off = np.zeros(nr * nv + 1, dtype=np.uint64)
        off[1:] = np.cumsum(lens, dtype=np.uint64)
        data = np.frombuffer(b"".join(parts) or b"\0", dtype=np.uint8).copy()
        sl = (C.c_uint32 * max(nv, 1))(*slots)
        out, info = C.c_void_p(), KbValuesInfo()
        self._check(lib().kb_values(self.h, sl, nv, nr, _ptr(undef) if len(undef) else None, _ptr(off), _ptr(data), C.byref(out), C.byref(info)))
        return Relation(self, out), info.as_dict()

    def bind_join(self, left: Relation, pat: KbPattern) -> Relation:
        """kb_bind_join: `left` joined with one store pattern (index lookup kernel when the index has a table for it)"""
        out = C.c_void_p()
        arr = patterns([pat])
        self._check(lib().kb_bind_join(self.h, left.h, arr, C.byref(out)))
        return Relation(self, out)

    def star_join(self, join_slot: int, pats: Sequence[KbPattern], filt: Optional[Sequence[KbFilterOp]] = None) -> Relation:
        a, n = filter_prog(filt)
        out = C.c_void_p()
        self._check(lib().kb_star_join(self.h, join_slot, patterns(pats), len(pats), a, n, C.byref(out)))
        return Relation(self, out)

    def bgp_execute(self, pats: Sequence[KbPattern], filt: Optional[Sequence[KbFilterOp]] = None, project: Optional[Sequence[int]] = None) -> Relation:
        a, n = filter_prog(filt)
        out = C.c_void_p()
        if project is not None:
            pr = (C.c_uint32 * max(len(project), 1))(*project)
            self._check(lib().kb_bgp_execute(self.h, patterns(pats), len(pats), a, n, pr, len(project), C.byref(out)))
        else:
            self._check(lib().kb_bgp_execute(self.h, patterns(pats), len(pats), a, n, None, 0, C.byref(out)))
        return Relation(self, out)

    def bgp_last_plan(self) -> dict:
        """kb_bgp_last_plan: the route, components, reduction rounds, rows per pattern, join order and intermediate sizes of the last
        successful bgp_execute"""
        info = KbBgpPlanInfo()
        self._check(lib().kb_bgp_last_plan(self.h, C.byref(info)))
        return info.as_dict()

    def rel_from_host(self, slots: Sequence[int], cols: Sequence[np.ndarray]) -> Relation:
        cols = [_u32(c) for c in cols]
        n = len(cols[0]) if cols else 0
        sl = (C.c_uint32 * max(len(slots), 1))(*slots)
        ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
        out = C.c_void_p()
        self._check(lib().kb_rel_from_host(self.h, sl, len(slots), ptrs, n, C.byref(out)))
        return Relation(self, out)

    def rel_from_device(self, slots: Sequence[int], ptrs_: Sequence[int], n: int) -> Relation:
        sl = (C.c_uint32 * max(len(slots), 1))(*slots)
        ptrs = (C.c_void_p * max(len(ptrs_), 1))(*ptrs_)
        out = C.c_void_p()
        self._check(lib().kb_rel_from_device(self.h, sl, len(slots), ptrs, n, C.byref(out)))
        return Relation(self, out)

    def order_by(self, rel: Relation, keys: Sequence[Tuple[int, bool]] = (), limit: int = 0) -> Tuple[Relation, dict]:
        """kb_order_by: `rel`'s rows sorted stably by keys = [(slot, descending)], then cut to `limit` rows when limit > 0.
        Returns (relation, kb_order_info as a dict). KB_E_UNSUPPORTED (a mixed key column, ...) raises: sort on the host."""
        arr = (KbOrderKey * max(len(keys), 1))(*[KbOrderKey(int(s_), 1 if d else 0) for s_, d in keys])
        out, info = C.c_void_p(), KbOrderInfo()
        self._check(lib().kb_order_by(self.h, rel.h, arr, len(keys), int(limit), C.byref(out), C.byref(info)))
        return Relation(self, out), info.as_dict(len(keys))

    def group_aggregate(self, rel: Relation, group_slots: Sequence[int], aggs: Sequence[tuple]):
        """aggs: [(kind, slot)] -> dict(keys=[cols], values=[cols], counts=array)"""
        gs = (C.c_uint32 * max(len(group_slots), 1))(*group_slots)
        ag = (KbAgg * max(len(aggs), 1))()
        for i, (k, s) in enumerate(aggs):
            ag[i] = KbAgg(k, s)
        g = C.c_void_p()
        self._check(lib().kb_group_aggregate(self.h, rel.h, gs, len(group_slots), ag, len(aggs), C.byref(g)))
        return self._groups_to_dict(g)

    def star_join_aggregate(self, join_slot: int, pats: Sequence[KbPattern], filt, group_slots: Sequence[int], aggs: Sequence[tuple]):
        """kb_star_join_aggregate: star join + GROUP BY without materialising the join when the fused path applies.
        Returns (groups dict as group_aggregate, joined row count)."""
        a, nf = filter_prog(filt)
        gs = (C.c_uint32 * max(len(group_slots), 1))(*group_slots)
        ag = (KbAgg * max(len(aggs), 1))()
        for i, (k, s) in enumerate(aggs):
            ag[i] = KbAgg(k, s)
        g = C.c_void_p()
        n_rows = C.c_uint64()
        self._check(lib().kb_star_join_aggregate(self.h, join_slot, patterns(pats), len(pats), a, nf, gs, len(group_slots), ag, len(aggs), C.byref(g), C.byref(n_rows)))
        return self._groups_to_dict(g), n_rows.value

    def star_join_aggregate_packed(self, join_slot: int, pats: Sequence[KbPattern], filt, group_slots: Sequence[int], aggs: Sequence[tuple]):
        """kb_star_join_aggregate, result left in its transport form (kb_groups_pack): what one rank contributes to a cross-rank
        GROUP BY. Returns (uint8 array, joined row count)."""
        a, nf = filter_prog(filt)
        gs = (C.c_uint32 * max(len(group_slots), 1))(*group_slots)
        ag = (KbAgg * max(len(aggs), 1))()
        for i, (k, s) in enumerate(aggs):
            ag[i] = KbAgg(k, s)
        g = C.c_void_p()
        n_rows = C.c_uint64()
        self._check(lib().kb_star_join_aggregate(self.h, join_slot, patterns(pats), len(pats), a, nf, gs, len(group_slots), ag, len(aggs), C.byref(g), C.byref(n_rows)))
        try:
            return self._groups_pack(g), n_rows.value
        finally:
            lib().kb_groups_free(g)

    def _groups_pack(self, g) -> np.ndarray:
        need = C.c_uint64()
        self._check(lib().kb_groups_pack(g, None, 0, C.byref(need)))
        buf = np.empty(need.value, dtype=np.uint8)
        self._check(lib().kb_groups_pack(g, _ptr(buf), need.value, C.byref(need)))
        return buf

    def groups_merge(self, parts: Sequence[np.ndarray]):
        """kb_groups_merge: fold the packed partial GROUP BY results of several ranks (device kernel); returns the groups dict"""
        parts = [np.ascontiguousarray(p_, dtype=np.uint8) for p_ in parts]
        ptrs = (C.c_void_p * len(parts))(*[p_.ctypes.data for p_ in parts])
        sizes = (C.c_uint64 * len(parts))(*[p_.nbytes for p_ in parts])
        g = C.c_void_p()
        self._check(lib().kb_groups_merge(self.h, ptrs, sizes, len(parts), C.byref(g)))
        return self._groups_to_dict(g)

    def prepare_star_join(self, join_slot: int, pats: Sequence[KbPattern], filt=None, group_slots: Sequence[int] = (), aggs: Sequence[tuple] = (), ring: int = 4) -> "Plan":
        """kb_star_join_prepare: resolve the query once; Plan.submit() is then one asynchronous kernel launch"""
        a, nf = filter_prog(filt)
        gs = (C.c_uint32 * max(len(group_slots), 1))(*group_slots)
        ag = (KbAgg * max(len(aggs), 1))()
        for i, (k, s) in enumerate(aggs):
            ag[i] = KbAgg(k, s)
        h = C.c_void_p()
        self._check(lib().kb_star_join_prepare(self.h, join_slot, patterns(pats), len(pats), a, nf, gs, len(group_slots), ag, len(aggs), ring, C.byref(h)))
        return Plan(self, h)

    def _groups_to_dict(self, g):
        try:
            n, ng, na = C.c_uint64(), C.c_uint32(), C.c_uint32()
            self._check(lib().kb_groups_info(g, C.byref(n), C.byref(ng), C.byref(na)))
            keys, vals = [], []
            for c in range(ng.value):
                p = C.POINTER(C.c_uint32)()
                self._check(lib().kb_groups_keys(g, c, C.byref(p)))
                keys.append(np.ctypeslib.as_array(p, shape=(n.value,)).copy() if n.value else np.empty(0, np.uint32))
            for a in range(na.value):
                p = C.POINTER(C.c_double)()
                self._check(lib().kb_groups_values(g, a, C.byref(p)))
                vals.append(np.ctypeslib.as_array(p, shape=(n.value,)).copy() if n.value else np.empty(0, np.float64))
            pc = C.POINTER(C.c_uint64)()
            self._check(lib().kb_groups_counts(g, C.byref(pc)))
            counts = np.ctypeslib.as_array(pc, shape=(n.value,)).copy() if n.value else np.empty(0, np.uint64)
            return {"keys": keys, "values": vals, "counts": counts}
        finally:
            lib().kb_groups_free(g)

    def datalog_fixpoint(self, rules: Sequence[dict], strategy: int = SEMI_NAIVE):
        """rules: [{'premise': [KbPattern], 'conclusion': [KbPattern], 'filters': [KbRuleFilter]}]"""
        arr, keep = make_rules(rules)
        out = C.c_void_p()
        st = KbFixpointStats()
        self._check(lib().kb_datalog_fixpoint(self.h, arr, len(rules), strategy, C.byref(out), C.byref(st)))
        return Relation(self, out), st

    def datalog_fixpoint_seed(self, rules: Sequence[dict], seed: Relation, strategy: int = SEMI_NAIVE):
        """kb_datalog_fixpoint_seed: the store is closed under `rules` already; `seed` (slots 0,1,2 = s,p,o) are facts to add. Returns
        (relation = the accepted seed facts followed by the facts inferred from them, number of accepted seed facts, stats)."""
        arr, keep = make_rules(rules)
        out = C.c_void_p()
        n_new = C.c_uint64()
        st = KbFixpointStats()
        self._check(lib().kb_datalog_fixpoint_seed(self.h, arr, len(rules), strategy, seed.h, C.byref(out), C.byref(n_new), C.byref(st)))
        return Relation(self, out), int(n_new.value), st

    def datalog_maintain(self, rules: Sequence[dict], evict_tags: Sequence[int] = (), add=None, add_tag: int = 0, strategy: int = SEMI_NAIVE):
        """kb_datalog_maintain: the store is closed under `rules` (an earlier datalog_fixpoint or datalog_maintain with the same rules and
        nothing changed since); the segments tagged `evict_tags` leave, `add` (a Relation with slots 0,1,2 = s,p,o, or an (n,3) uint32
        array; None: nothing added) becomes one segment tagged `add_tag`, and the inferred segment becomes the closure of the new base.
        Returns (inferred_removed, inferred_added, stats): the inferred facts that left and the ones that arrived (3-column relations)."""
        arr, keep = make_rules(rules)
        tags = (C.c_uint64 * max(len(evict_tags), 1))(*[int(t) for t in evict_tags])
        if add is not None and not isinstance(add, Relation):
            a = np.asarray(add, dtype=np.uint32)
            if a.ndim != 2:
                raise ValueError("add must be an (n, 3) array of (s, p, o)")
            add = self.rel_from_host(list(range(a.shape[1])), [a[:, j] for j in range(a.shape[1])])
        rem, new = C.c_void_p(), C.c_void_p()
        st = KbMaintainStats()
        self._check(lib().kb_datalog_maintain(self.h, arr, len(rules), strategy, tags, len(evict_tags), add.h if add is not None else None, add_tag,
                                              C.byref(rem), C.byref(new), C.byref(st)))
        return Relation(self, rem), Relation(self, new), st

    def datalog_query(self, rules: Sequence[dict], query: KbPattern, max_depth: int = BC_MAX_DEPTH):
        """kb_datalog_query: Reasoner::backward_chaining on the device. Returns (relation, stats): one column per distinct variable of
        `query` (s, p, o first-appearance order), each distinct binding of them over the facts with a proof of height <= max_depth once;
        a ground query gives no column and 0 or 1 rows. The store is left as it was."""
        arr, keep = make_rules(rules)
        out = C.c_void_p()
        st = KbBcStats()
        q = KbPattern(query.s, query.p, query.o)
        self._check(lib().kb_datalog_query(self.h, arr, len(rules), C.byref(q), max_depth, C.byref(out), C.byref(st)))
        return Relation(self, out), st

    def datalog_query_repairs(self, constraints: Sequence[dict], query: KbPattern):
        """kb_datalog_query_repairs: Reasoner::query_with_repairs on the device, under IAR semantics. `constraints` are rule dicts whose
        "premise" is read ("conclusion" and "filters" may be absent and are ignored). Returns (relation, stats): one column per distinct
        variable of `query` (s, p, o first-appearance order), each distinct binding of its matches over the store minus the facts of
        every minimal conflict once; a ground query gives no column and 0 or 1 rows. The store is left as it was."""
        arr, keep = make_rules([{"premise": r["premise"], "conclusion": r.get("conclusion", []), "filters": r.get("filters", [])}
                                for r in constraints])
        out = C.c_void_p()
        st = KbRepairStats()
        q = KbPattern(query.s, query.p, query.o)
        self._check(lib().kb_datalog_query_repairs(self.h, arr, len(constraints), C.byref(q), C.byref(out), C.byref(st)))
        return Relation(self, out), st

    def r2s(self, stream_op: int, slots: Sequence[int]) -> "StreamOperator":
        """kb_r2s_create: a Relation-to-Stream operator (RSTREAM / ISTREAM / DSTREAM) over rows of the variables `slots` (their order is
        the column order of what ISTREAM / DSTREAM emit)"""
        sl = (C.c_uint32 * max(len(slots), 1))(*slots)
        h = C.c_void_p()
        self._check(lib().kb_r2s_create(self.h, stream_op, sl, len(slots), C.byref(h)))
        return StreamOperator(self, h)

    def partition(self, rel: Relation, key_slot: int, n_parts: int):
        out = C.c_void_p()
        offs = (C.c_uint64 * (n_parts + 1))()
        self._check(lib().kb_partition(self.h, rel.h, key_slot, n_parts, C.byref(out), offs))
        return Relation(self, out), [offs[i] for i in range(n_parts + 1)]

    def partition_counts(self, rel: Relation, key_slot: int, n_parts: int) -> List[int]:
        cnt = (C.c_uint64 * n_parts)()
        self._check(lib().kb_partition_counts(self.h, rel.h, key_slot, n_parts, cnt))
        return [int(cnt[i]) for i in range(n_parts)]

    def shuffle_scatter(self, rel: Relation, key_slot: int, n_parts: int, peer_cols: Sequence[int], base: Sequence[int], capacity_rows: int):
        """kb_shuffle_scatter: peer_cols[d * n_cols + c] = address of column c of rank d's receive buffer (peer-mapped)"""
        pc = (C.c_void_p * len(peer_cols))(*peer_cols)
        bs = (C.c_uint64 * n_parts)(*base)
        self._check(lib().kb_shuffle_scatter(self.h, rel.h, key_slot, n_parts, pc, bs, capacity_rows))

    def shuffle_push(self, rel: Relation, key_slot: int, n_parts: int, peer_cols: Sequence[int], peer_cursors: Sequence[int], capacity_rows: int):
        """kb_shuffle_push: like shuffle_scatter, ranges reserved on the receivers' own cursors (peer_cursors[d] = address of rank d's
        u32 cursor in peer-mapped memory): no count pass, no count exchange"""
        pc = (C.c_void_p * len(peer_cols))(*peer_cols)
        cu = (C.c_void_p * n_parts)(*peer_cursors)
        self._check(lib().kb_shuffle_push(self.h, rel.h, key_slot, n_parts, pc, cu, capacity_rows))

    def rel_wrap_device(self, slots: Sequence[int], ptrs_: Sequence[int], n: int) -> Relation:
        """kb_rel_wrap_device: a relation over device columns the caller owns (no copy)"""
        sl = (C.c_uint32 * max(len(slots), 1))(*slots)
        ptrs = (C.c_void_p * max(len(ptrs_), 1))(*ptrs_)
        out = C.c_void_p()
        self._check(lib().kb_rel_wrap_device(self.h, sl, len(slots), ptrs, n, C.byref(out)))
        return Relation(self, out)

    def star_join_host(self, s, p, o, join_slot: int, pats: Sequence[KbPattern], filt=None):
        """One-shot host-buffer call (kb_star_join_host): upload + star join + download; result columns are malloc'd by the
        library and copied into numpy arrays here. Returns (rows x cols uint32 array, slots)."""
        s, p, o = _u32(s), _u32(p), _u32(o)
        a, nf = filter_prog(filt)
        n_cols, n_rows = C.c_uint32(), C.c_uint64(0)
        slots = (C.c_uint32 * KB_MAX_COLS)()
        cols = (C.c_void_p * KB_MAX_COLS)()
        self._check(lib().kb_star_join_host(self.h, _ptr(s), _ptr(p), _ptr(o), len(s), join_slot, patterns(pats), len(pats), a, nf,
                                            C.byref(n_cols), slots, cols, C.byref(n_rows)))
        libc = C.CDLL(None)
        libc.free.argtypes = [C.c_void_p]
        out = np.empty((n_rows.value, n_cols.value), dtype=np.uint32)
        for c in range(n_cols.value):
            if n_rows.value:
                out[:, c] = np.ctypeslib.as_array(C.cast(cols[c], C.POINTER(C.c_uint32)), shape=(n_rows.value,))
            libc.free(cols[c])
        return out, [slots[i] for i in range(n_cols.value)]

    # ---- stats
    def set_timing(self, on: bool):
        self._check(lib().kb_set_timing(self.h, 1 if on else 0))

    def get_stats(self, reset: bool = False) -> dict:
        st = KbStats()
        self._check(lib().kb_get_stats(self.h, C.byref(st), 1 if reset else 0))
        return st.as_dict()

    def synchronize(self):
        self._check(lib().kb_synchronize(self.h))

    def set_sharding(self, rank: int, world: int):
        """the store holds shard `rank` of `world` (sharded by subject with kb_shard_of): enables the dense key compaction"""
        self._check(lib().kb_set_sharding(self.h, rank, world))


class Plan:
    """kb_plan: a prepared star join with a ring of result buffers. submit() launches, collect(ticket) waits for that launch."""

    def __init__(self, ctx: Context, handle):
        self.ctx = ctx
        self.h = handle
        ring, cap, nc, grouped = C.c_uint32(), C.c_uint64(), C.c_uint32(), C.c_uint32()
        slots = (C.c_uint32 * KB_MAX_COLS)()
        ctx._check(lib().kb_plan_info(self.h, C.byref(ring), C.byref(cap), C.byref(nc), slots, C.byref(grouped)))
        self.ring, self.capacity_rows, self.grouped = ring.value, cap.value, bool(grouped.value)
        self.slots = [slots[i] for i in range(nc.value)]
        self._ticket = C.c_uint64()
        self._rows = C.c_uint64()
        ctx._plans.add(self)

    def submit(self) -> int:
        rc = lib().kb_plan_submit(self.ctx.h, self.h, C.byref(self._ticket))
        if rc != KB_OK:
            self.ctx._check(rc)
        return self._ticket.value

    def collect(self, ticket: int) -> int:
        """joined row count of the query `ticket` (waits for it)"""
        rc = lib().kb_plan_collect(self.ctx.h, self.h, ticket, C.byref(self._rows), None, None)
        if rc != KB_OK:
            self.ctx._check(rc)
        return self._rows.value

    def collect_rows(self, ticket: int) -> Relation:
        """the result as a Relation VIEW of the ring slot (valid until `ring` further submits)"""
        r = C.c_void_p()
        self.ctx._check(lib().kb_plan_collect(self.ctx.h, self.h, ticket, C.byref(self._rows), C.byref(r), None))
        return Relation(self.ctx, r)

    def collect_groups(self, ticket: int, packed: bool = False):
        """(groups dict — or the kb_groups_pack bytes when packed=True —, joined row count) of a grouped plan"""
        g = C.c_void_p()
        self.ctx._check(lib().kb_plan_collect(self.ctx.h, self.h, ticket, C.byref(self._rows), None, C.byref(g)))
        if packed:
            try:
                return self.ctx._groups_pack(g), self._rows.value
            finally:
                lib().kb_groups_free(g)
        return self.ctx._groups_to_dict(g), self._rows.value

    def peer_scratch_bytes(self) -> int:
        return int(lib().kb_plan_peer_scratch_bytes(self.h))

    def attach_peers(self, rank: int, world: int, peer_scratch: Sequence[int], keep=None):
        """kb_plan_attach_peers: peer_scratch[r] = device-visible address of rank r's zeroed scratch (peer_scratch_bytes() each);
        `keep` = whatever owns that memory (kept alive with the plan)"""
        ptrs = (C.c_void_p * world)(*peer_scratch)
        self.ctx._check(lib().kb_plan_attach_peers(self.ctx.h, self.h, rank, world, ptrs))
        self._keep = keep

    def free(self):
        if self.h:
            lib().kb_plan_free(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class StreamOperator:
    """kb_r2s: a Relation-to-Stream operator whose state (the previous evaluation's distinct rows) lives in device memory.
    eval(rel) returns the emitted rows as a Relation; info() = (distinct rows held, stream operator)."""

    def __init__(self, ctx: Context, handle):
        self.ctx = ctx
        self.h = handle
        ctx._plans.add(self)  # freed with the context's other handles, before the context itself

    def eval(self, rel: Relation) -> Relation:
        out = C.c_void_p()
        self.ctx._check(lib().kb_r2s_eval(self.ctx.h, self.h, rel.h, C.byref(out)))
        return Relation(self.ctx, out)

    def info(self) -> Tuple[int, int]:
        n, op = C.c_uint64(), C.c_uint32()
        self.ctx._check(lib().kb_r2s_info(self.h, C.byref(n), C.byref(op)))
        return n.value, op.value

    def free(self):
        if self.h:
            lib().kb_r2s_free(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def star_join_host_raw(ctx: Context, s_ptr: int, p_ptr: int, o_ptr: int, n: int, join_slot: int, pats, filt, out_ptrs: Sequence[int], out_cap: int):
    """kb_star_join_host_into with raw host pointers (pinned torch / numpy memory) for inputs and outputs. Returns (n_rows, slots)."""
    a, nf = filter_prog(filt)
    n_cols, n_rows = C.c_uint32(), C.c_uint64(0)
    slots = (C.c_uint32 * KB_MAX_COLS)()
    cols = (C.c_void_p * KB_MAX_COLS)()
    for i, ptr in enumerate(out_ptrs):
        cols[i] = ptr
    ctx._check(lib().kb_star_join_host_into(ctx.h, C.c_void_p(s_ptr), C.c_void_p(p_ptr), C.c_void_p(o_ptr), n, join_slot, patterns(pats), len(pats),
                                            a, nf, C.byref(n_cols), slots, cols, out_cap, C.byref(n_rows)))
    return n_rows.value, [slots[i] for i in range(n_cols.value)]


def make_rules(rules: Sequence[dict]):
    arr = (KbRule * max(len(rules), 1))()
    keep = []
    for i, r in enumerate(rules):
        prem = patterns(r["premise"])
        conc = patterns(r["conclusion"])
        fl = r.get("filters", [])
        farr = (KbRuleFilter * max(len(fl), 1))()
        for j, f in enumerate(fl):
            farr[j] = f
        keep += [prem, conc, farr]
        arr[i] = KbRule(C.cast(prem, C.POINTER(KbPattern)), len(r["premise"]), C.cast(farr, C.POINTER(KbRuleFilter)), len(fl),
                        C.cast(conc, C.POINTER(KbPattern)), len(r["conclusion"]))
    arr._keep = keep  # keep the nested arrays alive as long as the rule array
    return arr, keep


def legacy_hash_join_cuda(subjects, predicates, objects, predicate_filter: int, literal_filter: Optional[int] = None, libpath: Optional[str] = None) -> np.ndarray:
    """Replays exactly what Kolibrie's `hash_join_cuda` does (kolibrie/src/cuda/cuda_join.rs:28-60) against the legacy symbol."""
    L = lib() if libpath is None else C.CDLL(libpath)
    fn = L.perform_hash_join_cuda
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.POINTER(C.c_uint32)), C.POINTER(C.c_uint32)]
    s, p, o = _u32(subjects), _u32(predicates), _u32(objects)
    lit = C.c_uint32(literal_filter) if literal_filter is not None else None
    idx = C.POINTER(C.c_uint32)()
    cnt = C.c_uint32(0)
    fn(_ptr(s), _ptr(p), _ptr(o), len(s), predicate_filter, C.byref(lit) if lit is not None else None, C.byref(idx), C.byref(cnt))
    out = np.ctypeslib.as_array(idx, shape=(cnt.value,)).copy() if cnt.value else np.empty(0, np.uint32)
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    if idx:
        libc.free(C.cast(idx, C.c_void_p))  # the Rust side frees it through Vec's drop = libc free
    return out


def segment_write(path: str, s, p, o, tag: int = 0):
    """kb_segment_write (host only): three u32 columns as a columnar segment file"""
    s, p, o = _u32(s), _u32(p), _u32(o)
    rc = lib().kb_segment_write(path.encode(), _ptr(s), _ptr(p), _ptr(o), len(s), tag)
    if rc != KB_OK:
        raise KolibrieError(rc, f"cannot write {path}")


def segment_info(path: str):
    """kb_segment_info (host only): (n_triples, tag, cmin[3], cmax[3]) of a segment file"""
    n, tag = C.c_uint64(), C.c_uint64()
    lo, hi = (C.c_uint32 * 3)(), (C.c_uint32 * 3)()
    rc = lib().kb_segment_info(path.encode(), C.byref(n), C.byref(tag), lo, hi)
    if rc != KB_OK:
        raise KolibrieError(rc, f"{path} is not a segment file")
    return n.value, tag.value, list(lo), list(hi)
