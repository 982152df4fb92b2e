// kb_union.cu — SparqlDatabase::union and SparqlDatabase::par_join (kolibrie/src/sparql_database.rs:1874-2005): two device stores on
// one device combined into a third context's store, dictionary and quoted-triple table.
//
// kb_store_union runs five phases, each timed in kb_union_info.phase_ms:
//   sets        store_distinct (kb_serialize.cu) of b's live segments and of a's: each store as the BTreeSet the reference iterates.
//   terms       b's 3n ids in iteration order (s, p, o of each triple): union_first_kernel keeps, per id of b's dictionary, the smallest
//               position it occurs at (an atomicMin after a plain read, so a predicate met at every triple costs one atomic per warp
//               wave, not one per row) and raises a flag for an id b's dictionary does not map (a quoted id, an id past it: the
//               reference's decode(..).unwrap() panics). union_mark_kernel flags the positions k with first[id[k]] == k, an exclusive
//               scan of the flags (launch_exclusive_scan_u32, as dict_encode_device ranks its first occurrences) gives each its rank,
//               and union_terms_kernel writes the id at that rank: b's distinct terms in first-seen order, without a sort.
//   dictionary  decode_ids (Plain, from b's dictionary) renders the terms; dst's dictionary becomes a copy of a's (dict_copy) and
//               dict_encode_device encodes the terms into it. Distinct strings in first-seen order get exactly the ids the reference's
//               3n sequential encode(decode(..)) calls hand out: a string a holds keeps its id, every other one takes the next.
//   remap       union_remap_scatter_kernel writes each term's new id into a table over b's ids; union_remap_rows_kernel maps b's set
//               through it.
//   union       store_distinct of a's set and the remapped set: the union in ascending (s, p, o) order, dst's one new segment.
// kb_store_par_join runs four: the predicate's rows of both stores (scan_predicates, kb_scan.cu); the distinct (a.o, a.s) and (b.s, b.o)
// pairs and the distinct objects of B with the exact sizes of the join and of the semi-join (distinct_pairs / pair_join_count,
// kb_qbuilder.cu); the join a.o = b.s and the semi-join of a.o against B's objects (hash_join_impl, kb_join.cu); store_distinct of both.
// Nothing in dst changes until every refusal has been decided; the dictionary is restored if a later step fails, the quoted table and
// the store are replaced last.
#include <algorithm>

#include "kb_internal.hpp"

using kb::u32;
using kb::u64;

namespace kb {
namespace {

constexpr int UT = 256;                  // threads per block of every kernel here
constexpr u64 ROWS_MAX = 0xFFFFFFF0ull;  // 2^32 - 16: rows of one sort, and positions of b's id sequence

// id at position k of the sequence s0 p0 o0 s1 p1 o1 ... of a store_distinct result (S, PO)
__device__ __forceinline__ u32 term_at(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u32 k) {
    const u32 i = k / 3u, r = k - 3u * i;
    if (r == 0u) return __ldg(S + i);
    const unsigned long long po = __ldg(PO + i);
    return r == 1u ? (u32)(po >> 32) : (u32)po;
}

// first[id] = the smallest position of id among the m positions; *unmapped = 1 when an id is not below dict_ids
__global__ void __launch_bounds__(UT) union_first_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u32 m, u32 dict_ids,
                                                         u32* __restrict__ first, u32* unmapped) {
    bool bad = false;
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        const u32 id = term_at(S, PO, k);
        if (id >= dict_ids) bad = true;
        else if (__ldcg(first + id) > k) atomicMin(first + id, k);
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31u) == 0u) *unmapped = 1u;
}

// keep[k] = 1 when position k is its id's first (the id is mapped): the exclusive scan of keep is then the term's rank
__global__ void __launch_bounds__(UT) union_mark_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u32 m, u32 dict_ids,
                                                        const u32* __restrict__ first, u32* __restrict__ keep) {
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        const u32 id = term_at(S, PO, k);
        keep[k] = id < dict_ids && __ldg(first + id) == k ? 1u : 0u;
    }
}

// out[rank[k]] = the id at k for the positions that are their id's first: b's distinct terms in first-seen order
__global__ void __launch_bounds__(UT) union_terms_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u32 m, u32 dict_ids,
                                                         const u32* __restrict__ first, const u32* __restrict__ rank, u32* __restrict__ out) {
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        const u32 id = term_at(S, PO, k);
        if (id < dict_ids && __ldg(first + id) == k) out[rank[k]] = id;
    }
}

// the u32 offsets of decode_ids widened to the u64 offsets dict_encode_device reads
__global__ void __launch_bounds__(UT) union_widen_kernel(const u32* __restrict__ in, u32 n, unsigned long long* __restrict__ out) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = in[i];
}

// remap[terms[r]] = ids[r]
__global__ void __launch_bounds__(UT) union_remap_scatter_kernel(const u32* __restrict__ terms, const u32* __restrict__ ids, u32 d, u32* __restrict__ remap) {
    for (u32 r = blockIdx.x * blockDim.x + threadIdx.x; r < d; r += gridDim.x * blockDim.x) remap[terms[r]] = ids[r];
}

// row i of (S, PO) with every id mapped through remap, as three columns
__global__ void __launch_bounds__(UT) union_remap_rows_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u32 n,
                                                              const u32* __restrict__ remap, u32* __restrict__ s, u32* __restrict__ p, u32* __restrict__ o) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long po = PO[i];
        s[i] = __ldg(remap + S[i]);
        p[i] = __ldg(remap + (u32)(po >> 32));
        o[i] = __ldg(remap + (u32)po);
    }
}

auto U = [](const Buf& b) { return static_cast<u32*>(b->p); };

// what both entry points refuse before anything is read
kb_status check_contexts(kb_ctx* dst, const kb_ctx* a, const kb_ctx* b) {
    if (!a || !b) return fail(dst, KB_E_INVALID, "NULL context");
    if (dst == a || dst == b) return fail(dst, KB_E_INVALID, "dst must differ from a and from b (they are only read)");
    if (a->device != dst->device || b->device != dst->device)
        return fail(dst, KB_E_INVALID, "a is on device %d, b on device %d, dst on device %d: all three must share one", a->device, b->device, dst->device);
    if (dst->shard_world > 1 || a->shard_world > 1 || b->shard_world > 1) return fail(dst, KB_E_UNSUPPORTED, "a sharded context: the call reads and writes whole stores");
    return KB_OK;
}

// the n sorted distinct triples (S, PO) as dst's one segment, with its statistics
kb_status sorted_segment(kb_ctx* dst, const Buf& S, const Buf& PO, u32 n, Segment* sg) {
    *sg = Segment{};
    sg->n = n;
    KB_TRY(alloc_col(dst, n, &sg->s));
    KB_TRY(alloc_col(dst, n, &sg->p));
    KB_TRY(alloc_col(dst, n, &sg->o));
    KB_TRY(split_sorted(dst, S, PO, 0, n, sg->s.ptr, sg->p.ptr, sg->o.ptr));
    return segment_stats(dst, sg);
}

// the store's set: *n distinct triples, *S / *PO as store_distinct leaves them (empty store: n = 0, no buffers)
kb_status store_set(kb_ctx* dst, const kb_ctx* src, const char* what, Buf* S, Buf* PO, u32* n) {
    u64 n_raw = 0;
    const std::vector<ColSpan> spans = store_spans(src, &n_raw);
    *n = 0;
    if (n_raw >= ROWS_MAX) return fail(dst, KB_E_LIMIT, "%s holds %llu triples (limit 2^32 - 16)", what, (unsigned long long)n_raw);
    if (n_raw) KB_TRY(store_distinct(dst, spans, S, PO, n));
    return KB_OK;
}

// What follows the copy of a's dictionary into dst: b's terms encoded into it, b's set remapped, the union sorted, the quoted table
// copied and the store replaced. A failure returns before the store is replaced; the caller restores dst's dictionary.
struct UnionInput {
    Buf Sa, POa, Sb, POb, terms, off64, tbytes;
    u32 na = 0, nb = 0, d = 0, b_ids = 0;
    u64 total = 0;
};
kb_status union_commit(kb_ctx* dst, const kb_ctx* a, const UnionInput& in, kb_union_info* info, PhaseTimer<6>& pt) {
    Buf ids, remap;
    u32 n_new = 0;
    if (in.d) {
        KB_TRY(alloc_buf(dst, (size_t)in.d * sizeof(u32), &ids));
        KB_TRY(dict_encode_device(dst, static_cast<const u64*>(in.off64->p), static_cast<const unsigned char*>(in.tbytes->p), in.d, in.total, U(ids),
                                  &n_new, nullptr));
    }
    info->dict_new = n_new;
    pt.mark(dst->st);

    // ---- remap: b's set in dst's ids
    Col bcols[3];
    if (in.nb) {
        for (Col& c : bcols) KB_TRY(alloc_col(dst, in.nb, &c));
        KB_TRY(alloc_buf(dst, (size_t)in.b_ids * sizeof(u32), &remap));
        timer_begin(dst, F_OTHER, 2);
        union_remap_scatter_kernel<<<grid_1d(in.d, dst->n_sms, UT), UT, 0, dst->st>>>(U(in.terms), U(ids), in.d, U(remap));
        union_remap_rows_kernel<<<grid_1d(in.nb, dst->n_sms, UT), UT, 0, dst->st>>>(U(in.Sb), static_cast<const unsigned long long*>(in.POb->p), in.nb,
                                                                                  U(remap), bcols[0].ptr, bcols[1].ptr, bcols[2].ptr);
        timer_end(dst);
        KB_CUDA(dst, cudaGetLastError());
    }
    pt.mark(dst->st);

    // ---- union: a's set and b's remapped set, sorted and deduplicated, as dst's one segment
    std::vector<ColSpan> spans;
    Col acols[3];
    if (in.na) {
        for (Col& c : acols) KB_TRY(alloc_col(dst, in.na, &c));
        KB_TRY(split_sorted(dst, in.Sa, in.POa, 0, in.na, acols[0].ptr, acols[1].ptr, acols[2].ptr));
        spans.push_back({acols[0].ptr, acols[1].ptr, acols[2].ptr, in.na, nullptr});
    }
    if (in.nb) spans.push_back({bcols[0].ptr, bcols[1].ptr, bcols[2].ptr, in.nb, nullptr});
    Buf S, PO;
    u32 n = 0;
    if (!spans.empty()) KB_TRY(store_distinct(dst, spans, &S, &PO, &n));
    Segment sg;
    KB_TRY(sorted_segment(dst, S, PO, n, &sg));
    KB_TRY(quoted_copy(dst, a));  // D shares a's quoted-triple store
    pt.mark(dst->st);
    store_replace(dst, n ? std::vector<Segment>{sg} : std::vector<Segment>{});
    info->n_rows = n;
    return KB_OK;
}

kb_status store_union(kb_ctx* dst, const kb_ctx* a, const kb_ctx* b, kb_union_info* info) {
    KB_TRY(check_contexts(dst, a, b));
    u64 na_raw = 0, nb_raw = 0;
    store_spans(a, &na_raw);
    store_spans(b, &nb_raw);
    if (na_raw && !a->dict_ids) return fail(dst, KB_E_UNSUPPORTED, "a's store needs a's device dictionary strings (kb_dict_strings_load)");
    if (nb_raw && !b->dict_ids) return fail(dst, KB_E_UNSUPPORTED, "b's store needs b's device dictionary strings (kb_dict_strings_load)");
    KB_CUDA(dst, cudaStreamSynchronize(a->st));  // the last writes of a and b are done
    KB_CUDA(dst, cudaStreamSynchronize(b->st));
    info->dict_first = a->dict_ids;
    PhaseTimer<6> pt;
    pt.mark(dst->st);

    // ---- sets
    Buf Sa, POa, Sb, POb;
    u32 na = 0, nb = 0;
    KB_TRY(store_set(dst, b, "b", &Sb, &POb, &nb));
    if (3ull * nb >= ROWS_MAX) return fail(dst, KB_E_LIMIT, "b's %u triples give %llu ids to re-encode (limit 2^32 - 16)", nb, 3ull * nb);
    KB_TRY(store_set(dst, a, "a", &Sa, &POa, &na));
    info->n_a = na;
    info->n_b = nb;
    if ((u64)na + nb >= ROWS_MAX) return fail(dst, KB_E_LIMIT, "the union gives %llu rows before the dedup (limit 2^32 - 16)", (unsigned long long)na + nb);
    pt.mark(dst->st);

    // ---- terms: b's distinct ids in first-seen order over s, p, o of each triple
    Buf terms;
    u32 d = 0;
    if (nb) {
        const u32 m = 3u * nb;
        Buf first;
        KB_TRY(alloc_buf(dst, (size_t)b->dict_ids * sizeof(u32), &first));
        KB_TRY(alloc_buf(dst, (size_t)m * sizeof(u32), &terms));
        KB_CUDA(dst, cudaMemsetAsync(first->p, 0xFF, (size_t)b->dict_ids * sizeof(u32), dst->st));
        Buf rank, scratch;
        KB_TRY(alloc_buf(dst, ((size_t)m + 1) * sizeof(u32), &rank));
        KB_TRY(alloc_buf(dst, (((size_t)m + 1) / 2048 + 4) * sizeof(u32), &scratch));
        KB_CUDA(dst, cudaMemsetAsync(U(rank) + m, 0, sizeof(u32), dst->st));
        const u32 c = ctrl_alloc(dst, 2);  // [0] unmapped, [1] distinct terms (rank[m] after the scan)
        const unsigned long long* PO = static_cast<const unsigned long long*>(POb->p);
        const int grid = grid_1d(m, dst->n_sms, UT);
        timer_begin(dst, F_OTHER, 6);  // first, mark, the scan's three kernels, terms
        union_first_kernel<<<grid, UT, 0, dst->st>>>(U(Sb), PO, m, b->dict_ids, U(first), dst->ctrl + c);
        union_mark_kernel<<<grid, UT, 0, dst->st>>>(U(Sb), PO, m, b->dict_ids, U(first), U(rank));
        launch_exclusive_scan_u32(U(rank), m + 1, U(scratch), dst->st);
        union_terms_kernel<<<grid, UT, 0, dst->st>>>(U(Sb), PO, m, b->dict_ids, U(first), U(rank), U(terms));
        timer_end(dst);
        KB_CUDA(dst, cudaMemcpyAsync(dst->ctrl + c + 1, U(rank) + m, sizeof(u32), cudaMemcpyDeviceToDevice, dst->st));
        KB_CUDA(dst, cudaGetLastError());
        KB_TRY(ctrl_read(dst));
        if (dst->h_ctrl[c])
            return fail(dst, KB_E_INVALID, "b's store holds an id b's dictionary does not map (a quoted-triple id, or an id past its %u strings): "
                        "the reference's decode(..).unwrap() panics", b->dict_ids);
        d = dst->h_ctrl[c + 1];
    }
    info->n_terms = d;
    if ((u64)a->dict_ids + d >= 0x80000000ull)
        return fail(dst, KB_E_LIMIT, "a's %u strings and b's %u distinct terms could reach id 2^31 (reserved for quoted triples)", a->dict_ids, d);
    pt.mark(dst->st);

    // ---- dictionary: b's terms rendered from b's dictionary; dst's becomes a copy of a's, into which they are encoded
    UnionInput in;
    in.Sa = Sa; in.POa = POa; in.Sb = Sb; in.POb = POb; in.terms = terms;
    in.na = na; in.nb = nb; in.d = d; in.b_ids = b->dict_ids;
    if (d) {
        const DictTab bdict = dicttab(b);
        Buf toff;
        KB_TRY(decode_ids(dst, U(terms), d, 0, Decode::Plain, "b's terms", &toff, &in.tbytes, &in.total, &bdict));
        if (in.total >= ROWS_MAX) return fail(dst, KB_E_LIMIT, "b's terms take %llu bytes (limit 2^32 - 16)", (unsigned long long)in.total);
        KB_TRY(alloc_buf(dst, ((size_t)d + 1) * sizeof(u64), &in.off64));
        timer_begin(dst, F_OTHER, 1);
        union_widen_kernel<<<grid_1d((u64)d + 1, dst->n_sms, UT), UT, 0, dst->st>>>(U(toff), d + 1, static_cast<unsigned long long*>(in.off64->p));
        timer_end(dst);
        KB_CUDA(dst, cudaGetLastError());
    }
    DictState prev;
    KB_TRY(dict_copy(dst, a, &prev));
    const kb_status rc = union_commit(dst, a, in, info, pt);
    if (rc != KB_OK) {  // dst keeps the dictionary it had
        dict_restore(dst, std::move(prev));
        return rc;
    }
    KB_CUDA(dst, cudaStreamSynchronize(dst->st));
    for (int k = 0; k < 5; k++) info->phase_ms[k] = pt.ms(k);
    timers_flush(dst);
    return KB_OK;
}

kb_status store_par_join(kb_ctx* dst, const kb_ctx* a, const kb_ctx* b, u32 pred, kb_par_join_info* info) {
    KB_TRY(check_contexts(dst, a, b));
    if (pred == KB_ID_NONE) return fail(dst, KB_E_INVALID, "predicate KB_ID_NONE (reserved)");
    if (!a->dict_ids) return fail(dst, KB_E_UNSUPPORTED, "a's device dictionary strings are needed: the result shares a's dictionary (kb_dict_strings_load)");
    u64 na_raw = 0, nb_raw = 0;
    store_spans(a, &na_raw);
    store_spans(b, &nb_raw);
    if (na_raw >= ROWS_MAX || nb_raw >= ROWS_MAX)
        return fail(dst, KB_E_LIMIT, "a store of %llu triples (limit 2^32 - 16)", (unsigned long long)std::max(na_raw, nb_raw));
    KB_CUDA(dst, cudaStreamSynchronize(a->st));  // the last writes of a and b are done
    KB_CUDA(dst, cudaStreamSynchronize(b->st));
    PhaseTimer<5> pt;
    pt.mark(dst->st);

    // ---- select: (s, o) of the predicate's rows in each store
    std::vector<std::unique_ptr<kb_rel>> ra, rb;
    KB_TRY(scan_predicates(dst, a->segs, &pred, 1, ScanOut::Cols, &ra));
    KB_TRY(scan_predicates(dst, b->segs, &pred, 1, ScanOut::Cols, &rb));
    const kb_rel& A = *ra[0];
    const kb_rel& B = *rb[0];
    pt.mark(dst->st);

    // ---- the distinct pairs, and the exact sizes of the join and of the semi-join
    Buf lp, rp, yp;
    u32 nl = 0, nr = 0, ny = 0;
    const u32* as = A.cols[A.col_of(0)].ptr;
    const u32* ao = A.cols[A.col_of(1)].ptr;
    const u32* bs = B.cols[B.col_of(0)].ptr;
    const u32* bo = B.cols[B.col_of(1)].ptr;
    KB_TRY(distinct_pairs(dst, {{ao, as}}, {A.n}, &lp, &nl));  // (a.o << 32 | a.s)
    KB_TRY(distinct_pairs(dst, {{bs, bo}}, {B.n}, &rp, &nr));  // (b.s << 32 | b.o)
    KB_TRY(distinct_pairs(dst, {{bo, bo}}, {B.n}, &yp, &ny));  // B's distinct objects (y << 32 | y)
    info->n_a = nl;
    info->n_b = nr;
    u64 n_join = 0, n_semi = 0;
    KB_TRY(pair_join_count(dst, lp, nl, rp, nr, &n_join));
    KB_TRY(pair_join_count(dst, lp, nl, yp, ny, &n_semi));
    info->n_join = n_join;
    info->n_semi = n_semi;
    if (n_join + n_semi >= ROWS_MAX)
        return fail(dst, KB_E_LIMIT, "the join gives %llu rows before the dedup (limit 2^32 - 16)", (unsigned long long)(n_join + n_semi));
    pt.mark(dst->st);

    // ---- join a.o = b.s -> (a.s, P, b.o); semi-join a.o in B's objects -> (a.s, P, a.o). Slots: 0 a.s, 1 the key, 2 b.o, 3 y.
    std::unique_ptr<kb_rel> L, J, S2;
    std::vector<ColSpan> spans;
    Col pcol;
    KB_TRY(alloc_col(dst, std::max<u64>(n_join, n_semi), &pcol));
    if (n_join || n_semi) {
        launch_fill_u32(pcol.ptr, pred, std::max<u64>(n_join, n_semi), dst->st);
        dst->stats.kernel_launches++;
        KB_TRY(pair_rel(dst, lp, nl, 1, 0, &L));
    }
    if (n_join) {
        std::unique_ptr<kb_rel> R;
        KB_TRY(pair_rel(dst, rp, nr, 1, 2, &R));
        KB_TRY(hash_join_impl(dst, *L, *R, nullptr, &J));
        if (J->n != n_join) return fail(dst, KB_E_CUDA, "the join gave %llu rows, %llu counted", (unsigned long long)J->n, (unsigned long long)n_join);
        spans.push_back({J->cols[J->col_of(0)].ptr, pcol.ptr, J->cols[J->col_of(2)].ptr, J->n, nullptr});
    }
    if (n_semi) {
        std::unique_ptr<kb_rel> Y;
        KB_TRY(pair_rel(dst, yp, ny, 1, 3, &Y));
        KB_TRY(hash_join_impl(dst, *L, *Y, nullptr, &S2));
        if (S2->n != n_semi) return fail(dst, KB_E_CUDA, "the semi-join gave %llu rows, %llu counted", (unsigned long long)S2->n, (unsigned long long)n_semi);
        spans.push_back({S2->cols[S2->col_of(0)].ptr, pcol.ptr, S2->cols[S2->col_of(1)].ptr, S2->n, nullptr});
    }
    pt.mark(dst->st);

    // ---- sort + dedup into dst's one segment; dst's dictionary and quoted table become copies of a's
    Buf S, PO;
    u32 n = 0;
    if (!spans.empty()) KB_TRY(store_distinct(dst, spans, &S, &PO, &n));
    Segment sg;
    KB_TRY(sorted_segment(dst, S, PO, n, &sg));
    DictState prev;
    KB_TRY(dict_copy(dst, a, &prev));
    const kb_status rc = quoted_copy(dst, a);
    if (rc != KB_OK) {
        dict_restore(dst, std::move(prev));
        return rc;
    }
    pt.mark(dst->st);
    store_replace(dst, n ? std::vector<Segment>{sg} : std::vector<Segment>{});
    info->n_rows = n;
    KB_CUDA(dst, cudaStreamSynchronize(dst->st));
    for (int k = 0; k < 4; k++) info->phase_ms[k] = pt.ms(k);
    timers_flush(dst);
    return KB_OK;
}

}  // namespace
}  // namespace kb

extern "C" {

kb_status kb_store_union(kb_ctx* dst, const kb_ctx* a, const kb_ctx* b, kb_union_info* info) {
    KB_ENTER(dst);
    kb_union_info local{};
    if (!info) info = &local;
    *info = kb_union_info{};
    return kb::store_union(dst, a, b, info);
}

kb_status kb_store_par_join(kb_ctx* dst, const kb_ctx* a, const kb_ctx* b, uint32_t predicate, kb_par_join_info* info) {
    KB_ENTER(dst);
    kb_par_join_info local{};
    if (!info) info = &local;
    *info = kb_par_join_info{};
    return kb::store_par_join(dst, a, b, predicate, info);
}

}  // extern "C"
