// kb_serialize.cu — the device store as RDF text: SparqlDatabase::generate_ntriples and generate_turtle (sparql_database.rs:301-382),
// byte for byte, written in pieces so that the whole text is never resident.
//
// kb_serialize_begin does the ordering work and keeps, per distinct triple, what writing its UNIT needs (a unit is one N-Triples line,
// or one triple's share of the Turtle text with its separators):
//   sort      the live segments' s / p / o gathered into (s, packed p|o) and sorted by two stable LSD radix sorts (p|o first, then s):
//             ascending (s, p, o), the reference's BTreeSet<Triple> order (triple.rs:13-18); equal neighbours are dropped
//             (store_distinct, which kb_store_gather_stats and kb_qb_triples share)
//   render    every distinct id of the triples rendered once by the decode kernels of kb_rel_decode in their "missing -> empty" mode
//             (decode_any(..).unwrap_or_default()), with a class byte per term taken from its rendered bytes (starts with "<<", with
//             "http://" / "https://"); a triple holds the index of its three terms in the sorted distinct ids
//   ranks     Turtle: the dense rank of every rendered text (rank_values of kb_order.cu), then a stable radix sort of the id-ordered
//             triples by (rank of the subject text, rank of the predicate text): the BTreeMap<String, BTreeMap<String, Vec<_>>> order
//             with objects in id order inside a group; subject / predicate group boundaries become a flag byte per unit
//   units     the length of every unit from its terms' lengths and classes and its flags; a u64 exclusive scan gives their offsets
// kb_serialize_next finds the whole units that fit, writes them into a device staging buffer (one warp per 32 units, each unit's
// pieces copied by the lanes together, as decode_gather copies strings) and copies them to the caller's host buffer.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>

#include "kb_internal.hpp"

using kb::u32;
using kb::u64;
using kb::u8;

struct kb_serializer {
    kb_ctx* ctx = nullptr;
    int device = 0;
    u32 format = 0;
    u64 store_version = 0;
    std::string header;       // Turtle's @prefix lines: a unit of its own, written first
    bool header_done = false;
    u64 n = 0, cursor = 0;    // units (distinct triples) and the next one to write
    u64 max_unit = 0;
    kb::Buf ts, tp, to;       // u32 per unit: index of its subject / predicate / object among the rendered terms
    kb::Buf flags;            // Turtle: u8 per unit, SF_* bits
    kb::Buf uoff;             // u64 [n + 1]: exclusive prefix of the unit lengths
    kb::Buf toff, tbytes, tcls;  // rendered terms: u32 offsets [terms + 1], bytes, class byte
};

namespace kb {
namespace {

constexpr int ST = 256;  // threads per block of every kernel here
enum : u8 { TC_QUOTED = 1, TC_IRI = 2 };                   // term class: text starts with "<<"; with "http://" or "https://"
enum : u8 { SF_SUBJ = 1, SF_PRED = 2, SF_SUBJ_END = 4 };  // unit flags: first of its subject group, of its predicate group; last of its subject group


__global__ void __launch_bounds__(ST) ser_load_kernel(const u32* __restrict__ s, const u32* __restrict__ p, const u32* __restrict__ o, u64 n,
                                                      u32* __restrict__ S, unsigned long long* __restrict__ PO) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        S[i] = s[i];
        PO[i] = (unsigned long long)p[i] << 32 | o[i];
    }
}

__global__ void __launch_bounds__(ST) ser_distinct_flags_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u32 n,
                                                                u8* __restrict__ keep) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        keep[i] = i == 0u || S[i] != S[i - 1] || PO[i] != PO[i - 1];
}

// the three id columns of the distinct triples, one after the other: what the distinct terms are taken from
__global__ void __launch_bounds__(ST) ser_ids_kernel(const u32* __restrict__ S, const unsigned long long* __restrict__ PO, u32 n, u32* __restrict__ ids) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long po = PO[i];
        ids[i] = S[i];
        ids[(u64)n + i] = (u32)(po >> 32);
        ids[2ull * n + i] = (u32)po;
    }
}

__device__ __forceinline__ u32 lower_bound_u32(const u32* a, u32 n, u32 x) {
    u32 lo = 0, len = n;
    while (len > 0) {
        const u32 h = len >> 1;
        if (a[lo + h] < x) { lo += h + 1; len -= h + 1; }
        else len = h;
    }
    return lo;
}

// ids holds the triples' columns (ser_ids_kernel); each becomes the index of its id among the nu sorted distinct terms
__global__ void __launch_bounds__(ST) ser_term_index_kernel(u32* __restrict__ ids, u64 n3, const u32* __restrict__ terms, u32 nu) {
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < n3; i += (u64)gridDim.x * blockDim.x) ids[i] = lower_bound_u32(terms, nu, ids[i]);
}

__global__ void __launch_bounds__(ST) ser_class_kernel(const u32* __restrict__ off, const u8* __restrict__ bytes, u32 nu, u8* __restrict__ cls) {
    for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < nu; t += gridDim.x * blockDim.x) {
        const u32 a = off[t], len = off[t + 1] - a;
        auto starts = [&](const char* w, u32 k) {
            if (len < k) return false;
            for (u32 b = 0; b < k; b++)
                if (bytes[a + b] != (u8)w[b]) return false;
            return true;
        };
        cls[t] = starts("<<", 2) ? TC_QUOTED : (starts("http://", 7) || starts("https://", 8)) ? TC_IRI : (u8)0;
    }
}

// Turtle's order key of triple i: (rank of its subject text, rank of its predicate text)
__global__ void __launch_bounds__(ST) ser_group_key_kernel(const u32* __restrict__ ts, const u32* __restrict__ tp, u32 n, const u32* __restrict__ rank_of,
                                                           u32 rb, unsigned long long* __restrict__ key, u32* __restrict__ idx) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        key[i] = (unsigned long long)rank_of[ts[i]] << rb | rank_of[tp[i]];
        idx[i] = i;
    }
}

// unit k = the triple idx[k] of the id order; its flags from its key and its neighbours'
__global__ void __launch_bounds__(ST) ser_group_place_kernel(const unsigned long long* __restrict__ key, const u32* __restrict__ idx, u32 n, u32 rb,
                                                             const u32* __restrict__ ts, const u32* __restrict__ tp, const u32* __restrict__ to,
                                                             u32* __restrict__ os, u32* __restrict__ op, u32* __restrict__ oo, u8* __restrict__ flags) {
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const u32 i = idx[k];
        os[k] = ts[i];
        op[k] = tp[i];
        oo[k] = to[i];
        const unsigned long long x = key[k];
        u8 f = 0;
        if (k == 0u || (key[k - 1] >> rb) != (x >> rb)) f |= SF_SUBJ;
        if (k == 0u || key[k - 1] != x) f |= SF_PRED;
        if (k + 1u == n || (key[k + 1] >> rb) != (x >> rb)) f |= SF_SUBJ_END;
        flags[k] = f;
    }
}

struct UnitParams {
    const u32 *ts, *tp, *to;
    const u8* flags;  // null: N-Triples
    const u32* toff;
    const u8* tcls;
    u32 n;
};

// The pieces of one unit in output order: emit(src, len) per literal separator or term text.
//   N-Triples (sparql_database.rs:302-322): S " " "<" P ">" " " O " .\n"
//   Turtle (sparql_database.rs:325-382): [S] [(" " | " ;\n    ") "<" P ">" | " ,"] " " O [" .\n"]
// S is the text when it starts with "<<", else "<" text ">"; O the text when it starts with "<<", "<" text ">" when it starts with
// "http://" / "https://", else '"' text '"'.
template <class Emit>
__device__ __forceinline__ void unit_pieces(bool turtle, u32 f, const u8* sb, u32 sl, u32 sc, const u8* pb, u32 pl, const u8* ob, u32 ol, u32 oc,
                                            Emit emit) {
    auto L = [](const char* s) { return reinterpret_cast<const u8*>(s); };
    const u8 *lt = L("<"), *gt = L(">"), *sp = L(" "), *dq = L("\""), *semi = L(" ;\n    "), *comma = L(" ,"), *dot = L(" .\n");
    if (!turtle || (f & SF_SUBJ)) {
        if (sc & TC_QUOTED) emit(sb, sl);
        else { emit(lt, 1); emit(sb, sl); emit(gt, 1); }
    }
    if (!turtle || (f & SF_PRED)) {
        if (!turtle || (f & SF_SUBJ)) emit(sp, 1);
        else emit(semi, 7);
        emit(lt, 1); emit(pb, pl); emit(gt, 1);
    } else {
        emit(comma, 2);
    }
    emit(sp, 1);
    if (oc & TC_QUOTED) emit(ob, ol);
    else {
        const u8* w = (oc & TC_IRI) ? lt : dq;
        emit(w, 1); emit(ob, ol); emit((oc & TC_IRI) ? gt : dq, 1);
    }
    if (!turtle || (f & SF_SUBJ_END)) emit(dot, 3);
}

__global__ void __launch_bounds__(ST) ser_unit_len_kernel(const __grid_constant__ UnitParams P, unsigned long long* __restrict__ len,
                                                          unsigned long long* max_len, u32* groups) {
    unsigned long long mx = 0;
    u32 g = 0;
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < P.n; k += gridDim.x * blockDim.x) {
        const u32 s = P.ts[k], p = P.tp[k], o = P.to[k];
        const u32 f = P.flags ? P.flags[k] : 0u;
        unsigned long long l = 0;
        unit_pieces(P.flags != nullptr, f, nullptr, P.toff[s + 1] - P.toff[s], P.tcls[s], nullptr, P.toff[p + 1] - P.toff[p], nullptr,
                    P.toff[o + 1] - P.toff[o], P.tcls[o], [&](const u8*, u32 k2) { l += k2; });
        len[k] = l;
        mx = l > mx ? l : mx;
        g += (f & SF_SUBJ) ? 1u : 0u;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long y = __shfl_xor_sync(0xffffffffu, mx, o);
        mx = y > mx ? y : mx;
        g += __shfl_xor_sync(0xffffffffu, g, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (mx) atomicMax(max_len, mx);
        if (g) atomicAdd(groups, g);
    }
}

// the largest u1 in [u0, n] whose units [u0, u1) take at most `limit` bytes: out[0] = u1, out[1] = their bytes
__global__ void ser_fit_kernel(const unsigned long long* __restrict__ uoff, u64 u0, u64 n, u64 limit, unsigned long long* out) {
    const unsigned long long base = uoff[u0];
    u64 lo = u0, hi = n;  // uoff[lo] - base <= limit holds
    while (lo < hi) {
        const u64 mid = hi - ((hi - lo) >> 1);
        if (uoff[mid] - base <= limit) lo = mid;
        else hi = mid - 1;
    }
    out[0] = lo;
    out[1] = uoff[lo] - base;
}

// units [u0, u0 + m) into out (out[0] = the first byte of unit u0): one warp per 32 units; lane r's unit is broadcast and its pieces are
// copied by the whole warp, consecutive lanes on consecutive bytes
__global__ void __launch_bounds__(ST) ser_write_kernel(const __grid_constant__ UnitParams P, const u8* __restrict__ tbytes,
                                                       const unsigned long long* __restrict__ uoff, u64 u0, u32 m, u8* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const u32 warps = (gridDim.x * blockDim.x) >> 5;
    const u32 n_chunks = (m + 31u) >> 5;
    const unsigned long long base = uoff[u0];
    const bool turtle = P.flags != nullptr;
    for (u32 chunk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; chunk < n_chunks; chunk += warps) {
        const u32 j = chunk * 32u + (u32)lane;
        u32 f = 0, sa = 0, sl = 0, sc = 0, pa = 0, pl = 0, oa = 0, ol = 0, oc = 0;
        unsigned long long dst = 0;
        const bool live = j < m;
        if (live) {
            const u64 k = u0 + j;
            const u32 s = P.ts[k], p = P.tp[k], o = P.to[k];
            f = turtle ? P.flags[k] : 0u;
            sa = P.toff[s]; sl = P.toff[s + 1] - sa; sc = P.tcls[s];
            pa = P.toff[p]; pl = P.toff[p + 1] - pa;
            oa = P.toff[o]; ol = P.toff[o + 1] - oa; oc = P.tcls[o];
            dst = uoff[k] - base;
        }
        const u32 rows = min(32u, m - chunk * 32u);
        for (u32 r = 0; r < rows; r++) {
            const u32 rf = __shfl_sync(0xffffffffu, f, r), rsa = __shfl_sync(0xffffffffu, sa, r), rsl = __shfl_sync(0xffffffffu, sl, r),
                      rsc = __shfl_sync(0xffffffffu, sc, r), rpa = __shfl_sync(0xffffffffu, pa, r), rpl = __shfl_sync(0xffffffffu, pl, r),
                      roa = __shfl_sync(0xffffffffu, oa, r), rol = __shfl_sync(0xffffffffu, ol, r), roc = __shfl_sync(0xffffffffu, oc, r);
            u8* w = out + __shfl_sync(0xffffffffu, dst, r);
            unit_pieces(turtle, rf, tbytes + rsa, rsl, rsc, tbytes + rpa, rpl, tbytes + roa, rol, roc, [&](const u8* src, u32 k2) {
                for (u32 b = (u32)lane; b < k2; b += 32u) w[b] = src[b];
                w += k2;
            });
        }
    }
}

struct PhaseTimer {  // device time between marks on the context's stream
    ScopedEvent e[5];
    int at = 0;
    void mark(cudaStream_t st) { cudaEventRecord(e[at++], st); }
};

kb_status serialize_begin(kb_ctx* ctx, u32 format, const u64* poff, const u8* pbytes, u32 n_prefixes, std::unique_ptr<kb_serializer>* out,
                          kb_serialize_info* info) {
    auto ser = std::make_unique<kb_serializer>();
    ser->ctx = ctx;
    ser->device = ctx->device;
    ser->format = format;
    ser->store_version = ctx->store_version;
    if (format == KB_SER_TURTLE) {
        for (u32 k = 0; k < n_prefixes; k++) {
            const std::string name(reinterpret_cast<const char*>(pbytes) + poff[2 * k], poff[2 * k + 1] - poff[2 * k]);
            const std::string uri(reinterpret_cast<const char*>(pbytes) + poff[2 * k + 1], poff[2 * k + 2] - poff[2 * k + 1]);
            ser->header += "@prefix " + name + ": <" + uri + "> .\n";
        }
        if (n_prefixes) ser->header += "\n";
    }
    ser->header_done = ser->header.empty();
    ser->max_unit = ser->header.size();
    info->total_bytes = ser->header.size();
    u64 n_raw = 0;
    const std::vector<ColSpan> spans = store_spans(ctx, &n_raw);
    if (n_raw == 0) {
        *out = std::move(ser);
        return KB_OK;
    }
    if (n_raw * 3 >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "a store of %llu triples (serialize: limit (2^32 - 16) / 3)", (unsigned long long)n_raw);
    if (!ctx->dict_ids) return fail(ctx, KB_E_UNSUPPORTED, "serializing the store needs the device dictionary's strings (kb_dict_strings_load)");
    auto U = [](const Buf& b) { return static_cast<u32*>(b->p); };
    auto U64 = [](const Buf& b) { return static_cast<unsigned long long*>(b->p); };
    PhaseTimer pt;
    pt.mark(ctx->st);

    // ---- sort + dedup
    Buf S2, PO2;
    u32 n = 0;
    KB_TRY(store_distinct(ctx, spans, &S2, &PO2, &n));
    ser->n = n;
    const u32 c = ctrl_alloc(ctx, 1);  // distinct terms
    pt.mark(ctx->st);

    // ---- render: the distinct ids of the three columns, each rendered once
    Buf ids, sorted_ids, terms;
    const u64 n3 = 3ull * n;
    KB_TRY(alloc_buf(ctx, n3 * 4, &ids));
    KB_TRY(alloc_buf(ctx, n3 * 4, &sorted_ids));
    KB_TRY(alloc_buf(ctx, n3 * 4, &terms));
    timer_begin(ctx, F_OTHER, 3);
    ser_ids_kernel<<<grid_1d(n, ctx->n_sms, ST), ST, 0, ctx->st>>>(U(S2), U64(PO2), n, U(ids));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortKeys(t, b, U(ids), U(sorted_ids), (u32)n3, 0, 32, ctx->st); }));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceSelect::Unique(t, b, U(sorted_ids), U(terms), ctx->ctrl + c, (u32)n3, ctx->st); }));
    timer_end(ctx);
    S2.reset(); PO2.reset(); sorted_ids.reset();
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32 nu = ctx->h_ctrl[c];
    info->n_terms = nu;
    KB_TRY(decode_ids(ctx, U(terms), nu, 0, Decode::Empty, "the store", &ser->toff, &ser->tbytes, nullptr));
    KB_TRY(alloc_buf(ctx, (size_t)nu + 16, &ser->tcls));
    u8* tbytes = static_cast<u8*>(ser->tbytes->p);
    u8* tcls = static_cast<u8*>(ser->tcls->p);
    timer_begin(ctx, F_OTHER, 2);
    ser_class_kernel<<<grid_1d(nu, ctx->n_sms, ST), ST, 0, ctx->st>>>(U(ser->toff), tbytes, nu, tcls);
    ser_term_index_kernel<<<grid_1d(n3, ctx->n_sms, ST), ST, 0, ctx->st>>>(U(ids), n3, U(terms), nu);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    terms.reset();
    const u32* ts = U(ids);
    const u32* tp = U(ids) + n;
    const u32* to = U(ids) + 2ull * n;
    pt.mark(ctx->st);

    // ---- ranks (Turtle): units in (subject text, predicate text) order, stable over the id order
    const bool turtle = format == KB_SER_TURTLE;
    if (turtle) {
        Buf rank_of, key, key2, idx, idx2, placed;
        KB_TRY(alloc_buf(ctx, (size_t)nu * 4, &rank_of));
        u32 n_ranks = 0, rounds = 0;
        KB_TRY(rank_values(ctx, nu, nullptr, U(ser->toff), tbytes, U(rank_of), &n_ranks, &rounds));
        info->rank_rounds = rounds;
        const u32 rb = std::max(1u, bits_of(n_ranks - 1));
        for (Buf* b : {&key, &key2}) KB_TRY(alloc_buf(ctx, (size_t)n * 8, b));
        for (Buf* b : {&idx, &idx2}) KB_TRY(alloc_buf(ctx, (size_t)n * 4, b));
        KB_TRY(alloc_buf(ctx, n3 * 4, &placed));
        KB_TRY(alloc_buf(ctx, (size_t)n + 16, &ser->flags));
        timer_begin(ctx, F_OTHER, 3);
        ser_group_key_kernel<<<grid_1d(n, ctx->n_sms, ST), ST, 0, ctx->st>>>(ts, tp, n, U(rank_of), rb, U64(key), U(idx));
        KB_TRY(cub_run(ctx, [&](void* t, size_t& b) {
            return cub::DeviceRadixSort::SortPairs(t, b, U64(key), U64(key2), U(idx), U(idx2), n, 0, (int)(2 * rb), ctx->st);
        }));
        ser_group_place_kernel<<<grid_1d(n, ctx->n_sms, ST), ST, 0, ctx->st>>>(U64(key2), U(idx2), n, rb, ts, tp, to, U(placed), U(placed) + n,
                                                                           U(placed) + 2ull * n, static_cast<u8*>(ser->flags->p));
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        ids = placed;
        ts = U(ids);
        tp = U(ids) + n;
        to = U(ids) + 2ull * n;
    }
    ser->ts = ids;  // (tp / to live in the same buffer)
    pt.mark(ctx->st);

    // ---- units: lengths, the largest, subject groups, offsets
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * 8, &ser->uoff));
    const u32 cu = ctrl_alloc(ctx, 4);  // [0..1] u64 largest unit, [2] subject groups
    UnitParams P{ts, tp, to, turtle ? static_cast<const u8*>(ser->flags->p) : nullptr, U(ser->toff), tcls, n};
    KB_CUDA(ctx, cudaMemsetAsync(U64(ser->uoff) + n, 0, 8, ctx->st));
    timer_begin(ctx, F_OTHER, 2);
    ser_unit_len_kernel<<<grid_1d(n, ctx->n_sms, ST), ST, 0, ctx->st>>>(P, U64(ser->uoff), reinterpret_cast<unsigned long long*>(ctx->ctrl + cu), ctx->ctrl + cu + 2);
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, U64(ser->uoff), U64(ser->uoff), n + 1, ctx->st); }));
    timer_end(ctx);
    pt.mark(ctx->st);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    unsigned long long max_unit = 0, body = 0;
    memcpy(&max_unit, ctx->h_ctrl + cu, sizeof max_unit);
    KB_CUDA(ctx, cudaMemcpy(&body, U64(ser->uoff) + n, 8, cudaMemcpyDeviceToHost));
    ctx->stats.d2h_bytes += 8;
    if (max_unit > KB_SER_STAGING_BYTES) return fail(ctx, KB_E_LIMIT, "a unit of %llu bytes (limit KB_SER_STAGING_BYTES)", max_unit);
    ser->max_unit = std::max<u64>(ser->max_unit, max_unit);
    info->n_subject_groups = turtle ? ctx->h_ctrl[cu + 2] : 0u;
    info->total_bytes += body;
    for (int k = 0; k < 4; k++) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, pt.e[k], pt.e[k + 1]);
        info->phase_ms[k] = ms;
    }
    timers_flush(ctx);
    *out = std::move(ser);
    return KB_OK;
}

kb_status serialize_next(kb_ctx* ctx, kb_serializer* ser, u8* dst, u64 capacity, u64* written) {
    *written = 0;
    if (ser->ctx != ctx) return fail(ctx, KB_E_INVALID, "the serializer belongs to another context");
    if (ser->store_version != ctx->store_version) return fail(ctx, KB_E_INVALID, "the store changed since kb_serialize_begin");
    if (capacity < ser->max_unit)
        return fail(ctx, KB_E_LIMIT, "capacity %llu is below the largest unit (%llu bytes)", (unsigned long long)capacity, (unsigned long long)ser->max_unit);
    u64 w = 0;
    if (!ser->header_done) {
        memcpy(dst, ser->header.data(), ser->header.size());
        w = ser->header.size();
        ser->header_done = true;
    }
    if (ser->cursor < ser->n) {
        Buf staging;
        KB_TRY(alloc_buf(ctx, (size_t)std::min<u64>(capacity, KB_SER_STAGING_BYTES) + 16, &staging));
        const UnitParams P{static_cast<const u32*>(ser->ts->p), static_cast<const u32*>(ser->ts->p) + ser->n, static_cast<const u32*>(ser->ts->p) + 2 * ser->n,
                           ser->flags ? static_cast<const u8*>(ser->flags->p) : nullptr, static_cast<const u32*>(ser->toff->p),
                           static_cast<const u8*>(ser->tcls->p), (u32)ser->n};
        const auto* uoff = static_cast<const unsigned long long*>(ser->uoff->p);
        while (ser->cursor < ser->n) {
            const u64 limit = std::min<u64>(capacity - w, KB_SER_STAGING_BYTES);
            const u32 c = ctrl_alloc(ctx, 4);
            auto* fit = reinterpret_cast<unsigned long long*>(ctx->ctrl + c);
            timer_begin(ctx, F_OTHER, 1);
            ser_fit_kernel<<<1, 1, 0, ctx->st>>>(uoff, ser->cursor, ser->n, limit, fit);
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
            KB_TRY(ctrl_read(ctx));
            unsigned long long h[2];
            memcpy(h, ctx->h_ctrl + c, sizeof h);
            const u64 u1 = h[0], bytes = h[1];
            if (u1 == ser->cursor) break;  // the next unit does not fit what is left of `capacity`
            const u32 m = (u32)(u1 - ser->cursor);
            timer_begin(ctx, F_OTHER, 1);
            ser_write_kernel<<<grid_1d((u64)m * 32, ctx->n_sms, ST), ST, 0, ctx->st>>>(P, static_cast<const u8*>(ser->tbytes->p), uoff, ser->cursor, m,
                                                                                  static_cast<u8*>(staging->p));
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
            KB_CUDA(ctx, cudaMemcpyAsync(dst + w, staging->p, bytes, cudaMemcpyDeviceToHost, ctx->st));
            KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
            ctx->stats.d2h_bytes += bytes;
            w += bytes;
            ser->cursor = u1;
        }
        timers_flush(ctx);
    }
    *written = w;
    return KB_OK;
}

}  // namespace

std::vector<ColSpan> store_spans(const kb_ctx* ctx, u64* n_raw) {
    std::vector<ColSpan> spans;
    *n_raw = 0;
    for (const Segment& sg : ctx->segs) {
        if (!sg.n) continue;
        spans.push_back({sg.s.ptr, sg.p.ptr, sg.o.ptr, sg.n, sg.ready});
        *n_raw += sg.n;
    }
    return spans;
}

kb_status store_distinct(kb_ctx* ctx, const std::vector<ColSpan>& spans, Buf* S_out, Buf* PO_out, u32* n_out) {
    u64 n_raw = 0;
    for (const ColSpan& sp : spans) n_raw += sp.n;
    auto U = [](const Buf& b) { return static_cast<u32*>(b->p); };
    auto U64 = [](const Buf& b) { return static_cast<unsigned long long*>(b->p); };
    // (s, p|o) sorted by p|o, then stably by s; equal neighbours dropped
    Buf S, S2, PO, PO2;
    KB_TRY(alloc_buf(ctx, n_raw * 4, &S));
    KB_TRY(alloc_buf(ctx, n_raw * 4, &S2));
    KB_TRY(alloc_buf(ctx, n_raw * 8, &PO));
    KB_TRY(alloc_buf(ctx, n_raw * 8, &PO2));
    {
        u64 at = 0;
        for (const ColSpan& sp : spans) {
            if (!sp.n) continue;
            if (sp.ready) KB_CUDA(ctx, cudaStreamWaitEvent(ctx->st, sp.ready, 0));
            timer_begin(ctx, F_OTHER, 1);
            ser_load_kernel<<<grid_1d(sp.n, ctx->n_sms, ST), ST, 0, ctx->st>>>(sp.s, sp.p, sp.o, sp.n, U(S) + at, U64(PO) + at);
            timer_end(ctx);
            at += sp.n;
        }
    }
    const u32 nr = (u32)n_raw;
    timer_begin(ctx, F_OTHER, 2);
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, U64(PO), U64(PO2), U(S), U(S2), nr, 0, 64, ctx->st); }));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, U(S2), U(S), U64(PO2), U64(PO), nr, 0, 32, ctx->st); }));
    timer_end(ctx);
    Buf keep;
    KB_TRY(alloc_buf(ctx, n_raw, &keep));
    const u32 c = ctrl_alloc(ctx, 1);  // distinct triples
    timer_begin(ctx, F_OTHER, 3);
    ser_distinct_flags_kernel<<<grid_1d(nr, ctx->n_sms, ST), ST, 0, ctx->st>>>(U(S), U64(PO), nr, static_cast<u8*>(keep->p));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) {
        return cub::DeviceSelect::Flagged(t, b, U(S), static_cast<const u8*>(keep->p), U(S2), ctx->ctrl + c, nr, ctx->st);
    }));
    KB_TRY(cub_run(ctx, [&](void* t, size_t& b) {
        return cub::DeviceSelect::Flagged(t, b, U64(PO), static_cast<const u8*>(keep->p), U64(PO2), ctx->ctrl + c, nr, ctx->st);
    }));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    *n_out = ctx->h_ctrl[c];
    *S_out = S2;
    *PO_out = PO2;
    return KB_OK;
}

}  // namespace kb

extern "C" {

kb_status kb_serialize_begin(kb_ctx* ctx, uint32_t format, const uint64_t* prefix_offsets, const uint8_t* prefix_bytes, uint32_t n_prefixes,
                             kb_serializer** out, kb_serialize_info* info) {
    KB_ENTER(ctx);
    kb_serialize_info local{};
    if (!info) info = &local;
    *info = kb_serialize_info{};
    if (!out) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    if (format != KB_SER_NTRIPLES && format != KB_SER_TURTLE) return kb::fail(ctx, KB_E_INVALID, "unknown serialization format %u", format);
    if (n_prefixes) {
        if (!prefix_offsets) return kb::fail(ctx, KB_E_INVALID, "NULL prefix offsets");
        if (prefix_offsets[0] != 0 || (prefix_offsets[2ull * n_prefixes] && !prefix_bytes))
            return kb::fail(ctx, KB_E_INVALID, "prefix offsets must start at 0 and prefix bytes must not be NULL");
        for (kb::u64 i = 0; i < 2ull * n_prefixes; i++)
            if (prefix_offsets[i + 1] < prefix_offsets[i]) return kb::fail(ctx, KB_E_INVALID, "prefix offsets decrease at string %llu", (unsigned long long)i);
    }
    std::unique_ptr<kb_serializer> s;
    KB_TRY(kb::serialize_begin(ctx, format, prefix_offsets, prefix_bytes, n_prefixes, &s, info));
    info->n_triples = s->n;
    info->max_unit_bytes = s->max_unit;
    *out = s.release();
    return KB_OK;
}

kb_status kb_serialize_next(kb_ctx* ctx, kb_serializer* ser, uint8_t* host_dst, uint64_t capacity, uint64_t* bytes_written) {
    KB_ENTER(ctx);
    if (!ser || !bytes_written || (!host_dst && capacity)) return kb::fail(ctx, KB_E_INVALID, "NULL argument");
    return kb::serialize_next(ctx, ser, host_dst, capacity, bytes_written);
}

void kb_serialize_free(kb_serializer* ser) {
    if (!ser) return;
    kb::DeviceGuard guard(ser->device);
    delete ser;
}

}  // extern "C"
