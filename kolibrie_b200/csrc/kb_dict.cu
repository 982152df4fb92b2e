// kb_dict.cu — Dictionary::encode for a BATCH of terms on the device (SURVEY.md §8(f) rank 1, second half: the load-time encode of
// sparql_database.rs:1000-1013, which calls shared/src/dictionary.rs:32-48 once per term).
//
// dictionary.rs:32-48 hands out ids sequentially in first-seen order: encode(t) returns the id t already has, else next_id++. A batch of
// n terms therefore gets exactly these ids when (1) terms the dictionary already holds keep their id, (2) every other DISTINCT string
// gets base + (rank of its first occurrence among the first occurrences of the batch). That is a hash join + a scan, not a sequential
// loop:
//   K1 dict_hash_kernel        64-bit FNV-1a of every term (thread per term; neighbouring threads read neighbouring bytes)
//   K2 dict_resolve_kernel     probe the persistent index (hash tag + id, strings compared on a tag match); misses go into the batch
//                              table, whose slot keeps the SMALLEST position of the string in the batch (CAS to claim, atomicMin after)
//   K3 dict_mark_kernel        first[i] = 1 iff term i is the first occurrence of a new string (+ its length for the byte scan)
//      two exclusive scans     rank of the first occurrences, byte offsets of the new strings
//   K4 dict_assign_kernel      ids of the new terms = base + rank[first position]; first_pos[rank] = i; offsets of the new strings
//   K5 dict_append_kernel      the new strings' bytes appended to the device dictionary (warp per string)
//   K6 dict_index_insert_kernel  the new ids enter the persistent index (rebuilt larger beyond load 1/2)
// Both tables are tag-indexed (kb_tagtab.cuh). This file owns the device dictionary: its loads, its growth, the decode of ids into text
// (decode_ids: kb_rel_decode, string ORDER BY keys, the serializers, the QueryBuilder term lists) and its downloads.
#include "kb_internal.hpp"
#include "kb_tagtab.cuh"

#include <cstring>

namespace kb {

__device__ __forceinline__ u64 fnv1a64(const unsigned char* __restrict__ p, u64 len) {
    u64 h = 0xcbf29ce484222325ull;
    for (u64 i = 0; i < len; i++) { h ^= (u64)__ldg(p + i); h *= 0x100000001b3ull; }
    h ^= h >> 32;  // fold: FNV's low bits are weak for power-of-two tables
    h *= 0xd6e8feb86659fd93ull;
    h ^= h >> 32;
    return h;
}
__device__ __forceinline__ bool bytes_equal(const unsigned char* __restrict__ a, const unsigned char* __restrict__ b, u64 len) {
    for (u64 i = 0; i < len; i++) if (__ldg(a + i) != __ldg(b + i)) return false;
    return true;
}
// the payload of an entry: the id (persistent index) or a position in the batch (batch table)

__global__ void __launch_bounds__(256) dict_hash_kernel(const u64* __restrict__ off, const unsigned char* __restrict__ bytes, u32 n, u64* __restrict__ hash) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const u64 a = off[i];
        hash[i] = fnv1a64(bytes + a, off[i + 1] - a);
    }
}

struct DictResolveParams {
    const u64* off; const unsigned char* bytes; u32 n;           // the batch
    const u64* hash;
    const u64* index; u64 index_mask;                             // persistent index (null: empty dictionary)
    DictTab dict;
    u64* batch; u64 batch_mask;                                   // batch table, all empty
    u32* out_id;                                                  // id, or EMPTY32 for a term that is new
    u32* slot_of;                                                 // slot of the term's string in the batch table (new terms)
    u32* overflow;
};
__global__ void __launch_bounds__(256) dict_resolve_kernel(const __grid_constant__ DictResolveParams P) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        const u64 a = P.off[i], len = P.off[i + 1] - a;
        const unsigned char* s = P.bytes + a;
        const u64 h = P.hash[i];
        u32 id = EMPTY32;
        if (P.index)
            id = tag_find(P.index, P.index_mask, h, [&](u32 cand) {
                const unsigned long long ca = P.dict.off[cand];
                return P.dict.off[cand + 1] - ca == len && bytes_equal(P.dict.bytes + ca, s, len);
            });
        P.out_id[i] = id;
        if (id != EMPTY32) continue;
        // `rep`: some position of the slot's string (it may be lowered concurrently: always the same string)
        if (!tag_claim_min(P.batch, P.batch_mask, h, i, [&](u32 rep) {
                const u64 ra = P.off[rep];
                return P.off[rep + 1] - ra == len && bytes_equal(P.bytes + ra, s, len);
            }, &P.slot_of[i]))
            *P.overflow = 1u;
    }
}

__global__ void __launch_bounds__(256) dict_mark_kernel(const u64* __restrict__ off, u32 n, const u32* __restrict__ out_id, const u32* __restrict__ slot_of,
                                                        const u64* __restrict__ batch, u32* __restrict__ first, u32* __restrict__ first_len,
                                                        unsigned long long* total_new_bytes) {
    unsigned long long bytes = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        u32 f = 0, l = 0;
        if (out_id[i] == EMPTY32 && (u32)batch[slot_of[i]] == i) { f = 1u; l = (u32)(off[i + 1] - off[i]); bytes += l; }
        first[i] = f;
        first_len[i] = l;
    }
    for (int o = 16; o > 0; o >>= 1) bytes += __shfl_down_sync(0xffffffffu, bytes, o);
    if ((threadIdx.x & 31) == 0 && bytes) atomicAdd(total_new_bytes, bytes);
}

// first / first_len hold their exclusive prefixes here (n + 1 entries: the last one is the total)
__global__ void __launch_bounds__(256) dict_assign_kernel(const u64* __restrict__ off, u32 n, u32 base_id, unsigned long long base_bytes, u32* __restrict__ out_id,
                                                          const u32* __restrict__ slot_of, const u64* __restrict__ batch, const u32* __restrict__ rank,
                                                          const u32* __restrict__ byte_rank, u64* __restrict__ first_pos, unsigned long long* __restrict__ new_off) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (out_id[i] != EMPTY32) continue;
        const u32 fp = (u32)batch[slot_of[i]];
        const u32 r = rank[fp];
        out_id[i] = base_id + r;
        if (fp == i) {
            first_pos[r] = i;
            new_off[r] = base_bytes + byte_rank[i];  // dict_off[base_id + r]; the closing offset is written by the host
        }
    }
}

// one warp per new string: dict_bytes[new_off[r] ..) = the bytes of term first_pos[r]
__global__ void __launch_bounds__(256) dict_append_kernel(const u64* __restrict__ off, const unsigned char* __restrict__ bytes, const u64* __restrict__ first_pos,
                                                          const unsigned long long* __restrict__ new_off, u32 n_new, unsigned char* __restrict__ dict_bytes) {
    const int lane = threadIdx.x & 31;
    const u32 warps = (gridDim.x * blockDim.x) >> 5;
    for (u32 r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_new; r += warps) {
        const u64 i = first_pos[r];
        const u64 a = off[i], len = off[i + 1] - a;
        unsigned char* dst = dict_bytes + new_off[r];
        for (u64 b = (u64)lane; b < len; b += 32) dst[b] = __ldg(bytes + a + b);
    }
}

// ids [first, first + n) of the device dictionary enter the persistent index
__global__ void __launch_bounds__(256) dict_index_insert_kernel(const DictTab dict, u32 first, u32 n, u64* __restrict__ index, u64 mask, u32* overflow) {
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const u32 id = first + k;
        const unsigned long long a = dict.off[id];
        u32 slot;  // ids are distinct strings: nothing to compare
        if (!tag_claim_min(index, mask, fnv1a64(dict.bytes + a, dict.off[id + 1] - a), id, [](u32) { return false; }, &slot)) *overflow = 1u;
    }
}

enum { QW_OK = 0, QW_UNKNOWN = 1, QW_DEEP = 2 };
// Dictionary::decode_term of a quoted id (dictionary.rs:60-72) as an explicit depth-first walk: lit(text, bytes) for "<< ", " ", " >>",
// word(id) for every dictionary component, in output order. Like the reference's `?`, the walk stops at the first id that neither table
// holds (QW_UNKNOWN: the whole term is "unknown"); entering a level past KB_QUOTED_MAX_DEPTH gives QW_DEEP. The stack holds one table
// index per level and a 2-bit component cursor per level.
template <class Lit, class Word>
__device__ u32 quoted_walk(u32 id, u32 dict_ids, const QuotedTab& qt, Lit lit, Word word) {
    u32 ent[KB_QUOTED_MAX_DEPTH];
    u32 next = 0;  // bits 2d..2d+1: components of level d already emitted
    int d = 0;
    u32 cur = id;
    for (;;) {
        const u32 x = cur & 0x7FFFFFFFu;
        if (x >= qt.n || __ldg(qt.p + x) == EMPTY32) return QW_UNKNOWN;
        if (d == KB_QUOTED_MAX_DEPTH) return QW_DEEP;
        ent[d] = x;
        next &= ~(3u << (2 * d));
        d++;
        lit("<< ", 3u);
        for (;;) {
            const int top = d - 1;
            const u32 k = (next >> (2 * top)) & 3u;
            if (k == 3u) {
                lit(" >>", 3u);
                if (--d == 0) return QW_OK;
                continue;
            }
            next += 1u << (2 * top);
            if (k) lit(" ", 1u);
            const u32 e = ent[top];
            const u32 c = __ldg((k == 0u ? qt.s : k == 1u ? qt.p : qt.o) + e);
            if (c & 0x80000000u) { cur = c; break; }
            if (c >= dict_ids) return QW_UNKNOWN;
            word(c);
        }
    }
}

// decode_lengths_kernel: len[i] = length of the string of ids[i] ("unknown" = 7 bytes when the dictionary does not hold the id). A quoted id: without a table
// *quoted = 1; with one, the length of `<< s p o >>` walked with a bounded stack (dictionary.rs:60-72), "unknown" when any id on the walk
// is held by neither table, and *deep = 1 when the walk goes past KB_QUOTED_MAX_DEPTH levels first. *total += sum.
// missing_len: 7, or 0 when a term the tables do not hold renders as "" instead of "unknown" (decode_any(..).unwrap_or_default(), the serializers'
// rule, sparql_database.rs:301-322).
// plain: Dictionary::decode's rule, a quoted id is "none" (missing_len bytes) without a walk
__global__ void __launch_bounds__(256) decode_lengths_kernel(const u32* __restrict__ ids, u32 n, const DictTab dict, const QuotedTab qt, u32* __restrict__ len, unsigned long long* total, u32* quoted, u32* deep,
                                                             u32 missing_len, u32 plain) {
    const u32 stride = gridDim.x * blockDim.x;
    unsigned long long t = 0;
    bool q = false, dp = false;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const u32 id = ids[i];
        unsigned long long l = missing_len;  // "unknown" or ""
        if ((id & 0x80000000u) && !plain) {
            if (qt.n == 0u) {
                q = true;
            } else {
                unsigned long long acc = 0;
                const u32 r = quoted_walk(id, dict.ids, qt, [&](const char*, u32 k) { acc += k; },
                                          [&](u32 c) { acc += __ldg(dict.off + c + 1) - __ldg(dict.off + c); });
                dp = dp || r == QW_DEEP;
                if (r == QW_OK) l = acc;
            }
        } else if (id < dict.ids) {
            l = __ldg(dict.off + id + 1) - __ldg(dict.off + id);
        }
        len[i] = l > 0xFFFFFFFFull ? 0xFFFFFFFFu : (u32)l;  // (the total then exceeds 2^32-1: the caller refuses the column)
        t += l;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(total, t);
    if (q) *quoted = 1u;
    if (dp) *deep = 1u;
}
// out[off[i] .. off[i+1]) = bytes of the string of ids[i]; one warp per 32 rows, the lanes copy each dictionary string together; a quoted
// row is written by its own thread, walking the term again (a missing term is 7 bytes, "unknown", or 0: either way shorter than the
// 8 bytes of the shortest rendered quoted term)
__global__ void __launch_bounds__(256) decode_gather_kernel(const u32* __restrict__ ids, u32 n, const DictTab dict, const QuotedTab qt,
                                                            const u32* __restrict__ off, unsigned char* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const u32 warps = (gridDim.x * blockDim.x) >> 5;
    const u32 n_chunks = (n + 31u) >> 5;
    for (u32 chunk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; chunk < n_chunks; chunk += warps) {
        const u32 i = chunk * 32u + (u32)lane;
        u32 id = 0, dst = 0, l = 0;
        unsigned long long src = 0;
        bool known = false, walk = false;
        if (i < n) {
            id = ids[i];
            dst = off[i];
            l = off[i + 1] - dst;
            known = id < dict.ids;
            if (known) src = __ldg(dict.off + id);
            walk = (id & 0x80000000u) != 0u && l >= 8u;  // a rendered quoted term is at least 8 bytes: 7 is "unknown", 0 is ""
        }
        const u32 wl = walk ? 0u : l;
        for (int r = 0; r < 32; r++) {  // the warp copies row r of its chunk: consecutive lanes, consecutive bytes
            const u32 rl = __shfl_sync(0xffffffffu, wl, r);
            if (rl == 0u) continue;
            const u32 rdst = __shfl_sync(0xffffffffu, dst, r);
            const unsigned long long rsrc = __shfl_sync(0xffffffffu, src, r);
            const bool rknown = __shfl_sync(0xffffffffu, known ? 1 : 0, r) != 0;
            for (u32 b = (u32)lane; b < rl; b += 32u) out[rdst + b] = rknown ? __ldg(dict.bytes + rsrc + b) : (unsigned char)"unknown"[b];
        }
        if (walk) {  // a quoted term: this thread writes it, walking it again
            unsigned char* w = out + dst;
            quoted_walk(id, dict.ids, qt, [&](const char* s, u32 k) { for (u32 b = 0; b < k; b++) *w++ = (unsigned char)s[b]; },
                        [&](u32 c) {
                            const unsigned long long a = __ldg(dict.off + c), e = __ldg(dict.off + c + 1);
                            for (unsigned long long b = a; b < e; b++) *w++ = __ldg(dict.bytes + b);
                        });
        }
    }
}


}  // namespace kb

using namespace kb;

DictTab kb::dicttab(const kb_ctx* ctx) {
    DictTab t{};
    if (ctx->dict_ids) {
        t.off = static_cast<const unsigned long long*>(ctx->dict_off->p);
        t.bytes = static_cast<const unsigned char*>(ctx->dict_bytes->p);
        t.ids = ctx->dict_ids;
    }
    return t;
}

namespace {

// the persistent index holds every id and stays below load 1/2 with `extra` more
kb_status dict_index_ensure(kb_ctx* ctx, u64 extra) {
    const DictTab dict = dicttab(ctx);
    return tag_index_ensure(ctx, &ctx->dict_index, ctx->dict_ids, extra, "dictionary index", [&](u32 first, u32 n, u64* tab, u64 mask, u32* overflow) {
        dict_index_insert_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(dict, first, n, tab, mask, overflow);
    });
}

}  // namespace

// The body of kb_dict_encode over a batch already in device memory (kb_bind's CONCAT builds its concatenations there): term i =
// d_bytes[d_off[i] .. d_off[i+1]), d_off[n] = total. The ids go to d_out_ids (device, n entries); *first_pos (nullable) receives a device
// buffer whose entry k is the batch position of the term that introduced id (ids before the call) + k. Limits are checked before
// anything changes.
kb_status kb::dict_encode_device(kb_ctx* ctx, const u64* d_off, const unsigned char* d_bytes, u64 n_terms, u64 total, u32* d_out_ids, u32* n_new_out,
                             Buf* first_pos) {
    *n_new_out = 0;
    if (n_terms == 0) return KB_OK;
    if (n_terms >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "at most 2^32-16 terms per call");
    if (total > 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "at most 2^32-16 bytes of terms per call (split the batch)");
    if ((u64)ctx->dict_ids + n_terms >= 0x80000000ull) return fail(ctx, KB_E_LIMIT, "ids would reach bit 31 (reserved for quoted triples, quoted_triple_store.rs:28-55)");
    const u32 n = (u32)n_terms;
    Buf d_hash, d_batch, d_slot, d_first, d_flen, d_fpos, scratch;
    KB_TRY(dict_index_ensure(ctx, n));
    u64 bslots = 0;
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u64), &d_hash));
    KB_TRY(tag_batch_table(ctx, n, &d_batch, &bslots));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &d_slot));
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &d_first));
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &d_flen));
    KB_TRY(alloc_buf(ctx, (((size_t)n + 1) / 2048 + 4) * sizeof(u32), &scratch));
    const u32 c = ctrl_alloc(ctx, 4);  // [0] overflow, [2..3] u64 bytes of the new strings
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 4 * sizeof(u32), ctx->st));
    const int grid = grid_1d(n, ctx->n_sms);
    timer_begin(ctx, F_OTHER, 9);
    dict_hash_kernel<<<grid, 256, 0, ctx->st>>>(d_off, d_bytes, n, static_cast<u64*>(d_hash->p));
    DictResolveParams P{};
    P.off = d_off; P.bytes = d_bytes; P.n = n;
    P.hash = static_cast<const u64*>(d_hash->p);
    P.index = ctx->dict_ids ? static_cast<const u64*>(ctx->dict_index.tab->p) : nullptr;
    P.index_mask = ctx->dict_index.slots - 1;
    P.dict = dicttab(ctx);
    P.batch = static_cast<u64*>(d_batch->p); P.batch_mask = bslots - 1;
    P.out_id = d_out_ids; P.slot_of = static_cast<u32*>(d_slot->p);
    P.overflow = ctx->ctrl + c;
    dict_resolve_kernel<<<grid, 256, 0, ctx->st>>>(P);
    dict_mark_kernel<<<grid, 256, 0, ctx->st>>>(P.off, n, P.out_id, P.slot_of, P.batch, static_cast<u32*>(d_first->p), static_cast<u32*>(d_flen->p),
                                                reinterpret_cast<unsigned long long*>(ctx->ctrl + c + 2));
    KB_CUDA(ctx, cudaMemsetAsync(static_cast<u32*>(d_first->p) + n, 0, sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(static_cast<u32*>(d_flen->p) + n, 0, sizeof(u32), ctx->st));
    launch_exclusive_scan_u32(static_cast<u32*>(d_first->p), n + 1, static_cast<u32*>(scratch->p), ctx->st);
    launch_exclusive_scan_u32(static_cast<u32*>(d_flen->p), n + 1, static_cast<u32*>(scratch->p), ctx->st);
    timer_end(ctx);
    // the number of new strings (= first[n] after the scan) and their bytes
    const u32 c2 = ctrl_alloc(ctx, 4);
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->ctrl + c2, static_cast<u32*>(d_first->p) + n, sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    if (ctx->h_ctrl[c]) return fail(ctx, KB_E_LIMIT, "dictionary batch table overflow");
    const u32 n_new = ctx->h_ctrl[c2];
    unsigned long long new_bytes = 0;
    memcpy(&new_bytes, ctx->h_ctrl + c + 2, sizeof new_bytes);
    // grow the device dictionary: offsets [dict_ids + n_new + 1], bytes
    const u32 base_id = ctx->dict_ids;
    unsigned long long base_bytes = 0;
    if (ctx->dict_ids) {
        KB_CUDA(ctx, cudaMemcpyAsync(&base_bytes, static_cast<const unsigned long long*>(ctx->dict_off->p) + ctx->dict_ids, sizeof base_bytes, cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    }
    KB_TRY(alloc_buf(ctx, ((size_t)std::max(n_new, 1u)) * sizeof(u64), &d_fpos));
    Buf noff, nbytes;
    const size_t ids_after = (size_t)base_id + n_new;
    if (n_new) {
        // capacity with headroom (a bulk load encodes many batches): reallocate only when it runs out
        const size_t off_need = (ids_after + 1) * sizeof(u64), bytes_need = (size_t)base_bytes + new_bytes + 16;
        if (!ctx->dict_off || ctx->dict_off->bytes < off_need + 256) {
            KB_TRY(alloc_buf(ctx, off_need + off_need / 2, &noff));
            if (base_id) KB_CUDA(ctx, cudaMemcpyAsync(noff->p, ctx->dict_off->p, ((size_t)base_id + 1) * sizeof(u64), cudaMemcpyDeviceToDevice, ctx->st));
            else KB_CUDA(ctx, cudaMemsetAsync(noff->p, 0, sizeof(u64), ctx->st));
            ctx->dict_off = noff;
        }
        if (!ctx->dict_bytes || ctx->dict_bytes->bytes < bytes_need + 256) {
            KB_TRY(alloc_buf(ctx, bytes_need + bytes_need / 2, &nbytes));
            if (base_bytes) KB_CUDA(ctx, cudaMemcpyAsync(nbytes->p, ctx->dict_bytes->p, (size_t)base_bytes, cudaMemcpyDeviceToDevice, ctx->st));
            ctx->dict_bytes = nbytes;
        }
    }
    timer_begin(ctx, F_OTHER, n_new ? 2 : 1);
    dict_assign_kernel<<<grid, 256, 0, ctx->st>>>(P.off, n, base_id, base_bytes, P.out_id, P.slot_of, P.batch, static_cast<const u32*>(d_first->p),
                                                  static_cast<const u32*>(d_flen->p), static_cast<u64*>(d_fpos->p),
                                                  n_new ? static_cast<unsigned long long*>(ctx->dict_off->p) + base_id : nullptr);
    if (n_new) {
        const unsigned long long end = base_bytes + new_bytes;
        KB_CUDA(ctx, cudaMemcpyAsync(static_cast<unsigned long long*>(ctx->dict_off->p) + ids_after, &end, sizeof end, cudaMemcpyHostToDevice, ctx->st));
        dict_append_kernel<<<grid_1d((u64)n_new * 32, ctx->n_sms), 256, 0, ctx->st>>>(P.off, P.bytes, static_cast<const u64*>(d_fpos->p),
                                                                                     static_cast<const unsigned long long*>(ctx->dict_off->p) + base_id, n_new,
                                                                                     static_cast<unsigned char*>(ctx->dict_bytes->p));
    }
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));  // `end` (a stack variable) has been consumed
    ctx->dict_ids = (u32)ids_after;
    if (n_new) KB_TRY(dict_index_ensure(ctx, 0));  // the new ids enter the index
    *n_new_out = n_new;
    if (first_pos) *first_pos = d_fpos;
    return KB_OK;
}


kb_status kb::decode_ids(kb_ctx* ctx, const u32* ids, u32 n, u32 n_empty, Decode mode, const char* what, Buf* off_out, Buf* bytes_out,
                         u64* total_out, const DictTab* from) {
    const size_t m = (size_t)n + n_empty;
    Buf off, scratch, bytes;
    KB_TRY(alloc_buf(ctx, (m + 1) * sizeof(u32), &off));
    KB_TRY(alloc_buf(ctx, ((m + 1) / 2048 + 4) * sizeof(u32), &scratch));
    u32* d_off = static_cast<u32*>(off->p);
    KB_CUDA(ctx, cudaMemsetAsync(d_off + n, 0, ((size_t)n_empty + 1) * sizeof(u32), ctx->st));  // the scan runs over m + 1 entries: off[m] = total
    const u32 c = ctrl_alloc(ctx, 4);  // [0..1] u64 total bytes, [2] quoted-triple id seen without a table, [3] walk too deep
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 4 * sizeof(u32), ctx->st));
    const DictTab dict = from ? *from : dicttab(ctx);
    const QuotedTab qt = quotedtab(ctx);
    const int grid = grid_1d(n, ctx->n_sms);
    timer_begin(ctx, F_OTHER, 4);
    if (n)
        decode_lengths_kernel<<<grid, 256, 0, ctx->st>>>(ids, n, dict, mode == Decode::Plain ? QuotedTab{} : qt, d_off,
                                                         reinterpret_cast<unsigned long long*>(ctx->ctrl + c), ctx->ctrl + c + 2, ctx->ctrl + c + 3,
                                                         mode == Decode::Unknown ? 7u : 0u, mode == Decode::Plain ? 1u : 0u);
    launch_exclusive_scan_u32(d_off, (u32)m + 1, static_cast<u32*>(scratch->p), ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    unsigned long long total = 0;
    memcpy(&total, ctx->h_ctrl + c, sizeof total);
    if (ctx->h_ctrl[c + 2]) return fail(ctx, KB_E_UNSUPPORTED, "%s holds quoted-triple ids (bit 31) and no quoted-triple table is loaded (kb_quoted_load)", what);
    if (ctx->h_ctrl[c + 3]) return fail(ctx, KB_E_LIMIT, "a quoted-triple term nests deeper than %d levels", KB_QUOTED_MAX_DEPTH);
    if (total > 0xFFFFFFFFull) return fail(ctx, KB_E_LIMIT, "the text of %s would take %llu bytes (limit 2^32-1 per call)", what, total);
    KB_TRY(alloc_buf(ctx, (size_t)total + 16, &bytes));
    timer_begin(ctx, F_OTHER);
    if (n) decode_gather_kernel<<<grid, 256, 0, ctx->st>>>(ids, n, dict, mode == Decode::Plain ? QuotedTab{} : qt, d_off, static_cast<unsigned char*>(bytes->p));
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    *off_out = off;
    *bytes_out = bytes;
    if (total_out) *total_out = total;
    return KB_OK;
}

kb_status kb::dict_copy(kb_ctx* dst, const kb_ctx* src, DictState* prev) {
    DictState next;
    next.ids = src->dict_ids;
    if (src->dict_ids) {
        unsigned long long total = 0;
        KB_CUDA(dst, cudaMemcpyAsync(&total, static_cast<const unsigned long long*>(src->dict_off->p) + src->dict_ids, sizeof total, cudaMemcpyDeviceToHost, dst->st));
        KB_CUDA(dst, cudaStreamSynchronize(dst->st));
        KB_TRY(alloc_buf(dst, ((size_t)src->dict_ids + 1) * sizeof(u64), &next.off));
        KB_TRY(alloc_buf(dst, (size_t)total + 16, &next.bytes));
        KB_CUDA(dst, cudaMemcpyAsync(next.off->p, src->dict_off->p, ((size_t)src->dict_ids + 1) * sizeof(u64), cudaMemcpyDeviceToDevice, dst->st));
        if (total) KB_CUDA(dst, cudaMemcpyAsync(next.bytes->p, src->dict_bytes->p, (size_t)total, cudaMemcpyDeviceToDevice, dst->st));
    }
    prev->off = dst->dict_off;
    prev->bytes = dst->dict_bytes;
    prev->ids = dst->dict_ids;
    prev->index = dst->dict_index;
    dict_restore(dst, std::move(next));
    return KB_OK;
}

void kb::dict_restore(kb_ctx* dst, DictState&& prev) {
    dst->dict_off = std::move(prev.off);
    dst->dict_bytes = std::move(prev.bytes);
    dst->dict_ids = prev.ids;
    dst->dict_index = std::move(prev.index);
}

extern "C" {

kb_status kb_dict_encode(kb_ctx* ctx, const uint64_t* offsets, const uint8_t* bytes, uint64_t n_terms, uint32_t* out_ids, uint32_t* n_new_out,
                         uint64_t* new_first_pos) {
    KB_ENTER(ctx);
    if (n_new_out) *n_new_out = 0;
    if (n_terms == 0) return KB_OK;
    if (!offsets || !out_ids) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (n_terms >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "at most 2^32-16 terms per call");
    const u64 total = offsets[n_terms];
    if (offsets[0] != 0 || (total && !bytes)) return fail(ctx, KB_E_INVALID, "offsets must start at 0 and bytes must not be NULL");
    if (total > 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "at most 2^32-16 bytes of terms per call (split the batch)");
    if ((u64)ctx->dict_ids + n_terms >= 0x80000000ull) return fail(ctx, KB_E_LIMIT, "ids would reach bit 31 (reserved for quoted triples, quoted_triple_store.rs:28-55)");
    const u32 n = (u32)n_terms;
    // the batch on the device
    Buf d_off, d_bytes, d_ids, d_fpos;
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u64), &d_off));
    KB_TRY(alloc_buf(ctx, (size_t)total + 16, &d_bytes));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &d_ids));
    KB_CUDA(ctx, cudaMemcpyAsync(d_off->p, offsets, ((size_t)n + 1) * sizeof(u64), cudaMemcpyHostToDevice, ctx->st));
    if (total) KB_CUDA(ctx, cudaMemcpyAsync(d_bytes->p, bytes, (size_t)total, cudaMemcpyHostToDevice, ctx->st));
    ctx->stats.h2d_bytes += ((size_t)n + 1) * sizeof(u64) + total;
    u32 n_new = 0;
    KB_TRY(dict_encode_device(ctx, static_cast<const u64*>(d_off->p), static_cast<const unsigned char*>(d_bytes->p), n, total, static_cast<u32*>(d_ids->p),
                              &n_new, &d_fpos));
    KB_CUDA(ctx, cudaMemcpyAsync(out_ids, d_ids->p, (size_t)n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    if (new_first_pos && n_new) KB_CUDA(ctx, cudaMemcpyAsync(new_first_pos, d_fpos->p, (size_t)n_new * sizeof(u64), cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += (size_t)n * sizeof(u32) + (new_first_pos ? (size_t)n_new * sizeof(u64) : 0);
    if (n_new_out) *n_new_out = n_new;
    return KB_OK;
}

kb_status kb_dict_strings_info(kb_ctx* ctx, uint32_t* n_ids, uint64_t* n_bytes) {
    KB_ENTER(ctx);
    if (n_ids) *n_ids = ctx->dict_ids;
    if (n_bytes) {
        unsigned long long b = 0;
        if (ctx->dict_ids) {
            KB_CUDA(ctx, cudaMemcpyAsync(&b, static_cast<const unsigned long long*>(ctx->dict_off->p) + ctx->dict_ids, sizeof b, cudaMemcpyDeviceToHost, ctx->st));
            KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        }
        *n_bytes = b;
    }
    return KB_OK;
}

kb_status kb_dict_strings_load(kb_ctx* ctx, const uint64_t* offsets, const uint8_t* bytes, uint32_t n_ids) {
    KB_ENTER(ctx);
    ctx->dict_off.reset();
    ctx->dict_bytes.reset();
    ctx->dict_ids = 0;
    ctx->dict_index = TagIndex{};  // (kb_dict_encode rebuilds its string -> id index lazily)
    if (n_ids == 0) return KB_OK;
    if (!offsets) return fail(ctx, KB_E_INVALID, "NULL offsets");
    const uint64_t total = offsets[n_ids];
    if (offsets[0] != 0 || (total && !bytes)) return fail(ctx, KB_E_INVALID, "offsets must start at 0 and bytes must not be NULL");
    for (uint32_t i = 0; i < n_ids; i++) if (offsets[i + 1] < offsets[i]) return fail(ctx, KB_E_INVALID, "offsets decrease at id %u", i);
    KB_TRY(alloc_buf(ctx, ((size_t)n_ids + 1) * sizeof(uint64_t), &ctx->dict_off));
    KB_TRY(alloc_buf(ctx, (size_t)total + 16, &ctx->dict_bytes));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->dict_off->p, offsets, ((size_t)n_ids + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->st));
    if (total) KB_CUDA(ctx, cudaMemcpyAsync(ctx->dict_bytes->p, bytes, (size_t)total, cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.h2d_bytes += ((size_t)n_ids + 1) * sizeof(uint64_t) + total;
    ctx->dict_ids = n_ids;
    return KB_OK;
}

kb_status kb_rel_decode(kb_ctx* ctx, const kb_rel* r, uint32_t col, kb_strings** out) {
    KB_ENTER(ctx);
    if (!r || !out) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (col >= r->cols.size()) return fail(ctx, KB_E_INVALID, "column %u out of range", col);
    if (r->n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "relation too large");
    auto res = std::make_unique<kb_strings>();
    res->n = r->n;
    KB_TRY(decode_ids(ctx, r->cols[col].ptr, (u32)r->n, 0, Decode::Unknown, "the column", &res->off, &res->bytes, &res->total));
    *out = res.release();
    return KB_OK;
}
kb_status kb_strings_info(const kb_strings* s, uint64_t* n_strings, uint64_t* total_bytes) {
    if (!s) return KB_E_INVALID;
    if (n_strings) *n_strings = s->n;
    if (total_bytes) *total_bytes = s->total;
    return KB_OK;
}
kb_status kb_strings_download(kb_ctx* ctx, const kb_strings* s, uint64_t* offsets, uint8_t* bytes) {
    if (!ctx || !s) return KB_E_INVALID;
    DeviceGuard guard(ctx->device);
    if (offsets) {
        std::vector<u32> h((size_t)s->n + 1);
        KB_CUDA(ctx, cudaMemcpyAsync(h.data(), s->off->p, h.size() * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        for (size_t i = 0; i < h.size(); i++) offsets[i] = h[i];
    }
    if (bytes && s->total) {
        KB_CUDA(ctx, cudaMemcpyAsync(bytes, s->bytes->p, (size_t)s->total, cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    }
    ctx->stats.d2h_bytes += ((size_t)s->n + 1) * sizeof(u32) + s->total;
    return KB_OK;
}
void kb_strings_free(kb_ctx* ctx, kb_strings* s) {
    if (!s) return;
    if (ctx) { DeviceGuard guard(ctx->device); delete s; }
    else delete s;
}

kb_status kb_dict_strings_download(kb_ctx* ctx, uint32_t first, uint32_t n, uint64_t* offsets, uint8_t* bytes) {
    KB_ENTER(ctx);
    if (!offsets) return fail(ctx, KB_E_INVALID, "NULL offsets");
    if ((u64)first + n > ctx->dict_ids) return fail(ctx, KB_E_INVALID, "ids [%u, %llu) past the %u the device dictionary holds", first, (unsigned long long)first + n, ctx->dict_ids);
    offsets[0] = 0;
    if (n == 0) return KB_OK;
    KB_CUDA(ctx, cudaMemcpyAsync(offsets, static_cast<const unsigned long long*>(ctx->dict_off->p) + first, ((size_t)n + 1) * sizeof(u64), cudaMemcpyDeviceToHost, ctx->st));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    const u64 base = offsets[0];
    for (u32 k = 0; k <= n; k++) offsets[k] -= base;
    if (bytes && offsets[n]) {
        KB_CUDA(ctx, cudaMemcpyAsync(bytes, static_cast<const unsigned char*>(ctx->dict_bytes->p) + base, (size_t)offsets[n], cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    }
    ctx->stats.d2h_bytes += ((size_t)n + 1) * sizeof(u64) + (bytes ? offsets[n] : 0);
    return KB_OK;
}

}  // extern "C"
