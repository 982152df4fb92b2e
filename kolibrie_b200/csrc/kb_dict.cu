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
#include "kb_internal.hpp"
#include "kb_kernels.cuh"

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
constexpr u64 DEMPTY = 0xFFFFFFFFFFFFFFFFull;
// an entry = (hash tag in the high 32 bits, payload in the low 32): payload = id (persistent index) or position in the batch (batch table)
__device__ __forceinline__ u64 dentry(u64 h, u32 payload) { return (h & 0xFFFFFFFF00000000ull) | payload; }

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
    const unsigned long long* dict_off; const unsigned char* dict_bytes; u32 dict_ids;
    u64* batch; u64 batch_mask;                                   // batch table, all DEMPTY
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
        if (P.index) {
            for (u64 slot = h & P.index_mask, probes = 0; probes <= P.index_mask; probes++, slot = (slot + 1) & P.index_mask) {
                const u64 e = P.index[slot];
                if (e == DEMPTY) break;
                if ((e >> 32) != (h >> 32)) continue;
                const u32 cand = (u32)e;
                const unsigned long long ca = P.dict_off[cand];
                if (P.dict_off[cand + 1] - ca == len && bytes_equal(P.dict_bytes + ca, s, len)) { id = cand; break; }
            }
        }
        P.out_id[i] = id;
        if (id != EMPTY32) continue;
        bool placed = false;
        for (u64 slot = h & P.batch_mask, probes = 0; probes <= P.batch_mask; probes++, slot = (slot + 1) & P.batch_mask) {
            u64 e = *reinterpret_cast<volatile u64*>(&P.batch[slot]);
            if (e == DEMPTY) {
                e = atomicCAS(reinterpret_cast<unsigned long long*>(&P.batch[slot]), DEMPTY, dentry(h, i));
                if (e == DEMPTY) { P.slot_of[i] = (u32)slot; placed = true; break; }
            }
            if ((e >> 32) != (h >> 32)) continue;
            const u32 rep = (u32)e;  // some position of the slot's string (it may be lowered concurrently: always the same string)
            const u64 ra = P.off[rep];
            if (P.off[rep + 1] - ra == len && bytes_equal(P.bytes + ra, s, len)) {
                atomicMin(reinterpret_cast<unsigned long long*>(&P.batch[slot]), dentry(h, i));  // same tag: the minimum is over the position
                P.slot_of[i] = (u32)slot;
                placed = true;
                break;
            }
        }
        if (!placed) *P.overflow = 1u;
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
__global__ void __launch_bounds__(256) dict_index_insert_kernel(const unsigned long long* __restrict__ dict_off, const unsigned char* __restrict__ dict_bytes, u32 first, u32 n,
                                                                u64* __restrict__ index, u64 mask, u32* overflow) {
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
        const u32 id = first + k;
        const unsigned long long a = dict_off[id];
        const u64 h = fnv1a64(dict_bytes + a, dict_off[id + 1] - a);
        bool placed = false;
        for (u64 slot = h & mask, probes = 0; probes <= mask; probes++, slot = (slot + 1) & mask) {
            if (*reinterpret_cast<volatile u64*>(&index[slot]) != DEMPTY) continue;  // ids are distinct strings: nothing to compare
            if (atomicCAS(reinterpret_cast<unsigned long long*>(&index[slot]), DEMPTY, dentry(h, id)) == DEMPTY) { placed = true; break; }
        }
        if (!placed) *overflow = 1u;
    }
}

static int grid_1d(u64 n, int n_sms, int per_sm = 8) {
    const u64 want = (n + 255) / 256;
    const u64 cap = (u64)n_sms * per_sm;
    return (int)std::max<u64>(1, std::min(want, cap));
}

// (re)build the persistent index so that it holds every id and stays below load 1/2 with `extra` more
static kb_status dict_index_ensure(kb_ctx* ctx, u64 extra) {
    const u64 need = ((u64)ctx->dict_ids + extra) * 2 + 64;
    if (ctx->dict_index && ctx->dict_index_slots >= need && ctx->dict_indexed == ctx->dict_ids) return KB_OK;
    if (!ctx->dict_index || ctx->dict_index_slots < need) {
        u64 slots = 1024;
        while (slots < need + need / 2) slots <<= 1;  // headroom: the next batches extend it in place
        ctx->dict_index.reset();
        KB_TRY(alloc_buf(ctx, slots * sizeof(u64), &ctx->dict_index));
        KB_CUDA(ctx, cudaMemsetAsync(ctx->dict_index->p, 0xFF, slots * sizeof(u64), ctx->st));
        ctx->dict_index_slots = slots;
        ctx->dict_indexed = 0;
    }
    if (ctx->dict_indexed < ctx->dict_ids) {
        const u32 c = ctrl_alloc(ctx, 4);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 4 * sizeof(u32), ctx->st));
        const u32 n = ctx->dict_ids - ctx->dict_indexed;
        dict_index_insert_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(static_cast<const unsigned long long*>(ctx->dict_off->p),
                                                                                static_cast<const unsigned char*>(ctx->dict_bytes->p), ctx->dict_indexed, n,
                                                                                static_cast<u64*>(ctx->dict_index->p), ctx->dict_index_slots - 1, ctx->ctrl + c);
        ctx->stats.kernel_launches++;
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        if (ctx->h_ctrl[c]) return fail(ctx, KB_E_LIMIT, "dictionary index overflow");
        ctx->dict_indexed = ctx->dict_ids;
    }
    return KB_OK;
}

// The body of kb_dict_encode over a batch already in device memory (kb_bind's CONCAT builds its concatenations there): term i =
// d_bytes[d_off[i] .. d_off[i+1]), d_off[n] = total. The ids go to d_out_ids (device, n entries); *first_pos (nullable) receives a device
// buffer whose entry k is the batch position of the term that introduced id (ids before the call) + k. Limits are checked before
// anything changes.
kb_status dict_encode_device(kb_ctx* ctx, const u64* d_off, const unsigned char* d_bytes, u64 n_terms, u64 total, u32* d_out_ids, u32* n_new_out,
                             Buf* first_pos) {
    *n_new_out = 0;
    if (n_terms == 0) return KB_OK;
    if (n_terms >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "at most 2^32-16 terms per call");
    if (total > 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "at most 2^32-16 bytes of terms per call (split the batch)");
    if ((u64)ctx->dict_ids + n_terms >= 0x80000000ull) return fail(ctx, KB_E_LIMIT, "ids would reach bit 31 (reserved for quoted triples, quoted_triple_store.rs:28-55)");
    const u32 n = (u32)n_terms;
    Buf d_hash, d_batch, d_slot, d_first, d_flen, d_fpos, scratch;
    KB_TRY(dict_index_ensure(ctx, n));
    u64 bslots = 1024;
    while (bslots < 2ull * n) bslots <<= 1;
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u64), &d_hash));
    KB_TRY(alloc_buf(ctx, bslots * sizeof(u64), &d_batch));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &d_slot));
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &d_first));
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &d_flen));
    KB_TRY(alloc_buf(ctx, (((size_t)n + 1) / 2048 + 4) * sizeof(u32), &scratch));
    KB_CUDA(ctx, cudaMemsetAsync(d_batch->p, 0xFF, bslots * sizeof(u64), ctx->st));
    const u32 c = ctrl_alloc(ctx, 4);  // [0] overflow, [2..3] u64 bytes of the new strings
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 4 * sizeof(u32), ctx->st));
    const int grid = grid_1d(n, ctx->n_sms);
    timer_begin(ctx, F_OTHER, 5);
    dict_hash_kernel<<<grid, 256, 0, ctx->st>>>(d_off, d_bytes, n, static_cast<u64*>(d_hash->p));
    DictResolveParams P{};
    P.off = d_off; P.bytes = d_bytes; P.n = n;
    P.hash = static_cast<const u64*>(d_hash->p);
    P.index = ctx->dict_ids ? static_cast<const u64*>(ctx->dict_index->p) : nullptr;
    P.index_mask = ctx->dict_index_slots - 1;
    P.dict_off = ctx->dict_ids ? static_cast<const unsigned long long*>(ctx->dict_off->p) : nullptr;
    P.dict_bytes = ctx->dict_ids ? static_cast<const unsigned char*>(ctx->dict_bytes->p) : nullptr;
    P.dict_ids = ctx->dict_ids;
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
    ctx->stats.kernel_launches += 3;
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
    timer_begin(ctx, F_OTHER, 2);
    dict_assign_kernel<<<grid, 256, 0, ctx->st>>>(P.off, n, base_id, base_bytes, P.out_id, P.slot_of, P.batch, static_cast<const u32*>(d_first->p),
                                                  static_cast<const u32*>(d_flen->p), static_cast<u64*>(d_fpos->p),
                                                  n_new ? static_cast<unsigned long long*>(ctx->dict_off->p) + base_id : nullptr);
    ctx->stats.kernel_launches++;
    if (n_new) {
        const unsigned long long end = base_bytes + new_bytes;
        KB_CUDA(ctx, cudaMemcpyAsync(static_cast<unsigned long long*>(ctx->dict_off->p) + ids_after, &end, sizeof end, cudaMemcpyHostToDevice, ctx->st));
        dict_append_kernel<<<grid_1d((u64)n_new * 32, ctx->n_sms), 256, 0, ctx->st>>>(P.off, P.bytes, static_cast<const u64*>(d_fpos->p),
                                                                                     static_cast<const unsigned long long*>(ctx->dict_off->p) + base_id, n_new,
                                                                                     static_cast<unsigned char*>(ctx->dict_bytes->p));
        ctx->stats.kernel_launches++;
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


}  // namespace kb

using namespace kb;

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

}  // extern "C"
