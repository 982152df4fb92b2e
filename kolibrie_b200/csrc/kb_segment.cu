// kb_segment.cu — on-disk COLUMNAR segment of the device store (SURVEY.md §8 (f)4, second half). The reference persists an SSTable as a
// serialised UnifiedIndex of AoS triples (kolibrie/src/disk_storage/sstable.rs:40-85: id, level, index, min/max key, triple count); the
// device-side counterpart is the store's own layout written to disk: three u32 columns, each starting at a 4096-byte boundary (so that a
// column can be read or mapped page-aligned and copied to HBM without repacking), preceded by a header that carries what a load would
// otherwise have to compute with kernels (triple count, per-column id range) and a checksum per column.
//   [header 4096 B][s column, padded to 4096][p column, padded][o column, padded]
// kb_store_append_file streams a file into a new store segment through two pinned staging buffers (read of chunk i+1 overlaps the
// host->device copy of chunk i); kb_segment_save writes a store segment (or the whole store) out.
#include <cstdio>
#include <cstring>
#include <vector>

#include "kb_internal.hpp"

using namespace kb;

namespace {
constexpr uint64_t SEG_MAGIC = 0x31304745534B4Bull;  // "KKSEG01"
constexpr size_t PAGE = 4096;
struct SegHeader {
    uint64_t magic;
    uint64_t n_triples;
    uint64_t tag;
    uint32_t cmin[3], cmax[3];   // id range of s, p, o
    uint64_t checksum[3];        // sum of (word * (index + 1)) modulo 2^64 per column
    uint64_t col_offset[3];      // byte offset of each column in the file
    uint32_t version, reserved;
};
static_assert(sizeof(SegHeader) <= PAGE, "header fits its page");

inline size_t pad(size_t b) { return (b + PAGE - 1) / PAGE * PAGE; }
uint64_t checksum(const u32* a, uint64_t n, uint64_t first_index) {
    uint64_t c = 0;
    for (uint64_t i = 0; i < n; i++) c += (uint64_t)a[i] * (first_index + i + 1);
    return c;
}
struct File {
    FILE* f = nullptr;
    ~File() { if (f) fclose(f); }
};
}  // namespace

extern "C" {

// host only (no device needed): write three columns as a segment file
kb_status kb_segment_write(const char* path, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t tag) {
    if (!path || (n && (!s || !p || !o))) return KB_E_INVALID;
    File fh;
    fh.f = fopen(path, "wb");
    if (!fh.f) return KB_E_NOT_FOUND;
    SegHeader h{};
    h.magic = SEG_MAGIC; h.n_triples = n; h.tag = tag; h.version = 1;
    const u32* cols[3] = {s, p, o};
    uint64_t at = PAGE;
    for (int c = 0; c < 3; c++) {
        h.cmin[c] = 0xFFFFFFFFu; h.cmax[c] = 0;
        for (uint64_t i = 0; i < n; i++) { h.cmin[c] = std::min(h.cmin[c], cols[c][i]); h.cmax[c] = std::max(h.cmax[c], cols[c][i]); }
        h.checksum[c] = checksum(cols[c], n, 0);
        h.col_offset[c] = at;
        at += pad(n * sizeof(u32));
    }
    std::vector<char> page(PAGE, 0);
    memcpy(page.data(), &h, sizeof h);
    if (fwrite(page.data(), 1, PAGE, fh.f) != PAGE) return KB_E_CUDA;
    for (int c = 0; c < 3; c++) {
        const size_t bytes = n * sizeof(u32);
        if (bytes && fwrite(cols[c], 1, bytes, fh.f) != bytes) return KB_E_CUDA;
        std::vector<char> z(pad(bytes) - bytes, 0);
        if (!z.empty() && fwrite(z.data(), 1, z.size(), fh.f) != z.size()) return KB_E_CUDA;
    }
    return KB_OK;
}

kb_status kb_segment_info(const char* path, uint64_t* n_triples, uint64_t* tag, uint32_t* cmin /* [3] */, uint32_t* cmax /* [3] */) {
    if (!path) return KB_E_INVALID;
    File fh;
    fh.f = fopen(path, "rb");
    if (!fh.f) return KB_E_NOT_FOUND;
    SegHeader h{};
    if (fread(&h, 1, sizeof h, fh.f) != sizeof h || h.magic != SEG_MAGIC || h.version != 1) return KB_E_INVALID;
    if (n_triples) *n_triples = h.n_triples;
    if (tag) *tag = h.tag;
    for (int c = 0; c < 3; c++) { if (cmin) cmin[c] = h.cmin[c]; if (cmax) cmax[c] = h.cmax[c]; }
    return KB_OK;
}

kb_status kb_segment_save(kb_ctx* ctx, uint64_t tag, int whole_store, const char* path) {
    if (!ctx || !path) return KB_E_INVALID;
    DeviceGuard guard(ctx->device);
    KB_TRY(begin_call(ctx));
    uint64_t n = 0;
    for (auto& sg : ctx->segs) if (whole_store || sg.tag == tag) n += sg.n;
    std::vector<u32> s(n), p(n), o(n);
    uint64_t at = 0;
    bool any = false;
    for (auto& sg : ctx->segs) {
        if (!(whole_store || sg.tag == tag)) continue;
        any = true;
        if (!sg.n) continue;
        KB_CUDA(ctx, cudaMemcpyAsync(s.data() + at, sg.s.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(p.data() + at, sg.p.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(o.data() + at, sg.o.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        at += sg.n;
    }
    if (!any) return fail(ctx, KB_E_NOT_FOUND, "no segment with tag %llu", (unsigned long long)tag);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += 3 * n * sizeof(u32);
    const kb_status rc = kb_segment_write(path, s.data(), p.data(), o.data(), n, tag);
    if (rc != KB_OK) return fail(ctx, rc, "cannot write segment file %s", path);
    return KB_OK;
}

}  // extern "C"

extern "C" kb_status kb_store_append_file(kb_ctx* ctx, const char* path, uint64_t tag, int verify) {
    if (!ctx || !path) return KB_E_INVALID;
    DeviceGuard guard(ctx->device);
    KB_TRY(begin_call(ctx));
    File fh;
    fh.f = fopen(path, "rb");
    if (!fh.f) return fail(ctx, KB_E_NOT_FOUND, "cannot open %s", path);
    SegHeader h{};
    if (fread(&h, 1, sizeof h, fh.f) != sizeof h || h.magic != SEG_MAGIC || h.version != 1) return fail(ctx, KB_E_INVALID, "%s is not a segment file", path);
    const uint64_t n = h.n_triples;
    if (n) KB_TRY(refuse_reserved_id(ctx, h.cmax));
    if (ctx->n_triples + n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "store would exceed 2^32-16 triples");
    Segment sg;
    sg.tag = tag;
    sg.n = n;
    KB_TRY(alloc_col(ctx, n, &sg.s));
    KB_TRY(alloc_col(ctx, n, &sg.p));
    KB_TRY(alloc_col(ctx, n, &sg.o));
    // two pinned staging buffers: the file read of chunk i+1 overlaps the host->device copy of chunk i
    const size_t chunk_words = 4u << 20;  // 16 MiB
    u32* stage[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    auto cleanup = [&]() { for (int i = 0; i < 2; i++) { if (stage[i]) cudaFreeHost(stage[i]); if (done[i]) cudaEventDestroy(done[i]); } };
    for (int i = 0; i < 2; i++) {
        if (cudaMallocHost(reinterpret_cast<void**>(&stage[i]), chunk_words * sizeof(u32)) != cudaSuccess) { cleanup(); return fail(ctx, KB_E_OOM, "pinned staging buffer"); }
        cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming);
    }
    u32* dst[3] = {sg.s.ptr, sg.p.ptr, sg.o.ptr};
    int slot = 0;
    for (int c = 0; c < 3; c++) {
        if (fseek(fh.f, (long)h.col_offset[c], SEEK_SET) != 0) { cleanup(); return fail(ctx, KB_E_INVALID, "%s: truncated", path); }
        uint64_t sum = 0;
        for (uint64_t at = 0; at < n; at += chunk_words) {
            const uint64_t m = std::min<uint64_t>(chunk_words, n - at);
            cudaEventSynchronize(done[slot]);  // the copy that last used this staging buffer has drained
            if (fread(stage[slot], sizeof(u32), m, fh.f) != m) { cudaStreamSynchronize(ctx->st); cleanup(); return fail(ctx, KB_E_INVALID, "%s: truncated column %d", path, c); }
            if (verify) sum += checksum(stage[slot], m, at);
            cudaMemcpyAsync(dst[c] + at, stage[slot], m * sizeof(u32), cudaMemcpyHostToDevice, ctx->st);
            cudaEventRecord(done[slot], ctx->st);
            slot ^= 1;
        }
        if (verify && sum != h.checksum[c]) { cudaStreamSynchronize(ctx->st); cleanup(); return fail(ctx, KB_E_INVALID, "%s: checksum of column %d does not match", path, c); }
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    cleanup();
    ctx->stats.h2d_bytes += 3 * n * sizeof(u32);
    // the header carries the column ranges: no statistics kernels (sharded stores still verify ownership of the subjects)
    for (int c = 0; c < 3; c++) { sg.cmin[c] = h.cmin[c]; sg.cmax[c] = h.cmax[c]; }
    if (ctx->shard_world <= 1) { sg.has_stats = true; sg.stats_world = ctx->shard_world; sg.sharded_ok = true; }
    return store_add_device_segment(ctx, sg);
}
