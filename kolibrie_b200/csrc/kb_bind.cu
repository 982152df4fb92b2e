// kb_bind.cu — `PhysicalOperator::Bind` with the built-in functions of ExecutionEngine::execute_with_ids
// (kolibrie/src/streamertail_optimizer/execution/engine.rs:144-277) on a device relation, so that a BIND at the root of a plan does not
// send the scans, joins and filters beneath it back to the CPU. The semantics are in include/kolibrie_b200.h; here:
//   SUBJECT / PREDICATE / OBJECT  one gather pass over the quoted-triple table
//   isTRIPLE                      a pass for the first row that needs "true" / "false", the encode of those strings, a write pass
//   TRIPLE                        QuotedTripleStore::encode of the batch (quoted_encode, kb_quoted.cu)
//   CONCAT                        lengths, scan, byte gather, then kb_dict_encode's body on the concatenations (dict_encode_device)
#include <algorithm>
#include <cstring>

#include "kb_internal.hpp"

namespace kb {

// BIND built-ins (kb_bind, engine.rs:144-277). Every write pass takes `old` (the replaced column when the output variable was bound
// already, else null): a row the reference does not insert into keeps old[i], or gets EMPTY32; *n_unbound += rows left EMPTY32.
// SUBJECT / PREDICATE / OBJECT: out[i] = component `comp` of the table entry of arg[i] (a quoted id the table holds), else unbound
__global__ void __launch_bounds__(256) bind_component_kernel(const u32* __restrict__ arg, u32 n, const QuotedTab qt, u32 comp, const u32* __restrict__ old,
                                                             u32* __restrict__ out, unsigned long long* n_unbound) {
    const u32* __restrict__ tab = comp == 0u ? qt.s : comp == 1u ? qt.p : qt.o;
    const u32 stride = gridDim.x * blockDim.x;
    const u32 end = (n + 31u) & ~31u;  // whole warps for the ballot
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
        u32 v = EMPTY32;
        if (i < n) {
            const u32 id = arg[i], x = id & 0x7FFFFFFFu;
            if ((id & 0x80000000u) && x < qt.n) v = __ldg(tab + x);  // a hole holds EMPTY32; KB_ID_NONE has x = 2^31-1 >= qt.n
            if (v == EMPTY32 && old) v = old[i];
            out[i] = v;
        }
        bind_count_unbound(i < n && v == EMPTY32, n_unbound);
    }
}

// isTRIPLE, pass 1: first[0] = min row whose argument is a quoted id, first[1] = min row whose argument is bound and not quoted
// (first[] = EMPTY32 beforehand)
__global__ void __launch_bounds__(256) bind_istriple_first_kernel(const u32* __restrict__ arg, u32 n, u32* first) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 end = (n + 31u) & ~31u;
    u32 ft = EMPTY32, ff = EMPTY32;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
        if (i < n) {
            const u32 id = arg[i];
            if (id != EMPTY32) {
                if (id & 0x80000000u) ft = min(ft, i);
                else ff = min(ff, i);
            }
        }
    }
    ft = __reduce_min_sync(0xffffffffu, ft);
    ff = __reduce_min_sync(0xffffffffu, ff);
    if ((threadIdx.x & 31) == 0) {
        if (ft != EMPTY32) atomicMin(first, ft);
        if (ff != EMPTY32) atomicMin(first + 1, ff);
    }
}
// isTRIPLE, pass 2: out[i] = id_true / id_false, unbound where the argument is
__global__ void __launch_bounds__(256) bind_istriple_write_kernel(const u32* __restrict__ arg, u32 n, u32 id_true, u32 id_false, const u32* __restrict__ old,
                                                                  u32* __restrict__ out, unsigned long long* n_unbound) {
    const u32 stride = gridDim.x * blockDim.x;
    const u32 end = (n + 31u) & ~31u;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
        u32 v = EMPTY32;
        if (i < n) {
            const u32 id = arg[i];
            v = id == EMPTY32 ? (old ? old[i] : EMPTY32) : (id & 0x80000000u) ? id_true : id_false;
            out[i] = v;
        }
        bind_count_unbound(i < n && v == EMPTY32, n_unbound);
    }
}

// CONCAT: the pieces of row i are, per argument a, the dictionary string of col[a][i] ("" when the dictionary does not hold it) or the
// constant cbytes[coff[a] .. coff[a] + clen[a])
struct BindConcatParams {
    u32 n, n_args;
    const u32* col[KB_BIND_MAX_ARGS];  // null: a constant
    u64 coff[KB_BIND_MAX_ARGS];
    u32 clen[KB_BIND_MAX_ARGS];
    const unsigned char* cbytes;
    DictTab dict;
    u32* len;                          // lengths pass: [n + 1] (len[n] untouched); then their exclusive prefix
    unsigned long long* total;         // lengths pass: += bytes of all rows
    u64* off64;                        // gather pass: [n + 1] the prefix widened (the encode's offsets)
    unsigned char* out;
};
__device__ __forceinline__ void concat_piece(const BindConcatParams& P, u32 a, u32 i, const unsigned char** src, u32* len) {
    if (P.col[a]) {
        const u32 id = P.col[a][i];
        if (id < P.dict.ids) {  // Dictionary::decode: quoted ids (>= 2^31 > dict.ids), missing ids and KB_ID_NONE contribute ""
            const unsigned long long b = __ldg(P.dict.off + id);
            *src = P.dict.bytes + b;
            *len = (u32)(__ldg(P.dict.off + id + 1) - b);
        } else {
            *src = nullptr;
            *len = 0u;
        }
    } else {
        *src = P.cbytes + P.coff[a];
        *len = P.clen[a];
    }
}
__global__ void __launch_bounds__(256) bind_concat_lengths_kernel(const __grid_constant__ BindConcatParams P) {
    unsigned long long t = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
        unsigned long long l = 0;
        for (u32 a = 0; a < P.n_args; a++) {
            const unsigned char* src;
            u32 k;
            concat_piece(P, a, i, &src, &k);
            l += k;
        }
        P.len[i] = l > 0xFFFFFFFFull ? 0xFFFFFFFFu : (u32)l;  // (the total then exceeds the limit: the caller refuses the call)
        t += l;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0 && t) atomicAdd(P.total, t);
}
// one warp per 32 rows: the lanes copy each piece of a row together (decode_gather's access pattern)
__global__ void __launch_bounds__(256) bind_concat_gather_kernel(const __grid_constant__ BindConcatParams P) {
    const int lane = threadIdx.x & 31;
    const u32 warps = (gridDim.x * blockDim.x) >> 5;
    const u32 n_chunks = (P.n + 31u) >> 5;
    for (u32 chunk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; chunk < n_chunks; chunk += warps) {
        const u32 i = chunk * 32u + (u32)lane;
        u32 dst = 0;
        if (i < P.n) {
            dst = P.len[i];
            P.off64[i] = dst;
            if (i + 1u == P.n) P.off64[P.n] = P.len[P.n];
        }
        const u32 rows = min(32u, P.n - chunk * 32u);
        for (u32 r = 0; r < rows; r++) {  // the warp writes row r of its chunk, piece by piece: consecutive lanes, consecutive bytes
            const u32 row = chunk * 32u + r;
            u32 w = __shfl_sync(0xffffffffu, dst, (int)r);
            for (u32 a = 0; a < P.n_args; a++) {
                const unsigned char* src;
                u32 k;
                concat_piece(P, a, row, &src, &k);  // (the same address in every lane: one broadcast load)
                for (u32 b = (u32)lane; b < k; b += 32u) P.out[w + b] = __ldg(src + b);
                w += k;
            }
        }
    }
}

}  // namespace kb

using namespace kb;

namespace {

kb_status bind_is_triple(kb_ctx* ctx, const u32* arg, u32 n, const u32* old, u32* out, unsigned long long* n_unbound, kb_bind_info* info) {
    const u32 c = ctrl_alloc(ctx, 2);  // first row needing "true", first row needing "false"
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0xFF, 2 * sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER);
    bind_istriple_first_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(arg, n, ctx->ctrl + c);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    // the strings the rows need, in the order of the first row needing each (the reference encodes inside its row loop)
    std::vector<std::pair<u32, const char*>> need;
    if (ctx->h_ctrl[c] != EMPTY32) need.push_back({ctx->h_ctrl[c], "true"});
    if (ctx->h_ctrl[c + 1] != EMPTY32) need.push_back({ctx->h_ctrl[c + 1], "false"});
    std::sort(need.begin(), need.end());
    u32 ids[2] = {EMPTY32, EMPTY32};  // ids of the strings in `need` order
    info->dict_first = ctx->dict_ids;
    if (!need.empty()) {
        u64 h_off[3] = {0, 0, 0};
        std::string bytes;
        for (size_t k = 0; k < need.size(); k++) { bytes += need[k].second; h_off[k + 1] = bytes.size(); }
        Buf d_off, d_bytes, d_ids;
        KB_TRY(alloc_buf(ctx, sizeof h_off, &d_off));
        KB_TRY(alloc_buf(ctx, bytes.size(), &d_bytes));
        KB_TRY(alloc_buf(ctx, sizeof ids, &d_ids));
        KB_CUDA(ctx, cudaMemcpyAsync(d_off->p, h_off, sizeof h_off, cudaMemcpyHostToDevice, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(d_bytes->p, bytes.data(), bytes.size(), cudaMemcpyHostToDevice, ctx->st));
        ctx->stats.h2d_bytes += sizeof h_off + bytes.size();
        u32 n_new = 0;
        KB_TRY(dict_encode_device(ctx, static_cast<const u64*>(d_off->p), static_cast<const unsigned char*>(d_bytes->p), need.size(), bytes.size(),
                                  static_cast<u32*>(d_ids->p), &n_new, nullptr));
        KB_CUDA(ctx, cudaMemcpyAsync(ids, d_ids->p, need.size() * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));  // (h_off, bytes, ids: synchronised below)
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        info->dict_new = n_new;
    }
    u32 id_true = EMPTY32, id_false = EMPTY32;
    for (size_t k = 0; k < need.size(); k++) (need[k].second[0] == 't' ? id_true : id_false) = ids[k];
    timer_begin(ctx, F_OTHER);
    bind_istriple_write_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(arg, n, id_true, id_false, old, out, n_unbound);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

kb_status bind_concat(kb_ctx* ctx, const kb_bind_spec& spec, const u32* const* col, u32 n, u32* out, kb_bind_info* info) {
    BindConcatParams P{};
    P.n = n;
    P.n_args = spec.n_args;
    const u64 cbytes = spec.n_const ? spec.const_offsets[spec.n_const] : 0;
    Buf d_cbytes, len, scratch, off64, bytes;
    KB_TRY(alloc_buf(ctx, (size_t)cbytes, &d_cbytes));
    if (cbytes) {
        KB_CUDA(ctx, cudaMemcpyAsync(d_cbytes->p, spec.const_bytes, (size_t)cbytes, cudaMemcpyHostToDevice, ctx->st));
        ctx->stats.h2d_bytes += cbytes;
    }
    P.cbytes = static_cast<const unsigned char*>(d_cbytes->p);
    for (u32 a = 0; a < spec.n_args; a++) {
        P.col[a] = col[a];
        if (!col[a]) {
            const u32 k = spec.args[a].value;
            P.coff[a] = spec.const_offsets[k];
            P.clen[a] = (u32)(spec.const_offsets[k + 1] - spec.const_offsets[k]);
        }
    }
    P.dict = dicttab(ctx);
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &len));
    KB_TRY(alloc_buf(ctx, (((size_t)n + 1) / 2048 + 4) * sizeof(u32), &scratch));
    P.len = static_cast<u32*>(len->p);
    const u32 c = ctrl_alloc(ctx, 2);  // u64 total bytes
    P.total = reinterpret_cast<unsigned long long*>(ctx->ctrl + c);
    KB_CUDA(ctx, cudaMemsetAsync(P.total, 0, sizeof(unsigned long long), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(P.len + n, 0, sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER, 4);
    bind_concat_lengths_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(P);
    launch_exclusive_scan_u32(P.len, n + 1, static_cast<u32*>(scratch->p), ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    unsigned long long total = 0;
    memcpy(&total, ctx->h_ctrl + c, sizeof total);
    if (total > 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "CONCAT: %llu concatenated bytes (limit 2^32-16 per call)", total);
    if ((u64)ctx->dict_ids + n >= 0x80000000ull) return fail(ctx, KB_E_LIMIT, "CONCAT: dictionary ids would reach bit 31");
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u64), &off64));
    KB_TRY(alloc_buf(ctx, (size_t)total + 16, &bytes));
    P.off64 = static_cast<u64*>(off64->p);
    P.out = static_cast<unsigned char*>(bytes->p);
    timer_begin(ctx, F_OTHER);
    bind_concat_gather_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(P);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    info->dict_first = ctx->dict_ids;
    u32 n_new = 0;
    KB_TRY(dict_encode_device(ctx, P.off64, P.out, n, total, out, &n_new, nullptr));
    info->dict_new = n_new;
    return KB_OK;
}

}  // namespace

extern "C" {

kb_status kb_bind(kb_ctx* ctx, const kb_rel* in, const kb_bind_spec* spec, kb_rel** out, kb_bind_info* info) {
    KB_ENTER(ctx);
    if (!in || !spec || !out) return fail(ctx, KB_E_INVALID, "NULL argument");
    const u32 fn = spec->function;
    if (fn < KB_BIND_SUBJECT || fn > KB_BIND_CONCAT) return fail(ctx, KB_E_INVALID, "kb_bind: unknown function %u", fn);
    const u32 arity = fn == KB_BIND_TRIPLE ? 3u : fn == KB_BIND_CONCAT ? spec->n_args : 1u;
    if (spec->n_args != arity || spec->n_args > KB_BIND_MAX_ARGS)
        return fail(ctx, KB_E_INVALID, "kb_bind: %u arguments (SUBJECT, PREDICATE, OBJECT and isTRIPLE take 1, TRIPLE 3, CONCAT at most %d)", spec->n_args,
                    KB_BIND_MAX_ARGS);
    if (spec->n_args && !spec->args) return fail(ctx, KB_E_INVALID, "NULL arguments");
    if (in->pair) return fail(ctx, KB_E_INVALID, "internal relation layout");
    if (in->n >= 0xFFFFFFF0ull) return fail(ctx, KB_E_LIMIT, "kb_bind: relation too large (2^32-16 rows per call)");
    if (fn == KB_BIND_CONCAT && spec->n_const) {
        if (!spec->const_offsets || spec->const_offsets[0] != 0) return fail(ctx, KB_E_INVALID, "CONCAT constants: const_offsets must start at 0");
        for (u32 k = 0; k < spec->n_const; k++)
            if (spec->const_offsets[k + 1] < spec->const_offsets[k]) return fail(ctx, KB_E_INVALID, "CONCAT constants: offsets decrease at %u", k);
        if (spec->const_offsets[spec->n_const] && !spec->const_bytes) return fail(ctx, KB_E_INVALID, "CONCAT constants: NULL bytes");
    }
    const u32* col[KB_BIND_MAX_ARGS] = {};
    u32 cval[3] = {0, 0, 0};
    for (u32 a = 0; a < spec->n_args; a++) {
        const kb_term& t = spec->args[a];
        if (t.is_var == 1) {
            const int k = in->col_of(t.value);
            if (k < 0) return fail(ctx, KB_E_INVALID, "kb_bind: argument %u: slot %u is not a column of the input", a, t.value);
            col[a] = in->cols[k].ptr;
        } else if (t.is_var == 0 && fn == KB_BIND_TRIPLE) {
            if (t.value == KB_ID_NONE) return fail(ctx, KB_E_INVALID, "kb_bind: constant id 0xFFFFFFFF is reserved (KB_ID_NONE)");
            cval[a] = t.value;
        } else if (t.is_var == 0 && fn == KB_BIND_CONCAT) {
            if (t.value >= spec->n_const) return fail(ctx, KB_E_INVALID, "kb_bind: CONCAT constant %u of %u", t.value, spec->n_const);
        } else {
            return fail(ctx, KB_E_INVALID, "kb_bind: argument %u must be a variable%s", a, fn == KB_BIND_TRIPLE || fn == KB_BIND_CONCAT ? " or a constant" : "");
        }
    }
    const int oc = in->col_of(spec->out_slot);
    if (oc < 0 && in->slots.size() >= KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "kb_bind: more than %d columns", KB_MAX_COLS);
    if (fn == KB_BIND_TRIPLE && (!(spec->next_qt_id & 0x80000000u) || spec->next_qt_id == KB_ID_NONE || (spec->next_qt_id & 0x7FFFFFFFu) < ctx->quoted_slots))
        return fail(ctx, KB_E_INVALID, "kb_bind: next_qt_id 0x%08x is not a quoted-triple id above every id of the table (%u slots)", spec->next_qt_id,
                    ctx->quoted_slots);
    const u32 n = (u32)in->n;
    kb_bind_info inf{};
    inf.n_rows = n;
    inf.dict_first = ctx->dict_ids;
    Col res;
    KB_TRY(alloc_col(ctx, n, &res));
    const u32* old = oc >= 0 ? in->cols[oc].ptr : nullptr;
    const u32 c = ctrl_alloc(ctx, 2);  // u64 rows left unbound
    auto* n_unbound = reinterpret_cast<unsigned long long*>(ctx->ctrl + c);
    KB_CUDA(ctx, cudaMemsetAsync(n_unbound, 0, sizeof(unsigned long long), ctx->st));
    if (n) {
        switch (fn) {
        case KB_BIND_SUBJECT:
        case KB_BIND_PREDICATE:
        case KB_BIND_OBJECT:
            timer_begin(ctx, F_OTHER);
            bind_component_kernel<<<grid_1d(n, ctx->n_sms), 256, 0, ctx->st>>>(col[0], n, quotedtab(ctx), fn - KB_BIND_SUBJECT, old, res.ptr, n_unbound);
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
            break;
        case KB_BIND_IS_TRIPLE: KB_TRY(bind_is_triple(ctx, col[0], n, old, res.ptr, n_unbound, &inf)); break;
        case KB_BIND_TRIPLE: KB_TRY(quoted_encode(ctx, col, cval, n, spec->next_qt_id, old, res.ptr, n_unbound, &inf)); break;
        default: KB_TRY(bind_concat(ctx, *spec, col, n, res.ptr, &inf)); break;
        }
        KB_TRY(ctrl_read(ctx));
        memcpy(&inf.n_unbound, ctx->h_ctrl + c, sizeof inf.n_unbound);
    }
    auto r = std::make_unique<kb_rel>();
    r->slots = in->slots;
    r->cols = in->cols;
    r->n = in->n;
    if (oc >= 0) r->cols[oc] = res;
    else { r->slots.push_back(spec->out_slot); r->cols.push_back(res); }
    ctx->stats.rows_out = r->n;
    if (info) *info = inf;
    *out = r.release();
    return KB_OK;
}

}  // extern "C"
