// kb_bind.cu — `PhysicalOperator::Bind` with the built-in functions of ExecutionEngine::execute_with_ids
// (kolibrie/src/streamertail_optimizer/execution/engine.rs:144-277) on a device relation, so that a BIND at the root of a plan does not
// send the scans, joins and filters beneath it back to the CPU. The semantics are in include/kolibrie_b200.h; here:
//   SUBJECT / PREDICATE / OBJECT  one gather pass over the quoted-triple table
//   isTRIPLE                      a pass for the first row that needs "true" / "false", the encode of those strings, a write pass
//   TRIPLE                        QuotedTripleStore::encode of the batch: reverse-index probe, batch table of the misses (smallest row
//                                 wins), first-occurrence scan, ids next_qt_id + rank; the new entries join the table and the index
//   CONCAT                        lengths, scan, byte gather, then kb_dict_encode's body on the concatenations (dict_encode_device)
#include <algorithm>
#include <cstring>

#include "kb_internal.hpp"

using namespace kb;

namespace {

// the reverse index holds every entry of the table and stays below load 1/2 with `extra` more entries (rebuilt larger otherwise)
kb_status quoted_rev_ensure(kb_ctx* ctx, u64 extra) {
    const u64 need = ((u64)ctx->quoted_slots + extra) * 2 + 64;
    if (!ctx->quoted_rev || ctx->quoted_rev_slots < need) {
        u64 slots = 1024;
        while (slots < need + need / 2) slots <<= 1;  // headroom: the next batches insert in place
        ctx->quoted_rev.reset();
        KB_TRY(alloc_buf(ctx, slots * sizeof(u64), &ctx->quoted_rev));
        KB_CUDA(ctx, cudaMemsetAsync(ctx->quoted_rev->p, 0xFF, slots * sizeof(u64), ctx->st));
        ctx->quoted_rev_slots = slots;
        ctx->quoted_rev_indexed = 0;
    }
    if (ctx->quoted_rev_indexed < ctx->quoted_slots) {
        const u32 c = ctrl_alloc(ctx, 1);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, sizeof(u32), ctx->st));
        const u32 n = ctx->quoted_slots - ctx->quoted_rev_indexed;
        timer_begin(ctx, F_OTHER);
        launch_quoted_rev_insert(quotedtab(ctx), ctx->quoted_rev_indexed, n, static_cast<u64*>(ctx->quoted_rev->p), ctx->quoted_rev_slots - 1, ctx->ctrl + c,
                                 ctx->n_sms, ctx->st);
        timer_end(ctx);
        ctx->stats.kernel_launches++;
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        if (ctx->h_ctrl[c]) return fail(ctx, KB_E_LIMIT, "quoted-triple reverse index overflow");
        ctx->quoted_rev_indexed = ctx->quoted_slots;
    }
    return KB_OK;
}

// the table's buffers hold at least `slots` entries; new slots are EMPTY32. The buffers keep alloc_buf's padding past their capacity,
// which the match kernel's rounded-up TMA reads of the last tile rely on.
kb_status quoted_grow(kb_ctx* ctx, u32 slots) {
    if (slots <= ctx->quoted_cap) return KB_OK;
    const u32 cap = (u32)std::min<u64>(KB_QUOTED_MAX_SLOTS, std::max<u64>((u64)slots + slots / 2, 1024));
    Buf* cols[3] = {&ctx->quoted_s, &ctx->quoted_p, &ctx->quoted_o};
    Buf nb[3];
    for (int k = 0; k < 3; k++) {
        KB_TRY(alloc_buf(ctx, (size_t)cap * sizeof(u32), &nb[k]));
        launch_fill_u32(static_cast<u32*>(nb[k]->p), EMPTY32, cap, ctx->st);
        if (ctx->quoted_slots)
            KB_CUDA(ctx, cudaMemcpyAsync(nb[k]->p, (*cols[k])->p, (size_t)ctx->quoted_slots * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    }
    ctx->stats.kernel_launches += 3;
    KB_CUDA(ctx, cudaGetLastError());
    for (int k = 0; k < 3; k++) *cols[k] = nb[k];
    ctx->quoted_cap = cap;
    return KB_OK;
}

kb_status bind_triple(kb_ctx* ctx, const u32* const* col, const u32* cval, u32 n, u32 next_qt_id, const u32* old, u32* out, unsigned long long* n_unbound,
                      kb_bind_info* info) {
    KB_TRY(quoted_rev_ensure(ctx, n));
    u64 bslots = 1024;
    while (bslots < 2ull * n) bslots <<= 1;
    Buf batch, hit, slot_of, first, scratch;
    KB_TRY(alloc_buf(ctx, bslots * sizeof(u64), &batch));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &hit));
    KB_TRY(alloc_buf(ctx, (size_t)n * sizeof(u32), &slot_of));
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &first));
    KB_TRY(alloc_buf(ctx, (((size_t)n + 1) / 2048 + 4) * sizeof(u32), &scratch));
    KB_CUDA(ctx, cudaMemsetAsync(batch->p, 0xFF, bslots * sizeof(u64), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(static_cast<u32*>(first->p) + n, 0, sizeof(u32), ctx->st));
    BindTripleParams P{};
    for (int k = 0; k < 3; k++) { P.col[k] = col[k]; P.cval[k] = cval[k]; }
    P.n = n;
    P.qt = quotedtab(ctx);
    P.rev = static_cast<const u64*>(ctx->quoted_rev->p);
    P.rev_mask = ctx->quoted_rev_slots - 1;
    P.batch = static_cast<u64*>(batch->p);
    P.batch_mask = bslots - 1;
    P.hit = static_cast<u32*>(hit->p);
    P.slot_of = static_cast<u32*>(slot_of->p);
    P.first = static_cast<u32*>(first->p);
    const u32 c = ctrl_alloc(ctx, 2);  // [0] overflow, [1] new triples (first[n] after the scan)
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0, 2 * sizeof(u32), ctx->st));
    P.overflow = ctx->ctrl + c;
    timer_begin(ctx, F_OTHER, 3);
    launch_bind_triple_resolve(P, ctx->n_sms, ctx->st);
    launch_bind_triple_mark(P, ctx->n_sms, ctx->st);
    launch_exclusive_scan_u32(P.first, n + 1, static_cast<u32*>(scratch->p), ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches += 3;
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->ctrl + c + 1, P.first + n, sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    if (ctx->h_ctrl[c]) return fail(ctx, KB_E_LIMIT, "TRIPLE batch table overflow");
    const u32 n_new = ctx->h_ctrl[c + 1];
    const u32 base = next_qt_id & 0x7FFFFFFFu;
    if (n_new && (u64)base + n_new > KB_QUOTED_MAX_SLOTS)
        return fail(ctx, KB_E_LIMIT, "TRIPLE: %u new quoted triples from id 0x%08x would pass the table's %u slots", n_new, next_qt_id, KB_QUOTED_MAX_SLOTS);
    // nothing has changed so far (the reverse index is a cache of the table); from here on the table grows
    if (n_new) KB_TRY(quoted_grow(ctx, base + n_new));
    P.next_qt_id = next_qt_id;
    P.ws = n_new ? static_cast<u32*>(ctx->quoted_s->p) : nullptr;
    P.wp = n_new ? static_cast<u32*>(ctx->quoted_p->p) : nullptr;
    P.wo = n_new ? static_cast<u32*>(ctx->quoted_o->p) : nullptr;
    P.old = old;
    P.out = out;
    P.n_unbound = n_unbound;
    timer_begin(ctx, F_OTHER);
    launch_bind_triple_assign(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches++;
    KB_CUDA(ctx, cudaGetLastError());
    if (n_new) {
        ctx->quoted_slots = base + n_new;
        KB_TRY(quoted_rev_ensure(ctx, 0));  // the new entries enter the reverse index
    }
    info->quoted_first = n_new ? next_qt_id : 0;
    info->quoted_new = n_new;
    return KB_OK;
}

kb_status bind_is_triple(kb_ctx* ctx, const u32* arg, u32 n, const u32* old, u32* out, unsigned long long* n_unbound, kb_bind_info* info) {
    const u32 c = ctrl_alloc(ctx, 2);  // first row needing "true", first row needing "false"
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + c, 0xFF, 2 * sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER);
    launch_bind_istriple_first(arg, n, ctx->ctrl + c, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches++;
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
    launch_bind_istriple_write(arg, n, id_true, id_false, old, out, n_unbound, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches++;
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
    P.dict_off = ctx->dict_ids ? static_cast<const unsigned long long*>(ctx->dict_off->p) : nullptr;
    P.dict_bytes = ctx->dict_ids ? static_cast<const unsigned char*>(ctx->dict_bytes->p) : nullptr;
    P.dict_ids = ctx->dict_ids;
    KB_TRY(alloc_buf(ctx, ((size_t)n + 1) * sizeof(u32), &len));
    KB_TRY(alloc_buf(ctx, (((size_t)n + 1) / 2048 + 4) * sizeof(u32), &scratch));
    P.len = static_cast<u32*>(len->p);
    const u32 c = ctrl_alloc(ctx, 2);  // u64 total bytes
    P.total = reinterpret_cast<unsigned long long*>(ctx->ctrl + c);
    KB_CUDA(ctx, cudaMemsetAsync(P.total, 0, sizeof(unsigned long long), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(P.len + n, 0, sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER, 2);
    launch_bind_concat_lengths(P, ctx->n_sms, ctx->st);
    launch_exclusive_scan_u32(P.len, n + 1, static_cast<u32*>(scratch->p), ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches += 2;
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
    launch_bind_concat_gather(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches++;
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
            launch_bind_component(col[0], n, quotedtab(ctx), fn - KB_BIND_SUBJECT, old, res.ptr, n_unbound, ctx->n_sms, ctx->st);
            timer_end(ctx);
            ctx->stats.kernel_launches++;
            KB_CUDA(ctx, cudaGetLastError());
            break;
        case KB_BIND_IS_TRIPLE: KB_TRY(bind_is_triple(ctx, col[0], n, old, res.ptr, n_unbound, &inf)); break;
        case KB_BIND_TRIPLE: KB_TRY(bind_triple(ctx, col, cval, n, spec->next_qt_id, old, res.ptr, n_unbound, &inf)); break;
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

kb_status kb_quoted_download(kb_ctx* ctx, uint32_t first_id, uint32_t n, uint32_t* s, uint32_t* p, uint32_t* o) {
    KB_ENTER(ctx);
    if (n == 0) return KB_OK;
    if (!s || !p || !o) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (!(first_id & 0x80000000u)) return fail(ctx, KB_E_INVALID, "0x%08x is not a quoted-triple id", first_id);
    const u64 x = first_id & 0x7FFFFFFFu;
    if (x + n > 0x7FFFFFFFull) return fail(ctx, KB_E_INVALID, "id range past 0xFFFFFFFE");
    const u64 held = x < ctx->quoted_slots ? std::min<u64>(n, ctx->quoted_slots - x) : 0;
    uint32_t* dst[3] = {s, p, o};
    const Buf* src[3] = {&ctx->quoted_s, &ctx->quoted_p, &ctx->quoted_o};
    for (int k = 0; k < 3; k++) {
        if (held) KB_CUDA(ctx, cudaMemcpyAsync(dst[k], static_cast<const u32*>((*src[k])->p) + x, held * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        std::fill(dst[k] + held, dst[k] + n, KB_ID_NONE);
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    ctx->stats.d2h_bytes += held * 12u;
    return KB_OK;
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
