// kb_store.cu — the device triple store: its segments, the version that everything derived from it is keyed to (prepared plans, the
// seeded fixpoint's state, kb_datalog_maintain's closed token), the per-version hints of the star-join builds and the
// predicate-partitioned index. This file is the only writer of that state: every change to the store goes through store_replace,
// store_add_device_segment or store_evict_tag, which bump the version, drop the hints and maintain or drop the index.
#include <algorithm>
#include <chrono>
#include <cstdlib>

#include "kb_internal.hpp"

using namespace kb;

#define KB_ENTER(ctx)                                         \
    if (!(ctx)) return KB_E_INVALID;                          \
    kb::DeviceGuard _guard((ctx)->device);                    \
    KB_TRY(kb::begin_call(ctx))

namespace kb {

kb_status segment_stats(kb_ctx* ctx, Segment* sg) {
    if ((sg->has_stats && sg->stats_world == ctx->shard_world) || sg->n == 0) { sg->has_stats = true; sg->stats_world = ctx->shard_world; return KB_OK; }
    // one pass: column ranges, foreign subjects, distinct predicates + their row counts (segment_profile_kernel)
    const u32 off = ctrl_alloc(ctx, SEGP_WORDS);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0xFF, SEGP_MAX * sizeof(u32), ctx->st));
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off + SEGP_MAX, 0, (SEGP_WORDS - SEGP_MAX) * sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER);
    launch_segment_profile(sg->s.ptr, sg->p.ptr, sg->o.ptr, (u32)sg->n, ctx->shard_rank, ctx->shard_world, ctx->ctrl + off, ctx->n_sms, ctx->st);
    timer_end(ctx);
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32* h = ctx->h_ctrl + off;
    for (int c = 0; c < 3; c++) { sg->cmin[c] = h[SEGP_MIN + c]; sg->cmax[c] = h[SEGP_MAX + c]; }
    sg->sharded_ok = h[SEGP_FOREIGN] == 0;  // key compaction is only sound when every subject is ours
    sg->pred_rows.clear();
    sg->preds_overflow = h[SEGP_OVERFLOW] != 0;
    sg->has_preds = true;
    if (!sg->preds_overflow) {
        for (u32 i = 0; i < SEGP_SLOTS; i++) if (h[SEGP_SLOT + i] != EMPTY32) sg->pred_rows.push_back({h[SEGP_SLOT + i], h[SEGP_COUNT + i]});
        std::sort(sg->pred_rows.begin(), sg->pred_rows.end());
    }
    sg->stats_world = ctx->shard_world;
    sg->has_stats = true;
    return KB_OK;
}

// ---- store index, one chunk per (predicate, store segment)
// the rank column of a slice's subject table: xkey[compact(subject) - xtab_min] = rank of the object's value in the value order (slots
// without a key are never read: they stay unset)
static kb_status build_rank_column(kb_ctx* ctx, PredSlice& ps) {
    bool ok = false;
    KB_TRY(ensure_num_order(ctx, &ok));
    if (!ok) return KB_OK;
    KB_TRY(alloc_buf(ctx, (size_t)ps.xtab_range * sizeof(u32), &ps.xkey));
    for (auto& ch : ps.chunks) {
        if (!ch.n) continue;
        launch_pair_ranktab(reinterpret_cast<const uint2*>(ch.pairs.ptr), (u32)ch.n, numtab(ctx), static_cast<const double*>(ctx->numv->p),
                            (u32)ctx->h_numv.size(), static_cast<u32*>(ps.xkey->p), ps.xtab_min, ps.xtab_range, ps.tab_cshift, ctx->n_sms, ctx->st);
        ctx->stats.kernel_launches++;
    }
    ps.xkey_version = ctx->num_version;
    return KB_OK;
}

// (re)build or extend the persistent table of one column of a slice after `added` (index into ps.chunks; -1: all chunks) arrived.
// flag_word: control word the insert kernels raise on a duplicate key. Returns through *touched whether a flag has to be read.
// full_build: called by kb_store_build_index, which builds the rank columns itself once every chunk is in.
static kb_status slice_table_update(kb_ctx* ctx, PredSlice& ps, u32 y, int added, u32 cshift, u32 flag_off, bool full_build, bool* touched) {
    Buf& tab = y ? ps.ytab : ps.xtab;
    u32& tmin = y ? ps.ytab_min : ps.xtab_min;
    u32& tcap = y ? ps.ytab_range : ps.xtab_range;
    bool& tried = y ? ps.y_tried : ps.x_tried;
    bool& unique = y ? ps.y_unique : ps.x_unique;
    *touched = false;
    if (tried && !tab) return KB_OK;  // the column was found multi-valued or too sparse: no table, nothing to maintain
    const u32 cs = y ? 0u : cshift;    // only subjects are sharded
    const u32 lo = compact_key(y ? ps.ymin : ps.xmin, cs), hi = compact_key(y ? ps.ymax : ps.xmax, cs);
    const u64 range = (u64)hi - lo + 1;
    const bool fits = tab && lo >= tmin && (u64)hi < (u64)tmin + tcap && (y || ps.tab_cshift == cshift);
    if (!fits) {
        // (re)build over every chunk, with headroom above the largest key: dictionary ids grow, so appended segments bring larger ones
        tab.reset();
        if (!y) ps.xkey.reset();
        tried = true;
        unique = false;
        if (range > std::max<u64>(4 * ps.n + 65536, 1ull << 16) || range > (1ull << 28)) return KB_OK;  // not dense: keep no table
        // headroom: half the range for large tables, twice the range for small ones (a sliding window's ids move up by a slide per
        // slide: a 10-slide window then re-bases its tables every ~20 slides instead of every ~5)
        const u64 cap = std::min<u64>(range + (range <= (4ull << 20) ? 2 * range : range / 2) + 65536, 1ull << 29);
        KB_TRY(alloc_buf(ctx, cap * sizeof(u32), &tab));
        KB_CUDA(ctx, cudaMemsetAsync(tab->p, 0xFF, cap * sizeof(u32), ctx->st));
        tmin = lo;
        tcap = (u32)cap;
        if (!y) ps.tab_cshift = cshift;
        added = -1;
        unique = true;  // until a flag says otherwise
    }
    for (size_t c = 0; c < ps.chunks.size(); c++) {
        if (added >= 0 && (int)c != added) continue;
        const SliceChunk& ch = ps.chunks[c];
        if (!ch.n) continue;
        launch_build_direct_pairs(reinterpret_cast<const uint2*>(ch.pairs.ptr), y, (u32)ch.n, static_cast<u32*>(tab->p), tmin, tcap, cs, ctx->ctrl + flag_off, 0u,
                                  ctx->n_sms, ctx->st);
        ctx->stats.kernel_launches++;
        *touched = true;
    }
    // a subject table rebuilt outside the full build takes its rank column along (the table-mode probe filters on it)
    if (!y && !fits && !full_build && ctx->n_ids && ps.typed(ctx->num_version)) KB_TRY(build_rank_column(ctx, ps));
    return KB_OK;
}

// index the triples of ONE store segment: a chunk per predicate it carries, ranges, persistent tables, typed literal columns
// the slide-sized case of index_add_segment: the segment's predicates and their row counts are known from its profile pass, so the
// chunks are allocated exactly and ONE kernel files every triple (segment_split_kernel); one read-back
static kb_status index_add_segment_split(kb_ctx* ctx, const Segment& sg, u32 cshift) {
    const u32 k = (u32)sg.pred_rows.size();
    SplitParams P{};
    P.s = sg.s.ptr; P.p = sg.p.ptr; P.o = sg.o.ptr;
    P.n = (u32)sg.n;
    P.k = k;
    P.nt = numtab(ctx);
    const u32 off = ctrl_alloc(ctx, k * SPLIT_WORDS);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, k * SPLIT_WORDS * sizeof(u32), ctx->st));
    P.ctrl = ctx->ctrl + off;
    std::vector<SliceChunk> chs(k);
    bool rebuild[MAXP][2];
    for (u32 i = 0; i < k; i++) {
        PredSlice& ps = ctx->index[sg.pred_rows[i].first];
        SliceChunk& ch = chs[i];
        ch.tag = sg.tag;
        ch.n = sg.pred_rows[i].second;
        KB_TRY(alloc_col(ctx, 2 * ch.n, &ch.pairs));
        if (ctx->n_ids) KB_TRY(alloc_buf(ctx, ch.n * sizeof(double), &ch.ynum));
        SplitEntry& e = P.e[i];
        e.pred = sg.pred_rows[i].first;
        e.n = (u32)ch.n;
        e.pairs = reinterpret_cast<uint2*>(ch.pairs.ptr);
        e.ynum = ch.ynum ? static_cast<double*>(ch.ynum->p) : nullptr;
        const bool xok = ps.xtab && ps.tab_cshift == cshift;
        rebuild[i][0] = ps.xtab ? !xok : !ps.x_tried;
        rebuild[i][1] = !ps.ytab && !ps.y_tried;
        if (xok) { e.xtab = static_cast<u32*>(ps.xtab->p); e.xtab_min = ps.xtab_min; e.xtab_range = ps.xtab_range; e.cshift = cshift; }
        if (xok && ps.xkey && ps.xkey_version == ctx->num_version && ctx->numv_version == ctx->num_version && ctx->n_ids) {
            e.xkey = static_cast<u32*>(ps.xkey->p);
            P.numv = static_cast<const double*>(ctx->numv->p);
            P.n_numv = (u32)ctx->h_numv.size();
        } else ps.xkey.reset();
        if (ps.ytab) { e.ytab = static_cast<u32*>(ps.ytab->p); e.ytab_min = ps.ytab_min; e.ytab_range = ps.ytab_range; }
    }
    timer_begin(ctx, F_OTHER);
    launch_segment_split(P, ctx->n_sms, ctx->st);
    timer_end(ctx);
    ctx->stats.kernel_launches++;
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(ctrl_read(ctx));
    const u32 uoff = ctrl_alloc(ctx, 2 * MAXP);
    bool any_touched = false;
    std::vector<char> touched(2 * k, 0);
    std::vector<int> chunk_of(k, -1);
    for (u32 i = 0; i < k; i++) {
        const u32* h = ctx->h_ctrl + off + i * SPLIT_WORDS;
        PredSlice& ps = ctx->index[sg.pred_rows[i].first];
        SliceChunk& ch = chs[i];
        if (h[SPLIT_CURSOR] != ch.n) return fail(ctx, KB_E_CUDA, "index maintenance: predicate %u has %u rows, its profile said %llu", sg.pred_rows[i].first,
                                                  h[SPLIT_CURSOR], (unsigned long long)ch.n);
        ch.xmin = ~h[SPLIT_XMIN]; ch.ymin = ~h[SPLIT_YMIN]; ch.xmax = h[SPLIT_XMAX]; ch.ymax = h[SPLIT_YMAX];
        if (ch.ynum && h[SPLIT_NNUM] > 0) ch.ynum_version = ctx->num_version;
        else { ch.ynum.reset(); ps.xkey.reset(); }
        ps.xmin = std::min(ps.xmin, ch.xmin); ps.ymin = std::min(ps.ymin, ch.ymin);
        ps.xmax = std::max(ps.xmax, ch.xmax); ps.ymax = std::max(ps.ymax, ch.ymax);
        chunk_of[i] = (int)ps.chunks.size();
        ps.chunks.push_back(ch);
        ps.n += ch.n;
        if (ps.chunks.size() > 1) { ps.xoff.reset(); ps.xval.reset(); ps.yoff.reset(); ps.yval.reset(); }  // the directories describe one chunk
        if (h[SPLIT_XDUP]) { ps.x_unique = false; ps.xtab.reset(); ps.xkey.reset(); }  // a subject occurs twice
        if (h[SPLIT_YDUP]) { ps.y_unique = false; ps.ytab.reset(); }
        if (h[SPLIT_XOUT] && ps.xtab) rebuild[i][0] = true;  // a key outside the table: rebuild it over every chunk, with new headroom
        if (h[SPLIT_YOUT] && ps.ytab) rebuild[i][1] = true;
    }
    for (u32 i = 0; i < k; i++) {
        PredSlice& ps = ctx->index[sg.pred_rows[i].first];
        for (u32 y = 0; y < 2; y++) {
            if (!rebuild[i][y]) continue;
            if (!any_touched) { KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + uoff, 0, 2 * MAXP * sizeof(u32), ctx->st)); any_touched = true; }
            Buf& tab = y ? ps.ytab : ps.xtab;
            tab.reset();  // slice_table_update sees no table: a rebuild over all chunks (the new one included)
            if (y) ps.y_tried = false; else ps.x_tried = false;
            bool t = false;
            KB_TRY(slice_table_update(ctx, ps, y, chunk_of[i], cshift, uoff + 2 * i + y, /*full_build=*/false, &t));
            touched[2 * i + y] = t ? 1 : 0;
        }
    }
    if (any_touched) {
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        for (u32 i = 0; i < k; i++) {
            PredSlice& ps = ctx->index[sg.pred_rows[i].first];
            if (touched[2 * i] && ctx->h_ctrl[uoff + 2 * i]) { ps.x_unique = false; ps.xtab.reset(); }
            if (touched[2 * i + 1] && ctx->h_ctrl[uoff + 2 * i + 1]) { ps.y_unique = false; ps.ytab.reset(); }
        }
    }
    return KB_OK;
}

// full_build: kb_store_build_index indexes the store segment by segment
static kb_status index_add_segment(kb_ctx* ctx, size_t seg_idx, bool full_build, bool* indexable) {
    *indexable = true;
    Segment sg = ctx->segs[seg_idx];
    if (sg.n == 0) return KB_OK;
    static const bool split_ok = !(getenv("KOLIBRIE_INDEX_SPLIT") && getenv("KOLIBRIE_INDEX_SPLIT")[0] == '0');
    if (split_ok && !full_build && sg.has_stats && sg.stats_world == ctx->shard_world && sg.has_preds && !sg.preds_overflow &&
        sg.pred_rows.size() <= MAXP) {
        size_t n_new = 0;
        for (auto& pr : sg.pred_rows) n_new += ctx->index.count(pr.first) ? 0 : 1;
        if (ctx->index.size() + n_new <= 4096) {
            u32 cshift = 0;  // subject-sharded store: compact the subject keys (see compact_key)
            bool sharded = ctx->shard_world > 1 && (ctx->shard_world & (ctx->shard_world - 1)) == 0;
            for (auto& g : ctx->segs) if (g.n && g.has_stats && !g.sharded_ok) sharded = false;
            if (sharded) while ((1u << cshift) < ctx->shard_world) cshift++;
            return index_add_segment_split(ctx, sg, cshift);
        }
    }
    // 1. distinct predicates of the segment
    const u32 set_slots = 8192;
    Buf set;
    KB_TRY(alloc_buf(ctx, set_slots * sizeof(u32), &set));
    KB_CUDA(ctx, cudaMemsetAsync(set->p, 0xFF, set_slots * sizeof(u32), ctx->st));
    const u32 off = ctrl_alloc(ctx, 4);
    KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, 4 * sizeof(u32), ctx->st));
    timer_begin(ctx, F_OTHER);
    launch_distinct(sg.p.ptr, (u32)sg.n, static_cast<u32*>(set->p), set_slots, ctx->ctrl + off, ctx->n_sms, ctx->st);
    timer_end(ctx);
    std::vector<u32> hset(set_slots);
    KB_CUDA(ctx, cudaMemcpyAsync(hset.data(), set->p, set_slots * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
    KB_TRY(ctrl_read(ctx));
    std::vector<u32> preds;
    for (u32 v : hset) if (v != EMPTY32) preds.push_back(v);
    std::sort(preds.begin(), preds.end());
    {
        std::set<u32> all(preds.begin(), preds.end());
        for (auto& kv : ctx->index) all.insert(kv.first);
        if (ctx->h_ctrl[off] || all.size() > 4096) { *indexable = false; return KB_OK; }  // too many predicates: keep scanning
    }
    if (!sg.has_stats || sg.stats_world != ctx->shard_world) { KB_TRY(segment_stats(ctx, &ctx->segs[seg_idx])); sg = ctx->segs[seg_idx]; }
    u32 cshift = 0;  // subject-sharded store: compact the subject keys (see compact_key)
    {
        bool sharded = ctx->shard_world > 1 && (ctx->shard_world & (ctx->shard_world - 1)) == 0;
        for (auto& g : ctx->segs) if (g.n && g.has_stats && !g.sharded_ok) sharded = false;
        if (sharded) while ((1u << cshift) < ctx->shard_world) cshift++;
    }
    // 2. one fused scan of THIS segment per 8 predicates, pair output, shrunk to a chunk; id ranges of both halves
    const std::vector<Segment> one{sg};
    for (size_t b = 0; b < preds.size(); b += MAXP) {
        const u32 k = (u32)std::min<size_t>(MAXP, preds.size() - b);
        kb_pattern pats[MAXP];
        for (u32 i = 0; i < k; i++) { pats[i].s = kb_term{1, 0}; pats[i].p = kb_term{0, preds[b + i]}; pats[i].o = kb_term{1, 1}; }
        std::vector<std::unique_ptr<kb_rel>> rels;
        std::vector<FilterProg> none;
        KB_TRY(scan_impl(ctx, one, pats, k, none, /*use_index=*/false, false, true, &rels));
        const u32 soff = ctrl_alloc(ctx, 4 * MAXP);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + soff, 0, 4 * MAXP * sizeof(u32), ctx->st));
        for (u32 i = 0; i < k; i++) KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + soff + 4 * i, 0xFF, 2 * sizeof(u32), ctx->st));
        std::vector<int> chunk_of(k, -1);
        for (u32 i = 0; i < k; i++) {
            if (rels[i]->n == 0) continue;
            PredSlice& ps = ctx->index[preds[b + i]];
            SliceChunk ch;
            ch.tag = sg.tag;
            ch.n = rels[i]->n;
            KB_TRY(alloc_col(ctx, 2 * ch.n, &ch.pairs));
            KB_CUDA(ctx, cudaMemcpyAsync(ch.pairs.ptr, rels[i]->cols[0].ptr, ch.n * sizeof(uint2), cudaMemcpyDeviceToDevice, ctx->st));
            launch_pair_minmax(reinterpret_cast<const uint2*>(ch.pairs.ptr), (u32)ch.n, ctx->ctrl + soff + 4 * i, ctx->n_sms, ctx->st);
            ctx->stats.kernel_launches++;
            chunk_of[i] = (int)ps.chunks.size();
            ps.chunks.push_back(ch);
            ps.n += ch.n;
            if (ps.chunks.size() > 1) { ps.xoff.reset(); ps.xval.reset(); ps.yoff.reset(); ps.yval.reset(); }  // the directories describe one chunk
            if (!full_build) ps.xkey.reset();  // (kept in table order by the full build only)
        }
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        // 3. persistent tables (inserted in place; a duplicate key or a key outside the table ends / rebuilds it) and the typed literal
        //    column of the new chunk: the f64 value of every object, so that FILTER(?o <cmp> c) reads it sequentially instead of
        //    gathering num_or0[object] at random
        const u32 uoff = ctrl_alloc(ctx, 2 * MAXP);
        const u32 noff = ctrl_alloc(ctx, MAXP);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + uoff, 0, 2 * MAXP * sizeof(u32), ctx->st));
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + noff, 0, MAXP * sizeof(u32), ctx->st));
        std::vector<char> touched(2 * k, 0);
        for (u32 i = 0; i < k; i++) {
            if (chunk_of[i] < 0) continue;
            PredSlice& ps = ctx->index[preds[b + i]];
            {
                SliceChunk& ch = ps.chunks[chunk_of[i]];
                ch.xmin = ctx->h_ctrl[soff + 4 * i]; ch.ymin = ctx->h_ctrl[soff + 4 * i + 1];
                ch.xmax = ctx->h_ctrl[soff + 4 * i + 2]; ch.ymax = ctx->h_ctrl[soff + 4 * i + 3];
                ps.xmin = std::min(ps.xmin, ch.xmin); ps.ymin = std::min(ps.ymin, ch.ymin);
                ps.xmax = std::max(ps.xmax, ch.xmax); ps.ymax = std::max(ps.ymax, ch.ymax);
            }
            for (u32 y = 0; y < 2; y++) {
                bool t = false;
                KB_TRY(slice_table_update(ctx, ps, y, chunk_of[i], cshift, uoff + 2 * i + y, full_build, &t));
                touched[2 * i + y] = t ? 1 : 0;
            }
            if (ctx->n_ids) {
                SliceChunk& ch = ps.chunks[chunk_of[i]];
                KB_TRY(alloc_buf(ctx, ch.n * sizeof(double), &ch.ynum));
                launch_pair_numcol(reinterpret_cast<const uint2*>(ch.pairs.ptr), (u32)ch.n, numtab(ctx), static_cast<double*>(ch.ynum->p), ctx->ctrl + noff + i,
                                   ctx->n_sms, ctx->st);
                ctx->stats.kernel_launches++;
            }
        }
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(ctrl_read(ctx));
        for (u32 i = 0; i < k; i++) {
            if (chunk_of[i] < 0) continue;
            PredSlice& ps = ctx->index[preds[b + i]];
            SliceChunk& ch = ps.chunks[chunk_of[i]];
            if (ch.ynum && ctx->h_ctrl[noff + i] > 0) ch.ynum_version = ctx->num_version;
            else ch.ynum.reset();
            if (touched[2 * i] && ctx->h_ctrl[uoff + 2 * i]) { ps.x_unique = false; ps.xtab.reset(); }      // a subject occurs twice
            if (touched[2 * i + 1] && ctx->h_ctrl[uoff + 2 * i + 1]) { ps.y_unique = false; ps.ytab.reset(); }
        }
    }
    return KB_OK;
}

// eviction of the segment(s) tagged `tag`: their chunks leave the slices, their keys leave the persistent tables
static kb_status index_evict_tag(kb_ctx* ctx, u64 tag) {
    ClearParams C{};
    std::vector<SliceChunk> dying;  // kept until the clears are queued: their buffers are released stream-ordered behind them
    auto flush = [&]() {
        if (C.k) { launch_clear_chunks(C, ctx->n_sms, ctx->st); ctx->stats.kernel_launches++; }
        C.k = 0;
    };
    for (auto it = ctx->index.begin(); it != ctx->index.end();) {
        PredSlice& ps = it->second;
        bool hit = false;
        for (size_t c = 0; c < ps.chunks.size();) {
            SliceChunk& ch = ps.chunks[c];
            if (ch.tag != tag) { c++; continue; }
            hit = true;
            if ((ps.xtab || ps.ytab) && ch.n) {
                ClearEntry& e = C.e[C.k++];
                e = ClearEntry{};
                e.pairs = reinterpret_cast<const uint2*>(ch.pairs.ptr);
                e.n = (u32)ch.n;
                if (ps.xtab) { e.xtab = static_cast<u32*>(ps.xtab->p); e.xtab_min = ps.xtab_min; e.xtab_range = ps.xtab_range; e.cshift = ps.tab_cshift; }
                if (ps.ytab) { e.ytab = static_cast<u32*>(ps.ytab->p); e.ytab_min = ps.ytab_min; e.ytab_range = ps.ytab_range; }
                if (C.k == CLEAR_MAX) flush();
            }
            ps.n -= ch.n;
            dying.push_back(ch);
            ps.chunks.erase(ps.chunks.begin() + c);
            ps.xoff.reset(); ps.xval.reset(); ps.yoff.reset(); ps.yval.reset();  // (xkey stays: its slots are only read where xtab holds a key)
        }
        if (hit) {  // the slice's id ranges shrink to the surviving chunks': a long-running window does not walk its whole past
            ps.xmin = ps.ymin = 0xFFFFFFFFu;
            ps.xmax = ps.ymax = 0u;
            for (auto& ch : ps.chunks) {
                ps.xmin = std::min(ps.xmin, ch.xmin); ps.ymin = std::min(ps.ymin, ch.ymin);
                ps.xmax = std::max(ps.xmax, ch.xmax); ps.ymax = std::max(ps.ymax, ch.ymax);
            }
        }
        if (ps.chunks.empty()) it = ctx->index.erase(it);
        else ++it;
    }
    flush();
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

// ---- changes to the store: the only code that writes ctx->segs, n_triples, store_version, the hint sets and the index
static bool index_maintainable(const kb_ctx* ctx) {
    return ctx->index_maintain && ctx->index_version == ctx->store_version && !ctx->index.empty();
}
// a new store version: everything keyed to the old one is void, and what the star-join builds learnt about its predicates is forgotten
static void bump_version(kb_ctx* ctx) {
    ctx->store_version++;
    ctx->multi_valued.clear();
    ctx->single_valued.clear();
}
static void drop_index(kb_ctx* ctx) {
    ctx->index.clear();
    ctx->index_version = ~0ull;
}

void store_replace(kb_ctx* ctx, std::vector<Segment> segs) {
    ctx->segs = std::move(segs);
    ctx->n_triples = 0;
    for (auto& sg : ctx->segs) ctx->n_triples += sg.n;
    bump_version(ctx);
    drop_index(ctx);  // a replaced store: nothing to maintain
}

kb_status store_add_device_segment(kb_ctx* ctx, Segment& sg, bool keep_index) {
    if (keep_index && sg.n && !sg.has_stats) KB_TRY(segment_stats(ctx, &sg));
    const bool maintain = keep_index && index_maintainable(ctx);
    ctx->segs.push_back(sg);
    ctx->n_triples += sg.n;
    bump_version(ctx);
    if (maintain) {
        // the index stays alive across the mutation: the new segment becomes one more chunk of every predicate slice it touches and
        // its keys are inserted into the persistent tables in place (an RSP window slide keeps the one-kernel index path)
        bool indexable = true;
        const kb_status rc = index_add_segment(ctx, ctx->segs.size() - 1, /*full_build=*/false, &indexable);
        if (rc == KB_OK && indexable) { ctx->index_version = ctx->store_version; return KB_OK; }
        drop_index(ctx);
        return rc;
    }
    drop_index(ctx);  // the predicate-partitioned index describes the previous store version
    return KB_OK;
}

bool store_evict_tag(kb_ctx* ctx, u64 tag, bool keep_index) {
    bool found = false;
    for (size_t i = 0; i < ctx->segs.size();) {
        if (ctx->segs[i].tag == tag) {
            ctx->n_triples -= ctx->segs[i].n;
            ctx->segs.erase(ctx->segs.begin() + i);
            found = true;
        } else i++;
    }
    const bool maintain = keep_index && index_maintainable(ctx);
    bump_version(ctx);
    if (maintain && index_evict_tag(ctx, tag) == KB_OK) ctx->index_version = ctx->store_version;
    else drop_index(ctx);
    return found;
}
}  // namespace kb

extern "C" {

// ------------------------------------------------------------------ store
static kb_status store_add_segment(kb_ctx* ctx, const u32* s, const u32* p, const u32* o, u64 n, u64 tag, cudaMemcpyKind kind) {
    if (n && (!s || !p || !o)) return kb::fail(ctx, KB_E_INVALID, "NULL column pointer");
    if (ctx->n_triples + n >= 0xFFFFFFF0ull) return kb::fail(ctx, KB_E_LIMIT, "store would exceed 2^32-16 triples");
    kb::Segment sg;
    sg.tag = tag;
    sg.n = n;
    KB_TRY(kb::alloc_col(ctx, n, &sg.s));
    KB_TRY(kb::alloc_col(ctx, n, &sg.p));
    KB_TRY(kb::alloc_col(ctx, n, &sg.o));
    if (n) {
        static const bool trace = getenv("KOLIBRIE_TRACE") != nullptr;
        const auto t0 = std::chrono::steady_clock::now();
        // one stream, back to back: three concurrent H2D copies on three streams were several times SLOWER at 16 MB per column
        // and no faster at 4 MB
        KB_CUDA(ctx, cudaMemcpyAsync(sg.s.ptr, s, n * sizeof(u32), kind, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(sg.p.ptr, p, n * sizeof(u32), kind, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(sg.o.ptr, o, n * sizeof(u32), kind, ctx->st));
        if (trace) KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
        const auto t1 = std::chrono::steady_clock::now();
        if (kind == cudaMemcpyHostToDevice) ctx->stats.h2d_bytes += 3 * n * sizeof(u32);
        // the statistics pass ends with a read-back on the same stream: when it returns the copies are done too (the caller's
        // buffers are borrowed for this call only)
        KB_TRY(kb::segment_stats(ctx, &sg));
        if (trace)
            fprintf(stderr, "[kb trace] segment of %llu triples: copies %.3f ms, statistics %.3f ms\n", (unsigned long long)n,
                    std::chrono::duration<double, std::milli>(t1 - t0).count(),
                    std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count());
    }
    return kb::store_add_device_segment(ctx, sg);
}

kb_status kb_store_clear(kb_ctx* ctx) {
    KB_ENTER(ctx);
    kb::store_replace(ctx, {});
    return KB_OK;
}
// a load empties the store first: a rejected load leaves it empty, at a new version
kb_status kb_store_load(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n) {
    KB_ENTER(ctx);
    kb::store_replace(ctx, {});
    return store_add_segment(ctx, s, p, o, n, 0, cudaMemcpyHostToDevice);
}
kb_status kb_store_load_device(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n) {
    KB_ENTER(ctx);
    kb::store_replace(ctx, {});
    return store_add_segment(ctx, s, p, o, n, 0, cudaMemcpyDeviceToDevice);
}
kb_status kb_store_append(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t tag) {
    KB_ENTER(ctx);
    return store_add_segment(ctx, s, p, o, n, tag, cudaMemcpyHostToDevice);
}
kb_status kb_store_append_device(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n, uint64_t tag) {
    KB_ENTER(ctx);
    return store_add_segment(ctx, s, p, o, n, tag, cudaMemcpyDeviceToDevice);
}
kb_status kb_store_evict(kb_ctx* ctx, uint64_t tag) {
    KB_ENTER(ctx);
    const bool found = kb::store_evict_tag(ctx, tag, /*keep_index=*/true);
    return found ? KB_OK : kb::fail(ctx, KB_E_NOT_FOUND, "no segment with tag %llu", (unsigned long long)tag);
}
kb_status kb_set_use_index(kb_ctx* ctx, int enabled) {
    if (!ctx) return KB_E_INVALID;
    ctx->use_index = enabled != 0;
    return KB_OK;
}

kb_status kb_store_build_index(kb_ctx* ctx, uint32_t* n_predicates, double* build_ms) {
    KB_ENTER(ctx);
    if (n_predicates) *n_predicates = 0;
    if (build_ms) *build_ms = 0.0;
    kb::drop_index(ctx);
    if (ctx->n_triples == 0) return KB_OK;
    kb::ScopedEvent e0, e1;
    cudaEventRecord(e0, ctx->st);
    for (auto& sg : ctx->segs) if (sg.n && (!sg.has_stats || sg.stats_world != ctx->shard_world)) KB_TRY(kb::segment_stats(ctx, &sg));
    for (size_t g = 0; g < ctx->segs.size(); g++) {
        bool indexable = true;
        const kb_status rc = kb::index_add_segment(ctx, g, /*full_build=*/true, &indexable);
        if (rc != KB_OK || !indexable) {
            ctx->index.clear();
            if (rc != KB_OK) return rc;
            return KB_OK;  // too many predicates: keep scanning (n_predicates = 0)
        }
    }
    // value ranks in table order for subject tables whose slice is numeric: the table-mode probe reads FILTER operands sequentially
    for (auto& kv : ctx->index) {
        kb::PredSlice& ps = kv.second;
        if (!ps.xtab || !ctx->n_ids || !ps.typed(ctx->num_version)) continue;
        KB_TRY(kb::build_rank_column(ctx, ps));
    }
    // key-grouped directories (counting sort by the dense key) for the columns that did not get a direct table
    for (auto& kv : ctx->index) {
        kb::PredSlice& ps = kv.second;
        const kb::SliceChunk* ch = ps.single();
        if (!ch || ch->n == 0) continue;
        for (u32 y = 0; y < 2; y++) {
            if (y ? (bool)ps.ytab : (bool)ps.xtab) continue;  // unique column: the direct table answers the lookup
            const u32 lo = y ? ps.ymin : ps.xmin, hi = y ? ps.ymax : ps.xmax;
            const u64 range = (u64)hi - lo + 1;
            if (range > std::max<u64>(8 * ps.n, 1ull << 20) || range > (1ull << 28)) continue;  // sparse ids: no directory
            kb::Buf off, val, cursor, scratch;
            KB_TRY(kb::alloc_buf(ctx, (range + 1) * sizeof(u32), &off));
            KB_TRY(kb::alloc_buf(ctx, ch->n * sizeof(u32), &val));
            KB_TRY(kb::alloc_buf(ctx, range * sizeof(u32), &cursor));
            KB_TRY(kb::alloc_buf(ctx, ((range + 1) / 2048 + 4) * sizeof(u32), &scratch));
            KB_CUDA(ctx, cudaMemsetAsync(off->p, 0, (range + 1) * sizeof(u32), ctx->st));
            const uint2* pairs = reinterpret_cast<const uint2*>(ch->pairs.ptr);
            kb::launch_csr_count_pairs(pairs, y, (u32)ch->n, lo, static_cast<u32*>(off->p), ctx->n_sms, ctx->st);
            kb::launch_exclusive_scan_u32(static_cast<u32*>(off->p), (u32)range + 1, static_cast<u32*>(scratch->p), ctx->st);
            KB_CUDA(ctx, cudaMemcpyAsync(cursor->p, off->p, range * sizeof(u32), cudaMemcpyDeviceToDevice, ctx->st));
            kb::launch_csr_fill_pairs(pairs, y, (u32)ch->n, lo, static_cast<u32*>(cursor->p), static_cast<u32*>(val->p), ctx->n_sms, ctx->st);
            ctx->stats.kernel_launches += 5;
            if (y) { ps.yoff = off; ps.yval = val; ps.ycsr_min = lo; ps.ycsr_range = (u32)range; }
            else { ps.xoff = off; ps.xval = val; ps.xcsr_min = lo; ps.xcsr_range = (u32)range; }
        }
    }
    KB_CUDA(ctx, cudaGetLastError());
    cudaEventRecord(e1, ctx->st);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    ctx->index_version = ctx->store_version;
    if (n_predicates) *n_predicates = (uint32_t)ctx->index.size();
    if (build_ms) *build_ms = ms;
    return KB_OK;
}

kb_status kb_store_size(kb_ctx* ctx, uint64_t* n, uint32_t* n_seg) {
    if (!ctx) return KB_E_INVALID;
    if (n) *n = ctx->n_triples;
    if (n_seg) *n_seg = (uint32_t)ctx->segs.size();
    return KB_OK;
}

kb_status kb_store_delete(kb_ctx* ctx, const uint32_t* s, const uint32_t* p, const uint32_t* o, uint64_t n) {
    KB_ENTER(ctx);
    if (n == 0 || ctx->n_triples == 0) return KB_OK;
    if (!s || !p || !o) return kb::fail(ctx, KB_E_INVALID, "NULL column pointer");
    // 1. the delete set (96-bit keys), 2. mark matching triples by overwriting a copy of the predicate column with KB_ID_NONE,
    // 3. rescan every segment with (?s ?p ?o) — a row whose predicate is KB_ID_NONE can never equal a real constant, and the
    //    pattern's pushed-down filter NE_ID drops it.
    const u32 set_slots = kb::pow2_at_least(n * 2);
    kb::Buf set, ds, dp, dob;
    KB_TRY(kb::alloc_buf(ctx, (size_t)set_slots * sizeof(uint4), &set));
    KB_TRY(kb::alloc_buf(ctx, n * sizeof(u32), &ds));
    KB_TRY(kb::alloc_buf(ctx, n * sizeof(u32), &dp));
    KB_TRY(kb::alloc_buf(ctx, n * sizeof(u32), &dob));
    KB_CUDA(ctx, cudaMemsetAsync(set->p, 0, (size_t)set_slots * sizeof(uint4), ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(ds->p, s, n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(dp->p, p, n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    KB_CUDA(ctx, cudaMemcpyAsync(dob->p, o, n * sizeof(u32), cudaMemcpyHostToDevice, ctx->st));
    const u32 off = kb::ctrl_alloc(ctx, 4);
    kb::launch_set_insert(static_cast<uint4*>(set->p), set_slots, (const u32*)ds->p, (const u32*)dp->p, 0u, (const u32*)dob->p, (u32)n,
                          ctx->ctrl + off, ctx->n_sms, ctx->st);
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    kb_pattern pt{{1, 0}, {1, 1}, {1, 2}};
    kb::FilterProg keep;
    kb_filter_op ne{};
    ne.op = KB_F_NE_ID; ne.slot = 1; ne.id = KB_ID_NONE;  // true for every bound predicate; a marked one reads as unbound: false
    keep.ops.push_back(ne);
    const std::vector<kb::FilterProg> pd{keep};
    // the new segments are built aside: the store changes only when all of them are (a failure leaves it as it was)
    std::vector<kb::Segment> kept;
    for (auto& sg : ctx->segs) {
        kb::Segment marked = sg;
        if (sg.n) {
            KB_TRY(kb::alloc_col(ctx, sg.n, &marked.p));
            kb::launch_delete_mark(sg.s.ptr, sg.p.ptr, sg.o.ptr, (u32)sg.n, static_cast<const uint4*>(set->p), set_slots, marked.p.ptr,
                                   ctx->n_sms, ctx->st);
        }
        // rescan this one segment
        std::vector<std::unique_ptr<kb_rel>> rels;
        KB_TRY(kb::scan_impl(ctx, {marked}, &pt, 1, pd, /*use_index=*/false, false, false, &rels));
        kb::Segment ns;
        ns.tag = sg.tag;
        ns.n = rels[0]->n;
        ns.s = rels[0]->cols[0]; ns.p = rels[0]->cols[1]; ns.o = rels[0]->cols[2];
        kept.push_back(ns);
    }
    kb::store_replace(ctx, std::move(kept));
    return KB_OK;
}

kb_status kb_store_download(kb_ctx* ctx, uint32_t* s, uint32_t* p, uint32_t* o, uint64_t cap, uint64_t* n) {
    KB_ENTER(ctx);
    if (n) *n = ctx->n_triples;
    if (cap < ctx->n_triples) return kb::fail(ctx, KB_E_LIMIT, "buffer holds %llu triples, store has %llu", (unsigned long long)cap, (unsigned long long)ctx->n_triples);
    u64 off = 0;
    for (auto& sg : ctx->segs) {
        if (!sg.n) continue;
        KB_CUDA(ctx, cudaMemcpyAsync(s + off, sg.s.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(p + off, sg.p.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        KB_CUDA(ctx, cudaMemcpyAsync(o + off, sg.o.ptr, sg.n * sizeof(u32), cudaMemcpyDeviceToHost, ctx->st));
        off += sg.n;
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    return KB_OK;
}

}  // extern "C"
