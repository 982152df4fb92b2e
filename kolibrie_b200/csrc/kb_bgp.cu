// kb_bgp.cu — kb_bgp_execute's component route: every BGP that is not a star of at most KB_MAX_PATTERNS patterns. The semantics are
// in include/kolibrie_b200.h; here:
//   scans              scan_store in fused groups of at most MAXP patterns (index lookups with a valid index)
//   plan               components, GYO and the join order: kb_bgp_plan.hpp (host C++, shared with a CPU test driver)
//   domain reduction   components of three or more patterns. For every variable v that two or more of the component's patterns hold,
//                      D(v) is a bitmap over v's id range (the intersection of the segment profiles' ranges of the positions v
//                      takes). K1 bgp_reduce_kernel streams every relation once: a row survives iff each of its reduced variables has
//                      its bit in D(v) (ids beyond the bitmap pass); survivors are compacted with a warp ballot and one atomic per
//                      warp, and their values atomicOr-ed into the relation's own bitmap of v. K2 bgp_and_kernel ANDs those bitmaps into
//                      the next D(v). The first pass only marks (no row is dropped, nothing is written). Rounds repeat until no
//                      relation shrinks, at most one per pattern of the component. Dropping rows that join with nothing leaves the bag
//                      as it was.
//   joins              hash_join_impl inside a component in the planned order, then the components' cross joins, smallest first;
//                      the post-FILTER is fused into the last join
// Byte model of one filtering round over relation k (c_k columns, n_k rows in, n'_k out): 4·c_k·n_k read, 4·c_k·n'_k written, one bit
// probe and one atomicOr per surviving row and reduced variable (bitmaps: about 1 MB per variable at 10 M triples, L2-resident).
#include <algorithm>

#include "kb_bgp_plan.hpp"
#include "kb_internal.hpp"

namespace kb {
namespace {

constexpr int RED_MAXR = KB_BGP_MAX_PATTERNS;
constexpr int RED_THREADS = 256;
constexpr u64 RED_MAX_BITS = 1ull << 28;  // 32 MB per bitmap at most; ids beyond it pass

struct RedRel {
    const u32* in[3];
    u32* out[3];
    u32 n_cols, n;
    u64 base;           // first flat row of the relation: a multiple of 32, so a warp never spans two relations
    u32 n_red;          // columns checked against a bitmap
    u32 rcol[3];        // which columns
    u32 lo[3], nbits[3];  // the bitmap of rcol[j] covers ids [lo, lo + nbits)
    const u32* dom[3];  // D(v)
    u32* mark[3];       // this relation's bitmap of its survivors' values of v
};
struct ReduceParams {
    RedRel r[RED_MAXR];
    u32 n_rel;
    u32 filter;         // 0: mark every row (first pass); 1: drop rejected rows, write the survivors
    u64 total;          // flat rows, a multiple of 32
    u32* count;         // [n_rel] survivors
};
struct AndVar {
    u32* dom;
    u32 words, n_src;
    const u32* src[RED_MAXR];
};
struct AndParams {
    AndVar v[KB_MAX_COLS];
};

__device__ __forceinline__ u32 pick3(const u32 (&v)[3], u32 c) { return c == 0u ? v[0] : c == 1u ? v[1] : v[2]; }

__global__ void __launch_bounds__(RED_THREADS) bgp_reduce_kernel(const __grid_constant__ ReduceParams P) {
    const u32 lane = threadIdx.x & 31u;
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < P.total; g += (u64)gridDim.x * blockDim.x) {
        u32 r = 0;  // warp-uniform (bases and the stride are multiples of 32)
        while (r + 1 < P.n_rel && g >= P.r[r + 1].base) r++;
        const RedRel& R = P.r[r];
        const u64 i = g - R.base;
        const bool valid = i < R.n;
        u32 v[3] = {0u, 0u, 0u};
#pragma unroll
        for (u32 c = 0; c < 3; c++)
            if (valid && c < R.n_cols) v[c] = __ldg(R.in[c] + i);
        bool keep = valid;
        if (P.filter) {
#pragma unroll
            for (u32 j = 0; j < 3; j++) {
                if (j >= R.n_red) break;
                const u32 d = pick3(v, R.rcol[j]) - R.lo[j];
                if (keep && d < R.nbits[j]) keep = (__ldg(R.dom[j] + (d >> 5)) >> (d & 31u)) & 1u;
            }
        }
        if (keep) {
#pragma unroll
            for (u32 j = 0; j < 3; j++) {
                if (j >= R.n_red) break;
                const u32 d = pick3(v, R.rcol[j]) - R.lo[j];
                if (d < R.nbits[j]) atomicOr(R.mark[j] + (d >> 5), 1u << (d & 31u));
            }
        }
        if (!P.filter) continue;
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (!b) continue;
        u32 at = 0;
        if (lane == (u32)__ffs(b) - 1u) at = atomicAdd(P.count + r, (u32)__popc(b));
        at = __shfl_sync(0xffffffffu, at, __ffs(b) - 1);
        if (keep) {
            const u32 o = at + (u32)__popc(b & ((1u << lane) - 1u));
#pragma unroll
            for (u32 c = 0; c < 3; c++)
                if (c < R.n_cols) R.out[c][o] = v[c];
        }
    }
}

__global__ void __launch_bounds__(256) bgp_and_kernel(const __grid_constant__ AndParams P) {
    const AndVar& V = P.v[blockIdx.y];
    for (u32 w = blockIdx.x * blockDim.x + threadIdx.x; w < V.words; w += gridDim.x * blockDim.x) {
        u32 x = 0xFFFFFFFFu;
        for (u32 s = 0; s < V.n_src; s++) x &= __ldg(V.src[s] + w);
        V.dom[w] = x;
    }
}

struct RedVar {
    u32 slot;
    u32 lo, nbits, words;
    u32* dom;
    std::vector<std::pair<u32, u32*>> marks;  // (pattern, its bitmap of this variable)
};

// Domain reduction of the component `comp` in place (rels[k] replaced by its survivors). *rounds = filtering rounds run.
kb_status reduce_component(kb_ctx* ctx, const std::vector<u32>& comp, const std::vector<std::vector<u32>>& pv,
                           const std::vector<std::vector<u32>>& psrc, std::vector<std::unique_ptr<kb_rel>>* rels, u32* rounds,
                           kb_bgp_plan_info* info) {
    *rounds = 0;
    u32 smin[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, smax[3] = {0, 0, 0};  // id range of each position over the store
    for (auto& sg : ctx->segs) {
        if (sg.n == 0) continue;
        if (!sg.has_stats) KB_TRY(segment_stats(ctx, &sg));
        for (int c = 0; c < 3; c++) { smin[c] = std::min(smin[c], sg.cmin[c]); smax[c] = std::max(smax[c], sg.cmax[c]); }
    }
    std::vector<RedVar> vars;
    for (u32 k : comp)
        for (size_t i = 0; i < pv[k].size(); i++) {
            const u32 s = pv[k][i];
            auto it = std::find_if(vars.begin(), vars.end(), [&](const RedVar& x) { return x.slot == s; });
            if (it == vars.end()) { vars.push_back(RedVar{s, 0u, 0xFFFFFFFFu, 0u, nullptr, {}}); it = vars.end() - 1; }
            it->lo = std::max(it->lo, smin[psrc[k][i]]);
            it->nbits = std::min(it->nbits, smax[psrc[k][i]]);  // (the upper end until the loop below)
            it->marks.push_back({k, nullptr});
        }
    u64 words = 0;
    std::vector<RedVar> red;
    for (auto& v : vars) {
        if (v.marks.size() < 2 || v.lo > v.nbits) continue;  // held by one pattern, or no id can satisfy every position it takes
        v.nbits = (u32)std::min<u64>((u64)v.nbits - v.lo + 1, RED_MAX_BITS);
        v.words = (v.nbits + 31u) / 32u;
        words += (u64)v.words * (1 + v.marks.size());
        red.push_back(v);
    }
    if (red.empty()) return KB_OK;
    Buf bits;
    KB_TRY(alloc_buf(ctx, words * sizeof(u32), &bits));
    u32* cursor = static_cast<u32*>(bits->p);
    u32* marks_begin = nullptr;
    for (auto& v : red) { v.dom = cursor; cursor += v.words; }
    marks_begin = cursor;
    for (auto& v : red) for (auto& m : v.marks) { m.second = cursor; cursor += v.words; }
    const size_t mark_bytes = (size_t)(cursor - marks_begin) * sizeof(u32);

    ReduceParams P{};
    std::vector<u32> members;  // patterns in the launch: those with a reduced variable
    for (u32 k : comp) {
        RedRel& R = P.r[members.size()];
        const kb_rel& rel = *(*rels)[k];
        for (auto& v : red)
            for (auto& m : v.marks)
                if (m.first == k) {
                    R.rcol[R.n_red] = (u32)rel.col_of(v.slot);
                    R.lo[R.n_red] = v.lo;
                    R.nbits[R.n_red] = v.nbits;
                    R.dom[R.n_red] = v.dom;
                    R.mark[R.n_red] = m.second;
                    R.n_red++;
                }
        if (R.n_red) members.push_back(k);
        else R = RedRel{};
    }
    P.n_rel = (u32)members.size();
    AndParams A{};
    for (size_t j = 0; j < red.size(); j++) {
        A.v[j].dom = red[j].dom;
        A.v[j].words = red[j].words;
        for (auto& m : red[j].marks) A.v[j].src[A.v[j].n_src++] = m.second;
    }
    u32 max_words = 0;
    for (auto& v : red) max_words = std::max(max_words, v.words);
    const dim3 and_grid((unsigned)std::max<u64>(1, std::min<u64>(((u64)max_words + 255) / 256, (u64)ctx->n_sms * 4)), (unsigned)red.size());
    auto launch_and = [&]() -> kb_status {
        timer_begin(ctx, F_FILTER);
        bgp_and_kernel<<<and_grid, 256, 0, ctx->st>>>(A);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        return KB_OK;
    };
    // filter = false: the marking pass; otherwise the survivors go to `next` (one relation per member)
    auto launch_reduce = [&](std::vector<std::unique_ptr<kb_rel>>* next) -> kb_status {
        u64 base = 0;
        for (u32 m = 0; m < P.n_rel; m++) {
            RedRel& R = P.r[m];
            const kb_rel& rel = *(*rels)[members[m]];
            R.n_cols = (u32)rel.cols.size();
            R.n = (u32)rel.n;
            R.base = base;
            base += (rel.n + 31) & ~31ull;
            for (u32 c = 0; c < R.n_cols; c++) { R.in[c] = rel.cols[c].ptr; R.out[c] = next ? (*next)[m]->cols[c].ptr : nullptr; }
        }
        P.total = base;
        P.filter = next ? 1u : 0u;
        for (u32 m = 0; m < P.n_rel; m++) {  // the marking pass: an atomicOr per row, a filtering round: a probe per row (+ the
            info->reduce_bytes += 4ull * P.r[m].n_cols * P.r[m].n;  // survivors' writes and atomicOrs, once their count is known)
            info->reduce_bit_ops += (u64)P.r[m].n_red * P.r[m].n;
        }
        KB_CUDA(ctx, cudaMemsetAsync(marks_begin, 0, mark_bytes, ctx->st));
        const int grid = (int)std::max<u64>(1, std::min<u64>((P.total + RED_THREADS - 1) / RED_THREADS, (u64)ctx->n_sms * 8));
        timer_begin(ctx, F_FILTER);
        bgp_reduce_kernel<<<grid, RED_THREADS, 0, ctx->st>>>(P);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        return KB_OK;
    };
    KB_TRY(launch_reduce(nullptr));
    KB_TRY(launch_and());
    for (u32 round = 0; round < (u32)comp.size(); round++) {
        std::vector<std::unique_ptr<kb_rel>> next(P.n_rel);
        for (u32 m = 0; m < P.n_rel; m++) {
            const kb_rel& rel = *(*rels)[members[m]];
            next[m] = std::make_unique<kb_rel>();
            next[m]->slots = rel.slots;
            for (size_t c = 0; c < rel.cols.size(); c++) { Col col; KB_TRY(alloc_col(ctx, rel.n, &col)); next[m]->cols.push_back(col); }
        }
        const u32 off = ctrl_alloc(ctx, P.n_rel);
        KB_CUDA(ctx, cudaMemsetAsync(ctx->ctrl + off, 0, P.n_rel * sizeof(u32), ctx->st));
        P.count = ctx->ctrl + off;
        KB_TRY(launch_reduce(&next));
        KB_TRY(ctrl_read(ctx));
        ++*rounds;
        bool shrank = false;
        for (u32 m = 0; m < P.n_rel; m++) {
            next[m]->n = ctx->h_ctrl[off + m];
            info->reduce_bytes += 4ull * P.r[m].n_cols * next[m]->n;
            info->reduce_bit_ops += (u64)P.r[m].n_red * next[m]->n;
            if (next[m]->n == (*rels)[members[m]]->n) continue;
            shrank = true;
            (*rels)[members[m]] = std::move(next[m]);
        }
        if (!shrank) break;
        for (u32 m = 0; m < P.n_rel; m++) if ((*rels)[members[m]]->n == 0) return KB_OK;  // the component joins to nothing
        if (round + 1 < (u32)comp.size()) KB_TRY(launch_and());
    }
    return KB_OK;
}

}  // namespace

kb_status bgp_components(kb_ctx* ctx, const kb_pattern* pats, u32 n_pats, const kb_filter_op* filter, u32 n_ops,
                         const std::vector<std::vector<u32>>& pv, const std::vector<u32>& all_slots, std::unique_ptr<kb_rel>* out) {
    if (all_slots.size() > KB_MAX_COLS) return fail(ctx, KB_E_LIMIT, "more than %d variables", KB_MAX_COLS);
    std::vector<std::vector<u32>> psrc(n_pats);
    for (u32 k = 0; k < n_pats; k++) {
        KB_TRY(check_pattern(ctx, pats[k]));
        std::vector<u32> slots;
        pattern_vars(pats[k], &slots, &psrc[k]);
    }
    std::vector<FilterProg> pushdown;
    FilterProg post;
    KB_TRY(split_filter(ctx, filter, n_ops, pv, all_slots, &pushdown, &post));
    kb_bgp_plan_info info{};
    info.route = KB_BGP_COMPONENTS;
    info.n_patterns = n_pats;
    std::vector<std::unique_ptr<kb_rel>> rels;
    for (u32 g = 0; g < n_pats; g += (u32)MAXP) {
        const u32 m = std::min(n_pats - g, (u32)MAXP);
        std::vector<FilterProg> pd(pushdown.begin() + g, pushdown.begin() + g + m);
        std::vector<std::unique_ptr<kb_rel>> part;
        KB_TRY(scan_store(ctx, pats + g, m, pd, &part));
        for (auto& r : part) rels.push_back(std::move(r));
    }
    const std::vector<std::vector<u32>> comps = kb_bgp::components(pv);
    info.n_components = (u32)comps.size();
    bool empty = false;
    for (u32 c = 0; c < comps.size(); c++) for (u32 k : comps[c]) info.component[k] = c;
    for (u32 k = 0; k < n_pats; k++) {
        info.rows_scanned[k] = info.rows_reduced[k] = rels[k]->n;
        if (rels[k]->n == 0) empty = true;
    }
    auto finish_empty = [&]() -> kb_status {
        KB_TRY(empty_rel(ctx, all_slots, out));
        ctx->bgp_last = info;
        return KB_OK;
    };
    if (empty) return finish_empty();
    for (u32 c = 0; c < comps.size(); c++) {
        if (comps[c].size() < 3) continue;  // two patterns: their join is the semi-join already
        KB_TRY(reduce_component(ctx, comps[c], pv, psrc, &rels, &info.reduce_rounds[c], &info));
        for (u32 k : comps[c]) {
            info.rows_reduced[k] = rels[k]->n;
            if (rels[k]->n == 0) empty = true;
        }
        if (empty) return finish_empty();
    }
    u32 joins_left = n_pats - 1;  // the post-FILTER rides on the last one
    auto join = [&](std::unique_ptr<kb_rel>* cur, const kb_rel& r) -> kb_status {
        std::unique_ptr<kb_rel> j;
        KB_TRY(hash_join_impl(ctx, **cur, r, (--joins_left == 0 && !post.ops.empty()) ? &post : nullptr, &j));
        *cur = std::move(j);
        info.max_intermediate = std::max<u64>(info.max_intermediate, (*cur)->n);
        return KB_OK;
    };
    std::vector<uint64_t> rows(n_pats);
    for (u32 k = 0; k < n_pats; k++) rows[k] = rels[k]->n;
    std::vector<std::unique_ptr<kb_rel>> results(comps.size());
    u32 n_order = 0;
    for (u32 c = 0; c < comps.size(); c++) {
        std::vector<int> parent;
        const bool acyclic = kb_bgp::gyo(pv, comps[c], &parent);
        info.acyclic[c] = acyclic ? 1u : 0u;
        const std::vector<u32> order = kb_bgp::join_order(pv, comps[c], rows, acyclic, parent);
        if (order.size() != comps[c].size()) return fail(ctx, KB_E_INVALID, "internal: join order of component %u is incomplete", c);
        std::unique_ptr<kb_rel> cur = std::move(rels[order[0]]);
        info.join_order[n_order++] = order[0];
        for (size_t i = 1; i < order.size(); i++) {
            KB_TRY(join(&cur, *rels[order[i]]));
            info.join_order[n_order++] = order[i];
            info.component_max_rows[c] = std::max<u64>(info.component_max_rows[c], cur->n);
        }
        info.component_rows[c] = cur->n;
        info.component_max_rows[c] = std::max<u64>(info.component_max_rows[c], cur->n);
        results[c] = std::move(cur);
    }
    std::vector<u32> cross(comps.size());
    for (u32 c = 0; c < comps.size(); c++) cross[c] = c;
    std::stable_sort(cross.begin(), cross.end(), [&](u32 a, u32 b) { return results[a]->n < results[b]->n; });
    std::unique_ptr<kb_rel> cur = std::move(results[cross[0]]);
    for (size_t i = 1; i < cross.size(); i++) KB_TRY(join(&cur, *results[cross[i]]));
    for (u32 c = 0; c < comps.size(); c++) info.cross_order[c] = cross[c];
    if (n_pats == 1 && !post.ops.empty()) {
        std::unique_ptr<kb_rel> f;
        KB_TRY(filter_impl(ctx, *cur, post, &f));
        cur = std::move(f);
    }
    info.rows_unprojected = cur->n;
    *out = select_cols(*cur, all_slots);
    ctx->bgp_last = info;
    return KB_OK;
}

}  // namespace kb

extern "C" kb_status kb_bgp_last_plan(kb_ctx* ctx, kb_bgp_plan_info* out) {
    if (!ctx || !out) return KB_E_INVALID;
    *out = ctx->bgp_last;
    return KB_OK;
}
