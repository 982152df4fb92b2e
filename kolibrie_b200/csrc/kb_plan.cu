// kb_plan.cu — prepared star joins: kb_star_join_prepare resolves a query ONCE (patterns -> predicate slices and persistent tables of
// the store index, FILTER -> device programs, a ring of pre-allocated result buffers); kb_plan_submit is then one kernel launch with
// no allocation, no marshalling and no host synchronisation, and kb_plan_collect waits for exactly that launch. K queries run back to
// back on the device while the host stays `ring` launches ahead — the per-query host round trip of the synchronous operators
// (cudaMallocAsync, launch, cudaStreamSynchronize wake-up: tens of us next to a 0.1 ms kernel) disappears from the critical path.
// The reference's analogue is executing an already-optimised PhysicalOperator repeatedly (engine.rs:54); the plan is bound to the store
// and index version it was prepared on, like the reference's plan is to the statistics it was costed with.
#include <algorithm>

#include "kb_internal.hpp"

using namespace kb;

struct kb_plan {
    kb_ctx* ctx = nullptr;
    std::shared_ptr<Life> life;
    u64 store_version = 0, index_version = 0, num_version = 0;
    u32 shard_world = 1;
    IndexPlan ip;
    u32 ring = 0;
    struct Slot {
        std::vector<Col> cols;    // row plans: n_out columns of probe_rows rows (alloc_strided_cols)
        GroupTable tab;           // aggregate plans: the device group table of this slot (the overflow word rides behind it) ...
        char* h_rec = nullptr;    // ... and the mapped pinned list its groups are compacted into: {u32 count, u32 overflow, pad} + GroupRecord[cap]
        char* d_rec = nullptr;
        u32 rec_cap = 0;
        cudaEvent_t done = nullptr;
        u64 ticket = 0;
        bool busy = false;        // submitted, not yet collected
    };
    std::vector<Slot> slots;
    u32* h_totals = nullptr;  // mapped pinned: one 64-byte line per slot, word 0 = joined rows of the slot's last launch
    u32* d_totals = nullptr;
    u64 next_ticket = 1;
    kb_agg agg1{};
    // kb_plan_attach_peers: the partial group tables live in peer-mapped scratch (group_peer_table); after a device-side barrier a
    // merge kernel reads every rank's partial table over NVLink into the slot's local merged table
    bool attached = false;
    u32 rank = 0;
    std::vector<char*> peer_scratch;
    std::vector<GroupTable> merged;
};

namespace {
void plan_release(kb_plan* pl) {
    for (auto& s : pl->slots) {
        if (s.done) cudaEventDestroy(s.done);
        if (s.h_rec) cudaFreeHost(s.h_rec);
    }
    if (pl->h_totals) cudaFreeHost(pl->h_totals);

    delete pl;
}
}  // namespace

extern "C" {

kb_status kb_star_join_prepare(kb_ctx* ctx, uint32_t join_slot, const kb_pattern* pats, uint32_t n_pats, const kb_filter_op* filter, uint32_t n_ops,
                               const uint32_t* group_slots, uint32_t n_group, const kb_agg* aggs, uint32_t n_aggs, uint32_t ring, kb_plan** out) {
    KB_ENTER(ctx);
    if (!pats || !out) return fail(ctx, KB_E_INVALID, "NULL argument");
    if (ring == 0 || ring > 64) return fail(ctx, KB_E_LIMIT, "ring depth must be 1..64 (got %u)", ring);
    if ((n_group && !group_slots) || (n_aggs && !aggs)) return fail(ctx, KB_E_INVALID, "NULL argument");
    const bool grouped = n_group != 0;
    if (grouped && (n_group != 1 || n_aggs > 1))
        return fail(ctx, KB_E_UNSUPPORTED, "a prepared GROUP BY takes one variable and at most one aggregate (other shapes: kb_star_join + kb_group_aggregate)");
    if (!grouped && n_aggs) return fail(ctx, KB_E_INVALID, "aggregates without GROUP BY");
    if (grouped) KB_TRY(check_group_spec(ctx, group_slots, n_group, aggs, n_aggs));
    AggSpec spec(grouped ? group_slots[0] : 0u, n_aggs ? aggs : nullptr);
    auto pl = std::unique_ptr<kb_plan, void (*)(kb_plan*)>(new kb_plan, plan_release);
    KB_TRY(resolve_index_plan(ctx, join_slot, pats, n_pats, filter, n_ops, grouped ? &spec : nullptr, &pl->ip));
    if (!pl->ip.ok) return fail(ctx, KB_E_UNSUPPORTED, "prepared plans take the one-kernel index path only: %s", pl->ip.why);
    if (grouped && !pl->ip.agg) return fail(ctx, KB_E_UNSUPPORTED, "prepared GROUP BY: the group or aggregate variable is not bound by the join");
    pl->ctx = ctx;
    pl->life = ctx->life;
    pl->store_version = ctx->store_version;
    pl->index_version = ctx->index_version;
    pl->num_version = ctx->num_version;
    pl->shard_world = ctx->shard_world;
    pl->ring = ring;
    if (n_aggs) pl->agg1 = aggs[0];
    KB_CUDA(ctx, cudaHostAlloc(reinterpret_cast<void**>(&pl->h_totals), (size_t)ring * 64, cudaHostAllocMapped));
    memset(pl->h_totals, 0, (size_t)ring * 64);
    KB_CUDA(ctx, cudaHostGetDevicePointer(reinterpret_cast<void**>(&pl->d_totals), pl->h_totals, 0));
    pl->slots.resize(ring);
    const IndexPlan& ip = pl->ip;
    for (u32 i = 0; i < ring; i++) {
        kb_plan::Slot& s = pl->slots[i];
        KB_CUDA(ctx, cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
        if (ip.agg) {
            GroupParams G{};
            KB_TRY(group_table_create(ctx, 1u << 12, false, &G, &s.tab));  // the same 4096-slot table the synchronous fused path tries first
            s.rec_cap = (u32)s.tab.slots;
            KB_CUDA(ctx, cudaHostAlloc(reinterpret_cast<void**>(&s.h_rec), 16 + (size_t)s.rec_cap * sizeof(GroupRecord), cudaHostAllocMapped));
            memset(s.h_rec, 0, 16);
            KB_CUDA(ctx, cudaHostGetDevicePointer(reinterpret_cast<void**>(&s.d_rec), s.h_rec, 0));
        } else {
            KB_TRY(alloc_strided_cols(ctx, ip.probe_rows, ip.n_out, &s.cols));
        }
    }
    KB_TRY(ensure_tile_state(ctx, ip.P.n_tiles));  // a submit allocates nothing
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    *out = pl.release();
    return KB_OK;
}

kb_status kb_plan_submit(kb_ctx* ctx, kb_plan* pl, uint64_t* ticket) {
    if (!ctx || !pl || pl->ctx != ctx) return KB_E_INVALID;
    DeviceGuard guard(ctx->device);
    if (pl->store_version != ctx->store_version || pl->index_version != ctx->index_version || ctx->index_version != ctx->store_version ||
        pl->num_version != ctx->num_version || pl->shard_world != ctx->shard_world)
        return fail(ctx, KB_E_INVALID, "stale plan: the store, its index or the numeric table changed since kb_star_join_prepare");
    const u64 t = pl->next_ticket;
    kb_plan::Slot& s = pl->slots[t % pl->ring];
    if (s.busy) return fail(ctx, KB_E_LIMIT, "ring full: collect ticket %llu before submitting another query", (unsigned long long)s.ticket);
    ProbeIParams P = pl->ip.P;
    P.cb = ctx->fast_cb;  // launches of one context are serialised on its stream: they share the self-cleaning control block
    P.host_total = pl->d_totals + (t % pl->ring) * 16;
    if (pl->ip.agg) {
        GroupParams G = group_params(ctx, 1, &pl->agg1, pl->ip.has_agg ? 1u : 0u);
        const u32 si = (u32)(t % pl->ring);
        s.tab.point(&G, pl->attached ? group_peer_table(pl->peer_scratch[pl->rank], s.tab, si) : static_cast<char*>(s.tab.buf->p));
        KB_TRY(compact_setup(ctx, P.n_tiles, ctx->fast_cb, &P.c));
        P.c.ordered = 0;  // the rows are folded into groups: no output order to keep
        timer_begin(ctx, F_GROUP);
        launch_group_init(G, ctx->st);
        timer_end(ctx);
        timer_begin(ctx, F_PROBE);
        launch_probe_index(P, &G, ctx->n_sms, ctx->st);
        timer_end(ctx);
        KB_CUDA(ctx, cudaGetLastError());
        if (pl->attached) {
            // device-side barrier (every rank's partial table of this ticket is complete and visible), then ONE kernel folds all the
            // partial tables, read from the peers' memory, into this slot's merged table
            const PeerTables T = group_peer_tables(s.tab, pl->peer_scratch, pl->rank, si);
            GroupParams Gm = G;
            pl->merged[si].point(&Gm, static_cast<char*>(pl->merged[si].buf->p));
            timer_begin(ctx, F_GROUP, 3);
            launch_peer_barrier(T, (u32)t, ctx->st);
            launch_group_init(Gm, ctx->st);
            launch_group_merge_peers(Gm, T, ctx->n_sms, ctx->st);
            timer_end(ctx);
            launch_group_compact(Gm, reinterpret_cast<GroupRecord*>(s.d_rec + 16), reinterpret_cast<u32*>(s.d_rec), s.rec_cap, ctx->st);
            ctx->stats.kernel_launches++;
            KB_CUDA(ctx, cudaGetLastError());
        } else {
            timer_begin(ctx, F_GROUP);
            launch_group_compact(G, reinterpret_cast<GroupRecord*>(s.d_rec + 16), reinterpret_cast<u32*>(s.d_rec), s.rec_cap, ctx->st);
            timer_end(ctx);
            KB_CUDA(ctx, cudaGetLastError());
        }
    } else {
        KB_TRY(launch_index_rows(ctx, P, s.cols));
    }
    KB_CUDA(ctx, cudaEventRecord(s.done, ctx->st));
    ctx->stats.rows_probed += pl->ip.probe_rows;
    ctx->stats.index_joins++;
    s.busy = true;
    s.ticket = t;
    pl->next_ticket++;
    if (ticket) *ticket = t;
    return KB_OK;
}

kb_status kb_plan_collect(kb_ctx* ctx, kb_plan* pl, uint64_t ticket, uint64_t* n_rows, kb_rel** rows, kb_groups** groups) {
    if (!ctx || !pl || pl->ctx != ctx) return KB_E_INVALID;
    DeviceGuard guard(ctx->device);
    kb_plan::Slot& s = pl->slots[ticket % pl->ring];
    if (!s.busy || s.ticket != ticket)
        return fail(ctx, KB_E_NOT_FOUND, "ticket %llu is not in flight (already collected, or its ring slot was never submitted)", (unsigned long long)ticket);
    KB_CUDA(ctx, cudaEventSynchronize(s.done));
    timers_flush(ctx);
    s.busy = false;
    const u64 total = *reinterpret_cast<volatile u32*>(pl->h_totals + (ticket % pl->ring) * 16);
    ctx->stats.d2h_bytes += sizeof(u32);
    ctx->stats.rows_out = total;
    if (n_rows) *n_rows = total;
    if (pl->ip.agg) {
        // attached plans: the merged (GLOBAL) groups of all ranks; *n_rows stays this rank's own joined rows
        if (rows) *rows = nullptr;
        const u32* hdr = reinterpret_cast<const u32*>(s.h_rec);
        const u32 n_groups = reinterpret_cast<const volatile u32*>(hdr)[0], ovf = reinterpret_cast<const volatile u32*>(hdr)[1];
        ctx->stats.d2h_bytes += 16 + (u64)n_groups * sizeof(GroupRecord);
        if (ovf & 2u)
            return fail(ctx, KB_E_CUDA, "the cross-rank barrier of this query timed out: a rank did not submit it (all ranks must submit the same queries)");
        if (ovf)
            return fail(ctx, KB_E_LIMIT, "more than %llu groups%s: the prepared GROUP BY holds fixed tables (use kb_star_join + kb_group_aggregate)",
                        (unsigned long long)s.tab.slots, pl->attached ? " on some rank or in the merge" : "");
        if (groups) {
            auto g = std::make_unique<kb_groups>(1, &pl->agg1, pl->ip.has_agg ? 1u : 0u);
            const GroupRecord* rec = reinterpret_cast<const GroupRecord*>(s.h_rec + 16);
            for (u32 i = 0; i < n_groups; i++) g->add(rec[i].keys, rec[i].count, rec[i].raw);
            *groups = g.release();
        }
        return KB_OK;
    }
    if (groups) *groups = nullptr;
    if (rows) {
        // a VIEW of the ring slot (no copy): valid until the slot is submitted again, i.e. for the next ring-1 submits
        auto r = std::make_unique<kb_rel>();
        r->n = total;
        for (u32 sl : pl->ip.all_slots) {
            for (u32 c = 0; c < pl->ip.n_out; c++) if (pl->ip.out_slots[c] == sl) {
                r->slots.push_back(sl);
                r->cols.push_back(s.cols[c]);
                break;
            }
        }
        *rows = r.release();
    }
    return KB_OK;
}

uint64_t kb_plan_peer_scratch_bytes(const kb_plan* pl) {
    if (!pl || !pl->ip.agg) return 0;
    return group_peer_scratch_bytes(pl->slots[0].tab, pl->ring);
}

kb_status kb_plan_attach_peers(kb_ctx* ctx, kb_plan* pl, uint32_t rank, uint32_t world, void* const* peer_scratch) {
    if (!ctx || !pl || pl->ctx != ctx) return KB_E_INVALID;
    DeviceGuard guard(ctx->device);
    if (!pl->ip.agg) return fail(ctx, KB_E_UNSUPPORTED, "only grouped plans merge across ranks (row plans need no exchange for subject stars)");
    if (!peer_scratch || world == 0 || world > 64 || rank >= world) return fail(ctx, KB_E_INVALID, "rank %u / world %u (1..64 ranks)", rank, world);
    if (pl->ring < 2) return fail(ctx, KB_E_INVALID, "a plan that merges across ranks needs a ring of at least 2 (a slot must not be refilled while a peer still reads it)");
    if (pl->next_ticket != 1) return fail(ctx, KB_E_INVALID, "attach the peers before the first submit");
    for (u32 r = 0; r < world; r++) if (!peer_scratch[r]) return fail(ctx, KB_E_INVALID, "peer scratch %u is NULL", r);
    pl->rank = rank;
    pl->peer_scratch.assign(world, nullptr);
    for (u32 r = 0; r < world; r++) pl->peer_scratch[r] = static_cast<char*>(peer_scratch[r]);
    pl->merged.resize(pl->ring);
    for (u32 i = 0; i < pl->ring; i++) {
        GroupParams G{};
        // the GLOBAL result is bounded like a rank's: at most `slots` groups (the record list's capacity); the merged table holds
        // them at load <= 1/2, more distinct groups than that are reported as overflow by the compaction
        KB_TRY(group_table_create(ctx, 2 * pl->slots[0].tab.slots, false, &G, &pl->merged[i]));
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->st));
    pl->attached = true;
    return KB_OK;
}

kb_status kb_plan_info(const kb_plan* pl, uint32_t* ring, uint64_t* capacity_rows, uint32_t* n_cols, uint32_t* slots, uint32_t* grouped) {
    if (!pl) return KB_E_INVALID;
    if (ring) *ring = pl->ring;
    if (capacity_rows) *capacity_rows = pl->ip.probe_rows;
    if (n_cols) *n_cols = (uint32_t)pl->ip.all_slots.size();
    if (slots) for (size_t i = 0; i < pl->ip.all_slots.size() && i < KB_MAX_COLS; i++) slots[i] = pl->ip.all_slots[i];
    if (grouped) *grouped = pl->ip.agg ? 1u : 0u;
    return KB_OK;
}

void kb_plan_free(kb_ctx* ctx, kb_plan* pl) {
    if (!pl) return;
    if (pl->life && pl->life->alive && pl->ctx) {
        DeviceGuard guard(pl->ctx->device);
        cudaStreamSynchronize(pl->ctx->st);  // launches still reading the ring
        plan_release(pl);
    } else {
        plan_release(pl);
    }
    (void)ctx;
}

}  // extern "C"
