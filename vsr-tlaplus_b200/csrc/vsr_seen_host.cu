/*
 * vsr_seen_host.cu — the seen-set's host tier (VsrRunOpts::table_host_capacity; DESIGN §2 "Seen-set host tier"): delayed
 * duplicate detection for state spaces whose seen-set outgrows the HBM table.  Part of vsr_gpu.cu's translation unit.
 *
 *   eviction     at a level boundary where the table's resident entries pass the load threshold, the entries of levels
 *                older than the frontier are appended, unchanged, to the tier (pinned host memory, append-only), and the
 *                table is rebuilt from the frontier level's entries (compacted into the idle frontier buffer, re-inserted)
 *   false new    the expand kernel does not know the tier: a successor equal to an evicted state is inserted as new, flushed,
 *                traced, checked and counted like any new state
 *   tier pass    after the level (and its VIEW-tie patch), one kernel streams the tier against the table and marks those
 *                states; a second one drops them from the level, so everything that reads the level afterwards — its
 *                totals, VsrLevelInfo, the liveness store, collect_levels, the ranks' all-gather — sees exactly the states an
 *                HBM-only run finds
 * Every probe stays in HBM; host memory is read sequentially, once per level, and written once per entry.
 */

namespace {

/* Evict when the resident entries exceed this fraction of the table's slots.  The level expanded after an eviction inserts
   into a table holding only the frontier level, and the 7/8 limit applies to that level's new states plus those entries:
   at 1/2 a level may bring up to 3/8 of the slots (false new states included) before a 152, and a level that small
   after a boundary pays one tier pass per level.  Test hook VSR_B200_EVICT_LOAD (0: evict at every boundary). */
constexpr double EVICT_LOAD = 0.5;

double evict_load() {
    const char* s = getenv("VSR_B200_EVICT_LOAD");
    return s && s[0] ? strtod(s, nullptr) : EVICT_LOAD;
}

int grid_for(const VsrEngine* e, uint64_t n) {
    const uint64_t want = (n + 255) / 256, most = (uint64_t)e->sms * 8;
    return (int)std::max<uint64_t>(1, std::min(want, most));
}

} // namespace

cudaError_t seen_host_create(VsrEngine* e) {
    if (!e->opts.table_host_capacity) return cudaSuccess;
    cudaError_t ce = e->seen_host.alloc_hbm(0, 16, e->stream); /* no HBM part: rows of {fp, meta} */
    if (ce == cudaSuccess) ce = e->seen_host.alloc_host(e->opts.table_host_capacity);
    if (ce == cudaSuccess) ce = cudaMallocAsync((void**)&e->seen_host_ctr, 4 * sizeof(unsigned long long), e->stream);
    return ce;
}

void seen_host_destroy(VsrEngine* e) {
    if (e->seen_host_ctr) cudaFreeAsync(e->seen_host_ctr, e->stream);
    e->seen_host_ctr = nullptr;
    e->seen_host.release(e->stream);
}

int seen_host_filter(VsrEngine* e, LevelCounters& lc, size_t ctr_bytes, VsrLevelInfo& li) {
    const uint64_t n = lc.c.out_count;
    const int level = e->level + 1; /* the tag of the states just generated */
    const double t0 = now_s();
    CK(cudaMemsetAsync(e->seen_host_ctr, 0, 4 * sizeof(unsigned long long), e->stream));
    seen_host_pass_kernel<<<grid_for(e, e->seen_host_n), 256, 0, e->stream>>>((const uint64_t*)e->seen_host.host, e->seen_host_n, e->table,
                                                                                e->table_cap, level, e->seen_host_ctr, &e->ctr->collisions);
    CK(cudaGetLastError());
    unsigned long long marked = 0;
    CK(cudaMemcpyAsync(&marked, e->seen_host_ctr, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    const double t1 = now_s();
    if (marked) {
        SeenHostParams q;
        memset(&q, 0, sizeof q);
        q.rows = e->frontier[e->cur ^ 1].view();
        q.n = n;
        q.n_keep = n - marked;
        q.trace = e->trace.view();
        q.base = e->next_base;
        q.trace_cap = e->trace_cap;
        q.holes = e->frontier[e->cur].view_as(2); /* the level just expanded: idle until the next one is generated */
        q.count = e->seen_host_ctr + 1;
        q.cover = e->cov ? reinterpret_cast<LevelCounters*>(e->ctr)->cover : nullptr;
        q.table = e->table;
        q.table_cap = e->table_cap;
        q.fp_tab = e->fp_tab;
        q.run = e->m->run;
        q.level = level;
        CK(e->g->launch_seen_host_compact(q, e->sms, e->stream));
        q.phase = 1;
        q.count = e->seen_host_ctr + 2;
        CK(e->g->launch_seen_host_compact(q, e->sms, e->stream));
        const unsigned long long kept = q.n_keep;
        CK(cudaMemcpyAsync(&e->ctr->out_count, &kept, 8, cudaMemcpyHostToDevice, e->stream));
        if (lc.c.viol_id != ~0ull) { /* the level's verdict over the rows that stay: the patch pass without ties */
            static const unsigned long long ones = ~0ull;
            CK(cudaMemcpyAsync(&e->ctr->viol_id, &ones, 8, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemsetAsync(&e->ctr->viol_which, 0, sizeof(int), e->stream));
            ExpandParams p;
            fill_params(e, p);
            CK(e->g->launch_patch(p, e->ties, 0, kept, e->stream));
            e->st.kernel_launches++;
        }
        e->st.kernel_launches += 2;
        e->st.bytes_h2d += 8;
    }
    CK(cudaMemcpyAsync(&lc, e->ctr, ctr_bytes, cudaMemcpyDeviceToHost, e->stream)); /* the tier pass's collisions, the kept count */
    CK(cudaStreamSynchronize(e->stream));
    e->st.kernel_launches++;
    e->st.bytes_d2h += 8 + ctr_bytes;
    const double t2 = now_s();
    li.false_new = marked;
    li.ms_host_pass = (t1 - t0) * 1e3;
    li.ms_host_compact = (t2 - t1) * 1e3;
    e->st.host_false_new += marked;
    e->st.seconds_host_pass += t1 - t0;
    e->st.seconds_host_compact += t2 - t1;
    return 0;
}

int seen_host_evict(VsrEngine* e, VsrLevelInfo& li) {
    if ((double)e->table_resident <= evict_load() * (double)e->table_cap) return 0;
    const int d = e->level; /* depth of the frontier: its entries stay */
    const double t0 = now_s();
    const uint64_t room = e->seen_host.host_rows - e->seen_host_n;
    const SpillRows tier = {nullptr, e->seen_host.host + 4 * e->seen_host_n, 0};
    const SpillBuffer& scratch = e->frontier[e->cur ^ 1]; /* the level just expanded: idle */
    const uint64_t scratch_rows = scratch.capacity_as(4);
    unsigned long long* ctr = e->seen_host_ctr;
    CK(cudaMemsetAsync(ctr, 0, 4 * sizeof(unsigned long long), e->stream));
    /* tags below evict_floor are marked false new states, already in the tier: neither moved again nor kept */
    seen_compact_kernel<<<e->sms * 8, 256, 0, e->stream>>>(e->table, 0, e->table_cap, e->evict_floor, d, tier, room, ctr);
    seen_compact_kernel<<<e->sms * 8, 256, 0, e->stream>>>(e->table, 0, e->table_cap, d, 256, scratch.view_as(4), scratch_rows, ctr + 1);
    CK(cudaGetLastError());
    unsigned long long cnt[2] = {0, 0};
    CK(cudaMemcpyAsync(cnt, ctr, sizeof cnt, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    const uint64_t moved = cnt[0], kept = cnt[1];
    if (moved > room) {
        snprintf(e->last_error, sizeof e->last_error,
                 "capacity exceeded (seen-set host tier): %llu entries of depth < %d to move to host memory, the tier holds %llu of %llu entries",
                 (unsigned long long)moved, d, (unsigned long long)e->seen_host_n, (unsigned long long)e->seen_host.host_rows);
        li.overflow = 6;
        return VSR_RC_TOO_LARGE;
    }
    if (kept > scratch_rows) {
        snprintf(e->last_error, sizeof e->last_error, "seen-set eviction: %llu entries of depth %d, the idle frontier buffer holds %llu",
                 (unsigned long long)kept, d, (unsigned long long)scratch_rows);
        return VSR_RC_ERROR;
    }
    CK(cudaMemsetAsync(e->table, 0, e->table_cap * 16, e->stream));
    seen_reinsert_kernel<<<grid_for(e, kept), 256, 0, e->stream>>>(e->table, e->table_cap, scratch.view_as(4), kept, 64, 0, ctr + 2, nullptr);
    CK(cudaGetLastError());
    unsigned long long not_new = 0;
    CK(cudaMemcpyAsync(&not_new, ctr + 2, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (not_new) {
        snprintf(e->last_error, sizeof e->last_error, "seen-set eviction: %llu of %llu entries of depth %d were not new when re-inserted",
                 not_new, (unsigned long long)kept, d);
        return VSR_RC_ERROR;
    }
    e->seen_host_n += moved;
    e->table_resident = kept;
    e->evict_floor = d;
    e->st.kernel_launches += 3;
    e->st.bytes_d2h += 24;
    e->st.host_entries = e->seen_host_n;
    const double t1 = now_s();
    li.evicted = moved;
    li.ms_host_evict = (t1 - t0) * 1e3;
    e->st.seconds_host_evict += t1 - t0;
    if (e->opts.verbose)
        fprintf(stderr, "seen-set rank %d: %llu entries of depth < %d moved to host memory (%llu held, %.2f GB), %llu kept in HBM, %.3f ms\n",
                e->rank, (unsigned long long)moved, d, (unsigned long long)e->seen_host_n, e->seen_host_n * 16e-9, (unsigned long long)kept, li.ms_host_evict);
    return 0;
}

int seen_host_lookup(const VsrEngine* e, uint64_t fp, uint32_t check) {
    const uint64_t* t = (const uint64_t*)e->seen_host.host;
    for (uint64_t i = 0; i < e->seen_host_n; i++)
        if (t[2 * i] == fp && (uint32_t)t[2 * i + 1] == check) return (int)(t[2 * i + 1] >> 56);
    return 0;
}
