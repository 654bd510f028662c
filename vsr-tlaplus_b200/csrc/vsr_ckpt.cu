/*
 * vsr_ckpt.cu — checkpoint / recover of one rank's shard of the BFS (include/vsr_b200.h: vsr_engine_checkpoint,
 * vsr_engine_recover).  Stands in for TLC's `-checkpoint <minutes>` / `-recover <dir>` (SURVEY §8f item 4; the reference's
 * .gitignore:1 ignores TLC's states/ metadir): a multi-hour run of the README constants can be stopped and continued.
 *
 * A checkpoint is taken at a level boundary — every state of depth <= level is in the seen-set, the current frontier holds
 * exactly the states of depth `level`, nothing is in flight between ranks — and is ONE file per rank:
 *
 *   CkptHeader | VsrStats of this rank | VsrStats totals of the job | frontier: n_cur packed states | seen-set: n_entries x {fp, meta} | trace: next_base x 8 B
 *
 * The seen-set is written as its non-empty entries (compacted on the device into the idle frontier buffer, chunk by chunk)
 * and re-inserted on recovery with the BFS's own insert routine, so the table a run continues with may have another
 * capacity (or bucket layout) than the one it was checkpointed from.
 */
#include <errno.h>
#include <stdio.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <string>
#include <vector>

#include "vsr_engine.h"

using namespace vsr;

namespace {

constexpr uint64_t CKPT_MAGIC = 0x3154504B43525356ull; /* "VSRCKPT1" */
constexpr uint32_t CKPT_VERSION = 2; /* 2: VsrStats ends with the seen-set host tier's figures */

struct CkptHeader {
    uint64_t magic;
    uint32_t version, header_bytes, stats_bytes, state_bytes;
    int32_t R, V, K;                      /* layout */
    int32_t symmetry, use_view, invariant; /* RunCfg: another VIEW / SYMMETRY setting is another state graph */
    int32_t rank, world;
    int32_t level, keep_trace;
    uint64_t n_cur, cur_base, next_base;  /* frontier of depth `level`: local ids [cur_base, cur_base + n_cur) */
    uint64_t n_entries;                   /* seen-set entries that follow */
    uint64_t n_trace;                     /* trace records that follow (0 without keep_trace) */
    uint64_t records_sent, records_received;
};

/* old trace records renumbered into the new world's ids */
__global__ void ckpt_remap_trace_kernel(const uint64_t* __restrict__ in, unsigned long long n, const SpillRows out, const GidRemap m) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        *(uint64_t*)out.row<2>(i) = remap_trec(m, in[i]);
}

struct File {
    FILE* f = nullptr;
    ~File() { if (f) fclose(f); }
};

int io_error(VsrEngine* e, const char* what, const char* path) {
    snprintf(e->last_error, sizeof e->last_error, "checkpoint: %s %s: %s", what, path, strerror(errno));
    return VSR_RC_SYSTEM;
}

constexpr uint64_t IO_CHUNK = 64ull << 20; /* bytes per host staging round */

bool header_ok(const CkptHeader& h) {
    return h.magic == CKPT_MAGIC && h.version == CKPT_VERSION && h.header_bytes == sizeof h && h.stats_bytes == sizeof(VsrStats);
}

/* 1: a checkpoint header of this build, 0: something else, -1: the file cannot be opened */
int peek_header(const std::string& path, CkptHeader& h) {
    File in;
    in.f = fopen(path.c_str(), "rb");
    if (!in.f) return -1;
    return fread(&h, sizeof h, 1, in.f) == 1 && header_ok(h) ? 1 : 0;
}

/* file offsets of a checkpoint's sections */
constexpr uint64_t SECTIONS = sizeof(CkptHeader) + 2 * sizeof(VsrStats);
uint64_t entries_at(const CkptHeader& h) { return SECTIONS + h.n_cur * h.state_bytes; }
uint64_t trace_at(const CkptHeader& h) { return entries_at(h) + h.n_entries * 16; }

int seek(VsrEngine* e, File& f, uint64_t at, const char* path) {
    if (fseeko(f.f, (off_t)at, SEEK_SET) != 0) return io_error(e, "truncated", path);
    return 0;
}

/* the host tier holds seen-set entries a checkpoint file has no section for */
int refuse_host_tier(VsrEngine* e) {
    snprintf(e->last_error, sizeof e->last_error, "%s", HOST_TIER_NO_CHECKPOINT);
    return VSR_RC_CONFIG_ERROR;
}

} // namespace

extern "C" {

int vsr_engine_checkpoint(VsrEngine* e, const char* path, const VsrStats* totals) {
    if (!e || !path) return VSR_RC_ERROR;
    if (e->seen_host.host_rows) return refuse_host_tier(e);
    if (e->level_open) {
        snprintf(e->last_error, sizeof e->last_error, "checkpoint: only at a level boundary (after vsr_engine_finish_level)");
        return VSR_RC_ERROR;
    }
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    const uint64_t S = (uint64_t)e->g->bytes;
    const std::string tmp = std::string(path) + ".tmp";
    File out;
    out.f = fopen(tmp.c_str(), "wb");
    if (!out.f) return io_error(e, "cannot create", tmp.c_str());
    CkptHeader h;
    memset(&h, 0, sizeof h);
    h.magic = CKPT_MAGIC;
    h.version = CKPT_VERSION;
    h.header_bytes = sizeof h;
    h.stats_bytes = sizeof(VsrStats);
    h.state_bytes = (uint32_t)S;
    h.R = e->g->R; h.V = e->g->V; h.K = e->g->K;
    h.symmetry = e->m->run.symmetry; h.use_view = e->m->run.use_view; h.invariant = e->m->run.invariant;
    h.rank = e->rank; h.world = e->world;
    h.level = e->level;
    h.keep_trace = e->trace_cap ? 1 : 0;
    h.n_cur = e->n_cur; h.cur_base = e->cur_base; h.next_base = e->next_base;
    h.n_entries = e->st.distinct; /* checked against what the compaction finds */
    h.n_trace = std::min<uint64_t>(e->next_base, e->trace_cap);
    h.records_sent = e->records_sent; h.records_received = e->records_received;
    const VsrStats& tot = totals ? *totals : e->st;
    if (fwrite(&h, sizeof h, 1, out.f) != 1 || fwrite(&e->st, sizeof(VsrStats), 1, out.f) != 1 || fwrite(&tot, sizeof(VsrStats), 1, out.f) != 1)
        return io_error(e, "cannot write", tmp.c_str());
    std::vector<uint8_t> host;
    /* 1. the frontier of depth `level` */
    {
        const uint64_t per = std::max<uint64_t>(1, IO_CHUNK / S);
        host.resize(per * S);
        for (uint64_t first = 0; first < e->n_cur; first += per) {
            const uint64_t n = std::min(per, e->n_cur - first);
            CK(e->frontier[e->cur].to_host(first, n, host.data()));
            if (fwrite(host.data(), S, n, out.f) != n) return io_error(e, "cannot write", tmp.c_str());
        }
    }
    /* 2. the seen-set's entries, compacted into the idle frontier buffer (its HBM part) chunk by chunk */
    {
        uint64_t* scratch = (uint64_t*)e->frontier[e->cur ^ 1].hbm;
        const uint64_t slots_per_pass = std::max<uint64_t>(64, e->frontier[e->cur ^ 1].hbm_rows * S / 16);
        unsigned long long* dcount = &e->ctr->work_next; /* scratch word: the level's counters are reset when it opens */
        uint64_t written = 0;
        for (uint64_t first = 0; first < e->table_cap; first += slots_per_pass) {
            const uint64_t n = std::min(slots_per_pass, e->table_cap - first);
            CK(cudaMemsetAsync(dcount, 0, 8, e->stream));
            seen_compact_kernel<<<e->sms * 8, 256, 0, e->stream>>>(e->table, first, n, 0, 256, SpillRows{(uint32_t*)scratch, nullptr, ~0ull}, ~0ull, dcount);
            CK(cudaGetLastError());
            unsigned long long cnt = 0;
            CK(cudaMemcpyAsync(&cnt, dcount, 8, cudaMemcpyDeviceToHost, e->stream));
            CK(cudaStreamSynchronize(e->stream));
            const uint64_t per = IO_CHUNK / 16;
            host.resize(std::min<uint64_t>(per, std::max<uint64_t>(cnt, 1)) * 16);
            for (uint64_t o = 0; o < cnt; o += per) {
                const uint64_t k = std::min<uint64_t>(per, cnt - o);
                CK(cudaMemcpy(host.data(), scratch + 2 * o, k * 16, cudaMemcpyDeviceToHost));
                if (fwrite(host.data(), 16, k, out.f) != k) return io_error(e, "cannot write", tmp.c_str());
            }
            written += cnt;
        }
        if (written != h.n_entries) {
            snprintf(e->last_error, sizeof e->last_error, "checkpoint: the seen-set holds %llu entries, the run counted %llu distinct states",
                     (unsigned long long)written, (unsigned long long)h.n_entries);
            return VSR_RC_ERROR;
        }
        e->st.bytes_d2h += written * 16;
    }
    /* 3. the trace records */
    if (h.n_trace) {
        const uint64_t per = IO_CHUNK / 8;
        host.resize(std::min(per, h.n_trace) * 8);
        for (uint64_t o = 0; o < h.n_trace; o += per) {
            const uint64_t k = std::min(per, h.n_trace - o);
            CK(e->trace.to_host(o, k, host.data()));
            if (fwrite(host.data(), 8, k, out.f) != k) return io_error(e, "cannot write", tmp.c_str());
        }
        e->st.bytes_d2h += h.n_trace * 8;
    }
    e->st.bytes_d2h += e->n_cur * S;
    if (fflush(out.f) != 0 || fsync(fileno(out.f)) != 0) return io_error(e, "cannot write", tmp.c_str()); /* on disk before it replaces the previous one */
    fclose(out.f);
    out.f = nullptr;
    if (rename(tmp.c_str(), path) != 0) return io_error(e, "cannot rename to", path);
    return 0;
}

} /* extern "C" */

/* ------------------------------------------------------------------ recovery on any number of ranks
 * A checkpoint of W_old ranks continues on W_new ranks, both powers of two.  The owner is the top bits of fp x C
 * (owner_of), so the owners nest, and each new rank reads the bulk sections of its source files only:
 *   W_old = k W_new (k >= 1)  new rank r owns exactly what old ranks r k ... r k + k - 1 owned: it takes their seen-set
 *                             entries and frontiers whole, and their trace records stay where they were (k = 1: same ids)
 *   W_new = s W_old (s > 1)   new rank r's share lies in old file r / s: the entries and frontier states it owns
 *                             (reshard_frontier_kernel: the BFS's fingerprint and owner rule), and slice r % s of the file's
 *                             trace records, its frontier's records copied after the slice
 * Every rank still checks the headers, statistics and job totals of every old file, so that all the files are one
 * checkpoint.  Every stored global id is renumbered with one GidRemap (vsr_gpu.cuh).  The job's totals travel unchanged
 * (the violation id renumbered).  In the same world the rank continues its file's counters; in another world only
 * `distinct` (= entries it inserted, which its next checkpoint checks) carries over, the work counters start at 0. */
namespace {

/* <base> when one rank wrote it, <base>.rank0 ... <base>.rank(W_old - 1) when several did (W_old from <base>.rank0's
   header).  Both: the one of this world, 151 when neither is.  Anything else is the one file the loader names. */
int old_files(VsrEngine* e, const char* base, std::vector<std::string>& files) {
    const std::string P = base, P0 = P + ".rank0";
    CkptHeader h1, h0;
    const int k1 = peek_header(P, h1), k0 = peek_header(P0, h0), W = e->world;
    const bool one = k1 == 1 && h1.world == 1;
    if (one && k0 == 1 && W != 1 && W != h0.world) {
        snprintf(e->last_error, sizeof e->last_error, "recover: both %s (1 rank) and %s (%d ranks) exist and neither was written by %d ranks: remove one",
                 P.c_str(), P0.c_str(), h0.world, W);
        return VSR_RC_CONFIG_ERROR;
    }
    if (k0 == 1 && !(one && W == 1)) {
        if (h0.world < 1 || h0.world > MAX_WORLD || (h0.world & (h0.world - 1))) {
            snprintf(e->last_error, sizeof e->last_error, "recover: %s claims a world of %d ranks", P0.c_str(), h0.world);
            return VSR_RC_SPEC_ERROR;
        }
        for (int r = 0; r < h0.world; r++) files.push_back(P + ".rank" + std::to_string(r));
    } else {
        files.push_back(k1 == -1 && (k0 == 0 || W > 1) ? P0 : P); /* not a checkpoint, or missing: the loader says which */
    }
    return 0;
}

} // namespace

extern "C" int vsr_engine_recover(VsrEngine* e, const char* path, VsrStats* totals_out) {
    if (!e || !path) return VSR_RC_ERROR;
    if (e->seen_host.host_rows) return refuse_host_tier(e);
    CK(cudaSetDevice(e->device));
    std::vector<std::string> files;
    int rc = old_files(e, path, files);
    if (rc) return rc;
    const int Wold = (int)files.size(), W = e->world, me = e->rank;
    const uint64_t S = (uint64_t)e->g->bytes;
    const double t_start = now_s();
    double t_read = 0, t_insert = 0, t_frontier = 0, t_trace = 0;
    uint64_t bytes_read = 0;
    std::vector<File> in(Wold);
    std::vector<CkptHeader> h(Wold);
    VsrStats tot{}, mine{}, st, st_tot;
    /* 1. every old file: a checkpoint of this build and model, rank q of Wold, of the same level and job */
    for (int q = 0; q < Wold; q++) {
        const char* f = files[q].c_str();
        in[q].f = fopen(f, "rb");
        if (!in[q].f) return io_error(e, "cannot open", f);
        if (fread(&h[q], sizeof h[q], 1, in[q].f) != 1 || !header_ok(h[q])) {
            snprintf(e->last_error, sizeof e->last_error, "recover: %s is not a checkpoint of this build", f);
            return VSR_RC_SPEC_ERROR;
        }
        if (fread(&st, sizeof st, 1, in[q].f) != 1 || fread(&st_tot, sizeof st_tot, 1, in[q].f) != 1) return io_error(e, "truncated", f);
        const CkptHeader& x = h[q];
        if (x.state_bytes != S || x.R != e->g->R || x.V != e->g->V || x.K != e->g->K || x.symmetry != e->m->run.symmetry || x.use_view != e->m->run.use_view ||
            x.invariant != e->m->run.invariant) {
            snprintf(e->last_error, sizeof e->last_error,
                     "recover: %s was written for ReplicaCount=%d |Values|=%d StartViewOnTimerLimit=%d symmetry=%d view=%d invariants=%d: not this model", f,
                     x.R, x.V, x.K - 1, x.symmetry, x.use_view, x.invariant);
            return VSR_RC_SPEC_ERROR;
        }
        if (x.world != Wold || x.rank != q) {
            snprintf(e->last_error, sizeof e->last_error, "recover: %s is rank %d of %d, expected rank %d of %d", f, x.rank, x.world, q, Wold);
            return VSR_RC_SPEC_ERROR;
        }
        if (q && (x.level != h[0].level || x.keep_trace != h[0].keep_trace || memcmp(&st_tot, &tot, sizeof tot) != 0)) {
            snprintf(e->last_error, sizeof e->last_error, "recover: %s is not of the same checkpoint as %s (level, trace or job totals differ)", f, files[0].c_str());
            return VSR_RC_SPEC_ERROR;
        }
        if (x.next_base != x.cur_base + x.n_cur) {
            snprintf(e->last_error, sizeof e->last_error, "recover: %s holds a frontier of %llu states at local id %llu, its next id is %llu", f,
                     (unsigned long long)x.n_cur, (unsigned long long)x.cur_base, (unsigned long long)x.next_base);
            return VSR_RC_SPEC_ERROR;
        }
        if (x.n_trace && x.n_trace != x.next_base) {
            snprintf(e->last_error, sizeof e->last_error, "recover: %s holds %llu of its %llu trace records", f, (unsigned long long)x.n_trace,
                     (unsigned long long)x.next_base);
            return VSR_RC_SPEC_ERROR;
        }
        if (q == 0) tot = st_tot;
        if (q == me) mine = st;
    }
    /* 2. the source files [src, src + nsrc) and the id mapping */
    const bool grow = W > Wold;
    const int k = grow ? 1 : Wold / W, s = grow ? W / Wold : 1;
    const int src = grow ? me / s : me * k, nsrc = grow ? 1 : k;
    GidRemap m;
    memset(&m, 0, sizeof m);
    m.old_world = Wold;
    uint64_t T = 0;
    for (int g = 0; g < Wold; g += k) {
        uint64_t hist = 0, front = 0;
        for (int q = g; q < g + k; q++) front += h[q].cur_base;
        for (int q = g; q < g + k; q++) {
            T += h[q].next_base;
            m.to[q] = grow ? q * s : g / k;
            m.slice[q] = grow ? std::max<uint64_t>(1, (h[q].next_base + s - 1) / s) : REMAP_ALL;
            m.cut[q] = grow ? REMAP_ALL : h[q].cur_base;
            m.hist[q] = grow ? 0 : hist;
            m.front[q] = grow ? 0 : front;
            hist += h[q].cur_base;
            front += h[q].n_cur;
        }
    }
    if (e->trace_cap && !h[0].keep_trace && T) {
        snprintf(e->last_error, sizeof e->last_error, "recover: %s was written without trace records; continue it with keep_trace off (vsrmc -notrace)", files[0].c_str());
        return VSR_RC_CONFIG_ERROR;
    }
    const bool tr = e->trace_cap && h[0].keep_trace;
    /* this rank's old ids in each source file: grow, its slice of file src; else all of them */
    uint64_t lo = 0, hi = h[src].next_base;
    if (grow) {
        lo = std::min<uint64_t>(hi, (uint64_t)(me % s) * m.slice[src]);
        hi = std::min<uint64_t>(hi, lo + m.slice[src]);
    }
    const uint64_t cur_base = grow ? hi - lo : m.front[src]; /* the group's histories, then its frontiers */
    rc = vsr_engine_reset(e);
    if (rc) return rc;
    e->touched = true; /* from here on a failure leaves part of the checkpoint in the engine */
    CK(cudaStreamSynchronize(e->stream));
    std::vector<uint8_t> host;
    unsigned long long* d0 = &e->ctr->work_next; /* scratch words: the level's counters are reset when it opens */
    unsigned long long* d1 = &e->ctr->drain_next;
    uint8_t* scratch = (uint8_t*)e->frontier[1].hbm;
    const uint64_t scratch_bytes = e->frontier[1].hbm_rows * S;
    /* 3. the seen-set entries this rank owns.  Chunks of at most 1/16 of the table: the load is checked after every chunk,
       so a share that does not fit stops at 15/16 load, where inserts still end */
    const uint64_t limit = e->table_cap - e->table_cap / 8;
    unsigned long long counts[2] = {0, 0}; /* entries not new, entries owned */
    uint64_t n_entries = 0;
    for (int q = src; q < src + nsrc; q++) n_entries += h[q].n_entries;
    {
        const uint64_t per = std::max<uint64_t>(1, std::min<uint64_t>({IO_CHUNK / 16, scratch_bytes / 16, e->table_cap / 16}));
        CK(cudaMemsetAsync(d0, 0, 16, e->stream));
        host.resize(per * 16);
        for (int q = src; q < src + nsrc; q++) {
            if ((rc = seek(e, in[q], entries_at(h[q]), files[q].c_str()))) return rc;
            for (uint64_t o = 0; o < h[q].n_entries; o += per) {
                const uint64_t n = std::min(per, h[q].n_entries - o);
                double t = now_s();
                if (fread(host.data(), 16, n, in[q].f) != n) return io_error(e, "truncated", files[q].c_str());
                t_read += now_s() - t;
                t = now_s();
                CK(cudaMemcpyAsync(scratch, host.data(), n * 16, cudaMemcpyHostToDevice, e->stream));
                seen_reinsert_kernel<<<e->sms * 8, 256, 0, e->stream>>>(e->table, e->table_cap, SpillRows{(uint32_t*)scratch, nullptr, ~0ull}, n, e->owner_shift, me, d0, d1);
                CK(cudaGetLastError());
                CK(cudaMemcpyAsync(counts, d0, 16, cudaMemcpyDeviceToHost, e->stream));
                CK(cudaStreamSynchronize(e->stream)); /* `host` is reused by the next round */
                t_insert += now_s() - t;
                bytes_read += n * 16;
                if (counts[1] > limit) {
                    snprintf(e->last_error, sizeof e->last_error,
                             "capacity exceeded (recover): rank %d of %d owns more than %llu of the checkpoint's seen-set entries: 7/8 of its %llu slots", me, W,
                             (unsigned long long)limit, (unsigned long long)e->table_cap);
                    return VSR_RC_TOO_LARGE;
                }
            }
        }
        /* shrinking or the same world: every entry of a source file is this rank's */
        const unsigned long long bad = counts[0] + (grow ? 0 : n_entries - counts[1]);
        if (bad) {
            snprintf(e->last_error, sizeof e->last_error, "recover: %llu seen-set entries of %s could not be inserted as new (corrupt file?)", bad,
                     files[src].c_str());
            return VSR_RC_ERROR;
        }
    }
    const uint64_t owned = counts[1];
    /* 4. the frontier states, into buffer 0: shrinking or the same world, each source file's whole frontier in file order;
       growing, the states this rank owns, with their trace records after its slice */
    uint64_t kept = 0, launches = 0;
    {
        const uint64_t fcap_total = e->frontier[0].capacity();
        const bool copy = grow && tr;
        const uint64_t per = std::max<uint64_t>(1, (std::min(IO_CHUNK, scratch_bytes) - 16) / (S + 8));
        const uint64_t tr_off = (per * S + 15) & ~15ull;
        ReshardParams q;
        memset(&q, 0, sizeof q);
        q.in = (const uint32_t*)scratch;
        q.in_trace = copy ? (const uint64_t*)(scratch + tr_off) : nullptr;
        q.out = e->frontier[0].view();
        q.out_cap = fcap_total;
        q.trace = e->trace.view();
        q.trace_base = cur_base;
        q.trace_cap = copy ? e->trace.capacity() : 0;
        q.table = e->table;
        q.table_cap = e->table_cap;
        q.fp_tab = e->fp_tab;
        q.run = e->m->run;
        q.rank = me;
        q.owner_shift = e->owner_shift;
        q.level = h[0].level;
        q.place = !grow;
        q.remap = m;
        q.kept = d0;
        q.missing = d1;
        CK(cudaMemsetAsync(d0, 0, 16, e->stream));
        host.resize(per * (S + 8));
        uint64_t* host_tr = (uint64_t*)(host.data() + per * S);
        for (int r = src; r < src + nsrc; r++) {
            const uint64_t n_cur = h[r].n_cur;
            for (uint64_t o = 0; o < n_cur; o += per) {
                const uint64_t n = std::min(per, n_cur - o);
                double t = now_s();
                if ((rc = seek(e, in[r], SECTIONS + o * S, files[r].c_str()))) return rc;
                if (fread(host.data(), S, n, in[r].f) != n) return io_error(e, "truncated", files[r].c_str());
                if (copy) {
                    if ((rc = seek(e, in[r], trace_at(h[r]) + (h[r].cur_base + o) * 8, files[r].c_str()))) return rc;
                    if (fread(host_tr, 8, n, in[r].f) != n) return io_error(e, "truncated", files[r].c_str());
                }
                t_read += now_s() - t;
                t = now_s();
                CK(cudaMemcpyAsync(scratch, host.data(), n * S, cudaMemcpyHostToDevice, e->stream));
                if (copy) CK(cudaMemcpyAsync(scratch + tr_off, host_tr, n * 8, cudaMemcpyHostToDevice, e->stream));
                q.n = n;
                q.out_first = kept + o;
                CK(e->g->launch_reshard_frontier(q, e->sms, e->stream));
                CK(cudaStreamSynchronize(e->stream));
                launches++;
                t_frontier += now_s() - t;
                bytes_read += n * (S + (copy ? 8 : 0));
            }
            if (!grow) kept += n_cur;
        }
        CK(cudaMemcpy(counts, d0, 16, cudaMemcpyDeviceToHost));
        if (grow) kept = counts[0];
        if (kept > fcap_total) {
            snprintf(e->last_error, sizeof e->last_error, "capacity exceeded (recover): rank %d of %d owns %llu of the checkpoint's frontier states, its frontier holds %llu",
                     me, W, (unsigned long long)kept, (unsigned long long)fcap_total);
            return VSR_RC_TOO_LARGE;
        }
        if (counts[1]) {
            snprintf(e->last_error, sizeof e->last_error,
                     "recover: the checkpoint's frontier and seen-set disagree: %llu frontier states rank %d took are not in its seen-set at depth %d", counts[1], me,
                     h[0].level);
            return VSR_RC_ERROR;
        }
        if (tr && cur_base + kept > e->trace.capacity()) {
            snprintf(e->last_error, sizeof e->last_error,
                     "capacity exceeded (recover): rank %d needs %llu trace records (%llu of the checkpoint's %llu, then %llu frontier states), it holds %llu", me,
                     (unsigned long long)(cur_base + kept), (unsigned long long)cur_base, (unsigned long long)T, (unsigned long long)kept,
                     (unsigned long long)e->trace.capacity());
            return VSR_RC_TOO_LARGE;
        }
    }
    /* 5. this rank's old records [lo, hi) of each source file, renumbered on the device: each chunk lies on one side of
       the file's cut, where the new ids are consecutive */
    if (tr) {
        const uint64_t per = std::max<uint64_t>(1, std::min(IO_CHUNK, scratch_bytes) / 8);
        host.resize(per * 8);
        for (int r = src; r < src + nsrc; r++) {
            const uint64_t a = grow ? lo : 0, b = grow ? hi : h[r].next_base;
            if (a < b && (rc = seek(e, in[r], trace_at(h[r]) + a * 8, files[r].c_str()))) return rc;
            for (uint64_t o = a, n; o < b; o += n) {
                n = std::min(per, (o < m.cut[r] ? std::min<uint64_t>(b, m.cut[r]) : b) - o);
                double t = now_s();
                if (fread(host.data(), 8, n, in[r].f) != n) return io_error(e, "truncated", files[r].c_str());
                t_read += now_s() - t;
                t = now_s();
                const uint64_t row = remap_gid(m, make_gid(r, o)) & ((1ull << 40) - 1ull);
                CK(cudaMemcpyAsync(scratch, host.data(), n * 8, cudaMemcpyHostToDevice, e->stream));
                ckpt_remap_trace_kernel<<<e->sms * 4, 256, 0, e->stream>>>((const uint64_t*)scratch, n, e->trace.view().from(row, 2), m);
                CK(cudaGetLastError());
                CK(cudaStreamSynchronize(e->stream));
                t_trace += now_s() - t;
                bytes_read += n * 8;
            }
        }
    }
    /* the BFS position: the frontier of depth `level`, this rank's ids continue after it */
    if (W == Wold) { /* the same world: this rank's counters continue; capacities are this engine's */
        const VsrStats fresh = e->st;
        e->st = mine;
        e->st.table_capacity = fresh.table_capacity; e->st.frontier_capacity = fresh.frontier_capacity;
        e->st.bytes_table = fresh.bytes_table; e->st.bytes_frontier = fresh.bytes_frontier;
        e->records_sent = h[me].records_sent; e->records_received = h[me].records_received;
    } else {
        e->st.distinct = owned;
        e->st.kernel_launches = launches;
    }
    e->st.bytes_h2d += bytes_read;
    e->n_cur = kept;
    e->cur_base = cur_base;
    e->next_base = cur_base + kept;
    e->cur = 0;
    e->level = h[0].level;
    e->level_open = false;
    if (e->opts.collect_levels) e->collected.resize(h[0].level); /* depths up to the checkpoint's were collected by another run: empty */
    if (tot.violation_level) tot.violation_id = remap_gid(m, tot.violation_id);
    if (totals_out) *totals_out = tot;
    if (e->opts.verbose)
        fprintf(stderr,
                "recover: rank %d of %d took its share of %d checkpoint files (%llu bytes read) in %.3f s: %.3f s reading, %.3f s seen-set insert, %.3f s frontier, %.3f s trace; "
                "%llu seen-set entries, %llu frontier states\n",
                me, W, nsrc, (unsigned long long)bytes_read, now_s() - t_start, t_read, t_insert, t_frontier, t_trace, (unsigned long long)owned,
                (unsigned long long)kept);
    return 0;
}
