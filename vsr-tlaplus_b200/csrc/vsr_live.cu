/*
 * vsr_live.cu — the liveness pass: PROPERTY ViewChangeCompletes == []<>P under Spec == Init /\ [][Next]_vars /\ WF_vars(Next)
 * (VSR.tla:964-967), P = AllReplicasMoveToSameView.  On the finite (quotient) state graph the property is violated iff a
 * reachable not-P state has no successor but itself (stuttering forever there is fair: Next is disabled), or a reachable
 * cycle of not-P states with at least one real step exists (it satisfies WF_vars(Next)).  DESIGN "Liveness" has the argument,
 * SYMMETRY and VIEW included.
 *
 * Store: every finished BFS level appends its not-P states (live_collect_kernel) — words, BFS local id — and inserts them
 * into the live index.  Sweeps: after a complete BFS, one launch per level, deepest first; a stored state stays alive iff
 * one of its not-P successors other than itself is alive; repeat until a sweep removes nothing.  Most edges go from depth d
 * to d + 1, so deepest-first order settles an acyclic graph in few sweeps.  The first sweep also finds the sinks.
 * Counterexample: the BFS trace to the reported state, then (a cycle) a host walk along alive not-P successors until a state
 * repeats; TLC's lasso.  Kernels: vsr_live.cuh.
 */
#include <stdlib.h>

#include <map>
#include <utility>

#include "vsr_engine.h"

using namespace vsr;

namespace {

/* {fp, check} pairs looked up in the live index: out[i] = store index + 1 (0 = absent), bit 63 = alive */
__global__ void live_lookup_kernel(const uint64_t* index, unsigned long long cap, const uint32_t* alive, const unsigned long long* keys, int n,
                                   unsigned long long* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t meta = table_lookup(index, cap, keys[2 * i], (uint32_t)keys[2 * i + 1]);
    unsigned long long r = meta >> 32;
    if (r && ((alive[(r - 1) >> 5] >> ((r - 1) & 31)) & 1u)) r |= 1ull << 63;
    out[i] = r;
}

uint64_t env_u64(const char* name) {
    const char* s = getenv(name);
    return s && s[0] ? strtoull(s, nullptr, 10) : 0;
}

LiveParams live_params(VsrEngine* e) {
    LiveParams q;
    memset(&q, 0, sizeof q);
    q.words = e->live_words.view();
    q.cap = e->live_words.capacity();
    q.ids = e->live_ids;
    q.index = e->live_index;
    q.index_cap = e->live_index_cap;
    q.alive = e->live_alive;
    q.ctr = e->live_ctr;
    q.fp_tab = e->fp_tab;
    q.run = e->m->run;
    q.hooks = e->m->live_hooks;
    return q;
}

uint64_t live_stored(const VsrEngine* e) { return e->live_level_off.empty() ? 0 : e->live_level_off.back(); }

} // namespace

/* Sizes, up front: the store holds as many states as the seen-set (its load limit, plus its host tier), unless VSR_B200_LIVE_STATES says fewer;
   the live index has two slots per stored state (load <= 1/2), the local ids 8 B and the alive bits 1 bit per state in HBM.
   The words go to HBM as far as it has room (VSR_B200_LIVE_HBM_STATES caps that part, for tests) and continue in pinned host
   memory mapped into the device when the run allows host memory (frontier_host_capacity > 0, as for the frontier spill);
   otherwise the store ends there.  A level that does not fit is a 152, never a truncation. */
int live_create(VsrEngine* e, char* err, size_t errcap) {
    auto fail = [&](int rc, const char* fmt, unsigned long long a, unsigned long long b) {
        if (err && errcap) snprintf(err, errcap, fmt, a, b);
        return rc;
    };
    const uint64_t S = (uint64_t)e->g->bytes;
    uint64_t cap = e->table_cap - e->table_cap / 8 + e->opts.table_host_capacity; /* the seen-set with its host tier */
    if (const uint64_t want = env_u64("VSR_B200_LIVE_STATES")) cap = std::min(cap, want);
    cap = std::min<uint64_t>(cap, 0xFFFFFFFEull); /* the index's meta carries store index + 1 in 32 bits */
    cap = (cap + 31) & ~31ull;
    e->live_index_cap = (2 * cap + 63) & ~63ull;
    const uint64_t abytes = cap / 8;
    if ((cudaMallocAsync((void**)&e->live_index, e->live_index_cap * 16, e->stream)) != cudaSuccess ||
        (cudaMallocAsync((void**)&e->live_ids, cap * 8, e->stream)) != cudaSuccess ||
        (cudaMallocAsync((void**)&e->live_alive, abytes, e->stream)) != cudaSuccess ||
        (cudaMallocAsync((void**)&e->live_ctr, sizeof(LiveCtr), e->stream)) != cudaSuccess) {
        cudaGetLastError();
        return fail(VSR_RC_TOO_LARGE, "liveness store: the live index (%llu bytes) and ids (%llu bytes) do not fit in device memory beside the seen-set; "
                    "give a smaller table_capacity", (unsigned long long)(e->live_index_cap * 16), (unsigned long long)(cap * 8));
    }
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    const uint64_t margin = 512ull << 20;
    uint64_t dev = free_b > margin ? (free_b - margin) / S : 0;
    if (const uint64_t hbm = env_u64("VSR_B200_LIVE_HBM_STATES")) dev = std::min(dev, hbm);
    dev = std::min(dev, cap);
    const uint64_t host = e->opts.frontier_host_capacity ? cap - dev : 0;
    if (!host) cap = dev = dev & ~31ull; /* the store ends with its HBM part (whole words of alive bits) */
    if (e->live_words.alloc_hbm(dev, S, e->stream) != cudaSuccess) {
        cudaGetLastError();
        return fail(VSR_RC_TOO_LARGE, "liveness store: %llu states of %llu bytes do not fit in device memory", (unsigned long long)dev, (unsigned long long)S);
    }
    if (e->live_words.alloc_host(host) != cudaSuccess) {
        cudaGetLastError();
        return fail(VSR_RC_TOO_LARGE, "liveness store: %llu bytes of pinned host memory for its continuation (%llu states) cannot be allocated",
                    (unsigned long long)(host * S), (unsigned long long)host);
    }
    e->live_bytes_hbm = e->live_index_cap * 16 + cap * 8 + abytes + dev * S;
    e->live_bytes_host = host * S;
    const int rc = live_reset(e);
    if (rc && err && errcap) snprintf(err, errcap, "%s", e->last_error);
    return rc;
}

void live_destroy(VsrEngine* e) {
    if (e->live_index) cudaFreeAsync(e->live_index, e->stream);
    if (e->live_ids) cudaFreeAsync(e->live_ids, e->stream);
    if (e->live_alive) cudaFreeAsync(e->live_alive, e->stream);
    if (e->live_ctr) cudaFreeAsync(e->live_ctr, e->stream);
    e->live_words.release(e->stream);
    e->live_index = nullptr;
    e->live_ids = nullptr;
    e->live_alive = nullptr;
    e->live_ctr = nullptr;
}

int live_reset(VsrEngine* e) {
    if (!e->live_index) return 0;
    CK(cudaMemsetAsync(e->live_index, 0, e->live_index_cap * 16, e->stream));
    CK(cudaMemsetAsync(e->live_ctr, 0, sizeof(LiveCtr), e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->live_level_off.clear();
    return 0;
}

/* after vsr_engine_finish_level advanced: the level now current (depth e->level) goes into the store */
int live_collect(VsrEngine* e) {
    LiveParams q = live_params(e);
    q.in = e->frontier[e->cur].view();
    q.n_in = e->n_cur;
    q.in_base = e->cur_base;
    std::vector<uint64_t>& off = e->live_level_off; /* off[d - 1] .. off[d]: depth d */
    if (off.empty()) off.push_back(0);
    while (off.size() < (size_t)e->level) off.push_back(off.back());
    CK(e->g->launch_live_collect(q, e->sms, e->stream));
    e->st.kernel_launches++;
    LiveCtr c;
    CK(cudaMemcpyAsync(&c, e->live_ctr, sizeof c, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->st.bytes_d2h += sizeof c;
    off.push_back(std::min<uint64_t>(c.count, e->live_words.capacity()));
    if (c.overflow) {
        snprintf(e->last_error, sizeof e->last_error, "capacity exceeded (liveness %s): %llu not-P states at depth %d, the store holds %llu "
                 "(%llu in HBM; frontier_host_capacity > 0 lets it continue in host memory)", c.overflow == 1 ? "store" : "index",
                 (unsigned long long)c.count, e->level, (unsigned long long)e->live_words.capacity(), (unsigned long long)e->live_words.hbm_rows);
        return VSR_RC_TOO_LARGE;
    }
    if (c.error) {
        snprintf(e->last_error, sizeof e->last_error, "liveness store: error %d at depth %d (a state stored twice)", c.error, e->level);
        if (!e->st.error_code) e->st.error_code = c.error;
        return VSR_RC_ERROR;
    }
    return 0;
}

extern "C" {

int vsr_engine_liveness(VsrEngine* e, VsrLiveStats* out, uint32_t* cands_out, size_t cands_cap) {
    if (!e || !out) return VSR_RC_ERROR;
    memset(out, 0, sizeof *out);
    const double t0 = now_s();
    auto refuse = [&](int rc, const char* msg) {
        snprintf(e->last_error, sizeof e->last_error, "%s", msg);
        out->rc = rc;
        return rc;
    };
    if (!e->live_index) return refuse(VSR_RC_CONFIG_ERROR, "the model has no PROPERTY: there is nothing to check");
    if (e->world != 1) return refuse(VSR_RC_CONFIG_ERROR, "liveness is checked on one GPU only");
    if (e->level < 1 || e->n_cur != 0 || e->level_open)
        return refuse(VSR_RC_CONFIG_ERROR, "temporal properties are checked on a complete state graph only: the BFS has not finished");
    /* the level off table has one entry per level collected, + 1: off[d - 1] .. off[d] is depth d */
    const std::vector<uint64_t>& off = e->live_level_off;
    const int nlev = (int)off.size() - 1;
    const uint64_t stored = live_stored(e);
    out->stored = stored;
    out->capacity = e->live_words.capacity();
    out->bytes_hbm = e->live_bytes_hbm;
    out->bytes_host = e->live_bytes_host;
    out->violation_index = ~0ull;
    CK(cudaSetDevice(e->device));
    CK(cudaMemsetAsync(e->live_alive, 0xFF, e->live_words.capacity() / 8, e->stream));
    LiveParams q = live_params(e);
    LiveCtr c;
    memset(&c, 0, sizeof c);
    for (int sweep = 0; stored; sweep++) {
        LiveCtr z = c; /* count kept; the per-sweep fields cleared */
        z.killed = z.alive = 0;
        z.alive_min = ~0ull;
        if (sweep == 0) { z.sinks = 0; z.sink_min = ~0ull; }
        CK(cudaMemcpyAsync(e->live_ctr, &z, sizeof z, cudaMemcpyHostToDevice, e->stream));
        CK(cudaStreamSynchronize(e->stream)); /* z lives on this stack frame */
        q.first_sweep = sweep == 0;
        CK(cudaEventRecord(e->ev0, e->stream));
        for (int d = nlev; d >= 1; d--) { /* deepest first: a state's successors are mostly one level deeper, already swept */
            q.first = off[d - 1];
            q.n = off[d] - off[d - 1];
            CK(e->g->launch_live_sweep(q, e->sms, e->stream));
            e->st.kernel_launches++;
        }
        CK(cudaEventRecord(e->ev1, e->stream));
        CK(cudaMemcpyAsync(&c, e->live_ctr, sizeof c, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        float ms = 0;
        cudaEventElapsedTime(&ms, e->ev0, e->ev1);
        if (sweep < VSR_MAX_SWEEPS) out->ms_sweep[sweep] = ms;
        out->sweeps = sweep + 1;
        if (c.error) {
            out->error_code = c.error;
            if (!e->st.error_code) e->st.error_code = c.error;
            snprintf(e->last_error, sizeof e->last_error, "liveness sweep %d: error %d (%s)", sweep + 1, c.error,
                     c.error == E_LIVE_MISSING ? "a reachable not-P state is missing from the store: the BFS and the store disagree" : "a successor cannot be represented");
            out->rc = VSR_RC_ERROR;
            out->seconds_total = now_s() - t0;
            return VSR_RC_ERROR;
        }
        if (sweep == 0) out->sinks = c.sinks;
        if (c.sinks) break; /* a sink decides the verdict: no more sweeps */
        if (c.killed == 0) {
            out->survivors = c.alive;
            break;
        }
    }
    if (out->sinks) out->violation_index = c.sink_min;
    else if (out->survivors) out->violation_index = c.alive_min;
    if (out->violation_index == ~0ull) {
        out->seconds_total = now_s() - t0;
        return 0;
    }
    out->rc = VSR_RC_LIVENESS;
    const uint64_t vi = out->violation_index;
    for (int d = 1; d <= nlev; d++)
        if (vi >= off[d - 1] && vi < off[d]) out->violation_level = d;
    /* ---- the lasso: the BFS trace from Init to the reported state ... */
    const ModelOps* ops = e->m->ops;
    const RunCfg& run = e->m->run;
    const int S = ops->bytes, hooks = e->m->live_hooks;
    std::vector<uint32_t> prefix, walk;
    if (!e->trace_cap || !cands_out) { /* no parent records kept: the verdict without a counterexample */
        out->seconds_total = now_s() - t0;
        return VSR_RC_LIVENESS;
    }
    unsigned long long local_id = 0;
    CK(cudaMemcpy(&local_id, e->live_ids + vi, 8, cudaMemcpyDeviceToHost));
    if (walk_trace(e, local_id, prefix)) return VSR_RC_ERROR;
    uint32_t cur[VSR_MAX_STATE_BYTES / 4], nx[VSR_MAX_STATE_BYTES / 4], init[VSR_MAX_STATE_BYTES / 4];
    CK(e->live_words.to_host(vi, 1, cur));
    ops->init(init);
    auto key = [&](const uint32_t* w) {
        uint64_t fp = ops->fingerprint(w, run.use_view);
        return std::make_pair(fp ? fp : 1, e->g->check_hash(w, run.use_view));
    };
    int loop = 0, loop_action = 0;
    if (!out->sinks) { /* ... then, for a cycle, along the first alive not-P successor until a state repeats */
        std::map<std::pair<uint64_t, uint32_t>, int> seen; /* walk state -> its position (0 = the reported state) */
        seen[key(cur)] = 0;
        unsigned long long *dkeys = nullptr, *dres = nullptr;
        CK(cudaMalloc(&dkeys, 16ull * ops->ncand));
        CK(cudaMalloc(&dres, 8ull * ops->ncand));
        std::vector<unsigned long long> hkeys(2 * ops->ncand), hres(ops->ncand);
        std::vector<int> hcand(ops->ncand);
        bool restarted = false;
        int rc = 0;
        for (int steps = 0; !loop && !rc; steps++) {
            if (steps > (1 << 22)) { rc = VSR_RC_ERROR; break; }
            const auto me = key(cur);
            int n = 0, nonself = 0;
            for (int cnd = 0; cnd < ops->ncand; cnd++) {
                if (!ops->guard(&run, cur, cnd)) continue;
                if (ops->step(&run, cur, cnd, nx) <= 0) continue;
                const auto k = key(nx);
                if (k == me) continue;
                nonself++;
                if (ops->property(&run, nx, hooks)) continue;
                hkeys[2 * n] = k.first;
                hkeys[2 * n + 1] = k.second;
                hcand[n++] = cnd;
            }
            int pick = -1;
            if (n) {
                if (cudaMemcpy(dkeys, hkeys.data(), 16ull * n, cudaMemcpyHostToDevice) != cudaSuccess) { rc = VSR_RC_SYSTEM; break; }
                live_lookup_kernel<<<(n + 127) / 128, 128>>>(e->live_index, e->live_index_cap, e->live_alive, dkeys, n, dres);
                if (cudaMemcpy(hres.data(), dres, 8ull * n, cudaMemcpyDeviceToHost) != cudaSuccess) { rc = VSR_RC_SYSTEM; break; }
                for (int i = 0; i < n && pick < 0; i++)
                    if (hres[i] >> 63) pick = i;
            }
            if (pick < 0) {
                if (!nonself && (hooks & LIVE_HOOK_INIT_EDGE)) { /* the test hook's edge to Init: the loop starts over at Init */
                    if (restarted) { loop = 1; loop_action = 0; break; }
                    restarted = true;
                    prefix.clear();
                    walk.clear();
                    seen.clear();
                    memcpy(cur, init, S);
                    seen[key(cur)] = 0;
                    continue;
                }
                rc = VSR_RC_ERROR; /* an alive state without an alive successor: the sweeps did not reach their fixpoint */
                break;
            }
            ops->step(&run, cur, hcand[pick], nx);
            const auto k = key(nx);
            auto it = seen.find(k);
            if (it != seen.end()) {
                loop = (int)prefix.size() + it->second + 1;
                loop_action = ops->action_of(hcand[pick]);
                break;
            }
            walk.push_back((uint32_t)hcand[pick]);
            seen[k] = (int)walk.size();
            memcpy(cur, nx, S);
        }
        cudaFree(dkeys);
        cudaFree(dres);
        if (rc) {
            snprintf(e->last_error, sizeof e->last_error, "liveness: the lasso walk from store index %llu found no alive successor", (unsigned long long)vi);
            out->rc = rc;
            return rc;
        }
    }
    prefix.insert(prefix.end(), walk.begin(), walk.end());
    const size_t n = std::min(prefix.size(), cands_cap);
    memcpy(cands_out, prefix.data(), n * sizeof(uint32_t));
    out->trace_len = (int)n;
    out->trace_loop = loop;
    out->trace_loop_action = loop_action;
    out->seconds_total = now_s() - t0;
    return VSR_RC_LIVENESS;
}

} /* extern "C" */
