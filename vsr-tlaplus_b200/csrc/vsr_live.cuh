/*
 * vsr_live.cuh — device side of the liveness pass (PROPERTY ViewChangeCompletes; host side: vsr_live.cu).
 *
 *   live_collect_kernel  after a BFS level: appends the level's not-P states to the store (words, local id) and inserts
 *                        each into the live index, an open-addressed table of the seen-set's {fp, meta} entries (the same
 *                        table_insert / table_lookup) whose meta is (store index + 1) << 32 | check hash
 *   live_sweep_kernel    one elimination pass over one level of the store: a state stays alive iff some successor other
 *                        than itself (same fingerprint and check hash) is a not-P state that is alive.  Successors come from
 *                        the BFS's own step function (Ops::step), one thread per stored state over all candidates.
 */
#ifndef VSR_LIVE_CUH
#define VSR_LIVE_CUH

#include "vsr_gpu.cuh"

namespace vsr {

struct LiveCtr {
    unsigned long long count;     /* states stored (all levels) */
    unsigned long long killed;    /* per sweep: states found dead */
    unsigned long long alive;     /* per sweep: states found alive */
    unsigned long long alive_min; /* per sweep: smallest store index found alive */
    unsigned long long sinks;     /* first sweep: not-P states without a successor other than themselves */
    unsigned long long sink_min;  /* smallest store index of such a state (~0 = none) */
    int error;                    /* first E_* */
    int overflow;                 /* 1 store full, 2 live index full */
};

struct LiveParams {
    /* collect: the level just finished, n_in states of L::NW words */
    SpillRows in;
    unsigned long long n_in, in_base;
    /* the store: state s is words' row s */
    SpillRows words;
    unsigned long long cap;
    unsigned long long* ids;      /* local (BFS) id of each stored state */
    uint64_t* index;
    unsigned long long index_cap;
    uint32_t* alive;              /* one bit per store index */
    LiveCtr* ctr;
    const uint64_t* fp_tab;
    RunCfg run;
    int hooks;                    /* LIVE_HOOK_* (vsr_model.h) */
    int first_sweep;
    unsigned long long first, n;  /* sweep: store indices [first, first + n) */
};

template <class L> __global__ void live_collect_kernel(const LiveParams P) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    /* blockDim is a multiple of 32: a warp enters and leaves the loop together (the ballot needs all lanes) */
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i - lane < P.n_in; i += stride) {
        uint32_t w[L::NW];
        bool take = false;
        if (i < P.n_in) {
            const uint32_t* st = P.in.row<L::NW>(i);
            for (int j = 0; j < L::NW; j++) w[j] = st[j];
            take = !Ops<L>::live_pred(P.run, w, P.hooks);
        }
        const unsigned m = __ballot_sync(0xffffffffu, take);
        unsigned long long base = 0;
        if (lane == 0 && m) base = atomicAdd(&P.ctr->count, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (!take) continue;
        const unsigned long long s = base + __popc(m & ((1u << lane) - 1u));
        if (s >= P.cap) {
            atomicCAS(&P.ctr->overflow, 0, 1);
            continue;
        }
        uint32_t* dst = P.words.row<L::NW>(s);
        for (int j = 0; j < L::NW; j++) dst[j] = w[j];
        P.ids[s] = P.in_base + i;
        uint64_t fp = fp64_view8<L>(P.fp_tab, w, P.run.use_view != 0);
        if (fp == 0) fp = 1;
        const uint32_t chk = check_hash<L>(w, P.run.use_view != 0);
        unsigned probes = 0, coll = 0;
        const int r = table_insert(P.index, P.index_cap, fp, ((uint64_t)(s + 1) << 32) | chk, probes, coll);
        if (r == INS_FULL) atomicCAS(&P.ctr->overflow, 0, 2);
        else if (r != INS_NEW) atomicCAS(&P.ctr->error, 0, E_LIVE_DUP);
    }
}

/* one edge of the liveness graph from the state with (fps, chks) to `nx`: false for a self-loop (stuttering), else counts
   it in `nonself` and returns whether nx is a not-P state that is alive */
template <class L> __device__ __forceinline__ bool live_edge(const LiveParams& P, const uint32_t* nx, uint64_t fps, uint32_t chks, int& nonself) {
    uint64_t fp = fp64_view8<L>(P.fp_tab, nx, P.run.use_view != 0);
    if (fp == 0) fp = 1;
    const uint32_t chk = check_hash<L>(nx, P.run.use_view != 0);
    if (fp == fps && chk == chks) return false;
    nonself++;
    if (Ops<L>::live_pred(P.run, nx, P.hooks)) return false;
    const uint64_t meta = table_lookup(P.index, P.index_cap, fp, chk);
    if (!meta) { /* a reachable not-P state the store does not have: the BFS and the store disagree */
        atomicCAS(&P.ctr->error, 0, E_LIVE_MISSING);
        return false;
    }
    const unsigned long long j = (meta >> 32) - 1;
    return (P.alive[j >> 5] >> (j & 31)) & 1u;
}

template <class L> __global__ void live_sweep_kernel(const LiveParams P) {
    unsigned long long killed = 0, alive = 0, alive_min = ~0ull;
    const unsigned long long end = P.first + P.n;
    for (unsigned long long s = P.first + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s < end; s += (unsigned long long)gridDim.x * blockDim.x) {
        if (!((P.alive[s >> 5] >> (s & 31)) & 1u)) continue;
        uint32_t w[L::NW], nx[L::NW];
        const uint32_t* st = P.words.row<L::NW>(s);
        for (int j = 0; j < L::NW; j++) w[j] = st[j];
        uint64_t fps = fp64_view8<L>(P.fp_tab, w, P.run.use_view != 0);
        if (fps == 0) fps = 1;
        const uint32_t chks = check_hash<L>(w, P.run.use_view != 0);
        int nonself = 0;
        bool found = false;
        for (int c = 0; c < L::NCAND && !found; c++) {
            const int r = Ops<L>::template step<true>(P.run, (const uint32_t*)w, c, (uint32_t*)nx);
            if (r == 0) continue;
            if (r < 0) { atomicCAS(&P.ctr->error, 0, r); continue; }
            found = live_edge<L>(P, nx, fps, chks, nonself);
        }
        if (!found && nonself == 0 && (P.hooks & 2)) { /* test hook: a state without successors steps to Init */
            Ops<L>::init(nx);
            found = live_edge<L>(P, nx, fps, chks, nonself);
        }
        if (nonself == 0 && P.first_sweep) {
            atomicAdd(&P.ctr->sinks, 1ull);
            atomicMin(&P.ctr->sink_min, s);
        }
        if (found) {
            alive++;
            if (s < alive_min) alive_min = s;
        } else {
            atomicAnd(&P.alive[s >> 5], ~(1u << (s & 31)));
            killed++;
        }
    }
    for (int o = 16; o; o >>= 1) {
        killed += __shfl_xor_sync(0xffffffffu, killed, o);
        alive += __shfl_xor_sync(0xffffffffu, alive, o);
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, alive_min, o);
        if (other < alive_min) alive_min = other;
    }
    if ((threadIdx.x & 31) == 0) {
        if (killed) atomicAdd(&P.ctr->killed, killed);
        if (alive) {
            atomicAdd(&P.ctr->alive, alive);
            atomicMin(&P.ctr->alive_min, alive_min);
        }
    }
}

} // namespace vsr
#endif
