/*
 * vsr_gpu.cuh — device side of the BFS wavefront (sm_90a).
 *
 * One launch of expand_kernel<L> = TLC's worker loop (SURVEY §3.1 / §8a stages E1-E9) over one BFS
 * level of packed VSR.tla states:
 *   E1  successor enumeration   Ops<L>::step over the candidate (action, binding) index space
 *   E2  SYMMETRY                kept incrementally by step (canonical value labels)
 *   E3  VIEW                    mask of the aux bits inside fp64_view
 *   E4  fingerprint             FP64 (Rabin, slicing-by-8 tables in shared memory) of the packed VIEW bytes + a 32-bit check hash
 *   E5  seen-set                open-addressed HBM table of 16-byte {fp, meta} entries, one 128-bit load per
 *                               probe (issued as soon as the fingerprint is known), insertion by one 128-bit CAS
 *                               (ATOMG.E.CAS.128); probing is bounded, a full table is an error, never a spin
 *   E6  queue                   next frontier staged per warp in shared memory, flushed 32 states at a time
 *                               by a TMA bulk store (cp.async.bulk.global.shared::cta, UBLKCP)
 *   E7  invariant               evaluated inline on every newly inserted state
 *   E8  trace                   (parent id, candidate) per new state
 *   E9  deadlock                states with no enabled candidate
 * Work shape (SURVEY H5): a block takes 32*WARPS frontier states, one per thread.  SCAN: every thread copies its state
 * into registers and evaluates all guards of Next on it with compile-time candidate indices (Ops::enabled_group): one bit
 * per (action, binding); the enabled (state, candidate) pairs are written to a block pool grouped by action (packed warp
 * prefix sums, one shared atomic per warp and action group, one barrier).  APPLY: warps take batches of 32 pairs of ONE
 * action and apply them one per lane — the successor is built in a rotated shared-memory row, read once into registers,
 * fingerprinted, probed, inserted — so the expensive part runs with full lanes and without divergence between actions.
 */
#ifndef VSR_GPU_CUH
#define VSR_GPU_CUH

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vsr_flat.h" /* VSR_ACT_*, VSR_NUM_ACTIONS */
#include "vsr_actions.h"
#include "vsr_spill.cuh"

namespace vsr {

struct DevCounters {
    unsigned long long out_count;   /* states appended to the next frontier this level */
    unsigned long long generated;   /* successors generated (TLC's count: one per binding) */
    unsigned long long ties;        /* same-level VIEW ties with a different aux key */
    unsigned long long collisions;  /* fp equal, check hash different */
    unsigned long long probes;      /* table entries inspected */
    unsigned long long viol_id;     /* smallest global id of a violating new state (~0 = none) */
    unsigned long long dead_id;     /* smallest global id of an expanded state without successors */
    unsigned long long tie_count;   /* entries in the tie list */
    int error;                      /* first E_* raised */
    int overflow;                   /* next frontier / send buffer / tie list full */
    int viol_which;                 /* mask bit of the violated invariant */
    int _pad;
    /* per LAUNCH (one memset clears them): */
    unsigned long long work_next;   /* next round of frontier states to hand out */
    unsigned long long drain_next;  /* next chunk of inbox records to hand out */
    unsigned int send_count[8];     /* records pushed to each rank by this launch (MAX_WORLD) */
#ifdef VSR_EXP_ROUNDCLK
    unsigned long long roundclk[5]; /* warp-cycles of this launch by phase (CLK_*); printed per level by the host */
#endif
};
/* the engine's counter block: the coverage counters follow DevCounters, so that one memset clears and one copy reads both */
struct LevelCounters {
    DevCounters c;
    unsigned long long cover[2 * VSR_NUM_ACTIONS]; /* ExpandParams::cover */
};
#ifdef VSR_EXP_ROUNDCLK
/* phases of an expand warp's time: waiting at the end-of-round barrier, waiting at the scan's barriers (parents loaded,
   qcount final, pool written), applying batches, scanning (parent load, guards, pool layout), and the rest (start, drain, final flush) */
enum { CLK_END = 0, CLK_SCANBAR = 1, CLK_BATCH = 2, CLK_SCAN = 3, CLK_OTHER = 4 };
#endif

/* a same-level VIEW tie (SURVEY H2): header, then the candidate's L::NW packed words */
struct TieRec {
    uint64_t fp;
    uint64_t parent;
    uint32_t auxkey, cand, check, _pad;
};

/* record shipped to the owner rank of a successor: the state's words, then this 16-byte header.  The owner recomputes the
   check hash and the aux key from the words (a few dozen instructions); the 64-bit fingerprint travels because computing
   it is the expensive part and the sender needs it anyway to find the owner. */
struct RecHdr {
    uint64_t fp;
    uint64_t tm; /* trace record (parent global id << 12 | candidate, 56 bits) | mult << 56 */
};
constexpr int MAX_WORLD = 8;


struct ExpandParams {
    SpillRows in;                /* current frontier, n_in states of L::NW words (both frontiers may spill: vsr_spill.cuh) */
    unsigned long long n_in;
    unsigned long long in_base;  /* local id of in's row 0 */
    SpillRows out;               /* next frontier */
    unsigned long long out_cap;  /* states the next frontier holds in all (HBM part + host part) */
    unsigned long long out_base; /* local id of out's row 0 */
    uint64_t* table;             /* capacity entries of {fp, meta} */
    unsigned long long table_cap; /* entries: any multiple of VSR_BUCKET (not only powers of two: memory-bound configs size the seen-set to what is left) */
    SpillRows trace;             /* per local id: make_trec(parent global id, candidate), rows of 2 words (HBM, or host memory) */
    unsigned long long trace_cap; /* 0: no trace, never dereferenced */
    DevCounters* ctr;
    uint8_t* ties;               /* tie_cap entries of sizeof(TieRec) + L::BYTES */
    unsigned long long tie_cap;
    const uint64_t* fp_tab;      /* 8 x 256 FP64 slicing tables */
    RunCfg run;
    int level;                   /* depth of the states being GENERATED (Init = 1) */
    int check_deadlock;
    int rank, world, owner_shift;/* owner(fp) = owner_of(fp, owner_shift) (world a power of two; shift 64 when world = 1) */
    /* world > 1.  push[d] = where THIS rank's records for rank d go: its segment of rank d's inbox, in rank d's memory,
       mapped here over NVLink (CUDA IPC / peer access) — the expand kernel stores them there itself — or a local staging
       buffer when the host moves them with a collective.  Slots are taken from the local counters ctr->send_count[d]. */
    uint8_t* push[MAX_WORLD];
    unsigned long long push_cap; /* records per segment */
    /* records received from rank s in the previous step (the other half of the double-buffered inbox): inserted by this
       launch after its share of the frontier.  Init and vsr_engine_insert_records come this way too, as drain[0] of a
       launch with no frontier share */
    const uint8_t* drain[MAX_WORLD];
    unsigned int drain_n[MAX_WORLD];
    unsigned long long drain_total;
    /* action coverage (the COVER instantiation only; NULL otherwise): [2][VSR_NUM_ACTIONS] counters of the level being
       generated, by the action of the inserted record's candidate: sum of mult ("states generated"), then first arrivals */
    unsigned long long* cover;
};

/* ------------------------------------------------------------------ primitives */

__device__ __forceinline__ void cas128(uint64_t* p, uint64_t s0, uint64_t s1, uint64_t& o0, uint64_t& o1) {
    /* compare with {0,0} (empty slot), swap in {s0,s1}; returns the previous contents */
    asm volatile(
        "{\n\t.reg .b128 cmp, swp, old;\n\tmov.b128 cmp, {%2, %3};\n\tmov.b128 swp, {%4, %5};\n\t"
        "atom.global.relaxed.gpu.cas.b128 old, [%6], cmp, swp;\n\tmov.b128 {%0, %1}, old;\n\t}"
        : "=l"(o0), "=l"(o1)
        : "l"(0ull), "l"(0ull), "l"(s0), "l"(s1), "l"(p)
        : "memory");
}
__device__ __forceinline__ void ld128_cg(const uint64_t* p, uint64_t& a, uint64_t& b) {
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ uint64_t mix64(uint64_t x) { /* splitmix64 finaliser */
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
    x ^= x >> 27; x *= 0x94d049bb133111ebULL;
    x ^= x >> 31;
    return x;
}
template <class L, bool USE_VIEW, class W> VSR_HD uint32_t check_hash_t(const W& w) {
    /* second, independent 32-bit hash of the VIEW words (3 instructions per word + finaliser): lets the seen-set tell
       fp64 collisions apart instead of silently merging two states as a bare fingerprint set would */
    constexpr int full = L::VIEW_BITS >> 5, rem = L::VIEW_BITS & 31;
    constexpr int nw = USE_VIEW ? (full + (rem ? 1 : 0)) : L::NW;
    uint32_t h = 0x9747b28cu;
VSR_UNROLL
    for (int i = 0; i < nw; i++) {
        uint32_t k = rdw(w, i);
        if (USE_VIEW && i == full) k &= (1u << rem) - 1u;
        h ^= k;
        h = ((h << 13) | (h >> 19)) * 5u + 0xe6546b64u;
    }
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}
template <class L, class W> VSR_HD uint32_t check_hash(const W& w, bool use_view) {
    return use_view ? check_hash_t<L, true>(w) : check_hash_t<L, false>(w);
}

enum { INS_NEW = 0, INS_DUP = 1, INS_TIE = 2, INS_FULL = 3 };

/* global state id = rank << 40 | local id (44 bits; all ones = "no parent": Init); trace record = global id of the parent
   << 12 | candidate index (56 bits; bit 63 is a transient "violates the invariant" mark inside the staging area, bits
   56..59 carry mult in records that travel between ranks) */
constexpr unsigned long long GID_MASK = (1ull << 44) - 1ull, ROOT_GID = GID_MASK;
__host__ __device__ __forceinline__ uint64_t make_gid(int rank, unsigned long long local_id) { return ((uint64_t)rank << 40) | local_id; }
__host__ __device__ __forceinline__ uint64_t make_trec(uint64_t parent_gid, uint32_t cand) { return (parent_gid << 12) | (cand & 0xFFFu); }

__device__ __forceinline__ uint64_t make_meta(int level, uint32_t auxkey, uint32_t check) {
    return ((uint64_t)(uint32_t)level << 56) | ((uint64_t)(auxkey & 0xFFFFFFu) << 32) | check;
}

/* lock-free insert-if-absent over 16-byte entries {fp, meta}.  A probe reads one BUCKET of VSR_BUCKET consecutive entries
   (1: one 128-bit load; 2: one 32-byte sector; 4: two sectors, read by ld256_cg, all four 128-bit loads issued together) and
   walks to the next bucket only when every slot of this one holds another state.
   Slots of a bucket fill in order (no deletions), so a lookup may stop at the first empty slot.  The bucket's first entry
   (for VSR_BUCKET 4: all of it) is loaded by the caller as early as the fingerprint is known so that the HBM round trip
   overlaps the rest of the successor's work.  With 2-entry buckets the second entry is read only when the first holds
   another state: it is in L2 by then (same sector), and most inserts and duplicates end at the first entry.  Every
   128-bit load of a warp gathers 32 random sectors, and those gathers bind the kernel: reading the whole sector up front
   cost 9 % of the kernel time on an H100 (profiles/probe_gathers_h100.md). */
#ifndef VSR_BUCKET
#define VSR_BUCKET 2
#endif
struct Probe { uint64_t e[2 * VSR_BUCKET]; };
__device__ __forceinline__ void ld256_cg(const uint64_t* p, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
    /* one 32-byte sector.  sm_90 has no 256-bit load: two 128-bit loads of the same sector, issued back to back so that
       both are in flight together and cost one HBM round trip */
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%4];\n\tld.global.cg.v2.u64 {%2, %3}, [%4+16];"
                 : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p) : "memory");
}
__device__ __forceinline__ unsigned long long table_home(unsigned long long cap, uint64_t fp) {
    /* bucket = floor(hash * nbuckets / 2^64): any capacity, no division.  The hash is the fingerprint times an odd constant
       (the owner rank is the fingerprint's HIGH bits, so they must not select the bucket on their own) */
    return __umul64hi(fp * 0x9E3779B97F4A7C15ULL, cap / VSR_BUCKET) * VSR_BUCKET;
}
__device__ __forceinline__ void probe_load(const uint64_t* table, unsigned long long h, Probe& p) {
#if VSR_BUCKET == 1
    ld128_cg(table + 2 * h, p.e[0], p.e[1]);
#elif VSR_BUCKET == 2
    ld128_cg(table + 2 * h, p.e[0], p.e[1]); /* the bucket's first entry only: table_insert_from reads the second on demand */
#elif VSR_BUCKET == 4
    ld256_cg(table + 2 * h, p.e[0], p.e[1], p.e[2], p.e[3]);
    ld256_cg(table + 2 * h + 4, p.e[4], p.e[5], p.e[6], p.e[7]);
#else
#error "VSR_BUCKET must be 1, 2 or 4"
#endif
}
__device__ __forceinline__ int table_insert_from(uint64_t* table, unsigned long long cap, unsigned long long h, Probe p, uint64_t fp, uint64_t meta,
                                                 unsigned& probes, unsigned& collisions) {
    for (unsigned tries = 0;; tries++) {
        if (tries > (1u << 16)) return INS_FULL; /* the table is (nearly) full: never spin forever, the host aborts with 152 */
        probes++;
VSR_UNROLL
        for (int j = 0; j < VSR_BUCKET; j++) {
            uint64_t e0, e1;
            if (VSR_BUCKET == 2 && j == 1) {
                ld128_cg(table + 2 * (h + 1), e0, e1); /* the first entry holds another state */
            } else {
                e0 = p.e[2 * j];
                e1 = p.e[2 * j + 1];
            }
            if (e0 == 0) {
                cas128(table + 2 * (h + j), fp, meta, e0, e1);
                if (e0 == 0 && e1 == 0) return INS_NEW;
            }
            for (int again = 0; e1 == 0 && again < 64; again++) ld128_cg(table + 2 * (h + j), e0, e1); /* half-visible entry: look again */
            if (e0 == fp) {
                if ((uint32_t)e1 == (uint32_t)meta) {
                    const bool same_level = (e1 >> 56) == (meta >> 56);
                    const bool same_aux = ((e1 >> 32) & 0xFFFFFF) == ((meta >> 32) & 0xFFFFFF);
                    return (same_level && !same_aux) ? INS_TIE : INS_DUP;
                }
                collisions++;
            }
        }
        h += VSR_BUCKET;
        if (h >= cap) h = 0;
        probe_load(table, h, p);
    }
}
__device__ __forceinline__ int table_insert(uint64_t* table, unsigned long long cap, uint64_t fp, uint64_t meta,
                                            unsigned& probes, unsigned& collisions) {
    const unsigned long long h = table_home(cap, fp);
    Probe p;
    probe_load(table, h, p);
    return table_insert_from(table, cap, h, p, fp, meta, probes, collisions);
}

/* ------------------------------------------------------------------ expand kernel */

#ifdef VSR_QPS
constexpr int QPS = VSR_QPS;  /* tools/variants.sh "qps1": a pool so small that the overflow path (leftovers) runs all the time */
#else
constexpr int QPS = 10;       /* pool entries per parent state (pool = QPS * states per block round) */
#endif

/* a warp's staging area of ROWS rows: new states, packed back to back for the bulk store; its last 32 rows are the lanes'
   scratch rows while a batch builds its successors.  ROWS 64: flushed 32 states at a time (Expander::commit).  ROWS 32:
   every batch flushes all its new states, which halves the area; the two-pass round needs that space */
template <class L, int ROWS> struct WarpStage {
    alignas(16) uint32_t stage[ROWS * L::NW + 32]; /* (+ room for the skew of the scratch rows, Expander::scratch) */
    unsigned long long tstage[ROWS];             /* their trace records */
    /* per-warp running state.  It lives here, not in the Expander object: the big per-action routines are real calls
       (one copy of each in the instruction cache), and an object whose address is passed to them would be kept in
       local memory — 1024 threads x a few hundred bytes does not fit the L1 left beside 220 KB of shared memory. */
    int sn;                                      /* states currently staged */
};
template <class L, int WARPS, int PASSES> struct BlockSmemT {
    typedef WarpStage<L, PASSES == 2 ? 32 : 64> Stage;
    static constexpr int NS = WARPS * 32;        /* parent states per scan pass: one per thread */
    static constexpr int NR = PASSES * NS;       /* parent states per block round */
    static constexpr int NG = 13;                /* action groups (Ops<L>::NGRP) */
    uint64_t fp_tab[8 * 256];                    /* FP64 slicing-by-8 tables */
    uint32_t par[NR * (L::NW + 1)];              /* parents, row stride NW+1 (odd: bank-conflict-free column reads) */
    static constexpr int QCAP = QPS * NS;        /* pool entries per pass */
    uint16_t pool[PASSES * QCAP];                /* enabled (state, candidate) pairs, by pass, then grouped by action */
    int qcount[PASSES][NG];                      /* pairs found per pass and group (may exceed what the pool holds) */
    int take;
    unsigned long long round_first;
    Stage w[WARPS];
};
/* Block shape.  ONE block of up to 32 warps per SM when its shared memory fits (227 KB), else two blocks of 16 / 12 / 8 warps
   (2 x <= 113 KB).  One block of 32 warps — rounds of 1024 parents — rather than two blocks of 16 with the same 32 resident warps:
   the end-of-round tail (the barrier stall) halves, and all warps of the SM run the same phase, so they share the instruction
   cache lines of the scan.  The pool item keeps 16 bits: thread (10) | candidate offset in its group (6), which bounds a group at 63 candidates.
   Two scan passes per round when the shared memory holds them (one block per SM only): rounds of 2 x 32 x WARPS parents, so
   the end-of-round barrier, where every warp waits for the slowest warp's last batch, comes once per two passes.  It took
   12 % of the warp-cycles at one pass per round on an H100 (profiles/round_tail_h100.md).  The two-pass round uses the
   32-row staging area (a flush per batch) to fit; the warps are counted with the one-pass block, so both shapes have the
   same warps and register budget.  A flush per batch costs where a batch finds few new states: 6-9 % on five replicas
   (g ~ 7), so one-pass layouts keep the 64-row area. */
template <class L> struct ExpandCfg {
    static constexpr size_t SMEM_ONE = 227 * 1024 - 512, SMEM_TWO = 113 * 1024;
    static constexpr int max_grp() { int m = 0; for (int g = 0; g < Ops<L>::NGRP; g++) m = Ops<L>::grp_size(g) > m ? Ops<L>::grp_size(g) : m; return m; }
    template <int W> static constexpr int pick_one() { /* most warps (even) of ONE block per SM; 0: not even 18 fit */
        if constexpr (W < 18) return 0;
        else if constexpr (sizeof(BlockSmemT<L, W, 1>) <= SMEM_ONE) return W;
        else return pick_one<W - 2>();
    }
    static constexpr int W2 = sizeof(BlockSmemT<L, 16, 1>) <= SMEM_TWO ? 16 : (sizeof(BlockSmemT<L, 12, 1>) <= SMEM_TWO ? 12 : 8);
    static constexpr int W1 = max_grp() < 64 ? pick_one<32>() : 0;
#ifdef VSR_FORCE_WARPS
    static constexpr int WARPS = VSR_FORCE_WARPS; /* tuning experiments only */
#else
    static constexpr int WARPS = W1 >= 2 * W2 - 4 ? W1 : W2; /* one block unless it would cost more than 4 resident warps */
#endif
    static constexpr int BLOCKS = WARPS > 16 ? 1 : 2;
#ifdef VSR_ROUND_PASSES
    static constexpr int PASSES = VSR_ROUND_PASSES; /* A/B: tools/variants.sh "passes1" */
#else
    static constexpr int PASSES = BLOCKS == 1 && sizeof(BlockSmemT<L, WARPS, 2>) <= SMEM_ONE ? 2 : 1;
#endif
    typedef BlockSmemT<L, WARPS, PASSES> Smem;
    /* the compile-time limits a layout must meet (Expander and vsr_layout_plugin.cu assert them; tests/harness/layout_table.cu
       lists them for every layout) */
    static constexpr int NS = WARPS * 32;
    static constexpr int TBITS = NS <= 512 ? 9 : 10; /* pool item = thread (TBITS bits) | candidate offset in its group (the other 16 - TBITS) */
    static constexpr bool POOL_ITEM_FITS = NS <= (1 << TBITS) && max_grp() < (1 << (16 - TBITS));
    static constexpr bool POOL_COUNTERS_FIT = max_grp() * NS < 65536; /* 16-bit packed per-group counters of the scan */
    static constexpr size_t SMEM_SM = 227 * 1024;    /* shared memory of one SM that a block may have */
};

/*
 * Block-synchronous scan, action-pure apply.  A block takes NS = 32*WARPS frontier states (one per thread):
 *   scan   every thread copies its own state into registers and evaluates all of Next's guards on it with compile-time
 *          candidate indices: one bit per (action, binding).  The enabled (state, candidate) pairs are then laid out in
 *          a block pool grouped by action (packed warp prefix sums, one shared atomic per warp and group, one barrier).
 *   apply  after the second barrier, warps take batches of 32 pairs of ONE group and apply them one per lane: no
 *          divergence between actions inside a warp, full lanes except one partial batch per group.
 * Earlier forms: (1) every warp walking guards and effects on its own: 88 kB of SASS against the instruction cache;
 * (2) guards in a run-time loop over candidates with one ballot + barrier per group: 75 warp instructions per
 * (32 states, candidate) for slot decoding and shared-memory field reads; (3) this form: 16 per candidate.
 */
/* MULTI: the instantiation for several GPUs (push_records in emit, drain after the rounds), and for every launch that inserts
   records (Init, vsr_engine_insert_records).  The one-GPU expansion has none of that code: it costs the hot path registers
   (380 vs 140 bytes of spills in emit at the 64-register budget). */
/* COVER: the instantiation that also counts, per action of Next, what commit inserts (TLC's -coverage).  A run without
   coverage launches the instantiations without it: the same code as before the counters existed. */
template <class L, bool MULTI, bool COVER = false> struct Expander {
    typedef Ops<L> O_;
    typedef typename ExpandCfg<L>::Smem Smem;
    typedef typename Smem::Stage Stage;
    static constexpr int WARPS = ExpandCfg<L>::WARPS, NS = Smem::NS, PASSES = ExpandCfg<L>::PASSES;
    static constexpr int SROWS = PASSES == 2 ? 32 : 64; /* the staging area's rows (WarpStage) */
    const ExpandParams& P;
    Smem& B;
    Stage& S;
    const int lane, warp, tid;
    const uint32_t* mine = nullptr;
    bool have = false;
    int pass = 0; /* the round's scan pass in progress: this thread scans parent pass * NS + tid */
    __device__ __forceinline__ int pass_i() const { return PASSES == 1 ? 0 : pass; } /* a constant for one-pass layouts */

    __device__ Expander(const ExpandParams& p, Smem& b) : P(p), B(b), S(b.w[threadIdx.x >> 5]), lane(threadIdx.x & 31), warp(threadIdx.x >> 5), tid(threadIdx.x) {
#ifdef VSR_EXP_ROUNDCLK
        clk_t = clock64();
#endif
    }

#ifdef VSR_EXP_ROUNDCLK
    /* tools/variants.sh "roundclk": where each warp's cycles go.  clk_mark(i) books the cycles since the previous mark
       to phase i (CLK_*); finish() adds the warp's sums to DevCounters::roundclk */
    unsigned long long clk_t = 0, clk[5] = {};
    __device__ __forceinline__ void clk_mark(int i) {
        const unsigned long long t = clock64();
        clk[i] += t - clk_t;
        clk_t = t;
    }
#define VSR_CLK(X, i) (X).clk_mark(CLK_##i)
#else
#define VSR_CLK(X, i) ((void)0)
#endif

    /* flush the first n staged states (n <= 32) to the next frontier: one atomicAdd for the block of
       ids, one TMA bulk store for the states, then move the remainder (< 32 states) down */
    static __device__ __noinline__ void flush(const ExpandParams& P, Stage& S, int lane, int n) {
        const int sn = SROWS == 32 ? n : S.sn; /* 32 rows: the whole batch, nothing to move down */
        const SpillRows trace = P.trace; /* read before the atomic, whose latency hides these loads */
        const unsigned long long trace_cap = P.trace_cap;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(&P.ctr->out_count, (unsigned long long)n);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (lane < n) {
            const unsigned long long t = S.tstage[lane];
            if (t >> 63) { /* marked by the inline invariant check; now the id is known */
                atomicMin(&P.ctr->viol_id, P.out_base + base + lane);
                S.tstage[lane] = t & ~(1ull << 63);
            }
        }
        __syncwarp();
        if (base + n > P.out_cap) {
            if (lane == 0) atomicExch(&P.ctr->overflow, 1);
        } else {
            if (lane == 0) store_rows<L::NW>(P.out, base, S.stage, n);
            if (lane < n && P.out_base + base + lane < trace_cap) *(uint64_t*)trace.row<2>(P.out_base + base + lane) = S.tstage[lane];
        }
        __syncwarp();
        const int rest = sn - n;
        for (int i0 = 0; i0 < rest * L::NW; i0 += 32) {
            const int i = i0 + lane;
            uint32_t v = 0;
            if (i < rest * L::NW) v = S.stage[n * L::NW + i];
            __syncwarp();
            if (i < rest * L::NW) S.stage[i] = v;
        }
        unsigned long long t = 0;
        if (lane < rest) t = S.tstage[n + lane];
        __syncwarp();
        if (lane < rest) S.tstage[lane] = t;
        if (lane == 0) S.sn = rest;
        __syncwarp();
    }

    /* fingerprint, route, insert, stage: the part of apply that does not depend on the action */
    /* this lane's scratch row for the successor it builds: the last 32 staging rows are free whenever a batch starts (a
       64-row area holds fewer than 32 staged states then, a 32-row area none).  Plain rows, bank conflicts avoided by skewing the row STARTS (rather than
       rotating every access).  Rows of
       NW words collide every p = 32 / gcd(NW, 32) lanes; shifting lane l's row by l / p words puts the 32 lanes' word i in
       32 different banks, and an access is base + i: no per-access arithmetic. */
    typedef uint32_t* Row;
    static constexpr int gcd32(int a) { int g = 32; while (a % g) g >>= 1; return g; }
    static constexpr int SKEW_P = 32 / gcd32(L::NW);
    static __device__ __forceinline__ Row scratch(Stage& S, int lane) { return &S.stage[(SROWS - 32 + lane) * L::NW + lane / SKEW_P]; }

    /* Records for peer ranks (world > 1), pushed by the kernel itself: the lanes of the batch whose successor belongs to
       another rank lay their records out in destination order in the warp's 32 scratch rows (every lane has read its
       scratch row into registers by now, and the batch's new states are staged only after this), each destination's run
       takes its slots in that rank's inbox with ONE atomicAdd on a local counter, and the run leaves as ONE TMA bulk store
       (cp.async.bulk.global.shared::cta) to the peer's memory — over NVLink when push[] is a peer mapping.  Fire and
       forget: nothing waits for the remote write, the owner inserts the records in its next launch (drain).  The rows hold
       CAPREC records; a batch with more senders goes in two passes. */
    static __device__ __forceinline__ void push_records(const ExpandParams& P, Stage& S, int lane, const RegRow<L::NW>& v, int send_to, uint64_t fp,
                                                        uint64_t tm) {
        const unsigned senders = __ballot_sync(0xffffffffu, send_to >= 0);
        if (!senders) return;
        constexpr int RB = L::BYTES + (int)sizeof(RecHdr), RW = RB / 4;
        constexpr int CAPREC = (32 * L::BYTES) / RB;
        static_assert(CAPREC >= 16, "two passes must cover a batch");
        int off = 0, cnt = 0, rnk = 0; /* start of my destination's run in destination order, its length, my place in it */
        unsigned mymask = 0;
        for (int d = 0; d < P.world; d++) {
            const unsigned m = __ballot_sync(0xffffffffu, send_to == d);
            if (send_to > d) off += __popc(m);
            if (send_to == d) { mymask = m; cnt = __popc(m); rnk = __popc(m & ((1u << lane) - 1u)); }
        }
        unsigned base = 0;
        if (send_to >= 0 && rnk == 0) base = atomicAdd(&P.ctr->send_count[send_to], (unsigned)cnt);
        base = __shfl_sync(0xffffffffu, base, mymask ? __ffs(mymask) - 1 : 0);
        const bool fits = send_to >= 0 && (unsigned long long)base + (unsigned)cnt <= P.push_cap;
        if (send_to >= 0 && !fits && rnk == 0) atomicExch(&P.ctr->overflow, 3);
        const int pos = off + rnk, total = __popc(senders);
        uint32_t* sbuf = &S.stage[(SROWS - 32) * L::NW];
        for (int lo = 0; lo < total; lo += CAPREC) {
            const int hi = lo + CAPREC < total ? lo + CAPREC : total;
            if (send_to >= 0 && pos >= lo && pos < hi) {
                uint32_t* r = sbuf + (pos - lo) * RW;
                VSR_UNROLL
                for (int j = 0; j < L::NW; j++) r[j] = v.w[j];
                r[L::NW] = (uint32_t)fp; r[L::NW + 1] = (uint32_t)(fp >> 32);
                r[L::NW + 2] = (uint32_t)tm; r[L::NW + 3] = (uint32_t)(tm >> 32);
            }
            __syncwarp();
            if (fits) {
                const int st = off > lo ? off : lo, en = off + cnt < hi ? off + cnt : hi;
                if (pos == st && st < en)
                    bulk_store(P.push[send_to] + (size_t)(base + (unsigned)(st - off)) * RB, sbuf + (st - lo) * RW, (uint32_t)((en - st) * RB));
            }
            __syncwarp();
        }
    }

    /* ---- action coverage (COVER).  Counted where a state is inserted, so local successors, records drained from peers,
       Init and injected records are all counted once, at the owner (as `generated` is).  Per batch the warp aggregates by
       action — a batch of the pool holds one group, i.e. one or two actions; a drained chunk may hold more — and its first
       lane of each action adds the two sums to the block's table, which finish() adds to P.cover once per block.  The
       table is 320 bytes of static shared memory where the layout's block leaves them (cover_budget), else P.cover itself. */
    static constexpr int NCOV = 2 * VSR_NUM_ACTIONS;
    static constexpr size_t SMEM_SPARE = 512; /* static shared memory beside Smem: the round counter and the table */
    static_assert(NCOV * sizeof(unsigned long long) + sizeof(unsigned long long) <= SMEM_SPARE, "the table does not fit what ExpandCfg leaves beside Smem");
    static constexpr bool COVER_SHARED = sizeof(Smem) + SMEM_SPARE <= (ExpandCfg<L>::BLOCKS == 1 ? 227 * 1024 : 113 * 1024);
    static __device__ __forceinline__ unsigned long long* cover_table(const ExpandParams& P) {
        if constexpr (COVER_SHARED) {
            __shared__ unsigned long long tab[NCOV];
            return tab;
        } else {
            return P.cover;
        }
    }
    static __device__ __forceinline__ void cover_count(const ExpandParams& P, int lane, bool live, unsigned newmask, unsigned long long trec, unsigned gen) {
        const int a = !live ? -1 : (trec >> 12) == ROOT_GID ? (int)VSR_ACT_INIT : O_::action_of((int)(trec & 0xFFFu));
        unsigned long long* tab = cover_table(P);
        unsigned todo = __ballot_sync(0xffffffffu, a >= 0);
        while (todo) { /* warp-uniform: one turn per action present */
            const int first = __ffs(todo) - 1;
            const int act = __shfl_sync(0xffffffffu, a, first);
            const unsigned m = __ballot_sync(0xffffffffu, a == act);
            const unsigned g = __reduce_add_sync(0xffffffffu, a == act ? gen : 0u);
            if (lane == first) {
                atomicAdd(&tab[act], (unsigned long long)g);
                const int n = __popc(m & newmask);
                if (n) atomicAdd(&tab[VSR_NUM_ACTIONS + act], (unsigned long long)n);
            }
            todo &= ~m;
        }
    }

    /* the seen-set insert of one state per lane and everything after it — tie list, inline invariant, compaction of the
       survivors into the warp's staging area, flush — shared by the expansion (emit) and by the records of the drain
       (received from peers, Init, injected records): the only insert of a state in the library.  Returns this lane's
       counts for the run's statistics: successors generated (low half) | seen-set probes (high half); the caller keeps
       the running sums in registers (a warp reduction per batch cost 25 shuffles) */
    static __device__ __forceinline__ unsigned long long commit(const ExpandParams& P, Stage& S, int lane, const RegRow<L::NW>& v, bool live, uint64_t fp,
                                                                uint32_t chk, uint32_t auxkey, unsigned long long home, const Probe& first, unsigned long long trec,
                                                                unsigned mult) {
        unsigned gen = 0, probes = 0, coll = 0;
        int sn = SROWS == 32 ? 0 : S.sn;
        bool isnew = false;
        int bad = 0;
        if (live) {
            const uint64_t meta = make_meta(P.level, auxkey, chk);
            gen = mult;
            const int r = table_insert_from(P.table, P.table_cap, home, first, fp, meta, probes, coll);
            isnew = r == INS_NEW;
            if (r == INS_FULL) atomicExch(&P.ctr->overflow, 4);
            if (isnew) bad = O_::invariant(P.run, v);
            if (coll) atomicAdd(&P.ctr->collisions, (unsigned long long)coll); /* never seen so far */
            if (r == INS_TIE) {
                atomicAdd(&P.ctr->ties, 1ull);
                const unsigned long long t = atomicAdd(&P.ctr->tie_count, 1ull);
                if (t < P.tie_cap) {
                    TieRec rec;
                    rec.fp = fp; rec.parent = trec >> 12; rec.auxkey = auxkey; rec.cand = (uint32_t)(trec & 0xFFFu); rec.check = chk; rec._pad = 0;
                    uint8_t* dst = P.ties + t * (sizeof(TieRec) + L::BYTES);
                    *(TieRec*)dst = rec;
                    VSR_UNROLL
                    for (int j = 0; j < L::NW; j++) ((uint32_t*)(dst + sizeof(TieRec)))[j] = v.w[j];
                } else atomicExch(&P.ctr->overflow, 2);
            }
        }
        /* compaction of the survivors into the warp's staging area (one ballot, all lanes).  The survivors' final rows
           may overlap other lanes' scratch rows: every lane has read its row before anybody writes */
        const unsigned newmask = __ballot_sync(0xffffffffu, isnew);
        if constexpr (COVER) cover_count(P, lane, live, newmask, trec, gen);
        __syncwarp();
        if (isnew) {
            const int slot = sn + __popc(newmask & ((1u << lane) - 1u));
            VSR_UNROLL
            for (int j = 0; j < L::NW; j++) S.stage[slot * L::NW + j] = v.w[j];
            if (bad) {
                trec |= 1ull << 63;
                atomicOr(&P.ctr->viol_which, bad);
            }
            S.tstage[slot] = trec;
        }
        sn += __popc(newmask);
        __syncwarp();
        if constexpr (SROWS == 32) { /* flush the whole batch: nothing stays staged (S.sn stays 0) */
            if (newmask) flush(P, S, lane, sn);
        } else {
            if (lane == 0) S.sn = sn;
            __syncwarp();
            while (sn >= 32) {
                flush(P, S, lane, 32);
                sn -= 32;
            }
        }
        return (unsigned long long)gen | ((unsigned long long)probes << 32);
    }

    /* fingerprint and route one successor per lane: the part of apply that does not depend on the action */
    static __device__ __noinline__ unsigned long long emit(const ExpandParams& P, Smem& B, Stage& S, int lane, const Row n, int mult,
                                                           int cand, int si, bool act) {
        int send_to = -1;
        uint64_t fp = 0;
        uint32_t chk = 0, auxkey = 0;
        unsigned long long home = 0, trec = 0;
        Probe first = {};
        bool live = false;
        /* the successor's words, read once from the lane's scratch row: fingerprint, check hash, aux key, invariant and
           the copies to the staging area / a peer's inbox all work on registers (constant word indices) */
        RegRow<L::NW> v;
        if (act && mult > 0) {
            VSR_UNROLL
            for (int j = 0; j < L::NW; j++) v.w[j] = rdw(n, j);
        }
        if (act) {
            if (mult < 0) {
                atomicCAS(&P.ctr->error, 0, mult);
            } else if (mult > 0) {
                fp = fp64_view8<L>(B.fp_tab, v, P.run.use_view != 0);
                if (fp == 0) fp = 1;
                const int owner = MULTI ? owner_of(fp, P.owner_shift) : P.rank;
                trec = make_trec(make_gid(P.rank, P.in_base + B.round_first + si), (uint32_t)cand);
                if (owner == P.rank) {
                    /* start the seen-set probe now; the check hash, aux key and tags are computed under its latency */
                    live = true;
                    home = table_home(P.table_cap, fp);
                    probe_load(P.table, home, first);
                    chk = check_hash<L>(v, P.run.use_view != 0);
                    auxkey = O_::aux_key(v);
                } else {
                    send_to = owner; /* counted ("states generated") where it is inserted */
                }
            }
        }
        if (MULTI) {
            __syncwarp(); /* every lane has read its scratch row: that half of the staging area may now carry outgoing records */
            push_records(P, S, lane, v, send_to, fp, trec | ((uint64_t)(unsigned)mult << 56));
        }
        return commit(P, S, lane, v, live, fp, chk, auxkey, home, first, trec, (unsigned)mult);
    }

    /* ---- drain: one record per lane, after this block's share of the frontier: received from a peer (world > 1), or
       Init and the records of vsr_engine_insert_records (a launch with no frontier share, at any world size).  The
       sender computed the fingerprint; check hash and aux key are recomputed from the words; then the same seen-set insert
       / invariant / staging as a local successor.  drain_begin issues the header and bucket loads, drain_end consumes them.
       One record in flight per lane: more (2 or 4), or pipelining a chunk under every batch of the expansion, costs
       register spills in the hot loop (tools/drain_bench.py measures the drain). */
    struct DrainPre {
        uint64_t fp, tm;
        unsigned long long home;
        Probe first;
        const uint4* rec;
        bool have;
    };
    unsigned long long dchunk = ~0ull; /* inbox chunk this warp has claimed (>= nchunks: none left) */
    __device__ __forceinline__ unsigned long long drain_chunks() const { return (P.drain_total + 31) / 32; }
    __device__ __forceinline__ unsigned long long drain_claim() {
        unsigned long long c = 0;
        if (lane == 0) c = atomicAdd(&P.ctr->drain_next, 1ull);
        return c; /* lane 0's value; broadcast by the caller when it is needed (the atomic's latency hides under other work) */
    }
    __device__ __forceinline__ DrainPre drain_begin(unsigned long long chunk) {
        constexpr int RB = L::BYTES + (int)sizeof(RecHdr);
        DrainPre d;
        unsigned long long i = chunk * 32 + lane;
        d.have = chunk < drain_chunks() && i < P.drain_total;
        d.fp = d.tm = 0;
        d.home = 0;
        d.first = Probe{};
        d.rec = nullptr;
        if (d.have) {
            int s = 0;
            while (s < P.world - 1 && i >= P.drain_n[s]) { i -= P.drain_n[s]; s++; }
            d.rec = reinterpret_cast<const uint4*>(P.drain[s] + i * RB);
            const uint4 h = __ldcs(d.rec + L::NW / 4);
            d.fp = ((uint64_t)h.y << 32) | h.x;
            d.tm = ((uint64_t)h.w << 32) | h.z;
            d.home = table_home(P.table_cap, d.fp);
            probe_load(P.table, d.home, d.first);
        }
        return d;
    }
    __device__ __forceinline__ void drain_end(const DrainPre& d) {
        RegRow<L::NW> v;
        uint32_t chk = 0, auxkey = 0;
        if (d.have) {
            VSR_UNROLL
            for (int q = 0; q < L::NW / 4; q++) {
                const uint4 x = __ldcs(d.rec + q);
                v.w[4 * q] = x.x; v.w[4 * q + 1] = x.y; v.w[4 * q + 2] = x.z; v.w[4 * q + 3] = x.w;
            }
            chk = check_hash<L>(v, P.run.use_view != 0);
            auxkey = O_::aux_key(v);
        }
        tally(commit(P, S, lane, v, d.have, d.fp, chk, auxkey, d.home, d.first, d.tm & ((1ull << 56) - 1ull), (unsigned)((d.tm >> 56) & 0xFu)));
    }
    __device__ void drain() {
        const unsigned long long nchunks = drain_chunks();
        if (dchunk == ~0ull) dchunk = __shfl_sync(0xffffffffu, drain_claim(), 0);
        while (dchunk < nchunks) {
            const unsigned long long nx = drain_claim(); /* the next claim's latency hides under this chunk */
            const DrainPre d = drain_begin(dchunk);
            drain_end(d);
            dchunk = __shfl_sync(0xffffffffu, nx, 0);
        }
    }

    /* ---- scan: guards only, from registers.  Each thread copies its own state into registers and evaluates every guard
       of Next on it with compile-time candidate indices (Ops::enabled_group): a guard is a few bit tests on registers,
       not a decode of a run-time slot index plus shared-memory reads.  The result is one bit per candidate.  Then the
       (state, candidate) pairs are laid out in the block pool grouped by action: per-lane counts -> one packed warp
       prefix sum -> one shared atomic per (warp, group) -> barrier -> each lane writes its own pairs.  Two barriers per
       round instead of one per group. */
    static constexpr int NG = O_::NGRP;
    static __host__ __device__ constexpr int moff(int g) { int o = 0; for (int h = 0; h < g; h++) o += O_::grp_words(h); return o; }
    static constexpr int MW = moff(NG);       /* mask words per state */
    static constexpr int PW = (NG + 1) / 2;   /* packed 16-bit counters, two groups per word */
    static __host__ __device__ constexpr int max_grp() { int m = 0; for (int g = 0; g < NG; g++) m = O_::grp_size(g) > m ? O_::grp_size(g) : m; return m; }
    static constexpr int TBITS = ExpandCfg<L>::TBITS;
    static_assert(NS == ExpandCfg<L>::NS && max_grp() == ExpandCfg<L>::max_grp(), "ExpandCfg's limits are about this kernel");
    static_assert(ExpandCfg<L>::POOL_ITEM_FITS, "pool item does not fit 16 bits");
    static_assert(ExpandCfg<L>::POOL_COUNTERS_FIT, "16-bit packed counters");

    template <int G> __device__ __forceinline__ void guards(const RegRow<L::NW>& st, uint32_t* m, uint32_t* pc) {
        O_::template enabled_group<G>(P.run, st, m + moff(G));
        uint32_t c = 0;
        VSR_UNROLL
        for (int k = 0; k < O_::grp_words(G); k++) c += (uint32_t)__popc(m[moff(G) + k]);
        pc[G >> 1] += c << (16 * (G & 1));
        if constexpr (G + 1 < NG) guards<G + 1>(st, m, pc);
    }
    /* write this lane's pairs of group G (and the following groups) to the pool; pairs that do not fit stay in m */
    /* FAST: the whole round's pairs fit the pool (the caller has checked): no bound test per pair, nothing left over */
    template <int G, bool FAST> __device__ __forceinline__ void push(uint32_t* m, const uint32_t* ex, const uint32_t* wb, int st) {
        int pos = st + (int)((wb[G >> 1] >> (16 * (G & 1))) & 0xFFFFu) + (int)((ex[G >> 1] >> (16 * (G & 1))) & 0xFFFFu);
        VSR_UNROLL
        for (int k = 0; k < O_::grp_words(G); k++) {
            uint32_t mm = m[moff(G) + k], left = 0;
            while (mm) {
                const int bit = __ffs(mm) - 1;
                mm &= mm - 1;
                if (FAST || pos < Smem::QCAP) B.pool[pass_i() * Smem::QCAP + pos] = (uint16_t)(tid | ((k * 32 + bit) << TBITS));
                else left |= 1u << bit;
                pos++;
            }
            if (!FAST) m[moff(G) + k] = left;
        }
        if constexpr (G + 1 < NG) {
            const int q = B.qcount[pass_i()][G];
            const int nst = FAST ? st + q : (st + q < Smem::QCAP ? st + q : Smem::QCAP);
            push<G + 1, FAST>(m, ex, wb, nst);
        }
    }
    /* pool full (rare): the pairs left in m are applied right here by their own lanes, one group at a time */
    template <int G> __device__ __forceinline__ void leftovers(uint32_t* m) {
        VSR_UNROLL
        for (int k = 0; k < O_::grp_words(G); k++) {
            while (__any_sync(0xffffffffu, m[moff(G) + k] != 0)) {
                const bool inl = m[moff(G) + k] != 0;
                int cand = 0;
                if (inl) {
                    const int bit = __ffs(m[moff(G) + k]) - 1;
                    m[moff(G) + k] &= m[moff(G) + k] - 1;
                    cand = O_::grp_begin(G) + k * 32 + bit;
                }
                tally(apply<G>(P, B, S, lane, mine, cand, pass_i() * NS + tid, inl));
            }
        }
        if constexpr (G + 1 < NG) leftovers<G + 1>(m);
    }
    __device__ __forceinline__ void scan_all() {
        uint32_t m[MW], pc[PW];
        VSR_UNROLL
        for (int i = 0; i < MW; i++) m[i] = 0;
        VSR_UNROLL
        for (int i = 0; i < PW; i++) pc[i] = 0;
        if (have) {
            RegRow<L::NW> st;
            VSR_UNROLL
            for (int i = 0; i < L::NW; i++) st.w[i] = mine[i];
            guards<0>(st, m, pc);
        }
        /* warp prefix sums of the per-lane counts, two groups per word */
        uint32_t ex[PW], wb[PW];
        VSR_UNROLL
        for (int i = 0; i < PW; i++) ex[i] = pc[i];
        VSR_UNROLL
        for (int o = 1; o < 32; o <<= 1) {
            VSR_UNROLL
            for (int i = 0; i < PW; i++) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, ex[i], o);
                if (lane >= o) ex[i] += t;
            }
        }
        /* lane g reserves the warp's share of group g's pool segment */
        uint32_t mytot = 0, anyc = 0;
        VSR_UNROLL
        for (int g = 0; g < NG; g++) {
            const uint32_t t = (__shfl_sync(0xffffffffu, ex[g >> 1], 31) >> (16 * (g & 1))) & 0xFFFFu;
            if (lane == g) mytot = t;
        }
        VSR_UNROLL
        for (int i = 0; i < PW; i++) { anyc |= pc[i]; ex[i] -= pc[i]; } /* inclusive -> exclusive */
        uint32_t mybase = 0;
        if (lane < NG && mytot) mybase = (uint32_t)atomicAdd(&B.qcount[pass_i()][lane], (int)mytot);
        VSR_UNROLL
        for (int i = 0; i < PW; i++) wb[i] = 0;
        VSR_UNROLL
        for (int g = 0; g < NG; g++) wb[g >> 1] |= (__shfl_sync(0xffffffffu, mybase, g) & 0xFFFFu) << (16 * (g & 1));
        if (P.check_deadlock && have && !anyc) atomicMin(&P.ctr->dead_id, P.in_base + B.round_first + pass_i() * NS + tid);
        VSR_CLK(*this, SCAN);
        __syncthreads(); /* qcount[] final: group g's segment starts at min(sum of the groups before it, QCAP) */
        VSR_CLK(*this, SCANBAR);
#ifndef VSR_EXP_NO_PUSHFAST
        int all = 0;
        VSR_UNROLL
        for (int g = 0; g < NG; g++) all += B.qcount[pass_i()][g];
        if (all <= Smem::QCAP) { /* block-uniform: the usual case */
            push<0, true>(m, ex, wb, 0);
            return;
        }
#endif
        push<0, false>(m, ex, wb, 0);
        uint32_t rest = 0;
        VSR_UNROLL
        for (int i = 0; i < MW; i++) rest |= m[i];
        if (__any_sync(0xffffffffu, rest != 0)) leftovers<0>(m);
    }
    /* apply one (parent, candidate) pair of group G per lane; the only copy of that action's effect in the kernel */
    template <int G> static __device__ __noinline__ unsigned long long apply(const ExpandParams& P, Smem& B, Stage& S, int lane,
                                                                             const uint32_t* parent, int cand, int si, bool act) {
        const Row n = scratch(S, lane);
        int mult = 0;
        if (act) mult = O_::template step_grp<true, G>(P.run, parent, cand, n);
        return emit(P, B, S, lane, n, mult, cand, si, act);
    }
    /* one batch of <= 32 queued pairs of group G, pool[b .. b + k) (all of one pass) */
    template <int G> static __device__ __forceinline__ unsigned long long batch(const ExpandParams& P, Smem& B, Stage& S, int lane, int b,
                                                                                int k) {
        const bool act = lane < k;
        int cand = 0, si = 0;
        if (act) {
            const unsigned item = B.pool[b + lane];
            si = (PASSES == 1 ? 0 : b / Smem::QCAP) * NS + (int)(item & ((1 << TBITS) - 1));
            cand = O_::grp_begin(G) + (int)(item >> TBITS);
        }
        return apply<G>(P, B, S, lane, &B.par[si * (L::NW + 1)], cand, si, act);
    }
    unsigned long long acc_gen = 0, acc_probes = 0; /* this lane's share of the statistics, summed over the launch */
    __device__ __forceinline__ void tally(unsigned long long r) {
        acc_gen += (unsigned)r;
        acc_probes += r >> 32;
    }

    __device__ void run_round(unsigned long long first, int count) {
        /* coalesced load of `count` parent states into padded rows */
        const uint32_t* src = P.in.hbm + first * L::NW;
        if (P.in.in_hbm(first, count)) {
            for (int i = tid; i < count * L::NW; i += NS) B.par[(i / L::NW) * (L::NW + 1) + (i % L::NW)] = __ldg(src + i);
        } else { /* (part of) this round's parents are in the host part of the frontier */
            for (int i = tid; i < count * L::NW; i += NS) {
                const unsigned long long st = first + i / L::NW;
                const uint32_t* row = P.in.row<L::NW>(st);
                B.par[(i / L::NW) * (L::NW + 1) + (i % L::NW)] = __ldg(row + i % L::NW);
            }
        }
        if (tid < PASSES * Smem::NG) (&B.qcount[0][0])[tid] = 0;
        if (tid == 0) { B.round_first = first; B.take = 0; }
        VSR_CLK(*this, SCAN);
        __syncthreads();
        VSR_CLK(*this, SCANBAR);
#pragma unroll 1
        for (pass = 0; pass < PASSES; pass++) { /* a loop, not unrolled: one copy of the guards in the instruction cache */
            have = pass_i() * NS + tid < count;
            mine = &B.par[(have ? pass_i() * NS + tid : 0) * (L::NW + 1)];
            scan_all();
        }
        VSR_CLK(*this, SCAN);
        __syncthreads();
        VSR_CLK(*this, SCANBAR);
        /* batches: segment s = (pass s / NG, group s % NG) has ceil(|its part of the pass's pool| / 32) of them.  Lane s keeps
           segment s's pool range [st, en) and the index of its first batch, so mapping a batch number to (segment, offset) is
           one ballot and three shuffles. */
        static_assert(PASSES * Smem::NG <= 32, "one lane per segment");
        const int sp = lane / Smem::NG; /* this lane's pass */
        const int q = lane < PASSES * Smem::NG ? (&B.qcount[0][0])[lane] : 0;
        int inc = q;
        VSR_UNROLL
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        const int before = __shfl_sync(0xffffffffu, inc, sp * Smem::NG - 1 + (sp == 0)); /* pairs of the passes before this lane's */
        if (sp > 0) inc -= before;
        const int seg_st = sp * Smem::QCAP + (inc - q < Smem::QCAP ? inc - q : Smem::QCAP), seg_en = sp * Smem::QCAP + (inc < Smem::QCAP ? inc : Smem::QCAP);
        const int nb = (seg_en - seg_st + 31) >> 5;
        int binc = nb;
        VSR_UNROLL
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, binc, o);
            if (lane >= o) binc += t;
        }
        const int total = __shfl_sync(0xffffffffu, binc, 31);
        for (;;) {
            int t = 0;
            if (lane == 0) t = atomicAdd(&B.take, 1);
            t = __shfl_sync(0xffffffffu, t, 0);
            if (t >= total) break;
            const int s = __popc(__ballot_sync(0xffffffffu, lane < PASSES * Smem::NG && binc <= t)); /* segments that end before batch t */
            const int st = __shfl_sync(0xffffffffu, seg_st, s), en = __shfl_sync(0xffffffffu, seg_en, s);
            const int b = st + (t - __shfl_sync(0xffffffffu, binc - nb, s)) * 32;
            const int k = en - b < 32 ? en - b : 32;
            unsigned long long r;
            switch (s % Smem::NG) {
            case 0: r = batch<0>(P, B, S, lane, b, k); break;   case 1: r = batch<1>(P, B, S, lane, b, k); break;
            case 2: r = batch<2>(P, B, S, lane, b, k); break;   case 3: r = batch<3>(P, B, S, lane, b, k); break;
            case 4: r = batch<4>(P, B, S, lane, b, k); break;   case 5: r = batch<5>(P, B, S, lane, b, k); break;
            case 6: r = batch<6>(P, B, S, lane, b, k); break;   case 7: r = batch<7>(P, B, S, lane, b, k); break;
            case 8: r = batch<8>(P, B, S, lane, b, k); break;   case 9: r = batch<9>(P, B, S, lane, b, k); break;
            case 10: r = batch<10>(P, B, S, lane, b, k); break; case 11: r = batch<11>(P, B, S, lane, b, k); break;
            default: r = batch<12>(P, B, S, lane, b, k); break;
            }
            tally(r);
            VSR_CLK(*this, BATCH);
        }
        VSR_CLK(*this, BATCH);
    }

    __device__ void finish() {
        while (S.sn > 0) flush(P, S, lane, S.sn < 32 ? S.sn : 32);
#ifdef VSR_EXP_ROUNDCLK
        clk_mark(CLK_OTHER);
        VSR_UNROLL
        for (int i = 0; i < 5; i++)
            if (lane == 0) atomicAdd(&P.ctr->roundclk[i], clk[i]);
#endif
        for (int o = 16; o; o >>= 1) {
            acc_gen += __shfl_xor_sync(0xffffffffu, acc_gen, o);
            acc_probes += __shfl_xor_sync(0xffffffffu, acc_probes, o);
        }
        if (lane == 0) {
            atomicAdd(&P.ctr->generated, acc_gen);
            atomicAdd(&P.ctr->probes, acc_probes);
        }
        if constexpr (COVER && COVER_SHARED) {
            __syncthreads(); /* every warp's last batch is counted */
            const unsigned long long* tab = cover_table(P);
            if (tid < NCOV && tab[tid]) atomicAdd(&P.cover[tid], tab[tid]);
        }
    }
};

template <class L, bool MULTI, bool COVER = false> __global__ void __launch_bounds__(ExpandCfg<L>::WARPS * 32, ExpandCfg<L>::BLOCKS) expand_kernel(const __grid_constant__ ExpandParams P) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    typedef typename ExpandCfg<L>::Smem Smem;
    Smem& B = *reinterpret_cast<Smem*>(smem_raw);
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) B.fp_tab[i] = P.fp_tab[i];
    __shared__ unsigned long long next_round;
    Expander<L, MULTI, COVER> X(P, B);
    if ((threadIdx.x & 31) == 0) B.w[threadIdx.x >> 5].sn = 0;
    if constexpr (COVER && Expander<L, MULTI, COVER>::COVER_SHARED) { /* cleared before the loop's first barrier */
        if (threadIdx.x < Expander<L, MULTI, COVER>::NCOV) Expander<L, MULTI, COVER>::cover_table(P)[threadIdx.x] = 0;
    }
    const unsigned long long nrounds = (P.n_in + Smem::NR - 1) / Smem::NR;
    if (threadIdx.x == 0) next_round = atomicAdd(&P.ctr->work_next, 1ull);
    VSR_CLK(X, OTHER);
    for (;;) {
        __syncthreads();
        const unsigned long long c = next_round;
        __syncthreads();
        VSR_CLK(X, END);
        if (c >= nrounds) break;
        /* claim the round after this one now: the global atomic's latency hides under this round's work */
        if (threadIdx.x == 0) {
            next_round = atomicAdd(&P.ctr->work_next, 1ull);
            /* pull the next round's parents into L2 while this round runs */
            const unsigned long long nx = next_round;
            if (nx < nrounds && (nx + 1) * Smem::NR <= P.in.split) {
                const unsigned long long nfirst = nx * Smem::NR;
                const unsigned long long ncount = (P.n_in - nfirst) < (unsigned long long)Smem::NR ? (P.n_in - nfirst) : Smem::NR;
                asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(P.in.hbm + nfirst * L::NW), "r"((uint32_t)(ncount * L::BYTES)) : "memory");
            }
        }
        const unsigned long long first = c * Smem::NR;
        const int count = (int)((P.n_in - first) < (unsigned long long)Smem::NR ? (P.n_in - first) : Smem::NR);
        X.run_round(first, count);
    }
    if (MULTI && P.drain_total) X.drain();
    X.finish();
}

/* VIEW-tie patch pass (SURVEY H2; only launched for a level that reported ties).  `ties` holds, sorted by fp, ONE
   record per tied fingerprint: the smallest (aux_key, parent, candidate) among the late arrivals.  Every state of the
   new level looks itself up; if a tie record beats the first arrival's aux_key, the state and its trace record are
   replaced, so the survivor is "smallest aux_key wins" whatever the arrival order — the rule the oracle applies.
   The invariant is re-evaluated on every state of the level (the verdict may change with the aux variables). */
template <class L> __global__ void patch_ties_kernel(const ExpandParams P, const uint8_t* ties, unsigned long long ntie, unsigned long long n_out) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out) return;
    uint32_t w[L::NW];
    uint32_t* st = P.out.row<L::NW>(i);
    for (int j = 0; j < L::NW; j++) w[j] = st[j];
    uint64_t fp = fp64_view8<L>(P.fp_tab, w, P.run.use_view != 0);
    if (fp == 0) fp = 1;
    const uint32_t chk = check_hash<L>(w, P.run.use_view != 0);
    const size_t stride = sizeof(TieRec) + L::BYTES;
    unsigned long long lo = 0, hi = ntie;
    while (lo < hi) {
        const unsigned long long mid = (lo + hi) / 2;
        if (((const TieRec*)(ties + mid * stride))->fp < fp) lo = mid + 1; else hi = mid;
    }
    for (; lo < ntie; lo++) {
        const TieRec* t = (const TieRec*)(ties + lo * stride);
        if (t->fp != fp) break;
        if (t->check != chk) continue;
        if (t->auxkey < Ops<L>::aux_key(w)) {
            const uint32_t* tw = (const uint32_t*)((const uint8_t*)t + sizeof(TieRec));
            for (int j = 0; j < L::NW; j++) { w[j] = tw[j]; st[j] = tw[j]; }
            if (P.out_base + i < P.trace_cap) {
                uint64_t* rec = (uint64_t*)P.trace.row<2>(P.out_base + i);
                if (P.cover) { /* coverage follows the trace: the state now counts as found by the winner's action */
                    const uint64_t was = *rec;
                    const int a0 = (was >> 12) == ROOT_GID ? (int)VSR_ACT_INIT : Ops<L>::action_of((int)(was & 0xFFFu));
                    const int a1 = t->parent == ROOT_GID ? (int)VSR_ACT_INIT : Ops<L>::action_of((int)(t->cand & 0xFFFu));
                    if (a0 != a1) {
                        atomicAdd(&P.cover[VSR_NUM_ACTIONS + a0], ~0ull); /* - 1 */
                        atomicAdd(&P.cover[VSR_NUM_ACTIONS + a1], 1ull);
                    }
                }
                *rec = make_trec(t->parent, t->cand);
            }
        }
    }
    const int bad = Ops<L>::invariant(P.run, w);
    if (bad) {
        atomicMin(&P.ctr->viol_id, P.out_base + i);
        atomicOr(&P.ctr->viol_which, bad);
    }
}

/* meta of the seen-set entry holding (fp, check), 0 if absent (an entry's meta carries its level, >= 1).  The insert's
   probe order: entry by entry from the home bucket; the first empty slot ends the chain */
__device__ __forceinline__ uint64_t table_lookup(const uint64_t* table, unsigned long long cap, uint64_t fp, uint32_t check) {
    unsigned long long h = table_home(cap, fp);
    for (unsigned long long i = 0; i < cap; i++) {
        const uint64_t e0 = table[2 * h], e1 = table[2 * h + 1];
        if (e0 == 0) return 0;
        if (e0 == fp && (uint32_t)e1 == check) return e1;
        if (++h >= cap) h = 0;
    }
    return 0;
}

/* membership query (tests / golden-trace cross-check) */
static __global__ void lookup_kernel(const uint64_t* table, unsigned long long cap, uint64_t fp, uint32_t check, unsigned long long* meta_out) {
    *meta_out = table_lookup(table, cap, fp, check);
}

/* per-level audit (tests, vsr_engine_audit_level): seen-set entries tagged with a level, and the level's frontier looked up
   in the seen-set (table_lookup), plus order-independent digests of the frontier and of the tagged entries' fingerprints */
struct AuditSums {
    unsigned long long tagged, found, fp_sum, fp_xor, words_sum, words_xor, tagged_fp_sum, tagged_fp_xor;
};
__device__ __forceinline__ void audit_add(unsigned long long* dst, unsigned long long v, bool is_xor) {
    for (int o = 16; o; o >>= 1) v = is_xor ? v ^ __shfl_xor_sync(0xffffffffu, v, o) : v + __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) {
        if (is_xor) atomicXor(dst, v);
        else atomicAdd(dst, v);
    }
}
static __global__ void audit_table_kernel(const uint64_t* table, unsigned long long cap, int level, AuditSums* out) {
    unsigned long long n = 0, fs = 0, fx = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint64_t e0 = table[2 * i];
        if (e0 != 0 && (int)(table[2 * i + 1] >> 56) == level) {
            n++;
            fs += mix64(e0);
            fx ^= mix64(e0);
        }
    }
    audit_add(&out->tagged, n, false);
    audit_add(&out->tagged_fp_sum, fs, false);
    audit_add(&out->tagged_fp_xor, fx, true);
}
template <class L> __global__ void audit_frontier_kernel(const ExpandParams P, const SpillRows level, unsigned long long n_states, AuditSums* out) {
    unsigned long long found = 0, fs = 0, fx = 0, ws = 0, wx = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_states; i += (unsigned long long)gridDim.x * blockDim.x) {
        uint32_t w[L::NW];
        const uint32_t* st = level.row<L::NW>(i);
        uint64_t hw = 0;
        for (int j = 0; j < L::NW; j++) {
            w[j] = st[j];
            hw = mix64(hw ^ ((uint64_t)j << 32 | w[j]));
        }
        uint64_t fp = fp64_view8<L>(P.fp_tab, w, P.run.use_view != 0);
        if (fp == 0) fp = 1;
        const uint32_t chk = check_hash<L>(w, P.run.use_view != 0);
        found += (int)(table_lookup(P.table, P.table_cap, fp, chk) >> 56) == P.level;
        fs += mix64(fp);
        fx ^= mix64(fp);
        ws += hw;
        wx ^= hw;
    }
    audit_add(&out->found, found, false);
    audit_add(&out->fp_sum, fs, false);
    audit_add(&out->fp_xor, fx, true);
    audit_add(&out->words_sum, ws, false);
    audit_add(&out->words_xor, wx, true);
}

/* ------------------------------------------------------------------ recovering a checkpoint (vsr_ckpt.cu)
   A checkpoint written by W_old ranks, continued by W_new ranks (both powers of two).  Old record l of old rank q gets its
   new global id from five per-old-rank numbers:
     l < cut[q]:  rank to[q] + l / slice[q], local id hist[q] + l % slice[q]
     else:        rank to[q], local id front[q] + l - cut[q]
   Shrinking or the same world (W_old = k W_new): new rank q / k holds its group's histories (slice and cut: hist = ids of
   the group's earlier files, cut = cur_base), then its group's frontiers (front); with k = 1 this is the identity.  Growing
   (W_new = s W_old): file q's records are cut into s slices of ceil(next_base / s) (cut = infinity).  Every stored global
   id (trace parents, the totals' violation id) is renumbered with this one function, so the parent walk reads the new ids
   as it read the old ones. */
constexpr unsigned long long REMAP_ALL = ~0ull; /* slice or cut: infinity */
struct GidRemap {
    unsigned long long slice[MAX_WORLD], hist[MAX_WORLD], cut[MAX_WORLD], front[MAX_WORLD];
    int to[MAX_WORLD];
    int old_world, _pad;
};
__host__ __device__ __forceinline__ uint64_t remap_gid(const GidRemap& m, uint64_t gid) {
    if (gid == ROOT_GID) return ROOT_GID;
    const int r = (int)(gid >> 40), q = r < m.old_world ? r : 0;
    const unsigned long long l = gid & ((1ull << 40) - 1ull);
    return l < m.cut[q] ? make_gid(m.to[q] + (int)(l / m.slice[q]), m.hist[q] + l % m.slice[q]) : make_gid(m.to[q], m.front[q] + l - m.cut[q]);
}
__host__ __device__ __forceinline__ uint64_t remap_trec(const GidRemap& m, uint64_t t) {
    return make_trec(remap_gid(m, (t >> 12) & GID_MASK), (uint32_t)(t & 0xFFFu));
}

/* one chunk of an old rank's frontier, with the trace records of those states (NULL without a trace) */
struct ReshardParams {
    const uint32_t* in;                /* n states of L::NW words */
    const uint64_t* in_trace;          /* their records in the old numbering */
    unsigned long long n;
    SpillRows out;                     /* frontier buffer 0 */
    unsigned long long out_cap;
    unsigned long long out_first;      /* place: state i goes to row out_first + i */
    SpillRows trace;                   /* record of kept state j goes to row trace_base + j */
    unsigned long long trace_base, trace_cap; /* trace_cap 0: no trace (or place: the records are already in place) */
    const uint64_t* table;             /* this rank's seen-set, already filled from its source files */
    unsigned long long table_cap;
    const uint64_t* fp_tab;
    RunCfg run;
    int rank, owner_shift, level, place; /* place: shrinking or the same world, where every state of the chunk is this rank's */
    GidRemap remap;
    unsigned long long* kept;          /* !place: states this rank owns, over all chunks (their positions in buffer 0) */
    unsigned long long* missing;       /* states kept that are not in the seen-set with the checkpoint's level (place: or not owned) */
};
/* Keep the states this rank owns — the expand kernel's fingerprint and owner rule.  place: every state of the chunk is this
   rank's and goes to its row, with no atomics and no record copy (its record was loaded with the trace).  Else the owned
   states are appended to frontier buffer 0 (one atomic per warp), each with its trace record renumbered.  Every kept state
   must already be in the seen-set at the checkpoint's level: a miss (or, placed, a state of another rank) means the files
   disagree, and the host refuses the recovery. */
template <class L> __global__ void reshard_frontier_kernel(const ReshardParams P) {
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long rounds = (P.n + stride - 1) / stride;
    const int lane = threadIdx.x & 31;
    unsigned long long miss = 0;
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (unsigned long long rd = 0; rd < rounds; rd++, i += stride) { /* whole warps stay in the loop: the ballot is warp-wide */
        uint32_t w[L::NW];
        bool mine = false;
        if (i < P.n) {
            for (int j = 0; j < L::NW; j++) w[j] = P.in[i * L::NW + j];
            uint64_t fp = fp64_view8<L>(P.fp_tab, w, P.run.use_view != 0);
            if (fp == 0) fp = 1;
            mine = owner_of(fp, P.owner_shift) == P.rank;
            if (mine ? (int)(table_lookup(P.table, P.table_cap, fp, check_hash<L>(w, P.run.use_view != 0)) >> 56) != P.level : P.place != 0) miss++;
        }
        unsigned long long pos;
        if (P.place) { /* the same for the whole grid: no ballot below */
            if (i >= P.n) continue;
            pos = P.out_first + i;
        } else {
            const unsigned m = __ballot_sync(0xffffffffu, mine);
            if (!m) continue;
            unsigned long long base = 0;
            const int leader = __ffs(m) - 1;
            if (lane == leader) base = atomicAdd(P.kept, (unsigned long long)__popc(m));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (!mine) continue;
            pos = base + __popc(m & ((1u << lane) - 1u));
        }
        if (pos >= P.out_cap) continue; /* counted: the host reports the frontier's size */
        uint32_t* dst = P.out.row<L::NW>(pos);
        for (int j = 0; j < L::NW; j++) dst[j] = w[j];
        if (P.trace_base + pos < P.trace_cap) *(uint64_t*)P.trace.row<2>(P.trace_base + pos) = remap_trec(P.remap, P.in_trace[i]);
    }
    for (int o = 16; o; o >>= 1) miss += __shfl_xor_sync(0xffffffffu, miss, o);
    if (lane == 0 && miss) atomicAdd(P.missing, miss);
}

/* ------------------------------------------------------------------ simulation mode (TLC `-simulate`)
   One thread per random walk from Init, `depth` states long at most; the invariant is checked on every state reached.
   The first violating (walk, depth) is kept (smallest walk index wins), and with check_deadlock the first (walk, depth) of
   a state without successors before the bound; the host re-walks the smaller of the two for the trace. */
struct SimParams {
    unsigned long long num_walks, seed;
    int depth, check_deadlock;
    RunCfg run;
    unsigned long long* first_bad; /* walk << 16 | depth of the state that violates (~0 = none) */
    unsigned long long* first_dead; /* walk << 16 | depth of the state without successors (~0 = none); check_deadlock only */
    unsigned long long* steps;     /* transitions taken */
    unsigned long long* dead_ends; /* walks that stopped in a state without successors */
    unsigned long long* probe_out; /* optional: for walks 0 .. probe_walks-1, fingerprint of the last state and transitions taken */
    unsigned long long probe_walks;
    const uint64_t* fp_tab;
};
template <class L> __global__ void simulate_kernel(const SimParams Q) {
    unsigned long long steps = 0, dead = 0;
    for (unsigned long long wk = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; wk < Q.num_walks; wk += (unsigned long long)gridDim.x * blockDim.x) {
        uint64_t rng = Q.seed ^ (wk * 0xD1B54A32D192ED03ULL);
        uint32_t a[L::NW], b[L::NW];
        Ops<L>::init((uint32_t*)a);
        unsigned long long mysteps = 0;
        for (int d = 2; d <= Q.depth; d++) {
            const int cand = Ops<L>::random_enabled(Q.run, (const uint32_t*)a, rng);
            if (cand < 0) {
                dead++;
                if (Q.check_deadlock) atomicMin(Q.first_dead, (wk << 16) | (unsigned long long)(d - 1));
                break;
            }
            if (Ops<L>::template step<true>(Q.run, (const uint32_t*)a, cand, (uint32_t*)b) <= 0) break;
            for (int j = 0; j < L::NW; j++) a[j] = b[j];
            steps++;
            mysteps++;
            if (Ops<L>::invariant(Q.run, (const uint32_t*)a)) {
                atomicMin(Q.first_bad, (wk << 16) | (unsigned long long)d);
                break;
            }
        }
        if (wk < Q.probe_walks) {
            Q.probe_out[2 * wk] = fp64_view<L>(Q.fp_tab, (const uint32_t*)a, false);
            Q.probe_out[2 * wk + 1] = mysteps;
        }
    }
    for (int o = 16; o; o >>= 1) {
        steps += __shfl_xor_sync(0xffffffffu, steps, o);
        dead += __shfl_xor_sync(0xffffffffu, dead, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(Q.steps, steps);
        atomicAdd(Q.dead_ends, dead);
    }
}

/* seen-set micro-benchmark (SURVEY §8d): n splitmix64 keys, a fraction of them duplicates, inserted with the same
   table_insert the BFS uses; nothing else in the loop, so its rate is the random-probe ceiling of this table design */
static __global__ void probe_bench_kernel(uint64_t* table, unsigned long long cap, unsigned long long n, unsigned long long distinct,
                                   unsigned long long seed, unsigned long long* new_count, unsigned long long* probe_count) {
    unsigned long long mine_new = 0;
    unsigned probes = 0, coll = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long z = seed + (i % distinct) * 0x9E3779B97F4A7C15ULL; /* splitmix64 of the key index */
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        z ^= z >> 31;
        if (z == 0) z = 1;
        mine_new += table_insert(table, cap, z, make_meta(1, 0, (uint32_t)(z >> 32) | 1u), probes, coll) == INS_NEW;
    }
    for (int o = 16; o; o >>= 1) {
        mine_new += __shfl_xor_sync(0xffffffffu, mine_new, o);
        probes += __shfl_xor_sync(0xffffffffu, probes, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(new_count, mine_new);
        atomicAdd(probe_count, (unsigned long long)probes);
    }
}

} // namespace vsr
#endif
