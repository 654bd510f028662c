/*
 * vsr_seen_host.cuh — device side of the seen-set's entries outside the table: the compaction of a level window of the
 * table into a row buffer and the re-insertion of such rows (a checkpoint's seen-set section, vsr_ckpt.cu; the host tier's
 * eviction, vsr_seen_host.cu), and the host tier's two kernels:
 *   seen_host_pass_kernel          streams the tier once (16-byte coalesced reads of pinned host memory) and looks every entry
 *                                  up in the HBM table; a hit tagged with the level just generated is a state inserted as new
 *                                  that the tier already held: its tag becomes the tier entry's level, which marks it
 *   seen_host_compact_kernel<L>    drops the marked rows from that level: rows that stay move into the holes below the kept
 *                                  count, with their trace records, so ids stay dense
 */
#ifndef VSR_SEEN_HOST_CUH
#define VSR_SEEN_HOST_CUH

#include "vsr_gpu.cuh"

namespace vsr {

/* non-empty entries of table slots [first, first + n) whose level tag lies in [lo, hi) appended to rows of `out` (16-byte
   rows, order is irrelevant); *count counts them all, only the first out_cap are written.  One atomic per warp */
static __global__ void seen_compact_kernel(const uint64_t* __restrict__ table, unsigned long long first, unsigned long long n, int lo, int hi,
                                           const SpillRows out, unsigned long long out_cap, unsigned long long* count) {
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long rounds = (n + stride - 1) / stride;
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    for (unsigned long long r = 0; r < rounds; r++, i += stride) { /* whole warps stay in the loop: the ballot below is warp-wide */
        uint64_t e0 = 0, e1 = 0;
        if (i < n) {
            e0 = table[2 * (first + i)];
            e1 = table[2 * (first + i) + 1];
        }
        const int lvl = (int)(e1 >> 56);
        const bool take = e0 != 0 && lvl >= lo && lvl < hi;
        const unsigned m = __ballot_sync(0xffffffffu, take);
        if (!m) continue;
        unsigned long long base = 0;
        const int leader = __ffs(m) - 1;
        if (lane == leader) base = atomicAdd(count, (unsigned long long)__popc(m));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (take) {
            const unsigned long long pos = base + __popc(m & ((1u << lane) - 1u));
            if (pos < out_cap) {
                uint64_t* d = (uint64_t*)out.row<4>(pos);
                d[0] = e0;
                d[1] = e1;
            }
        }
    }
}

/* n rows of `ents` back into a table: every one must be new.  owner_shift < 64 (a checkpoint of another number of ranks):
   only the entries this rank owns, counted in *owned; 64 inserts every entry */
static __global__ void seen_reinsert_kernel(uint64_t* table, unsigned long long cap, const SpillRows ents, unsigned long long n, int owner_shift, int rank,
                                            unsigned long long* not_new, unsigned long long* owned) {
    unsigned long long bad = 0, mine = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint64_t* r = (const uint64_t*)ents.row<4>(i);
        const uint64_t fp = r[0], meta = r[1];
        if (owner_shift < 64 && owner_of(fp, owner_shift) != rank) continue;
        unsigned probes = 0, coll = 0;
        mine++;
        if (table_insert(table, cap, fp, meta, probes, coll) != INS_NEW) bad++;
    }
    if (bad) atomicAdd(not_new, bad);
    if (owned && mine) atomicAdd(owned, mine);
}

/* The tier pass: tier entries [0, n) against the table, in the insert's probe order.  A hit on (fp, check) tagged `level` is
   marked by one CAS of its meta to the tier entry's level (the CAS makes each state count once in *marked).  Entries with
   the same fingerprint, another check hash and the tag `level` are fingerprint collisions no insert has seen (the other
   state was in host memory when this one was inserted), counted once, in the level that inserted them */
static __global__ void seen_host_pass_kernel(const uint64_t* __restrict__ tier, unsigned long long n, uint64_t* table, unsigned long long cap, int level,
                                             unsigned long long* marked, unsigned long long* collisions) {
    unsigned long long hits = 0, coll = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const ulonglong2 t = ((const ulonglong2*)tier)[i];
        const uint64_t fp = t.x;
        const uint32_t chk = (uint32_t)t.y;
        unsigned long long h = table_home(cap, fp);
        for (unsigned long long k = 0; k < cap; k++) {
            const uint64_t e0 = table[2 * h], e1 = table[2 * h + 1];
            if (e0 == 0) break;
            if (e0 == fp && (int)(e1 >> 56) == level) {
                if ((uint32_t)e1 != chk) {
                    coll++;
                } else {
                    const uint64_t mark = (e1 & ((1ull << 56) - 1)) | (t.y & ~((1ull << 56) - 1));
                    hits += atomicCAS((unsigned long long*)&table[2 * h + 1], (unsigned long long)e1, (unsigned long long)mark) == e1;
                    break;
                }
            } else if (e0 == fp && (uint32_t)e1 == chk) {
                break;
            }
            if (++h >= cap) h = 0;
        }
    }
    if (hits) atomicAdd(marked, hits);
    if (coll) atomicAdd(collisions, coll);
}

/* the level's compaction, in two launches of one kernel over the level's rows.  keep(row) = its seen-set entry still carries
   the level's tag.  Phase 0, rows [0, n_keep): every dropped row is a hole, appended to `holes`.  Phase 1, rows
   [n_keep, n): every kept row j moves, with its trace record, into hole number atomicAdd(count) — as many holes as such
   rows, and no row is both, so no scratch copy of the rows is needed.  A dropped row takes its distinct count back from
   its action's coverage counter (cover != NULL), so the counters stay the histogram of the kept rows' trace records. */
struct SeenHostParams {
    SpillRows rows;               /* the level's states */
    unsigned long long n, n_keep;
    SpillRows trace;              /* trace record of row i at local id base + i (trace_cap 0: none) */
    unsigned long long base, trace_cap;
    SpillRows holes;              /* 2-word rows: row indices */
    unsigned long long* count;
    unsigned long long* cover;    /* ExpandParams::cover, NULL = off */
    const uint64_t* table;
    unsigned long long table_cap;
    const uint64_t* fp_tab;
    RunCfg run;
    int level, phase;
};

template <class L> __global__ void seen_host_compact_kernel(const SeenHostParams P) {
    const unsigned long long lo = P.phase ? P.n_keep : 0, hi = P.phase ? P.n : P.n_keep;
    for (unsigned long long i = lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (unsigned long long)gridDim.x * blockDim.x) {
        uint32_t w[L::NW];
        uint32_t* src = P.rows.row<L::NW>(i);
        for (int j = 0; j < L::NW; j++) w[j] = src[j];
        uint64_t fp = fp64_view8<L>(P.fp_tab, w, P.run.use_view != 0);
        if (fp == 0) fp = 1;
        const uint32_t chk = check_hash<L>(w, P.run.use_view != 0);
        const bool keep = (int)(table_lookup(P.table, P.table_cap, fp, chk) >> 56) == P.level;
        const bool has_rec = P.base + i < P.trace_cap;
        if (!keep && P.cover && has_rec) {
            const uint64_t t = *(const uint64_t*)P.trace.row<2>(P.base + i);
            const int a = (t >> 12) == ROOT_GID ? (int)VSR_ACT_INIT : Ops<L>::action_of((int)(t & 0xFFFu));
            atomicAdd(&P.cover[VSR_NUM_ACTIONS + a], ~0ull); /* - 1 */
        }
        if (P.phase == 0) {
            if (!keep) *(unsigned long long*)P.holes.row<2>(atomicAdd(P.count, 1ull)) = i;
        } else if (keep) {
            const unsigned long long d = *(const unsigned long long*)P.holes.row<2>(atomicAdd(P.count, 1ull));
            uint32_t* dst = P.rows.row<L::NW>(d);
            for (int j = 0; j < L::NW; j++) dst[j] = w[j];
            if (has_rec) *(uint64_t*)P.trace.row<2>(P.base + d) = *(const uint64_t*)P.trace.row<2>(P.base + i);
        }
    }
}

} // namespace vsr
#endif
