/*
 * vsr_layout.h — the packed fixed-width bit-vector encoding of one VSR.tla state.
 *
 * A state (the 20 VARIABLES of vsr-revisited/paper/VSR.tla:119-138) is stored as NW 32-bit words
 * holding bit-arrays of power-of-two element width (1, 2, 4 or 8 bits), so no element ever straddles
 * a word and every access is one shift+mask with a compile-time base and width.
 *
 * The message bag (VSR.tla:135, helpers :227-275) is stored by SLOT, not as a list.  With
 * RestartEmptyLimit = 0 every message that can ever be sent has a unique key:
 *   SVC(v, src, dest)           one per view increase of src                 (:293-297, :587, :611, :686)
 *   DVC(v, src)  dest=Primary(v) one per (src, v), payload log/lnv/commit     (:654-666)
 *   SV(v)        src=Primary(v)  one per view, payload log/commit, per dest   (:752-758)
 *   Prepare(x)   one per value x (each value is requested once, :370), payload view/req/op/commit
 *   PrepareOk(v, n, src) dest=Primary(v)                                     (:422-426, :786-790)
 *   GetState(v, src) payload (op_number, dest)                               (:510-514)
 *   NewState(v, dest) = the reply to GetState(v, dest), payload log/commit   (:533-541)
 * and DiscardFunc keeps the key with count 0 (:244-245), so a slot has three states:
 * 0 absent, 1 pending (count 1), 2 consumed (count 0).  A log entry record is determined by its
 * value (the Prepare slot holds its view and request number), so logs are sequences of value ids.
 * Every one of these uniqueness facts is CHECKED at run time: an action that would need a second
 * message in a slot returns an error instead of a state, and the oracle audits them independently.
 *
 * rep_op_number[r] is not stored: it always equals Len(rep_log[r]) (audited by the oracle).
 */
#ifndef VSR_LAYOUT_H
#define VSR_LAYOUT_H

#include <stdint.h>

#if defined(__CUDACC__)
#define VSR_HD __host__ __device__ __forceinline__
#define VSR_UNROLL _Pragma("unroll")
#else
#define VSR_HD inline
#define VSR_UNROLL
#endif

namespace vsr {

/* Owner rank of a fingerprint (world a power of two; shift = 64 - log2(world), 64 when world = 1): the high bits of the
   fingerprint TIMES AN ODD CONSTANT, not of the fingerprint itself.  FP64 is linear over GF(2): a successor differs from its
   parent in a handful of bits d, so fp(successor) = fp(parent) ^ A*d, and with plain high bits the destination of a rank's
   successors would be owner(parent) ^ (a few constants) — measured on the shipped VSR.cfg with 8 ranks: some (sender, owner)
   pairs carry 10x the records of others (24.5 k vs 2.4 k of 104 k), which overflowed inbox segments sized for the average and
   loads NVLink unevenly.  The carry chains of an integer multiplication are not linear: the same count is 12.8 - 13.3 k for
   every pair.  A different constant than table_home's, so that the bucket inside a shard stays uniform. */
VSR_HD int owner_of(uint64_t fp, int shift) {
    return shift >= 64 ? 0 : (int)((fp * 0xD6E8FEB86659FD93ULL) >> shift);
}

constexpr int pow2_width(int maxval) { return maxval < 2 ? 1 : (maxval < 4 ? 2 : (maxval < 16 ? 4 : 8)); }
constexpr int align_up(int x, int a) { return (x + a - 1) / a * a; }

/* slot states */
enum { ST_ABSENT = 0, ST_PENDING = 1, ST_CONSUMED = 2 };
/* aux_client_acked codes */
enum { ACK_ABSENT = 0, ACK_FALSE = 1, ACK_TRUE = 2 };

/* error codes returned by step() / pack() (negative) */
enum {
    E_SLOT_OCCUPIED = -1,   /* a send needs a slot that already holds a message (count would be 2, or 2 payloads) */
    E_OVERFLOW = -2,        /* a field exceeds its width (view > K, request number > |Values|, log longer than |Values|) */
    E_NOT_PRIMARY = -3,     /* SendSV by a replica that is not Primary(view): source is implied by the slot */
    E_STALE_RECV = -4,      /* SendGetState with non-empty received sets: their view would go stale */
    E_PREPKEY_CLASH = -5,   /* two created values share (view, op_number): canonical labelling undefined */
    E_MISSING_PAYLOAD = -6, /* a received DVC whose slot is absent */
    E_UNSUPPORTED = -7,     /* state not representable (pack): restart variables, count > 1, ... */
    /* liveness pass (vsr_live.cu): the BFS and the store of not-P states disagree */
    E_LIVE_MISSING = -8,    /* a not-P successor of a stored state is not in the live index */
    E_LIVE_DUP = -9         /* a state was stored twice */
};

#define VSR_FIELD(name, W, N, prev)                           \
    static constexpr int name##_W = (W);                      \
    static constexpr int name##_N = (N);                      \
    static constexpr int name##_B = align_up(prev##_E, (W));  \
    static constexpr int name##_E = name##_B + (W) * (N);

template <int R_, int V_, int K_> struct Layout {
    static constexpr int R = R_, V = V_, K = K_, L = K_ - 1;
    static_assert(R >= 2 && R <= 7, "ReplicaCount 2..7");
    static_assert(V >= 1 && V <= 7, "|Values| 1..7");
    static_assert(K >= 1 && K <= 15, "StartViewOnTimerLimit 0..14");
    static constexpr int VB = pow2_width(K);     /* view numbers 0..K */
    static constexpr int OB = pow2_width(V);     /* op/commit/request numbers and value ids 0..V */
    static constexpr int RB = pow2_width(R - 1); /* replica index 0..R-1 */
    static constexpr int O = R - 1;              /* "other replicas" of a given one */
    static constexpr int NV2 = K - 1;            /* views 2..K */
    static constexpr int NSVC = NV2 * R * O;
    static constexpr int NDVC = NV2 * O;
    static constexpr int NSV = NV2 * O;
    static constexpr int NPOK = K * V * O;
    static constexpr int NGS = NV2 * O;
    static constexpr int START_E = 0;
    /* --- per-replica variables */
    VSR_FIELD(STATUS, 2, R, START)
    VSR_FIELD(VIEWN, VB, R, STATUS)
    VSR_FIELD(COMMIT, OB, R, VIEWN)
    VSR_FIELD(LNV, VB, R, COMMIT)
    VSR_FIELD(SENT_DVC, 1, R, LNV)
    VSR_FIELD(SENT_SV, 1, R, SENT_DVC)
    VSR_FIELD(SVC_MASK, 1, R * R, SENT_SV)   /* rep_svc_recv[r] as a set of sources */
    VSR_FIELD(DVC_MASK, 1, R * R, SVC_MASK)  /* rep_dvc_recv[r] as a set of sources */
    VSR_FIELD(PEER, OB, R * R, DVC_MASK)
    VSR_FIELD(CT_REQ, OB, R, PEER)
    VSR_FIELD(CT_OP, OB, R, CT_REQ)
    VSR_FIELD(CT_EXEC, 1, R, CT_OP)
    VSR_FIELD(SELF_LNV, VB, R, CT_EXEC)      /* payload of r's own DVC in rep_dvc_recv[r] (:662-664) */
    VSR_FIELD(SELF_COMMIT, OB, R, SELF_LNV)
    /* --- all logs, contiguous (value ids; 0 = no entry) so relabelling is one sweep */
    VSR_FIELD(LOG, OB, R * V, SELF_COMMIT)
    VSR_FIELD(SELF_LOG, OB, R * V, LOG)
    VSR_FIELD(DVC_LOG, OB, NDVC * V, SELF_LOG)
    VSR_FIELD(SV_LOG, OB, NV2 * V, DVC_LOG)
    VSR_FIELD(NS_LOG, OB, NGS * V, SV_LOG)
    static constexpr int ALL_LOGS_B = LOG_B;
    static constexpr int ALL_LOGS_N = (NS_LOG_E - LOG_B) / OB;
    /* --- message slots */
    VSR_FIELD(SVC_ST, 2, NSVC, NS_LOG)
    VSR_FIELD(DVC_ST, 2, NDVC, SVC_ST)
    VSR_FIELD(DVC_LNV, VB, NDVC, DVC_ST)
    VSR_FIELD(DVC_COMMIT, OB, NDVC, DVC_LNV)
    VSR_FIELD(SV_ST, 2, NSV, DVC_COMMIT)
    VSR_FIELD(SV_COMMIT, OB, NV2, SV_ST)
    VSR_FIELD(PR_VIEW, VB, V, SV_COMMIT)     /* 0 = value not requested yet */
    VSR_FIELD(PR_REQ, OB, V, PR_VIEW)
    VSR_FIELD(PR_OP, OB, V, PR_REQ)
    VSR_FIELD(PR_COMMIT, OB, V, PR_OP)
    VSR_FIELD(PR_CONS, 1, V * O, PR_COMMIT)  /* 1 = the copy to that destination was consumed */
    VSR_FIELD(POK_ST, 2, NPOK, PR_CONS)
    VSR_FIELD(GS_ST, 2, NGS, POK_ST)
    VSR_FIELD(GS_T, OB, NGS, GS_ST)
    VSR_FIELD(GS_DEST, RB, NGS, GS_T)
    VSR_FIELD(NS_ST, 2, NGS, GS_DEST)
    VSR_FIELD(NS_COMMIT, OB, NGS, NS_ST)
    /* --- aux variables (not part of VIEW, VSR.tla:145,149-150): last, so the view part is a prefix */
    static constexpr int VIEW_BITS = NS_COMMIT_E;
    VSR_FIELD(AUX_SVC, pow2_width(K - 1 > 0 ? K - 1 : 1), 1, NS_COMMIT)
    VSR_FIELD(ACKED, 2, V, AUX_SVC)
    static constexpr int TOTAL_BITS = ACKED_E;
    static constexpr int NW = align_up(align_up(TOTAL_BITS, 32) / 32, 4); /* whole 16-byte units */
    static constexpr int BYTES = NW * 4;

    /* candidate (action, binding) index space: one entry per binding TLC's nested \E would try */
    static constexpr int C_TIMER = 0;                      /* r */
    static constexpr int C_HSVC = C_TIMER + R;             /* SVC slot */
    static constexpr int C_MSVC = C_HSVC + NSVC;           /* SVC slot */
    static constexpr int C_SDVC = C_MSVC + NSVC;           /* r */
    static constexpr int C_HDVC = C_SDVC + R;              /* DVC slot */
    static constexpr int C_MDVC = C_HDVC + NDVC;           /* DVC slot */
    static constexpr int C_SSV = C_MDVC + NDVC;            /* r */
    static constexpr int C_RSV = C_SSV + R;                /* SV slot */
    static constexpr int C_CREQ = C_RSV + NSV;             /* r * V + value index */
    static constexpr int C_RPREP = C_CREQ + R * V;         /* value * O + dest' */
    static constexpr int C_RPOK = C_RPREP + V * O;         /* PrepareOk slot */
    static constexpr int C_EXEC = C_RPOK + NPOK;           /* r */
    static constexpr int C_SGS = C_EXEC + R;               /* (value * O + dest') * O + rDest' */
    static constexpr int C_RGS = C_SGS + V * O * O;        /* GetState slot */
    static constexpr int C_RNS = C_RGS + NGS;              /* NewState slot */
    static constexpr int NCAND = C_RNS + NGS;
};

/* --- word access.  A state is normally a plain word pointer; the expand kernel also builds successors in a
   rotated shared-memory row (SwzRow) so that the 32 lanes of a warp, each owning one row, do not hit the same
   banks.  Everything above this layer goes through rdw()/wrw(). */
VSR_HD uint32_t rdw(const uint32_t* w, int i) { return w[i]; }
VSR_HD void wrw(uint32_t* w, int i, uint32_t v) { w[i] = v; }
template <int NW> struct SwzRow {
    uint32_t* base; /* NW words */
    int rot;        /* word i lives at base[(i + rot) mod NW] */
};
template <int NW> VSR_HD uint32_t rdw(const SwzRow<NW>& w, int i) {
    int x = i + w.rot;
    if (x >= NW) x -= NW;
    return w.base[x];
}
template <int NW> VSR_HD void wrw(const SwzRow<NW>& w, int i, uint32_t v) {
    int x = i + w.rot;
    if (x >= NW) x -= NW;
    w.base[x] = v;
}

/* A state held in registers (the expand kernel's guard scan).  A register array cannot be indexed at run time, so a
   read names the words it may touch — [LO, HI], known from the field's base, width and element count — and selects
   among them; with a compile-time index (the scan is fully unrolled) the chain folds to the one register. */
template <int NW> struct RegRow {
    uint32_t w[NW];
};
template <int LO, int HI, class S> VSR_HD uint32_t rdwr(const S& w, int i) { return rdw(w, i); }
template <int LO, int HI, int NW> VSR_HD uint32_t rdwr(const RegRow<NW>& r, int i) {
    constexpr int lo = HI < 0 ? 0 : LO, hi = HI < 0 ? NW - 1 : (HI < NW ? HI : NW - 1);
    uint32_t v = r.w[lo];
VSR_UNROLL
    for (int k = lo + 1; k <= hi; k++) v = i == k ? r.w[k] : v;
    return v;
}
template <int NW> VSR_HD uint32_t rdw(const RegRow<NW>& r, int i) { return rdwr<0, -1>(r, i); }

/* --- element access (base, width and element count compile-time; index run-time).  N = 0: count not given. */
template <int B, int W, int N = 0, class S> VSR_HD uint32_t fget(const S& w, int idx) {
    const int b = B + idx * W;
    return (rdwr<(B >> 5), (N > 0 ? ((B + W * N - 1) >> 5) : -1)>(w, b >> 5) >> (b & 31)) & ((1u << W) - 1u);
}
template <int B, int W, class S> VSR_HD void fset(const S& w, int idx, uint32_t val) {
    const int b = B + idx * W;
    const uint32_t m = ((1u << W) - 1u) << (b & 31);
    wrw(w, b >> 5, (rdw(w, b >> 5) & ~m) | ((val << (b & 31)) & m));
}
#define VGET(Lt, F, w, i) ::vsr::fget<Lt::F##_B, Lt::F##_W, Lt::F##_N>((w), (i))
#define VSET(Lt, F, w, i, v) ::vsr::fset<Lt::F##_B, Lt::F##_W>((w), (i), (uint32_t)(v))

} // namespace vsr
#endif
