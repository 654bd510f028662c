/*
 * vsr_actions.h — the Next relation of vsr-revisited/paper/VSR.tla:896-918 hand-lowered onto the
 * packed encoding of vsr_layout.h.  One source for host (C ABI: vsr_successors, trace replay) and
 * device (the BFS expand kernel).
 *
 * step<L, APPLY>(run, s, cand, out):
 *   cand indexes one binding of one action's \E (Layout::C_* ranges, textual order of Next);
 *   returns 0 if that binding's guard is false, a negative E_* code if the successor cannot be
 *   represented, else the number of TLC bindings this successor stands for (1, or the number of
 *   unused values for ReceiveClientRequest under SYMMETRY, where all unused values are one orbit).
 *   With APPLY = false only the guard is evaluated (out untouched).
 *
 * Recovery actions (RestartEmpty, ReceivesRecoveryMsg, ReceivesRecoveryResponseMsg, CompleteRecovery,
 * VSR.tla:813-894) are guarded by aux_restart < RestartEmptyLimit / status = Recovering and cannot
 * fire with RestartEmptyLimit = 0 (every shipped config, VSR.cfg:8); the loader rejects other values.
 */
#ifndef VSR_ACTIONS_H
#define VSR_ACTIONS_H

#include <utility>

#include "vsr_layout.h"

namespace vsr {

struct RunCfg {
    int symmetry;  /* SYMMETRY symmValues (VSR.cfg:31, VSR.tla:151) */
    int use_view;  /* VIEW view (VSR.cfg:29, VSR.tla:149-150) */
    int invariant; /* bitmask of INVARIANT names: 1 AcknowledgedWriteNotLost, 2 AcknowledgedWritesExistOnMajority,
                      4 NoLogDivergence, 8 TestInv (VSR.tla:926-952); 256 = test hook (see Ops::invariant) */
};

template <class L> struct Ops {
    static constexpr int R = L::R, V = L::V, K = L::K, O = L::O;

    static VSR_HD int primary(int v) { return (v - 1) % R; }             /* Primary, VSR.tla:287-288 (0-based) */
    static VSR_HD int oidx(int a, int b) { return b < a ? b : b - 1; }   /* index of b among replicas \ {a} */
    static VSR_HD int oinv(int a, int i) { return i < a ? i : i + 1; }

    template <int B, int N = 0, class W> static VSR_HD int loglen(const W& w, int row) { /* N: rows x V elements of the field */
        int n = 0;
        for (int i = 0; i < V; i++) {
            if (fget<B, L::OB, N>(w, row * V + i) == 0) break;
            n++;
        }
        return n;
    }
    template <int BD, int BS, class WD, class WS> static VSR_HD void logcopy(const WD& wd, int rowd, const WS& ws, int rows) {
        for (int i = 0; i < V; i++) fset<BD, L::OB>(wd, rowd * V + i, fget<BS, L::OB>(ws, rows * V + i));
    }
    template <int B, class W> static VSR_HD void logclear(const W& w, int row) {
        for (int i = 0; i < V; i++) fset<B, L::OB>(w, row * V + i, 0);
    }
    template <class W> static VSR_HD int popmask_svc(const W& w, int r) {
        int n = 0;
        for (int s = 0; s < R; s++) n += (int)VGET(L, SVC_MASK, w, r * R + s);
        return n;
    }
    template <class W> static VSR_HD int popmask_dvc(const W& w, int r) {
        int n = 0;
        for (int s = 0; s < R; s++) n += (int)VGET(L, DVC_MASK, w, r * R + s);
        return n;
    }
    /* ResetRecvMsgs, VSR.tla:299-301 (the self-DVC payload lives and dies with rep_dvc_recv[r]) */
    template <class W> static VSR_HD void reset_recv(const W& w, int r) {
        for (int s = 0; s < R; s++) {
            VSET(L, SVC_MASK, w, r * R + s, 0);
            VSET(L, DVC_MASK, w, r * R + s, 0);
        }
        logclear<L::SELF_LOG_B>(w, r);
        VSET(L, SELF_LNV, w, r, 0);
        VSET(L, SELF_COMMIT, w, r, 0);
    }
    template <class W> static VSR_HD void reset_dvc_only(const W& w, int r) {
        for (int s = 0; s < R; s++) VSET(L, DVC_MASK, w, r * R + s, 0);
        logclear<L::SELF_LOG_B>(w, r);
        VSET(L, SELF_LNV, w, r, 0);
        VSET(L, SELF_COMMIT, w, r, 0);
    }
    template <class W> static VSR_HD void reset_sent(const W& w, int r) { /* ResetSentVars :303-305 */
        VSET(L, SENT_DVC, w, r, 0);
        VSET(L, SENT_SV, w, r, 0);
    }
    static VSR_HD int svc_slot(int v, int s, int d) { return ((v - 2) * R + s) * O + oidx(s, d); }
    /* Broadcast(NewSVCMessage(r, v), r): BroadcastFunc :233-240 */
    template <class W> static VSR_HD int broadcast_svc(const W& w, int v, int s) {
        for (int dp = 0; dp < O; dp++) {
            const int idx = ((v - 2) * R + s) * O + dp;
            if (VGET(L, SVC_ST, w, idx) != ST_ABSENT) return E_SLOT_OCCUPIED;
            VSET(L, SVC_ST, w, idx, ST_PENDING);
        }
        return 0;
    }
    template <class W> static VSR_HD int ncreated(const W& w) {
        int c = 0;
        for (int x = 0; x < V; x++) c += VGET(L, PR_VIEW, w, x) != 0;
        return c;
    }

    /* ---------------------------------------------------------------- the step function */
    /* candidate groups: the blocks of the cascade below, in Next's textual order */
    static constexpr int NGRP = 13;
    static VSR_HD constexpr int grp_begin(int g) {
        const int b[NGRP + 1] = {L::C_TIMER, L::C_HSVC, L::C_SDVC, L::C_HDVC, L::C_SSV, L::C_RSV, L::C_CREQ, L::C_RPREP,
                                 L::C_RPOK, L::C_EXEC, L::C_SGS, L::C_RGS, L::C_RNS, L::NCAND};
        return b[g];
    }
    template <bool APPLY, class S, class N> static VSR_HD int step(const RunCfg& run, const S& s, int cand, const N& n) {
        return cand < L::C_HSVC ? step_grp<APPLY, 0, S, N>(run, s, cand, n) : cand < L::C_SDVC ? step_grp<APPLY, 1, S, N>(run, s, cand, n)
             : cand < L::C_HDVC ? step_grp<APPLY, 2, S, N>(run, s, cand, n) : cand < L::C_SSV ? step_grp<APPLY, 3, S, N>(run, s, cand, n)
             : cand < L::C_RSV ? step_grp<APPLY, 4, S, N>(run, s, cand, n) : cand < L::C_CREQ ? step_grp<APPLY, 5, S, N>(run, s, cand, n)
             : cand < L::C_RPREP ? step_grp<APPLY, 6, S, N>(run, s, cand, n) : cand < L::C_RPOK ? step_grp<APPLY, 7, S, N>(run, s, cand, n)
             : cand < L::C_EXEC ? step_grp<APPLY, 8, S, N>(run, s, cand, n) : cand < L::C_SGS ? step_grp<APPLY, 9, S, N>(run, s, cand, n)
             : cand < L::C_RGS ? step_grp<APPLY, 10, S, N>(run, s, cand, n) : cand < L::C_RNS ? step_grp<APPLY, 11, S, N>(run, s, cand, n)
             : step_grp<APPLY, 12, S, N>(run, s, cand, n);
    }
    /* one group's guard (+ effect when APPLY): only this group's code is instantiated, so the device can scan a
       group's candidates in a tight loop */
    template <bool APPLY, int GRP, class S, class N> static VSR_HD int step_grp(const RunCfg& run, const S& s, int cand, const N& n) {
        if constexpr (APPLY) {
            for (int i = 0; i < L::NW; i++) wrw(n, i, rdw(s, i));
        }
        /* ---- TimerSendSVC, VSR.tla:578-590 */
        if constexpr (GRP == 0) {
            const int r = cand - L::C_TIMER;
            const int aux = (int)VGET(L, AUX_SVC, s, 0);
            if (!(aux < L::L)) return 0;
            const int v = (int)VGET(L, VIEWN, s, r);
            if (primary(v) == r) return 0;
            if (!APPLY) return 1;
            if (v + 1 > K) return E_OVERFLOW;
            VSET(L, VIEWN, n, r, v + 1);
            VSET(L, STATUS, n, r, 1);
            reset_recv(n, r);
            reset_sent(n, r);
            VSET(L, AUX_SVC, n, 0, aux + 1);
            const int e = broadcast_svc(n, v + 1, r);
            return e ? e : 1;
        }
        /* ---- ReceiveHigherSVC :602-613 / ReceiveMatchingSVC :625-634 */
        if constexpr (GRP == 1) {
            const bool higher = cand < L::C_MSVC;
            const int idx = cand - (higher ? L::C_HSVC : L::C_MSVC);
            if (VGET(L, SVC_ST, s, idx) != ST_PENDING) return 0; /* ReceivableMsg :272-275 */
            const int dp = idx % O, src = (idx / O) % R, v = idx / (O * R) + 2;
            const int r = oinv(src, dp);
            const int vr = (int)VGET(L, VIEWN, s, r);
            if (higher) {
                if (!(v > vr)) return 0;
                if (!APPLY) return 1;
                VSET(L, VIEWN, n, r, v);
                VSET(L, STATUS, n, r, 1);
                reset_recv(n, r);
                VSET(L, SVC_MASK, n, r * R + src, 1);
                reset_sent(n, r);
                VSET(L, SVC_ST, n, idx, ST_CONSUMED); /* DiscardAndBroadcast :260-265 */
                const int e = broadcast_svc(n, v, r);
                return e ? e : 1;
            } else {
                if (!(v == vr)) return 0;
                if (VGET(L, STATUS, s, r) != 1) return 0;
                if (!APPLY) return 1;
                VSET(L, SVC_MASK, n, r * R + src, 1);
                VSET(L, SVC_ST, n, idx, ST_CONSUMED);
                return 1;
            }
        }
        /* ---- SendDVC :648-669 */
        if constexpr (GRP == 2) {
            const int r = cand - L::C_SDVC;
            if (VGET(L, STATUS, s, r) != 1) return 0;
            if (VGET(L, SENT_DVC, s, r) != 0) return 0;
            if (!(popmask_svc(s, r) >= R / 2)) return 0;
            if (!APPLY) return 1;
            const int v = (int)VGET(L, VIEWN, s, r);
            if (v < 2) return E_OVERFLOW;
            VSET(L, SENT_DVC, n, r, 1);
            const int p = primary(v);
            if (p == r) {
                if (VGET(L, DVC_MASK, s, r * R + r)) return E_SLOT_OCCUPIED;
                VSET(L, DVC_MASK, n, r * R + r, 1);
                logcopy<L::SELF_LOG_B, L::LOG_B>(n, r, s, r);
                VSET(L, SELF_LNV, n, r, VGET(L, LNV, s, r));
                VSET(L, SELF_COMMIT, n, r, VGET(L, COMMIT, s, r));
            } else {
                const int idx = (v - 2) * O + oidx(p, r);
                if (VGET(L, DVC_ST, s, idx) != ST_ABSENT) return E_SLOT_OCCUPIED;
                VSET(L, DVC_ST, n, idx, ST_PENDING);
                logcopy<L::DVC_LOG_B, L::LOG_B>(n, idx, s, r);
                VSET(L, DVC_LNV, n, idx, VGET(L, LNV, s, r));
                VSET(L, DVC_COMMIT, n, idx, VGET(L, COMMIT, s, r));
            }
            return 1;
        }
        /* ---- ReceiveHigherDVC :677-688 / ReceiveMatchingDVC :696-703 */
        if constexpr (GRP == 3) {
            const bool higher = cand < L::C_MDVC;
            const int idx = cand - (higher ? L::C_HDVC : L::C_MDVC);
            if (VGET(L, DVC_ST, s, idx) != ST_PENDING) return 0;
            const int v = idx / O + 2;
            const int r = primary(v); /* dest of every DVC(v) :660 */
            const int src = oinv(r, idx % O);
            const int vr = (int)VGET(L, VIEWN, s, r);
            if (higher) {
                if (!(v > vr)) return 0;
                if (!APPLY) return 1;
                VSET(L, VIEWN, n, r, v);
                VSET(L, STATUS, n, r, 1);
                reset_recv(n, r);
                VSET(L, DVC_MASK, n, r * R + src, 1);
                reset_sent(n, r);
                VSET(L, DVC_ST, n, idx, ST_CONSUMED);
                const int e = broadcast_svc(n, v, r);
                return e ? e : 1;
            } else {
                if (!(vr == v)) return 0;
                if (!APPLY) return 1;
                VSET(L, DVC_MASK, n, r * R + src, 1);
                VSET(L, DVC_ST, n, idx, ST_CONSUMED);
                return 1;
            }
        }
        /* ---- SendSV :735-760 with HighestLog/HighestOpNumber/HighestCommitNumber :716-733 */
        if constexpr (GRP == 4) {
            const int r = cand - L::C_SSV;
            if (VGET(L, STATUS, s, r) != 1) return 0;
            if (VGET(L, SENT_SV, s, r) != 0) return 0;
            if (!(popmask_dvc(s, r) >= R / 2 + 1)) return 0;
            if (!APPLY) return 1;
            const int v = (int)VGET(L, VIEWN, s, r);
            if (v < 2 || primary(v) != r) return E_NOT_PRIMARY;
            /* CHOOSE :717-721 = first, in TLC's set order, of the DVCs maximal on (last_normal_vn,
               op_number).  Tied records differ first in commit_number, then in source (SURVEY H3). */
            int best = -1, b_lnv = 0, b_op = 0, b_cn = 0, max_cn = 0;
            for (int src = 0; src < R; src++) {
                if (!VGET(L, DVC_MASK, s, r * R + src)) continue;
                int lnv, op, cn;
                if (src == r) {
                    lnv = (int)VGET(L, SELF_LNV, s, r);
                    cn = (int)VGET(L, SELF_COMMIT, s, r);
                    op = loglen<L::SELF_LOG_B>(s, r);
                } else {
                    const int di = (v - 2) * O + oidx(r, src);
                    if (VGET(L, DVC_ST, s, di) == ST_ABSENT) return E_MISSING_PAYLOAD;
                    lnv = (int)VGET(L, DVC_LNV, s, di);
                    cn = (int)VGET(L, DVC_COMMIT, s, di);
                    op = loglen<L::DVC_LOG_B>(s, di);
                }
                if (cn > max_cn) max_cn = cn;
                const bool better = best < 0 || lnv > b_lnv || (lnv == b_lnv && op > b_op) ||
                                    (lnv == b_lnv && op == b_op && cn < b_cn);
                if (better) { best = src; b_lnv = lnv; b_op = op; b_cn = cn; }
            }
            VSET(L, STATUS, n, r, 0);
            if (best == r) logcopy<L::LOG_B, L::SELF_LOG_B>(n, r, s, r);
            else logcopy<L::LOG_B, L::DVC_LOG_B>(n, r, s, (v - 2) * O + oidx(r, best));
            for (int p = 0; p < R; p++) VSET(L, PEER, n, r * R + p, 0);
            VSET(L, COMMIT, n, r, max_cn);
            VSET(L, SENT_SV, n, r, 1);
            VSET(L, LNV, n, r, v);
            for (int dp = 0; dp < O; dp++) {
                const int si = (v - 2) * O + dp;
                if (VGET(L, SV_ST, s, si) != ST_ABSENT) return E_SLOT_OCCUPIED;
                VSET(L, SV_ST, n, si, ST_PENDING);
            }
            logcopy<L::SV_LOG_B, L::LOG_B>(n, v - 2, n, r);
            VSET(L, SV_COMMIT, n, v - 2, max_cn);
            return 1;
        }
        /* ---- ReceiveSV :773-793 */
        if constexpr (GRP == 5) {
            const int idx = cand - L::C_RSV;
            if (VGET(L, SV_ST, s, idx) != ST_PENDING) return 0;
            const int v = idx / O + 2;
            const int p = primary(v);
            const int r = oinv(p, idx % O);
            if (!(v >= (int)VGET(L, VIEWN, s, r))) return 0;
            if (!APPLY) return 1;
            const int old_commit = (int)VGET(L, COMMIT, s, r);
            const int mop = loglen<L::SV_LOG_B>(s, v - 2);
            VSET(L, STATUS, n, r, 0);
            VSET(L, VIEWN, n, r, v);
            logcopy<L::LOG_B, L::SV_LOG_B>(n, r, s, v - 2);
            VSET(L, COMMIT, n, r, VGET(L, SV_COMMIT, s, v - 2));
            VSET(L, LNV, n, r, v);
            reset_recv(n, r);
            reset_sent(n, r);
            VSET(L, SV_ST, n, idx, ST_CONSUMED);
            if (old_commit < mop) { /* the OLD commit number :785 */
                const int pi = ((v - 1) * V + (mop - 1)) * O + oidx(p, r);
                if (VGET(L, POK_ST, s, pi) != ST_ABSENT) return E_SLOT_OCCUPIED;
                VSET(L, POK_ST, n, pi, ST_PENDING);
            }
            return 1;
        }
        /* ---- ReceiveClientRequest :366-394 */
        if constexpr (GRP == 6) {
            const int r = (cand - L::C_CREQ) / V, vi = (cand - L::C_CREQ) % V;
            const int v = (int)VGET(L, VIEWN, s, r);
            if (primary(v) != r) return 0;
            if (VGET(L, STATUS, s, r) != 0) return 0;
            if (!VGET(L, CT_EXEC, s, r)) return 0;
            int mult = 1, slot;
            if (run.symmetry) {
                /* all unused values are one symmetry orbit: one successor stands for V - created bindings */
                const int c = ncreated(s);
                if (vi != 0 || c >= V) return 0;
                mult = V - c;
                slot = c; /* provisional: last; moved to its sorted place below */
            } else {
                if (VGET(L, PR_VIEW, s, vi) != 0) return 0; /* v \notin DOMAIN aux_client_acked :370 */
                slot = vi;
            }
            if (!APPLY) return mult;
            const int req = (int)VGET(L, CT_REQ, s, r) + 1;
            const int op = loglen<L::LOG_B, L::LOG_N>(s, r) + 1;
            if (req > V || op > V) return E_OVERFLOW;
            if (run.symmetry) {
                /* canonical labels: created values ordered by the (view, op_number) of their Prepare */
                int p = 0;
                for (int x = 0; x < slot; x++) {
                    const int xv = (int)VGET(L, PR_VIEW, s, x), xo = (int)VGET(L, PR_OP, s, x);
                    if (xv == v && xo == op) return E_PREPKEY_CLASH;
                    if (xv < v || (xv == v && xo < op)) p = x + 1;
                }
                if (p < slot) {
                    for (int x = slot; x > p; x--) { /* shift Prepare slots and acked p..slot-1 up by one */
                        VSET(L, PR_VIEW, n, x, VGET(L, PR_VIEW, n, x - 1));
                        VSET(L, PR_REQ, n, x, VGET(L, PR_REQ, n, x - 1));
                        VSET(L, PR_OP, n, x, VGET(L, PR_OP, n, x - 1));
                        VSET(L, PR_COMMIT, n, x, VGET(L, PR_COMMIT, n, x - 1));
                        for (int dp = 0; dp < O; dp++) VSET(L, PR_CONS, n, x * O + dp, VGET(L, PR_CONS, n, (x - 1) * O + dp));
                        VSET(L, ACKED, n, x, VGET(L, ACKED, n, x - 1));
                    }
                    for (int i = 0; i < L::ALL_LOGS_N; i++) { /* value ids > p move up by one */
                        const uint32_t e = fget<L::ALL_LOGS_B, L::OB>(n, i);
                        if (e > (uint32_t)p) fset<L::ALL_LOGS_B, L::OB>(n, i, e + 1);
                    }
                    slot = p;
                }
            }
            VSET(L, PR_VIEW, n, slot, v);
            VSET(L, PR_REQ, n, slot, req);
            VSET(L, PR_OP, n, slot, op);
            VSET(L, PR_COMMIT, n, slot, VGET(L, COMMIT, s, r));
            for (int dp = 0; dp < O; dp++) VSET(L, PR_CONS, n, slot * O + dp, 0);
            VSET(L, LOG, n, r * V + (op - 1), slot + 1);
            VSET(L, CT_REQ, n, r, req);
            VSET(L, CT_OP, n, r, op);
            VSET(L, CT_EXEC, n, r, 0);
            VSET(L, ACKED, n, slot, ACK_FALSE);
            return mult;
        }
        /* ---- ReceivePrepareMsg :405-428 */
        if constexpr (GRP == 7) {
            const int x = (cand - L::C_RPREP) / O, dp = (cand - L::C_RPREP) % O;
            const int pv = (int)VGET(L, PR_VIEW, s, x);
            if (pv == 0) return 0;
            if (VGET(L, PR_CONS, s, x * O + dp)) return 0;
            const int src = primary(pv);
            const int r = oinv(src, dp);
            if (VGET(L, STATUS, s, r) != 0) return 0;
            if (pv != (int)VGET(L, VIEWN, s, r)) return 0;
            const int mop = (int)VGET(L, PR_OP, s, x);
            if (mop != loglen<L::LOG_B, L::LOG_N>(s, r) + 1) return 0;
            if (!APPLY) return 1;
            const int mcn = (int)VGET(L, PR_COMMIT, s, x);
            VSET(L, LOG, n, r * V + (mop - 1), x + 1);
            VSET(L, COMMIT, n, r, mcn);
            VSET(L, CT_REQ, n, r, VGET(L, PR_REQ, s, x));
            VSET(L, CT_OP, n, r, mop);
            VSET(L, CT_EXEC, n, r, mop <= mcn ? 1 : 0);
            VSET(L, PR_CONS, n, x * O + dp, 1);
            const int pi = ((pv - 1) * V + (mop - 1)) * O + oidx(src, r);
            if (VGET(L, POK_ST, s, pi) != ST_ABSENT) return E_SLOT_OCCUPIED;
            VSET(L, POK_ST, n, pi, ST_PENDING);
            return 1;
        }
        /* ---- ReceivePrepareOkMsg :437-447 */
        if constexpr (GRP == 8) {
            const int idx = cand - L::C_RPOK;
            if (VGET(L, POK_ST, s, idx) != ST_PENDING) return 0;
            const int sp = idx % O, nn = (idx / O) % V + 1, v = idx / (O * V) + 1;
            const int r = primary(v);
            const int src = oinv(r, sp);
            if (v != (int)VGET(L, VIEWN, s, r)) return 0; /* IsPrimary(r) follows from r = Primary(v) = Primary(View(r)) */
            if (VGET(L, STATUS, s, r) != 0) return 0;
            if (!(nn > (int)VGET(L, PEER, s, r * R + src))) return 0;
            if (!APPLY) return 1;
            VSET(L, PEER, n, r * R + src, nn);
            VSET(L, POK_ST, n, idx, ST_CONSUMED);
            return 1;
        }
        /* ---- ExecuteOp :462-476, IsCommitted :457-460 */
        if constexpr (GRP == 9) {
            const int r = cand - L::C_EXEC;
            if (primary((int)VGET(L, VIEWN, s, r)) != r) return 0;
            if (VGET(L, STATUS, s, r) != 0) return 0;
            const int cn = (int)VGET(L, COMMIT, s, r);
            if (!(cn < loglen<L::LOG_B, L::LOG_N>(s, r))) return 0;
            int q = 0;
            for (int p = 0; p < R; p++) q += (int)VGET(L, PEER, s, r * R + p) >= cn + 1;
            if (!(q >= R / 2)) return 0;
            if (!APPLY) return 1;
            VSET(L, COMMIT, n, r, cn + 1);
            VSET(L, CT_EXEC, n, r, 1);
            const int x = (int)VGET(L, LOG, s, r * V + cn); /* rep_log[r][cn+1].operation */
            VSET(L, ACKED, n, x - 1, ACK_TRUE);
            return 1;
        }
        /* ---- SendGetState :496-516 */
        if constexpr (GRP == 10) {
            const int c = cand - L::C_SGS;
            const int j = c % O, dp = (c / O) % O, x = c / (O * O);
            const int pv = (int)VGET(L, PR_VIEW, s, x);
            if (pv == 0) return 0;
            if (VGET(L, PR_CONS, s, x * O + dp)) return 0;
            const int src = primary(pv);
            const int r = oinv(src, dp);
            const int rdest = oinv(r, j);
            const int vr = (int)VGET(L, VIEWN, s, r);
            if (primary(vr) == r) return 0;
            if (VGET(L, STATUS, s, r) != 0) return 0;
            if (!(pv > vr)) return 0;
            const int len = loglen<L::LOG_B, L::LOG_N>(s, r);
            if (!((int)VGET(L, PR_OP, s, x) > len + 1)) return 0;
            const int cn = (int)VGET(L, COMMIT, s, r);
            const int t = cn <= len ? cn : len; /* MinVal :307-308 */
            const int gi = (pv - 2) * O + oidx(src, r);
            if (VGET(L, GS_ST, s, gi) != ST_ABSENT) {
                /* SendOnce :250-252: the same record already in DOMAIN messages disables the action */
                if ((int)VGET(L, GS_T, s, gi) == t && (int)VGET(L, GS_DEST, s, gi) == rdest) return 0;
                return APPLY ? E_SLOT_OCCUPIED : 1;
            }
            if (!APPLY) return 1;
            if (popmask_svc(s, r) != 0 || popmask_dvc(s, r) != 0) return E_STALE_RECV;
            for (int i = t; i < V; i++) VSET(L, LOG, n, r * V + i, 0); /* TruncateLogToCommitNumber :491-494 */
            VSET(L, VIEWN, n, r, pv);
            VSET(L, LNV, n, r, pv);
            VSET(L, GS_ST, n, gi, ST_PENDING);
            VSET(L, GS_T, n, gi, t);
            VSET(L, GS_DEST, n, gi, rdest);
            return 1;
        }
        /* ---- ReceiveGetState :526-543 */
        if constexpr (GRP == 11) {
            const int gi = cand - L::C_RGS;
            if (VGET(L, GS_ST, s, gi) != ST_PENDING) return 0;
            const int v = gi / O + 2;
            const int r = (int)VGET(L, GS_DEST, s, gi);
            if ((int)VGET(L, VIEWN, s, r) != v) return 0;
            if (VGET(L, STATUS, s, r) != 0) return 0;
            const int t = (int)VGET(L, GS_T, s, gi);
            const int len = loglen<L::LOG_B, L::LOG_N>(s, r);
            if (!(len > t)) return 0;
            if (!APPLY) return 1;
            VSET(L, GS_ST, n, gi, ST_CONSUMED);
            if (VGET(L, NS_ST, s, gi) != ST_ABSENT) return E_SLOT_OCCUPIED;
            VSET(L, NS_ST, n, gi, ST_PENDING);
            for (int i = 0; i < V; i++) VSET(L, NS_LOG, n, gi * V + i, (i >= t && i < len) ? VGET(L, LOG, s, r * V + i) : 0);
            VSET(L, NS_COMMIT, n, gi, VGET(L, COMMIT, s, r));
            return 1;
        }
        /* ---- ReceiveNewState :551-567 */
        if constexpr (GRP == 12) {
            const int gi = cand - L::C_RNS;
            if (VGET(L, NS_ST, s, gi) != ST_PENDING) return 0;
            const int v = gi / O + 2;
            const int r = oinv(primary(v), gi % O); /* dest of NewState = source of the GetState */
            if ((int)VGET(L, VIEWN, s, r) != v) return 0;
            if (VGET(L, STATUS, s, r) != 0) return 0;
            const int t = (int)VGET(L, GS_T, s, gi); /* first_op - 1 */
            if (loglen<L::LOG_B, L::LOG_N>(s, r) != t) return 0;
            if (!APPLY) return 1;
            for (int i = t; i < V; i++) VSET(L, LOG, n, r * V + i, VGET(L, NS_LOG, s, gi * V + i));
            VSET(L, NS_ST, n, gi, ST_CONSUMED);
            return 1;
        }
        return 0;
    }

    /* Guards of one group on a state whose words are in registers (RegRow): bit i of mask[i / 32] is set iff candidate
       grp_begin(G) + i is enabled.  The candidate index is a compile-time constant in every guard, so slot decoding,
       word indices and shifts fold away: a guard is a handful of bit tests on registers.  Same guards as step_grp<false>
       (it IS step_grp<false>); tests/harness compares the masks with the one-candidate-at-a-time form on the host. */
    static VSR_HD constexpr int grp_size(int g) { return grp_begin(g + 1) - grp_begin(g); }
    static VSR_HD constexpr int grp_words(int g) { return (grp_size(g) + 31) / 32; }
    template <int G, class S, int... I>
    static VSR_HD void enabled_seq(const RunCfg& run, const S& s, uint32_t* mask, std::integer_sequence<int, I...>) {
        ((mask[I >> 5] |= (uint32_t)(step_grp<false, G>(run, s, grp_begin(G) + I, (uint32_t*)nullptr) > 0) << (I & 31)), ...);
    }
    template <int G, class S> static VSR_HD void enabled_group(const RunCfg& run, const S& s, uint32_t* mask) {
        enabled_seq<G>(run, s, mask, std::make_integer_sequence<int, grp_size(G)>());
    }

    /* the enabled candidates of a state, in candidate order, through the register-mask form (host side of the C ABI's
       vsr_enabled_candidates, which cross-checks it against the one-candidate form) */
    template <int G> static VSR_HD int list_group(const RunCfg& run, const RegRow<L::NW>& st, uint32_t* out, int n) {
        uint32_t m[grp_words(G) > 0 ? grp_words(G) : 1] = {}; /* StartViewOnTimerLimit = 0 leaves the view-change groups empty */
        enabled_group<G>(run, st, m);
        for (int i = 0; i < grp_size(G); i++)
            if ((m[i >> 5] >> (i & 31)) & 1u) out[n++] = (uint32_t)(grp_begin(G) + i);
        if constexpr (G + 1 < NGRP) return list_group<G + 1>(run, st, out, n);
        else return n;
    }
    static VSR_HD int enabled_list(const RunCfg& run, const uint32_t* w, uint32_t* out /* NCAND entries */) {
        RegRow<L::NW> st;
        for (int i = 0; i < L::NW; i++) st.w[i] = w[i];
        return list_group<0>(run, st, out, 0);
    }

    /* action id (VSR_ACT_*, = textual position in Next) of a candidate index */
    static VSR_HD int action_of(int cand) {
        return cand < L::C_HSVC ? 1 : cand < L::C_MSVC ? 2 : cand < L::C_SDVC ? 3 : cand < L::C_HDVC ? 4
             : cand < L::C_MDVC ? 5 : cand < L::C_SSV ? 6 : cand < L::C_RSV ? 7 : cand < L::C_CREQ ? 8
             : cand < L::C_RPREP ? 9 : cand < L::C_RPOK ? 10 : cand < L::C_EXEC ? 11 : cand < L::C_SGS ? 12
             : cand < L::C_RGS ? 13 : cand < L::C_RNS ? 14 : 15;
    }

    /* Init, VSR.tla:323-348 */
    static VSR_HD void init(uint32_t* w) {
        for (int i = 0; i < L::NW; i++) w[i] = 0;
        for (int r = 0; r < R; r++) {
            VSET(L, VIEWN, w, r, 1);
            VSET(L, CT_EXEC, w, r, 1); /* EmptyClientTableRow :318-321 */
        }
    }

    /* invariants, VSR.tla:926-952; returns the mask of the selected ones the state violates (0 = all hold).  Every value is
       visited: a state can violate both, and which one TLC names depends on the INVARIANT order (vsr_reported_invariant) */
    template <class W> static VSR_HD int invariant(const RunCfg& run, const W& w) {
        int bad = 0;
        if (run.invariant & 256) { /* test hook, not a spec invariant (only reachable through vsr_model_create): "no replica has
                                      committed every value" — violated often, so tests can exercise the violation paths */
            for (int r = 0; r < R; r++)
                if ((int)VGET(L, COMMIT, w, r) == V) bad = 256;
        }
        if (!(run.invariant & 3)) return bad; /* NoLogDivergence is vacuous (r1/r1, :931), TestInv is TRUE */
        for (int x = 0; x < V; x++) {
            if (VGET(L, ACKED, w, x) != ACK_TRUE) continue;
            int holders = 0;
            for (int r = 0; r < R; r++) {
                int has = 0;
                for (int i = 0; i < V; i++) has |= (int)VGET(L, LOG, w, r * V + i) == x + 1; /* ReplicaHasOp :933-935 */
                holders += has;
            }
            if ((run.invariant & 1) && holders == 0) bad |= 1;         /* AcknowledgedWriteNotLost :945-950 */
            if ((run.invariant & 2) && holders < R / 2 + 1) bad |= 2;  /* AcknowledgedWritesExistOnMajority :937-943 */
        }
        return bad;
    }

    /* AllReplicasMoveToSameView, VSR.tla:958-962: every replica is Normal and all have the same view number.  The state
       predicate under ViewChangeCompletes == []<>AllReplicasMoveToSameView; reads only rep_status and rep_view_number */
    template <class W> static VSR_HD bool all_same_view_normal(const RunCfg&, const W& w) {
        const uint32_t v0 = VGET(L, VIEWN, w, 0);
        for (int r = 0; r < R; r++)
            if (VGET(L, STATUS, w, r) != 0 || VGET(L, VIEWN, w, r) != v0) return false;
        return true;
    }
    /* test hook of the liveness pass (vsr_model_create only), not a spec predicate: "some replica has committed" — false
       at Init, and some reachable states where it is false have no successor, so tests reach the violation paths */
    template <class W> static VSR_HD bool some_commit(const W& w) {
        for (int r = 0; r < R; r++)
            if (VGET(L, COMMIT, w, r) >= 1) return true;
        return false;
    }
    /* the predicate the liveness pass checks: P, or Q when the test hook (LIVE_HOOK_Q of vsr_model.h, bit 1) is on */
    template <class W> static VSR_HD bool live_pred(const RunCfg& run, const W& w, int live_hooks) {
        return (live_hooks & 1) ? some_commit(w) : all_same_view_normal(run, w);
    }

    /* label-independent key of the aux variables for same-level VIEW ties (DESIGN.md §H2); same
       number the oracle's aux_key() computes */
    template <class W> static VSR_HD uint32_t aux_key(const W& w) {
        uint32_t k = VGET(L, AUX_SVC, w, 0);
        k = k * 16u; /* aux_restart = 0 */
        for (int x = 0; x < V; x++) k = k * 3u + VGET(L, ACKED, w, x);
        return k;
    }

    /* Counterexamples are replayed with literal value names (TLC prints the un-permuted states).  The
       engine's candidate indices refer to canonical labels (created values in (view, op_number) order
       of their Prepare); this maps such an index to the candidate index on a literally labelled
       state w.  Returns -1 if there is no such candidate. */
    static VSR_HD int literal_cand(const uint32_t* w, int cand) {
        if (cand < L::C_CREQ || cand >= L::C_RGS || (cand >= L::C_RPOK && cand < L::C_SGS)) return cand;
        if (cand < L::C_RPREP) { /* ReceiveClientRequest: "the next unused value" */
            const int r = (cand - L::C_CREQ) / V;
            for (int x = 0; x < V; x++)
                if (VGET(L, PR_VIEW, w, x) == 0) return L::C_CREQ + r * V + x;
            return -1;
        }
        int order[V > 0 ? V : 1], nc = 0;
        for (int x = 0; x < V; x++)
            if (VGET(L, PR_VIEW, w, x)) order[nc++] = x;
        for (int i = 1; i < nc; i++) {
            const int x = order[i];
            const int kx = (int)VGET(L, PR_VIEW, w, x) * 16 + (int)VGET(L, PR_OP, w, x);
            int j = i - 1;
            while (j >= 0 && (int)VGET(L, PR_VIEW, w, order[j]) * 16 + (int)VGET(L, PR_OP, w, order[j]) > kx) { order[j + 1] = order[j]; j--; }
            order[j + 1] = x;
        }
        if (cand < L::C_RPOK) {
            const int c = cand - L::C_RPREP, x = c / O;
            return x < nc ? L::C_RPREP + order[x] * O + c % O : -1;
        }
        const int c = cand - L::C_SGS, x = c / (O * O);
        return x < nc ? L::C_SGS + order[x] * O * O + c % (O * O) : -1;
    }

    /* Simulation mode (TLC `-simulate`, README.md:22 of the reference): one step of a random walk.  Picks uniformly among
       the enabled (action, binding) candidates by reservoir sampling — one pass, one draw per enabled candidate — so host
       and device walk identically for the same generator state.  Returns the chosen candidate, -1 if none is enabled. */
    static VSR_HD uint64_t rng_next(uint64_t& x) { /* splitmix64 */
        uint64_t z = (x += 0x9E3779B97F4A7C15ULL);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        return z ^ (z >> 31);
    }
    static VSR_HD int random_enabled(const RunCfg& run, const uint32_t* s, uint64_t& rng) {
        int chosen = -1, n = 0;
        for (int cand = 0; cand < L::NCAND; cand++) {
            if (step<false>(run, s, cand, (uint32_t*)nullptr) <= 0) continue;
            n++;
            if (rng_next(rng) % (uint64_t)n == 0) chosen = cand;
        }
        return chosen;
    }

    /* General canonicalisation under SYMMETRY for an arbitrarily labelled packed state: relabel the
       created values in (view, op_number) order of their Prepare.  step() keeps states canonical
       incrementally; this is for pack() and for tests.  Returns 0 or E_PREPKEY_CLASH. */
    static VSR_HD int canonicalize(uint32_t* w) {
        int order[V > 0 ? V : 1], nc = 0; /* created slots sorted by key */
        for (int x = 0; x < V; x++)
            if (VGET(L, PR_VIEW, w, x)) order[nc++] = x;
        for (int i = 1; i < nc; i++) { /* insertion sort */
            const int x = order[i];
            const int kx = (int)VGET(L, PR_VIEW, w, x) * 16 + (int)VGET(L, PR_OP, w, x);
            int j = i - 1;
            while (j >= 0) {
                const int y = order[j];
                const int ky = (int)VGET(L, PR_VIEW, w, y) * 16 + (int)VGET(L, PR_OP, w, y);
                if (ky == kx) return E_PREPKEY_CLASH;
                if (ky < kx) break;
                order[j + 1] = y;
                j--;
            }
            order[j + 1] = x;
        }
        int newlab[V + 1];
        newlab[0] = 0;
        for (int x = 0; x < V; x++) newlab[x + 1] = 0;
        for (int i = 0; i < nc; i++) newlab[order[i] + 1] = i + 1;
        bool ident = true;
        for (int i = 0; i < nc; i++) ident = ident && order[i] == i;
        if (ident) return 0;
        uint32_t o[L::NW];
        for (int i = 0; i < L::NW; i++) o[i] = w[i];
        for (int x = 0; x < V; x++) {
            VSET(L, PR_VIEW, w, x, 0); VSET(L, PR_REQ, w, x, 0); VSET(L, PR_OP, w, x, 0); VSET(L, PR_COMMIT, w, x, 0);
            for (int dp = 0; dp < O; dp++) VSET(L, PR_CONS, w, x * O + dp, 0);
            VSET(L, ACKED, w, x, 0);
        }
        for (int i = 0; i < nc; i++) {
            const int x = order[i];
            VSET(L, PR_VIEW, w, i, VGET(L, PR_VIEW, o, x)); VSET(L, PR_REQ, w, i, VGET(L, PR_REQ, o, x));
            VSET(L, PR_OP, w, i, VGET(L, PR_OP, o, x)); VSET(L, PR_COMMIT, w, i, VGET(L, PR_COMMIT, o, x));
            for (int dp = 0; dp < O; dp++) VSET(L, PR_CONS, w, i * O + dp, VGET(L, PR_CONS, o, x * O + dp));
            VSET(L, ACKED, w, i, VGET(L, ACKED, o, x));
        }
        for (int i = 0; i < L::ALL_LOGS_N; i++) {
            const uint32_t e = fget<L::ALL_LOGS_B, L::OB>(o, i);
            fset<L::ALL_LOGS_B, L::OB>(w, i, (uint32_t)newlab[e]);
        }
        return 0;
    }
};

/* ---------------------------------------------------------------- FP64 (TLC's Rabin fingerprint)
 * TLC's tlc2.util.FP64 is not in the reference (external tool); this restates its published
 * construction (SURVEY App. B.1): 64-bit Rabin fingerprint over GF(2), polynomial Polys[0] =
 * 0x911498AE0E66BAD6 (TLC's `-fp 0`), bit 63 = x^0, one byte per step through ByteModTable_7:
 *     fp = (fp >>> 8) ^ T[(b ^ fp) & 0xFF],   initial fp = the polynomial.
 * It is applied to the bytes of the packed VIEW projection (little-endian words), not to TLC's
 * own value serialisation — fingerprint VALUES therefore differ from a TLC run (they also differ
 * between TLC runs: model values hash by intern index).  tests/ check the polynomial is irreducible.
 */
constexpr uint64_t FP64_POLY = 0x911498AE0E66BAD6ULL;

/* Test builds only (tests/test_fp_collisions.py, tools/variants.sh "weakfp"): -DVSR_WEAK_FP_BITS=k keeps the low k bits
   of both fingerprint forms, host and device alike, so that different states share fingerprints all the time and the
   seen-set has to keep them apart by their check hash.  k = 0 gives every state fingerprint 0 (1 after the usual remap):
   one probe chain.  The product build never defines it. */
#ifdef VSR_WEAK_FP_BITS
static_assert(VSR_WEAK_FP_BITS >= 0 && VSR_WEAK_FP_BITS <= 63, "VSR_WEAK_FP_BITS: 0..63");
VSR_HD uint64_t fp64_weaken(uint64_t fp) { return fp & ((1ull << VSR_WEAK_FP_BITS) - 1ull); }
#else
VSR_HD uint64_t fp64_weaken(uint64_t fp) { return fp; }
#endif

inline void fp64_build_table(uint64_t tab[256]) {
    uint64_t power[72];
    uint64_t t = 0x8000000000000000ULL;
    for (int i = 0; i < 72; i++) {
        power[i] = t;
        t = (t >> 1) ^ ((t & 1) ? FP64_POLY : 0);
    }
    for (int j = 0; j < 256; j++) {
        uint64_t v = 0;
        for (int k = 0; k < 8; k++)
            if (j & (1 << k)) v ^= power[127 - 56 - k];
        tab[j] = v;
    }
}

template <class L> VSR_HD uint64_t fp64_view(const uint64_t* __restrict__ tab, const uint32_t* w, bool use_view) {
    /* byte-at-a-time form (the definition) */
    uint64_t fp = FP64_POLY;
    constexpr int full = L::VIEW_BITS >> 5, rem = L::VIEW_BITS & 31;
    const int nw = use_view ? (full + (rem ? 1 : 0)) : L::NW;
    for (int i = 0; i < nw; i++) {
        uint32_t x = w[i];
        if (use_view && i == full) x &= (1u << rem) - 1u;
        for (int b = 0; b < 4; b++) {
            fp = (fp >> 8) ^ tab[(x ^ (uint32_t)fp) & 0xFF];
            x >>= 8;
        }
    }
    return fp64_weaken(fp);
}

/* Slicing-by-8: the same function eight bytes per step.  S[j][b] = state after byte b followed by j zero bytes,
   so fp' = S7[y0] ^ S6[y1] ^ ... ^ S0[y7] with y = fp ^ (next 8 bytes, little-endian).  The eight lookups of a
   step are independent (the byte form is a chain of 4*NW dependent shared-memory loads). */
inline void fp64_build_slices(uint64_t s8[8 * 256]) {
    fp64_build_table(s8);
    for (int j = 1; j < 8; j++)
        for (int b = 0; b < 256; b++) {
            const uint64_t p = s8[(j - 1) * 256 + b];
            s8[j * 256 + b] = (p >> 8) ^ s8[p & 0xFF];
        }
}

template <class L, bool USE_VIEW, class W> VSR_HD uint64_t fp64_view8_t(const uint64_t* __restrict__ s8, const W& w) {
    static_assert(L::NW % 2 == 0, "whole 64-bit words");
#ifdef VSR_EXP_FASTHASH
    /* experiment only (tools/variants.sh): what the 48-lookup FP64 walk costs.  A multiply-xorshift hash of the same
       words; NOT TLC's fingerprint function, so never the default. */
    {
        constexpr int full_ = L::VIEW_BITS >> 5, rem_ = L::VIEW_BITS & 31;
        constexpr int nw_ = USE_VIEW ? (full_ + (rem_ ? 1 : 0)) : L::NW;
        uint64_t h = FP64_POLY;
        VSR_UNROLL
        for (int i = 0; i < nw_; i += 2) {
            uint32_t lo = rdw(w, i), hi = i + 1 < nw_ ? rdw(w, i + 1) : 0u;
            if (USE_VIEW && i == full_) lo &= (1u << rem_) - 1u;
            if (USE_VIEW && i + 1 == full_) hi &= (1u << rem_) - 1u;
            h ^= ((uint64_t)hi << 32) | lo;
            h *= 0x9E3779B97F4A7C15ULL;
            h ^= h >> 29;
        }
        h *= 0xBF58476D1CE4E5B9ULL;
        h ^= h >> 32;
        (void)s8;
        return h;
    }
#endif
    uint64_t fp = FP64_POLY;
    constexpr int full = L::VIEW_BITS >> 5, rem = L::VIEW_BITS & 31;
    /* bytes of whole zero words after the VIEW prefix are not hashed by the byte form either: hash ceil(nw/2) pairs,
       but an odd word count must not pull in the next word: mask it to zero and stop the byte count there */
    constexpr int nw = USE_VIEW ? (full + (rem ? 1 : 0)) : L::NW;
    int i = 0;
VSR_UNROLL
    for (; i + 1 < nw; i += 2) {
        uint32_t lo = rdw(w, i), hi = rdw(w, i + 1);
        if (USE_VIEW && i + 1 == full) hi &= (1u << rem) - 1u;
        const uint64_t y = fp ^ (((uint64_t)hi << 32) | lo);
        fp = s8[7 * 256 + (y & 0xFF)] ^ s8[6 * 256 + ((y >> 8) & 0xFF)] ^ s8[5 * 256 + ((y >> 16) & 0xFF)] ^
             s8[4 * 256 + ((y >> 24) & 0xFF)] ^ s8[3 * 256 + ((y >> 32) & 0xFF)] ^ s8[2 * 256 + ((y >> 40) & 0xFF)] ^
             s8[1 * 256 + ((y >> 48) & 0xFF)] ^ s8[(y >> 56) & 0xFF];
    }
    if (nw & 1) { /* one trailing 32-bit word: four bytes */
        uint32_t x = rdw(w, nw - 1);
        if (USE_VIEW && nw - 1 == full) x &= (1u << rem) - 1u;
        const uint32_t y = x ^ (uint32_t)fp;
        fp = (fp >> 32) ^ s8[3 * 256 + (y & 0xFF)] ^ s8[2 * 256 + ((y >> 8) & 0xFF)] ^ s8[1 * 256 + ((y >> 16) & 0xFF)] ^ s8[(y >> 24) & 0xFF];
    }
    return fp64_weaken(fp);
}
template <class L, class W> VSR_HD uint64_t fp64_view8(const uint64_t* __restrict__ s8, const W& w, bool use_view) {
    return use_view ? fp64_view8_t<L, true>(s8, w) : fp64_view8_t<L, false>(s8, w);
}

} // namespace vsr
#endif
