/*
 * vsr_oracle.cpp — semantics of VSR.tla restated on the CPU (see vsr_oracle.h header comment:
 * test infrastructure only; pinned to state_transfer_violation_trace.txt and, through oracle/tla_eval.py,
 * to the text of VSR.tla itself; TLC's fingerprint values and the totals of the big configurations unpinned).
 * Every function cites the lines of the reference's vsr-revisited/paper/VSR.tla it follows.
 */
#include "vsr_oracle.h"

#include <algorithm>
#include <cassert>
#include <cstring>

namespace orc {

/* ------------------------------------------------------------------ value order (TLC compareTo) */

int cmp_entry(const Entry& a, const Entry& b) {
    /* record fields in first-interned order: view_number, operation, client_id, request_number
       (VSR.tla:157-161; order evidenced by state_transfer_violation_trace.txt:32) */
    if (a.view != b.view) return a.view < b.view ? -1 : 1;
    if (a.operation != b.operation) return a.operation < b.operation ? -1 : 1;
    if (a.client != b.client) return a.client < b.client ? -1 : 1;
    if (a.req != b.req) return a.req < b.req ? -1 : 1;
    return 0;
}

/* field-name intern order evidenced by the trace file (SURVEY §4, App. B.3):
   view_number(0) operation(1) client_id(2) request_number(3) type(4) message(5) op_number(6)
   commit_number(7) dest(8) source(9) log(10) last_normal_vn(11) x(12) executed(13) first_op(14) */
enum { F_VIEW = 0, F_TYPE = 4, F_MESSAGE = 5, F_OP = 6, F_COMMIT = 7, F_DEST = 8, F_SRC = 9, F_LOG = 10,
       F_LNV = 11, F_X = 12, F_FIRSTOP = 14 };

static int field_names(const Msg& m, int* names) {
    int n = 0;
    if (m.view != ABSENT) names[n++] = F_VIEW;
    names[n++] = F_TYPE;
    if (m.has_entry) names[n++] = F_MESSAGE;
    if (m.op != ABSENT) names[n++] = F_OP;
    if (m.commit != ABSENT) names[n++] = F_COMMIT;
    if (m.dest != ABSENT) names[n++] = F_DEST;
    if (m.src != ABSENT) names[n++] = F_SRC;
    if (m.has_log) names[n++] = F_LOG;
    if (m.lnv != ABSENT) names[n++] = F_LNV;
    if (m.x != ABSENT) names[n++] = F_X;
    if (m.first_op != ABSENT) names[n++] = F_FIRSTOP;
    return n;
}

static inline int cmp_int_or_nil(int a, int b) {
    /* a model value (Nil) sorts before any non-model value */
    if (a == b) return 0;
    if (a == NIL) return -1;
    if (b == NIL) return 1;
    return a < b ? -1 : 1;
}

static int cmp_log(const Msg& a, const Msg& b) {
    if (a.has_log != b.has_log) return a.has_log == 2 ? -1 : 1; /* Nil first */
    if (a.has_log == 2) return 0;
    /* function order: domain size, then (key, value) pairs */
    if (a.log.size() != b.log.size()) return a.log.size() < b.log.size() ? -1 : 1;
    for (size_t i = 0; i < a.log.size(); i++) {
        int ka = a.log_lo + (int)i, kb = b.log_lo + (int)i;
        if (ka != kb) return ka < kb ? -1 : 1;
        int c = cmp_entry(a.log[i], b.log[i]);
        if (c) return c;
    }
    return 0;
}

int cmp_msg(const Msg& a, const Msg& b) {
    int na[12], nb[12];
    int ca = field_names(a, na), cb = field_names(b, nb);
    if (ca != cb) return ca < cb ? -1 : 1;
    for (int i = 0; i < ca; i++) {
        if (na[i] != nb[i]) return na[i] < nb[i] ? -1 : 1;
        int c = 0;
        switch (na[i]) {
        case F_VIEW: c = cmp_int_or_nil(a.view, b.view); break;
        case F_TYPE: c = cmp_int_or_nil(a.type, b.type); break;
        case F_MESSAGE: c = cmp_entry(a.entry, b.entry); break;
        case F_OP: c = cmp_int_or_nil(a.op, b.op); break;
        case F_COMMIT: c = cmp_int_or_nil(a.commit, b.commit); break;
        case F_DEST: c = cmp_int_or_nil(a.dest, b.dest); break;
        case F_SRC: c = cmp_int_or_nil(a.src, b.src); break;
        case F_LOG: c = cmp_log(a, b); break;
        case F_LNV: c = cmp_int_or_nil(a.lnv, b.lnv); break;
        case F_X: c = cmp_int_or_nil(a.x, b.x); break;
        case F_FIRSTOP: c = cmp_int_or_nil(a.first_op, b.first_op); break;
        }
        if (c) return c;
    }
    return 0;
}

/* ------------------------------------------------------------------ helpers (VSR.tla:227-308) */

static inline int Primary(const Params& p, int v) { return 1 + ((v - 1) % p.R); } /* :287-288 */
static inline int View(const State& s, int r) { return s.view[r - 1]; }           /* :281-282 */
static inline bool IsPrimary(const Params& p, const State& s, int r) {            /* :290-291 */
    return Primary(p, View(s, r)) == r;
}

static void SendFunc(const Msg& m, MsgBag& msgs) { /* :228-231 */
    auto it = msgs.find(m);
    if (it != msgs.end()) it->second += 1;
    else msgs.emplace(m, 1);
}
static void BroadcastFunc(const Params& p, Msg msg, int source, MsgBag& msgs) { /* :233-240 */
    for (int r = 1; r <= p.R; r++) {
        if (r == source) continue;
        msg.dest = r;
        SendFunc(msg, msgs); /* existing key: +1; new key: 1 — same result as the two-part definition */
    }
}
static void DiscardFunc(const Msg& m, MsgBag& msgs) { /* :244-245 — the key stays, count drops */
    auto it = msgs.find(m);
    assert(it != msgs.end());
    it->second -= 1;
}
static inline bool ReceivableMsg(const Msg& m, int count, int type, int r) { /* :272-275 */
    return m.type == type && m.dest == r && count > 0;
}
static Msg NewSVCMessage(int r, int view_number) { /* :293-297 */
    Msg m;
    m.type = VSR_MT_SVC;
    m.view = view_number;
    m.dest = NIL; /* replaced in broadcast */
    m.src = r;
    return m;
}
static void ResetRecvMsgs(State& s, int r) { /* :299-301 */
    s.svc_recv[r - 1].clear();
    s.dvc_recv[r - 1].clear();
}
static void ResetSentVars(State& s, int r) { /* :303-305 */
    s.sent_dvc[r - 1] = 0;
    s.sent_sv[r - 1] = 0;
}
static inline int MinVal(int a, int b) { return a <= b ? a : b; } /* :307-308 */

/* ------------------------------------------------------------------ Init (VSR.tla:323-348) */

State init_state(const Params& p) {
    State s;
    int R = p.R, C = p.C;
    s.status.assign(R, VSR_NORMAL);
    s.log.assign(R, {});
    s.view.assign(R, 1);
    s.op.assign(R, 0);
    s.commit.assign(R, 0);
    s.peer_op.assign(R, std::vector<int>(R, 0));
    s.client_table.assign(R, std::vector<ClientRow>(C)); /* EmptyClientTableRow :318-321 */
    s.svc_recv.assign(R, MsgSet());
    s.dvc_recv.assign(R, MsgSet());
    s.sent_dvc.assign(R, 0);
    s.sent_sv.assign(R, 0);
    s.lnv.assign(R, 0);
    s.rec_recv.assign(R, MsgSet());
    s.rec_number.assign(R, 0);
    s.aux_svc = 0;
    s.aux_restart = 0;
    return s;
}

/* ------------------------------------------------------------------ the 19 actions */

/* TimerSendSVC, VSR.tla:578-590 */
static void TimerSendSVC(const Params& p, const State& s, std::vector<Succ>& out) {
    if (!(s.aux_svc < p.L)) return;
    for (int r = 1; r <= p.R; r++) {
        if (IsPrimary(p, s, r)) continue;
        State n = s;
        n.view[r - 1] = View(s, r) + 1;
        n.status[r - 1] = VSR_VIEWCHANGE;
        ResetRecvMsgs(n, r);
        ResetSentVars(n, r);
        n.aux_svc = s.aux_svc + 1;
        BroadcastFunc(p, NewSVCMessage(r, View(s, r) + 1), r, n.messages);
        out.push_back({std::move(n), VSR_ACT_TIMER_SEND_SVC});
    }
}

/* ReceiveHigherSVC, VSR.tla:602-613 */
static void ReceiveHigherSVC(const Params& p, const State& s, std::vector<Succ>& out) {
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        for (int r = 1; r <= p.R; r++) {
            if (!ReceivableMsg(m, kv.second, VSR_MT_SVC, r)) continue;
            if (!(m.view > s.view[r - 1])) continue;
            State n = s;
            n.view[r - 1] = m.view;
            n.status[r - 1] = VSR_VIEWCHANGE;
            n.svc_recv[r - 1].clear();
            n.svc_recv[r - 1].insert(m);
            n.dvc_recv[r - 1].clear();
            ResetSentVars(n, r);
            /* DiscardAndBroadcast :260-265 (guards hold: m in DOMAIN, count > 0) */
            DiscardFunc(m, n.messages);
            BroadcastFunc(p, NewSVCMessage(r, m.view), r, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_HIGHER_SVC});
        }
    }
}

/* ReceiveMatchingSVC, VSR.tla:625-634 */
static void ReceiveMatchingSVC(const Params& p, const State& s, std::vector<Succ>& out) {
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        for (int r = 1; r <= p.R; r++) {
            if (!ReceivableMsg(m, kv.second, VSR_MT_SVC, r)) continue;
            if (!(m.view == View(s, r))) continue;
            if (!(s.status[r - 1] == VSR_VIEWCHANGE)) continue;
            State n = s;
            n.svc_recv[r - 1].insert(m);
            DiscardFunc(m, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_MATCHING_SVC});
        }
    }
}

/* SendDVC, VSR.tla:648-669 */
static void SendDVC(const Params& p, const State& s, std::vector<Succ>& out) {
    for (int r = 1; r <= p.R; r++) {
        if (!(s.status[r - 1] == VSR_VIEWCHANGE)) continue;
        if (!(s.sent_dvc[r - 1] == 0)) continue;
        if (!((int)s.svc_recv[r - 1].size() >= p.R / 2)) continue;
        State n = s;
        n.sent_dvc[r - 1] = 1;
        Msg msg;
        msg.type = VSR_MT_DVC;
        msg.view = View(s, r);
        msg.has_log = 1;
        msg.log_lo = 1;
        msg.log = s.log[r - 1];
        msg.lnv = s.lnv[r - 1];
        msg.op = s.op[r - 1];
        msg.commit = s.commit[r - 1];
        msg.dest = Primary(p, View(s, r));
        msg.src = r;
        if (Primary(p, View(s, r)) == r) n.dvc_recv[r - 1].insert(msg);
        else SendFunc(msg, n.messages);
        out.push_back({std::move(n), VSR_ACT_SEND_DVC});
    }
}

/* ReceiveHigherDVC, VSR.tla:677-688 */
static void ReceiveHigherDVC(const Params& p, const State& s, std::vector<Succ>& out) {
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        for (int r = 1; r <= p.R; r++) {
            if (!ReceivableMsg(m, kv.second, VSR_MT_DVC, r)) continue;
            if (!(m.view > s.view[r - 1])) continue;
            State n = s;
            n.view[r - 1] = m.view;
            n.status[r - 1] = VSR_VIEWCHANGE;
            n.svc_recv[r - 1].clear();
            n.dvc_recv[r - 1].clear();
            n.dvc_recv[r - 1].insert(m);
            ResetSentVars(n, r);
            DiscardFunc(m, n.messages);
            BroadcastFunc(p, NewSVCMessage(r, m.view), r, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_HIGHER_DVC});
        }
    }
}

/* ReceiveMatchingDVC, VSR.tla:696-703 (no status guard) */
static void ReceiveMatchingDVC(const Params& p, const State& s, std::vector<Succ>& out) {
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        for (int r = 1; r <= p.R; r++) {
            if (!ReceivableMsg(m, kv.second, VSR_MT_DVC, r)) continue;
            if (!(View(s, r) == m.view)) continue;
            State n = s;
            n.dvc_recv[r - 1].insert(m);
            DiscardFunc(m, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_MATCHING_DVC});
        }
    }
}

/* HighestLog, VSR.tla:716-722: CHOOSE = first element in TLC's set order that satisfies the body */
static const Msg* HighestLogMsg(const MsgSet& dvcs, Assumptions* as) {
    const Msg* chosen = nullptr;
    for (const Msg& m : dvcs) {
        bool beaten = false;
        for (const Msg& m1 : dvcs) {
            if (m1.lnv > m.lnv || (m1.lnv == m.lnv && m1.op > m.op)) { beaten = true; break; }
        }
        if (beaten) continue;
        if (!chosen) chosen = &m;
        else if (as) {
            /* a second maximal element: the CHOOSE tie-break decided; does it matter? */
            bool same = chosen->log.size() == m.log.size();
            for (size_t i = 0; same && i < m.log.size(); i++) same = cmp_entry(chosen->log[i], m.log[i]) == 0;
            if (!same) as->choose_tie_diff_logs++;
        }
    }
    return chosen;
}

/* SendSV, VSR.tla:735-760 */
static void SendSV(const Params& p, const State& s, std::vector<Succ>& out, Assumptions* as) {
    for (int r = 1; r <= p.R; r++) {
        if (!(s.status[r - 1] == VSR_VIEWCHANGE)) continue;
        if (!(s.sent_sv[r - 1] == 0)) continue;
        const MsgSet& dvcs = s.dvc_recv[r - 1];
        if (!((int)dvcs.size() >= p.R / 2 + 1)) continue;
        const Msg* hm = HighestLogMsg(dvcs, as);
        std::vector<Entry> new_log = hm->log;                 /* HighestLog :716-722 */
        int new_on = new_log.empty() ? 0 : (int)new_log.size(); /* HighestOpNumber :724-727 */
        int new_cn = 0;                                        /* HighestCommitNumber :729-733 */
        for (const Msg& m : dvcs) new_cn = std::max(new_cn, m.commit);
        State n = s;
        n.status[r - 1] = VSR_NORMAL;
        n.view[r - 1] = View(s, r);
        n.log[r - 1] = new_log;
        n.op[r - 1] = new_on;
        n.peer_op[r - 1].assign(p.R, 0);
        n.commit[r - 1] = new_cn;
        n.sent_sv[r - 1] = 1;
        n.lnv[r - 1] = View(s, r);
        Msg msg;
        msg.type = VSR_MT_SV;
        msg.view = View(s, r);
        msg.has_log = 1;
        msg.log_lo = 1;
        msg.log = new_log;
        msg.op = new_on;
        msg.commit = new_cn;
        msg.dest = NIL;
        msg.src = r;
        BroadcastFunc(p, msg, r, n.messages);
        out.push_back({std::move(n), VSR_ACT_SEND_SV});
    }
}

/* ReceiveSV, VSR.tla:773-793 */
static void ReceiveSV(const Params& p, const State& s, std::vector<Succ>& out) {
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        for (int r = 1; r <= p.R; r++) {
            if (!ReceivableMsg(m, kv.second, VSR_MT_SV, r)) continue;
            if (!(m.view >= View(s, r))) continue;
            State n = s;
            n.status[r - 1] = VSR_NORMAL;
            n.view[r - 1] = m.view;
            n.log[r - 1] = m.log;
            n.op[r - 1] = m.op;
            n.commit[r - 1] = m.commit;
            n.lnv[r - 1] = m.view;
            ResetRecvMsgs(n, r);
            ResetSentVars(n, r);
            if (s.commit[r - 1] < m.op) { /* the OLD commit number, :785 */
                Msg ok;
                ok.type = VSR_MT_PREPAREOK;
                ok.view = m.view;
                ok.op = m.op;
                ok.dest = Primary(p, m.view);
                ok.src = r;
                DiscardFunc(m, n.messages); /* DiscardAndSend :267-270 */
                SendFunc(ok, n.messages);
            } else {
                DiscardFunc(m, n.messages);
            }
            out.push_back({std::move(n), VSR_ACT_RECEIVE_SV});
        }
    }
}

/* ReceiveClientRequest, VSR.tla:366-394 */
static void ReceiveClientRequest(const Params& p, const State& s, std::vector<Succ>& out) {
    for (int r = 1; r <= p.R; r++)
        for (int c = 1; c <= p.C; c++)
            for (int v = 1; v <= p.V; v++) {
                if (!IsPrimary(p, s, r)) continue;
                if (!(s.status[r - 1] == VSR_NORMAL)) continue;
                if (s.acked.count(v)) continue;
                if (!s.client_table[r - 1][c - 1].executed) continue;
                int req_number = s.client_table[r - 1][c - 1].req + 1;
                int op_number = (int)s.log[r - 1].size() + 1;
                Entry e{View(s, r), v, c, req_number};
                State n = s;
                n.log[r - 1].push_back(e);
                n.op[r - 1] = op_number;
                n.client_table[r - 1][c - 1] = ClientRow{req_number, op_number, false};
                Msg msg;
                msg.type = VSR_MT_PREPARE;
                msg.view = View(s, r);
                msg.has_entry = true;
                msg.entry = e;
                msg.op = op_number;
                msg.commit = s.commit[r - 1];
                msg.dest = NIL;
                msg.src = r;
                BroadcastFunc(p, msg, r, n.messages);
                n.acked[v] = false;
                out.push_back({std::move(n), VSR_ACT_RECEIVE_CLIENT_REQUEST});
            }
}

/* ReceivePrepareMsg, VSR.tla:405-428 */
static void ReceivePrepareMsg(const Params& p, const State& s, std::vector<Succ>& out) {
    for (int r = 1; r <= p.R; r++)
        for (const auto& kv : s.messages) {
            const Msg& m = kv.first;
            if (!ReceivableMsg(m, kv.second, VSR_MT_PREPARE, r)) continue;
            if (!(s.status[r - 1] == VSR_NORMAL)) continue;
            if (!(m.view == View(s, r))) continue;
            if (!(m.op == s.op[r - 1] + 1)) continue;
            State n = s;
            n.log[r - 1].push_back(m.entry);
            n.op[r - 1] = m.op;
            n.commit[r - 1] = m.commit;
            for (int c = 1; c <= p.C; c++) {
                if (c == m.entry.client)
                    n.client_table[r - 1][c - 1] = ClientRow{m.entry.req, m.op, m.op <= m.commit};
                /* else branch reads the non-existent field m.commit (:421): TLC would abort;
                   Params with C >= 2 are rejected before we get here (SURVEY H9) */
            }
            Msg ok;
            ok.type = VSR_MT_PREPAREOK;
            ok.view = View(s, r);
            ok.op = m.op;
            ok.dest = m.src;
            ok.src = r;
            DiscardFunc(m, n.messages);
            SendFunc(ok, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_PREPARE});
        }
}

/* ReceivePrepareOkMsg, VSR.tla:437-447 */
static void ReceivePrepareOkMsg(const Params& p, const State& s, std::vector<Succ>& out) {
    for (int r = 1; r <= p.R; r++)
        for (const auto& kv : s.messages) {
            const Msg& m = kv.first;
            if (!ReceivableMsg(m, kv.second, VSR_MT_PREPAREOK, r)) continue;
            if (!IsPrimary(p, s, r)) continue;
            if (!(s.status[r - 1] == VSR_NORMAL)) continue;
            if (!(m.view == View(s, r))) continue;
            if (!(m.op > s.peer_op[r - 1][m.src - 1])) continue;
            State n = s;
            n.peer_op[r - 1][m.src - 1] = m.op;
            DiscardFunc(m, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_PREPARE_OK});
        }
}

/* IsCommitted, VSR.tla:457-460 (Quantify = number of elements satisfying the predicate) */
static bool IsCommitted(const Params& p, const State& s, int r, int op_number) {
    int q = 0;
    for (int peer = 1; peer <= p.R; peer++)
        if (s.peer_op[r - 1][peer - 1] >= op_number) q++;
    return q >= p.R / 2;
}

/* ExecuteOp, VSR.tla:462-476 */
static void ExecuteOp(const Params& p, const State& s, std::vector<Succ>& out, Assumptions* as) {
    for (int r = 1; r <= p.R; r++) {
        if (!IsPrimary(p, s, r)) continue;
        if (!(s.status[r - 1] == VSR_NORMAL)) continue;
        if (!(s.commit[r - 1] < s.op[r - 1])) continue;
        if (!IsCommitted(p, s, r, s.commit[r - 1] + 1)) continue;
        int op_number = s.commit[r - 1] + 1;
        if (op_number > (int)s.log[r - 1].size()) { /* rep_log[r][op_number] undefined: TLC would abort */
            if (as) as->op_ne_loglen++;
            continue;
        }
        Entry op = s.log[r - 1][op_number - 1];
        State n = s;
        n.commit[r - 1] = op_number;
        n.client_table[r - 1][op.client - 1].executed = true;
        n.acked[op.operation] = true;
        out.push_back({std::move(n), VSR_ACT_EXECUTE_OP});
    }
}

/* SendGetState, VSR.tla:496-516 (TruncateLogToCommitNumber :491-494) */
static void SendGetState(const Params& p, const State& s, std::vector<Succ>& out) {
    for (int r = 1; r <= p.R; r++)
        for (int rDest = 1; rDest <= p.R; rDest++)
            for (const auto& kv : s.messages) {
                const Msg& m = kv.first;
                if (IsPrimary(p, s, r)) continue;
                if (r == rDest) continue;
                if (!ReceivableMsg(m, kv.second, VSR_MT_PREPARE, r)) continue;
                if (!(s.status[r - 1] == VSR_NORMAL)) continue;
                if (!(m.view > View(s, r))) continue;
                if (!(m.op > s.op[r - 1] + 1)) continue;
                int truncate_to = MinVal(s.commit[r - 1], (int)s.log[r - 1].size());
                Msg gs;
                gs.type = VSR_MT_GETSTATE;
                gs.view = m.view;
                gs.op = truncate_to;
                gs.dest = rDest;
                gs.src = r;
                if (s.messages.count(gs)) continue; /* SendOnce :250-252 */
                State n = s;
                n.log[r - 1].resize(truncate_to);
                n.op[r - 1] = truncate_to;
                n.view[r - 1] = m.view;
                n.lnv[r - 1] = m.view;
                SendFunc(gs, n.messages);
                out.push_back({std::move(n), VSR_ACT_SEND_GET_STATE});
            }
}

/* ReceiveGetState, VSR.tla:526-543 */
static void ReceiveGetState(const Params& p, const State& s, std::vector<Succ>& out, Assumptions* as) {
    for (int r = 1; r <= p.R; r++)
        for (const auto& kv : s.messages) {
            const Msg& m = kv.first;
            if (!ReceivableMsg(m, kv.second, VSR_MT_GETSTATE, r)) continue;
            if (!(View(s, r) == m.view)) continue;
            if (!(s.status[r - 1] == VSR_NORMAL)) continue;
            if (!(s.op[r - 1] > m.op)) continue;
            if (s.op[r - 1] > (int)s.log[r - 1].size()) { /* rep_log[r][on] undefined */
                if (as) as->op_ne_loglen++;
                continue;
            }
            Msg ns;
            ns.type = VSR_MT_NEWSTATE;
            ns.view = View(s, r);
            ns.has_log = 1;
            ns.log_lo = m.op + 1;
            for (int on = m.op + 1; on <= s.op[r - 1]; on++) ns.log.push_back(s.log[r - 1][on - 1]);
            ns.first_op = m.op + 1;
            ns.op = s.op[r - 1];
            ns.commit = s.commit[r - 1];
            ns.dest = m.src;
            ns.src = r;
            State n = s;
            DiscardFunc(m, n.messages);
            SendFunc(ns, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_GET_STATE});
        }
}

/* ReceiveNewState, VSR.tla:551-567 */
static void ReceiveNewState(const Params& p, const State& s, std::vector<Succ>& out) {
    for (int r = 1; r <= p.R; r++)
        for (const auto& kv : s.messages) {
            const Msg& m = kv.first;
            if (!ReceivableMsg(m, kv.second, VSR_MT_NEWSTATE, r)) continue;
            if (!(View(s, r) == m.view)) continue;
            if (!(s.status[r - 1] == VSR_NORMAL)) continue;
            if (!(s.op[r - 1] == m.first_op - 1)) continue;
            State n = s;
            std::vector<Entry> nl;
            for (int on = 1; on <= m.op; on++) {
                if (on <= s.op[r - 1]) nl.push_back(s.log[r - 1][on - 1]);
                else nl.push_back(m.log[on - m.log_lo]);
            }
            n.log[r - 1] = nl;
            n.op[r - 1] = m.op;
            DiscardFunc(m, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVE_NEW_STATE});
        }
}

/* UniqueNumber, VSR.tla:802-811 */
static int UniqueNumber(const State& s) {
    int hi = 0;
    bool any = false;
    for (const auto& kv : s.messages)
        if (kv.first.type == VSR_MT_RECOVERY) { any = true; hi = std::max(hi, kv.first.x); }
    return any ? hi + 1 : 1;
}

/* RestartEmpty, VSR.tla:813-837 (no golden coverage anywhere in the reference) */
static void RestartEmpty(const Params& p, const State& s, std::vector<Succ>& out) {
    if (!(s.aux_restart < p.restart_limit)) return;
    for (int r = 1; r <= p.R; r++) {
        State n = s;
        n.log[r - 1].clear();
        n.view[r - 1] = 1;
        n.op[r - 1] = 0;
        n.commit[r - 1] = 0;
        n.peer_op[r - 1].assign(p.R, 0);
        n.client_table[r - 1].assign(p.C, ClientRow());
        n.svc_recv[r - 1].clear();
        n.dvc_recv[r - 1].clear();
        n.sent_dvc[r - 1] = 0;
        n.sent_sv[r - 1] = 0;
        n.lnv[r - 1] = 0;
        n.rec_recv[r - 1].clear();
        n.status[r - 1] = VSR_RECOVERING;
        n.rec_number[r - 1] = UniqueNumber(s);
        n.aux_restart = s.aux_restart + 1;
        Msg msg;
        msg.type = VSR_MT_RECOVERY;
        msg.x = UniqueNumber(s);
        msg.dest = NIL;
        msg.src = r;
        BroadcastFunc(p, msg, r, n.messages);
        out.push_back({std::move(n), VSR_ACT_RESTART_EMPTY});
    }
}

/* ReceivesRecoveryMsg, VSR.tla:842-858 */
static void ReceivesRecoveryMsg(const Params& p, const State& s, std::vector<Succ>& out) {
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        for (int r = 1; r <= p.R; r++) {
            if (!ReceivableMsg(m, kv.second, VSR_MT_RECOVERY, r)) continue;
            if (!(s.status[r - 1] == VSR_NORMAL)) continue;
            Msg rr;
            rr.type = VSR_MT_RECOVERYRESPONSE;
            rr.view = View(s, r);
            rr.x = m.x;
            if (IsPrimary(p, s, r)) {
                rr.has_log = 1;
                rr.log_lo = 1;
                rr.log = s.log[r - 1];
                rr.op = s.op[r - 1];
                rr.commit = s.commit[r - 1];
            } else {
                rr.has_log = 2;
                rr.op = NIL;
                rr.commit = NIL;
            }
            rr.dest = m.src;
            rr.src = r;
            State n = s;
            DiscardFunc(m, n.messages);
            SendFunc(rr, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVES_RECOVERY});
        }
    }
}

/* ReceivesRecoveryResponseMsg, VSR.tla:864-872 */
static void ReceivesRecoveryResponseMsg(const Params& p, const State& s, std::vector<Succ>& out) {
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        for (int r = 1; r <= p.R; r++) {
            if (!ReceivableMsg(m, kv.second, VSR_MT_RECOVERYRESPONSE, r)) continue;
            if (!(s.rec_number[r - 1] == m.x)) continue;
            if (!(s.status[r - 1] == VSR_RECOVERING)) continue;
            State n = s;
            n.rec_recv[r - 1].insert(m);
            DiscardFunc(m, n.messages);
            out.push_back({std::move(n), VSR_ACT_RECEIVES_RECOVERY_RESPONSE});
        }
    }
}

/* CompleteRecovery, VSR.tla:878-894 */
static void CompleteRecovery(const Params& p, const State& s, std::vector<Succ>& out) {
    for (int r = 1; r <= p.R; r++) {
        if (!(s.status[r - 1] == VSR_RECOVERING)) continue;
        if (!((int)s.rec_recv[r - 1].size() > p.R / 2)) continue;
        const Msg* m = nullptr;
        for (const Msg& c : s.rec_recv[r - 1])
            if (c.has_log != 2) { m = &c; break; } /* CHOOSE :883 = first in set order */
        if (!m) continue;
        State n = s;
        n.status[r - 1] = VSR_NORMAL;
        n.view[r - 1] = m->view;
        n.lnv[r - 1] = m->view;
        n.log[r - 1] = m->log;
        n.op[r - 1] = m->op;
        n.commit[r - 1] = m->commit;
        n.rec_recv[r - 1].clear();
        out.push_back({std::move(n), VSR_ACT_COMPLETE_RECOVERY});
    }
}

/* Next, VSR.tla:896-918 — the disjuncts in textual order */
void successors(const Params& p, const State& s, std::vector<Succ>& out, Assumptions* as) {
    TimerSendSVC(p, s, out);
    ReceiveHigherSVC(p, s, out);
    ReceiveMatchingSVC(p, s, out);
    SendDVC(p, s, out);
    ReceiveHigherDVC(p, s, out);
    ReceiveMatchingDVC(p, s, out);
    SendSV(p, s, out, as);
    ReceiveSV(p, s, out);
    ReceiveClientRequest(p, s, out);
    ReceivePrepareMsg(p, s, out);
    ReceivePrepareOkMsg(p, s, out);
    ExecuteOp(p, s, out, as);
    SendGetState(p, s, out);
    ReceiveGetState(p, s, out, as);
    ReceiveNewState(p, s, out);
    RestartEmpty(p, s, out);
    ReceivesRecoveryMsg(p, s, out);
    ReceivesRecoveryResponseMsg(p, s, out);
    CompleteRecovery(p, s, out);
}

/* ------------------------------------------------------------------ invariants (VSR.tla:926-952) */

static bool ReplicaHasOp(const State& s, int r, int v) { /* :933-935 */
    for (const Entry& e : s.log[r - 1])
        if (e.operation == v) return true;
    return false;
}

bool invariant_holds(const Params& p, const State& s) {
    switch (p.invariant) {
    case 1: /* AcknowledgedWriteNotLost :945-950 */
        for (const auto& kv : s.acked) {
            if (!kv.second) continue;
            bool any = false;
            for (int r = 1; r <= p.R && !any; r++) any = ReplicaHasOp(s, r, kv.first);
            if (!any) return false;
        }
        return true;
    case 2: /* AcknowledgedWritesExistOnMajority :937-943 */
        for (const auto& kv : s.acked) {
            if (!kv.second) continue;
            int q = 0;
            for (int r = 1; r <= p.R; r++) q += ReplicaHasOp(s, r, kv.first) ? 1 : 0;
            if (!(q >= p.R / 2 + 1)) return false;
        }
        return true;
    case 3: /* NoLogDivergence :926-931 compares rep_log[r1][op] with itself: always TRUE */
        return true;
    default: /* TestInv :952, or none */
        return true;
    }
}

/* ------------------------------------------------------------------ assumption audit */

void check_assumptions(const Params& p, const State& s, Assumptions& as) {
    int K = 1 + p.L;
    std::map<int, Entry> seen_entry; /* value -> the one LogEntry record that may exist for it */
    auto note_entry = [&](const Entry& e) {
        auto it = seen_entry.find(e.operation);
        if (it == seen_entry.end()) seen_entry[e.operation] = e;
        else if (cmp_entry(it->second, e) != 0) as.entry_not_unique++;
    };
    auto note_log = [&](const std::vector<Entry>& lg) {
        if ((int)lg.size() > p.V) as.dup_value_in_log++;
        for (size_t i = 0; i < lg.size(); i++) {
            note_entry(lg[i]);
            for (size_t j = i + 1; j < lg.size(); j++)
                if (lg[i].operation == lg[j].operation) as.dup_value_in_log++;
        }
    };
    for (int r = 1; r <= p.R; r++) {
        if (s.op[r - 1] != (int)s.log[r - 1].size()) as.op_ne_loglen++;
        if (s.view[r - 1] > K || s.lnv[r - 1] > K) as.view_gt_max++;
        note_log(s.log[r - 1]);
        for (const Msg& m : s.svc_recv[r - 1])
            if (m.view != s.view[r - 1] || m.dest != r) as.recv_view_mismatch++;
        for (const Msg& m : s.dvc_recv[r - 1]) {
            if (m.view != s.view[r - 1] || m.dest != r) as.recv_view_mismatch++;
            if (m.op != (int)m.log.size()) as.op_ne_loglen++;
            note_log(m.log);
            /* a non-self DVC in the set must still be a key of the bag with identical payload */
            if (m.src != r && !s.messages.count(m)) as.slot_clash++;
        }
    }
    /* slot uniqueness: one message per (type, view, source[, dest]) etc. */
    std::set<std::vector<int>> slots;
    std::map<int, std::pair<int, int>> prep_key; /* value -> (view, op) */
    for (const auto& kv : s.messages) {
        const Msg& m = kv.first;
        if (kv.second > 1 || kv.second < 0) as.bag_count_gt1++;
        if (m.view != ABSENT && m.view > K) as.view_gt_max++;
        std::vector<int> key;
        switch (m.type) {
        case VSR_MT_SVC: key = {m.type, m.view, m.src, m.dest}; break;
        case VSR_MT_DVC:
            key = {m.type, m.view, m.src};
            if (m.dest != Primary(p, m.view) || m.src == m.dest) as.slot_clash++;
            if (m.op != (int)m.log.size()) as.op_ne_loglen++;
            note_log(m.log);
            break;
        case VSR_MT_SV:
            key = {m.type, m.view, m.dest};
            if (m.src != Primary(p, m.view)) as.slot_clash++;
            if (m.op != (int)m.log.size()) as.op_ne_loglen++;
            note_log(m.log);
            break;
        case VSR_MT_PREPARE: {
            key = {m.type, m.entry.operation, m.dest};
            if (m.src != Primary(p, m.view) || m.entry.view != m.view) as.slot_clash++;
            note_entry(m.entry);
            auto it = prep_key.find(m.entry.operation);
            if (it == prep_key.end()) prep_key[m.entry.operation] = {m.view, m.op};
            else if (it->second != std::make_pair(m.view, m.op)) as.slot_clash++;
            break;
        }
        case VSR_MT_PREPAREOK:
            key = {m.type, m.view, m.op, m.src};
            if (m.dest != Primary(p, m.view) || m.src == m.dest) as.slot_clash++;
            break;
        case VSR_MT_GETSTATE:
            key = {m.type, m.view, m.src};
            if (m.src == Primary(p, m.view)) as.slot_clash++;
            break;
        case VSR_MT_NEWSTATE: {
            key = {m.type, m.view, m.dest};
            note_log(m.log);
            if (m.op != m.log_lo + (int)m.log.size() - 1 || m.first_op != m.log_lo) as.slot_clash++;
            /* must answer a GetState that is still a key of the bag */
            Msg gs;
            gs.type = VSR_MT_GETSTATE;
            gs.view = m.view;
            gs.op = m.first_op - 1;
            gs.dest = m.src;
            gs.src = m.dest;
            if (!s.messages.count(gs)) as.slot_clash++;
            break;
        }
        default: key = {m.type, m.x, m.src, m.dest, m.view == ABSENT ? 0 : m.view}; break;
        }
        if (!slots.insert(key).second) as.slot_clash++;
    }
    /* every value in DOMAIN aux_client_acked has its Prepare in the bag, and vice versa */
    for (const auto& kv : s.acked)
        if (!prep_key.count(kv.first)) as.slot_clash++;
    for (const auto& kv : prep_key)
        if (!s.acked.count(kv.first)) as.slot_clash++;
    std::set<std::pair<int, int>> keys;
    for (const auto& kv : prep_key)
        if (!keys.insert(kv.second).second) as.prepare_key_clash++;
}

/* ------------------------------------------------------------------ state order, symmetry */

template <class T> static int cmp_scalar(T a, T b) { return a < b ? -1 : (a > b ? 1 : 0); }
static int cmp_ivec(const std::vector<int>& a, const std::vector<int>& b) {
    if (a.size() != b.size()) return a.size() < b.size() ? -1 : 1;
    for (size_t i = 0; i < a.size(); i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}
static int cmp_cvec(const std::vector<char>& a, const std::vector<char>& b) {
    for (size_t i = 0; i < a.size(); i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}
static int cmp_logv(const std::vector<Entry>& a, const std::vector<Entry>& b) {
    if (a.size() != b.size()) return a.size() < b.size() ? -1 : 1;
    for (size_t i = 0; i < a.size(); i++) {
        int c = cmp_entry(a[i], b[i]);
        if (c) return c;
    }
    return 0;
}
static int cmp_msgset(const MsgSet& a, const MsgSet& b) {
    if (a.size() != b.size()) return a.size() < b.size() ? -1 : 1;
    auto ia = a.begin(), ib = b.begin();
    for (; ia != a.end(); ++ia, ++ib) {
        int c = cmp_msg(*ia, *ib);
        if (c) return c;
    }
    return 0;
}

/* lexicographic over the variables in declaration order, VSR.tla:119-138 */
int cmp_state(const State& a, const State& b, bool with_aux) {
    int c;
    size_t R = a.status.size();
    if ((c = cmp_ivec(a.status, b.status))) return c;
    for (size_t r = 0; r < R; r++)
        if ((c = cmp_logv(a.log[r], b.log[r]))) return c;
    if ((c = cmp_ivec(a.view, b.view))) return c;
    if ((c = cmp_ivec(a.op, b.op))) return c;
    if ((c = cmp_ivec(a.commit, b.commit))) return c;
    for (size_t r = 0; r < R; r++)
        if ((c = cmp_ivec(a.peer_op[r], b.peer_op[r]))) return c;
    for (size_t r = 0; r < R; r++)
        for (size_t k = 0; k < a.client_table[r].size(); k++) {
            const ClientRow &x = a.client_table[r][k], &y = b.client_table[r][k];
            if ((c = cmp_scalar(x.req, y.req))) return c;
            if ((c = cmp_scalar(x.op, y.op))) return c;
            if ((c = cmp_scalar((int)x.executed, (int)y.executed))) return c;
        }
    if ((c = cmp_ivec(a.lnv, b.lnv))) return c;
    for (size_t r = 0; r < R; r++)
        if ((c = cmp_msgset(a.svc_recv[r], b.svc_recv[r]))) return c;
    for (size_t r = 0; r < R; r++)
        if ((c = cmp_msgset(a.dvc_recv[r], b.dvc_recv[r]))) return c;
    if ((c = cmp_cvec(a.sent_dvc, b.sent_dvc))) return c;
    if ((c = cmp_cvec(a.sent_sv, b.sent_sv))) return c;
    if ((c = cmp_ivec(a.rec_number, b.rec_number))) return c;
    for (size_t r = 0; r < R; r++)
        if ((c = cmp_msgset(a.rec_recv[r], b.rec_recv[r]))) return c;
    if (a.messages.size() != b.messages.size()) return a.messages.size() < b.messages.size() ? -1 : 1;
    {
        auto ia = a.messages.begin(), ib = b.messages.begin();
        for (; ia != a.messages.end(); ++ia, ++ib) {
            if ((c = cmp_msg(ia->first, ib->first))) return c;
            if ((c = cmp_scalar(ia->second, ib->second))) return c;
        }
    }
    if (!with_aux) return 0;
    if ((c = cmp_scalar(a.aux_svc, b.aux_svc))) return c;
    if ((c = cmp_scalar(a.aux_restart, b.aux_restart))) return c;
    if (a.acked.size() != b.acked.size()) return a.acked.size() < b.acked.size() ? -1 : 1;
    {
        auto ia = a.acked.begin(), ib = b.acked.begin();
        for (; ia != a.acked.end(); ++ia, ++ib) {
            if ((c = cmp_scalar(ia->first, ib->first))) return c;
            if ((c = cmp_scalar((int)ia->second, (int)ib->second))) return c;
        }
    }
    return 0;
}

static Entry perm_entry(Entry e, const std::vector<int>& perm) {
    e.operation = perm[e.operation - 1];
    return e;
}
static Msg perm_msg(Msg m, const std::vector<int>& perm) {
    if (m.has_entry) m.entry = perm_entry(m.entry, perm);
    for (Entry& e : m.log) e = perm_entry(e, perm);
    return m;
}
static MsgSet perm_set(const MsgSet& s, const std::vector<int>& perm) {
    MsgSet o;
    for (const Msg& m : s) o.insert(perm_msg(m, perm));
    return o;
}

State permute(const State& s, const std::vector<int>& perm) {
    State n = s;
    size_t R = s.status.size();
    for (size_t r = 0; r < R; r++) {
        for (Entry& e : n.log[r]) e = perm_entry(e, perm);
        n.svc_recv[r] = perm_set(s.svc_recv[r], perm);
        n.dvc_recv[r] = perm_set(s.dvc_recv[r], perm);
        n.rec_recv[r] = perm_set(s.rec_recv[r], perm);
    }
    n.messages.clear();
    for (const auto& kv : s.messages) n.messages.emplace(perm_msg(kv.first, perm), kv.second);
    n.acked.clear();
    for (const auto& kv : s.acked) n.acked[perm[kv.first - 1]] = kv.second;
    return n;
}

/* min over Permutations(Values) of the whole state, variables in declaration order (aux last, so the
   VIEW part is minimised first) — SURVEY App. B.4 */
State canonical(const Params& p, const State& s) {
    if (!p.symmetry || p.V <= 1) return s;
    std::vector<int> perm(p.V);
    for (int i = 0; i < p.V; i++) perm[i] = i + 1;
    State best = s;
    while (std::next_permutation(perm.begin(), perm.end())) {
        State c = permute(s, perm);
        if (cmp_state(c, best, true) < 0) best = std::move(c);
    }
    return best;
}

uint32_t aux_key(const Params& p, const State& s) {
    /* created values in an order that does not depend on their labels: by the (view, op_number) of
       their Prepare broadcast when SYMMETRY is on, by value index otherwise */
    std::vector<std::pair<std::pair<int, int>, int>> order; /* ((view, op), value) */
    for (const auto& kv : s.acked) {
        std::pair<int, int> key(0, kv.first);
        if (p.symmetry) {
            for (const auto& mk : s.messages)
                if (mk.first.type == VSR_MT_PREPARE && mk.first.entry.operation == kv.first) {
                    key = {mk.first.view, mk.first.op};
                    break;
                }
        }
        order.push_back({key, kv.first});
    }
    std::sort(order.begin(), order.end());
    uint32_t k = (uint32_t)s.aux_svc;
    k = k * 16u + (uint32_t)s.aux_restart;
    for (int i = 0; i < p.V; i++) {
        uint32_t code = 0;
        if (p.symmetry) {
            if (i < (int)order.size()) code = s.acked.at(order[i].second) ? 2u : 1u;
        } else {
            auto it = s.acked.find(i + 1); /* no SYMMETRY: values keep their identity, position = value index */
            if (it != s.acked.end()) code = it->second ? 2u : 1u;
        }
        k = k * 3u + code;
    }
    return k;
}

/* ------------------------------------------------------------------ serialisation */

static inline void put(std::string& o, int v) {
    o.push_back((char)(uint8_t)(v == ABSENT ? 0xFF : (v == NIL ? 0xFE : v)));
}
static inline int get(const std::string& in, size_t& i) {
    uint8_t b = (uint8_t)in[i++];
    return b == 0xFF ? ABSENT : (b == 0xFE ? NIL : (int)b);
}
static void put_entry(std::string& o, const Entry& e) { put(o, e.view); put(o, e.operation); put(o, e.client); put(o, e.req); }
static Entry get_entry(const std::string& in, size_t& i) {
    Entry e;
    e.view = get(in, i); e.operation = get(in, i); e.client = get(in, i); e.req = get(in, i);
    return e;
}
static void put_msg(std::string& o, const Msg& m) {
    put(o, m.type); put(o, m.view); put(o, m.src); put(o, m.dest); put(o, m.op); put(o, m.commit);
    put(o, m.lnv); put(o, m.first_op); put(o, m.x);
    put(o, m.has_entry ? 1 : 0);
    if (m.has_entry) put_entry(o, m.entry);
    put(o, m.has_log);
    if (m.has_log == 1) {
        put(o, m.log_lo);
        put(o, (int)m.log.size());
        for (const Entry& e : m.log) put_entry(o, e);
    }
}
static Msg get_msg(const std::string& in, size_t& i) {
    Msg m;
    m.type = get(in, i); m.view = get(in, i); m.src = get(in, i); m.dest = get(in, i); m.op = get(in, i);
    m.commit = get(in, i); m.lnv = get(in, i); m.first_op = get(in, i); m.x = get(in, i);
    m.has_entry = get(in, i) != 0;
    if (m.has_entry) m.entry = get_entry(in, i);
    m.has_log = get(in, i);
    if (m.has_log == 1) {
        m.log_lo = get(in, i);
        int n = get(in, i);
        for (int k = 0; k < n; k++) m.log.push_back(get_entry(in, i));
    }
    return m;
}
static void put_set(std::string& o, const MsgSet& s) {
    put(o, (int)s.size());
    for (const Msg& m : s) put_msg(o, m);
}
static void get_set(const std::string& in, size_t& i, MsgSet& s) {
    int n = get(in, i);
    for (int k = 0; k < n; k++) s.insert(s.end(), get_msg(in, i));
}

void serialize(const State& s, bool with_aux, std::string& o) {
    o.clear();
    size_t R = s.status.size();
    for (size_t r = 0; r < R; r++) {
        put(o, s.status[r]); put(o, s.view[r]); put(o, s.op[r]); put(o, s.commit[r]); put(o, s.lnv[r]);
        put(o, s.rec_number[r]); put(o, s.sent_dvc[r]); put(o, s.sent_sv[r]);
        put(o, (int)s.log[r].size());
        for (const Entry& e : s.log[r]) put_entry(o, e);
        for (int x : s.peer_op[r]) put(o, x);
        for (const ClientRow& c : s.client_table[r]) { put(o, c.req); put(o, c.op); put(o, c.executed ? 1 : 0); }
        put_set(o, s.svc_recv[r]);
        put_set(o, s.dvc_recv[r]);
        put_set(o, s.rec_recv[r]);
    }
    put(o, (int)(s.messages.size() & 0x7F));
    put(o, (int)(s.messages.size() >> 7));
    for (const auto& kv : s.messages) { put_msg(o, kv.first); put(o, kv.second); }
    if (with_aux) {
        put(o, s.aux_svc);
        put(o, s.aux_restart);
        put(o, (int)s.acked.size());
        for (const auto& kv : s.acked) { put(o, kv.first); put(o, kv.second ? 1 : 0); }
    }
}

State deserialize(const Params& p, const std::string& in) {
    State s = init_state(p);
    size_t i = 0;
    for (int r = 0; r < p.R; r++) {
        s.status[r] = get(in, i); s.view[r] = get(in, i); s.op[r] = get(in, i); s.commit[r] = get(in, i);
        s.lnv[r] = get(in, i); s.rec_number[r] = get(in, i); s.sent_dvc[r] = (char)get(in, i);
        s.sent_sv[r] = (char)get(in, i);
        int n = get(in, i);
        for (int k = 0; k < n; k++) s.log[r].push_back(get_entry(in, i));
        for (int k = 0; k < p.R; k++) s.peer_op[r][k] = get(in, i);
        for (int k = 0; k < p.C; k++) {
            s.client_table[r][k].req = get(in, i);
            s.client_table[r][k].op = get(in, i);
            s.client_table[r][k].executed = get(in, i) != 0;
        }
        get_set(in, i, s.svc_recv[r]);
        get_set(in, i, s.dvc_recv[r]);
        get_set(in, i, s.rec_recv[r]);
    }
    int n = get(in, i);
    n |= get(in, i) << 7;
    for (int k = 0; k < n; k++) {
        Msg m = get_msg(in, i);
        int c = get(in, i);
        s.messages.emplace_hint(s.messages.end(), std::move(m), c);
    }
    if (i < in.size()) {
        s.aux_svc = get(in, i);
        s.aux_restart = get(in, i);
        int na = get(in, i);
        for (int k = 0; k < na; k++) {
            int v = get(in, i);
            s.acked[v] = get(in, i) != 0;
        }
    }
    return s;
}

/* MurmurHash3 x64 128 (public-domain algorithm by Austin Appleby), used only to key the oracle's
   seen-set by 128 bits of an exact serialisation */
static inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static inline uint64_t fmix64(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
    return k;
}
void digest128(const std::string& bytes, uint64_t out[2]) {
    const uint8_t* data = (const uint8_t*)bytes.data();
    const size_t len = bytes.size();
    const size_t nblocks = len / 16;
    uint64_t h1 = 0x9E3779B97F4A7C15ULL, h2 = 0xD1B54A32D192ED03ULL;
    const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
    for (size_t i = 0; i < nblocks; i++) {
        uint64_t k1, k2;
        memcpy(&k1, data + 16 * i, 8);
        memcpy(&k2, data + 16 * i + 8, 8);
        k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
        h1 = rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
        k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
        h2 = rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
    }
    const uint8_t* tail = data + nblocks * 16;
    uint64_t k1 = 0, k2 = 0;
    size_t rem = len & 15;
    for (size_t i = rem; i > 8; i--) k2 ^= (uint64_t)tail[i - 1] << ((i - 9) * 8);
    if (rem > 8) { k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2; }
    for (size_t i = std::min<size_t>(rem, 8); i > 0; i--) k1 ^= (uint64_t)tail[i - 1] << ((i - 1) * 8);
    if (rem > 0) { k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1; }
    h1 ^= len; h2 ^= len;
    h1 += h2; h2 += h1;
    h1 = fmix64(h1); h2 = fmix64(h2);
    h1 += h2; h2 += h1;
    out[0] = h1; out[1] = h2;
}

/* ------------------------------------------------------------------ flat form */

static void msg_to_flat(const Msg& m, int count, VsrMsg* f) {
    memset(f, 0, sizeof(*f));
    auto b = [](int v) -> uint8_t { return v == ABSENT ? VSR_ABSENT : (v == NIL ? VSR_NIL : (uint8_t)v); };
    f->type = (uint8_t)m.type;
    f->view = b(m.view); f->src = b(m.src); f->dest = b(m.dest); f->op = b(m.op); f->commit = b(m.commit);
    f->lnv = b(m.lnv); f->first_op = b(m.first_op); f->x = b(m.x);
    f->has_entry = m.has_entry ? 1 : 0;
    if (m.has_entry) f->entry = VsrEntry{(uint8_t)m.entry.view, (uint8_t)m.entry.operation, (uint8_t)m.entry.client, (uint8_t)m.entry.req};
    f->has_log = (uint8_t)m.has_log;
    if (m.has_log == 1) {
        f->log_lo = (uint8_t)m.log_lo;
        f->log_n = (uint8_t)m.log.size();
        for (size_t i = 0; i < m.log.size() && i < VSR_MAX_V; i++)
            f->log[i] = VsrEntry{(uint8_t)m.log[i].view, (uint8_t)m.log[i].operation, (uint8_t)m.log[i].client, (uint8_t)m.log[i].req};
    }
    f->count = (uint8_t)count;
}
static Msg msg_from_flat(const VsrMsg* f) {
    Msg m;
    auto b = [](uint8_t v) -> int { return v == VSR_ABSENT ? ABSENT : (v == VSR_NIL ? NIL : (int)v); };
    m.type = f->type;
    m.view = b(f->view); m.src = b(f->src); m.dest = b(f->dest); m.op = b(f->op); m.commit = b(f->commit);
    m.lnv = b(f->lnv); m.first_op = b(f->first_op); m.x = b(f->x);
    m.has_entry = f->has_entry != 0;
    if (m.has_entry) m.entry = Entry{f->entry.view, f->entry.operation, f->entry.client, f->entry.req};
    m.has_log = f->has_log;
    if (m.has_log == 1) {
        m.log_lo = f->log_lo;
        for (int i = 0; i < f->log_n; i++) m.log.push_back(Entry{f->log[i].view, f->log[i].operation, f->log[i].client, f->log[i].req});
    }
    return m;
}

void to_flat(const Params& p, const State& s, VsrFlatState* f) {
    memset(f, 0, sizeof(*f));
    f->R = (uint8_t)p.R; f->C = (uint8_t)p.C; f->V = (uint8_t)p.V;
    f->aux_svc = (uint8_t)s.aux_svc; f->aux_restart = (uint8_t)s.aux_restart;
    for (const auto& kv : s.acked) f->acked[kv.first - 1] = kv.second ? 2 : 1;
    for (int r = 0; r < p.R; r++) {
        VsrReplica& q = f->rep[r];
        q.status = (uint8_t)s.status[r]; q.view = (uint8_t)s.view[r]; q.op = (uint8_t)s.op[r];
        q.commit = (uint8_t)s.commit[r]; q.lnv = (uint8_t)s.lnv[r]; q.sent_dvc = (uint8_t)s.sent_dvc[r];
        q.sent_sv = (uint8_t)s.sent_sv[r]; q.rec_number = (uint8_t)s.rec_number[r];
        q.log_n = (uint8_t)s.log[r].size();
        for (size_t i = 0; i < s.log[r].size() && i < VSR_MAX_V; i++)
            q.log[i] = VsrEntry{(uint8_t)s.log[r][i].view, (uint8_t)s.log[r][i].operation, (uint8_t)s.log[r][i].client, (uint8_t)s.log[r][i].req};
        for (int k = 0; k < p.R; k++) q.peer_op[k] = (uint8_t)s.peer_op[r][k];
        for (int k = 0; k < p.C; k++) {
            q.client_table[k].req = (uint8_t)s.client_table[r][k].req;
            q.client_table[k].op = (uint8_t)s.client_table[r][k].op;
            q.client_table[k].executed = s.client_table[r][k].executed ? 1 : 0;
        }
        for (const Msg& m : s.svc_recv[r]) msg_to_flat(m, 0, &q.svc_recv[q.n_svc++]);
        for (const Msg& m : s.dvc_recv[r]) msg_to_flat(m, 0, &q.dvc_recv[q.n_dvc++]);
        for (const Msg& m : s.rec_recv[r]) msg_to_flat(m, 0, &q.rec_recv[q.n_rec++]);
    }
    for (const auto& kv : s.messages) {
        if (f->n_msgs >= VSR_MAX_MSGS) break;
        msg_to_flat(kv.first, kv.second, &f->msgs[f->n_msgs++]);
    }
}

State from_flat(const VsrFlatState* f) {
    Params p;
    p.R = f->R; p.C = f->C; p.V = f->V;
    State s = init_state(p);
    s.aux_svc = f->aux_svc; s.aux_restart = f->aux_restart;
    for (int v = 0; v < f->V; v++)
        if (f->acked[v]) s.acked[v + 1] = f->acked[v] == 2;
    for (int r = 0; r < p.R; r++) {
        const VsrReplica& q = f->rep[r];
        s.status[r] = q.status; s.view[r] = q.view; s.op[r] = q.op; s.commit[r] = q.commit; s.lnv[r] = q.lnv;
        s.sent_dvc[r] = (char)q.sent_dvc; s.sent_sv[r] = (char)q.sent_sv; s.rec_number[r] = q.rec_number;
        for (int i = 0; i < q.log_n; i++) s.log[r].push_back(Entry{q.log[i].view, q.log[i].operation, q.log[i].client, q.log[i].req});
        for (int k = 0; k < p.R; k++) s.peer_op[r][k] = q.peer_op[k];
        for (int k = 0; k < p.C; k++) s.client_table[r][k] = ClientRow{q.client_table[k].req, q.client_table[k].op, q.client_table[k].executed != 0};
        for (int i = 0; i < q.n_svc; i++) s.svc_recv[r].insert(msg_from_flat(&q.svc_recv[i]));
        for (int i = 0; i < q.n_dvc; i++) s.dvc_recv[r].insert(msg_from_flat(&q.dvc_recv[i]));
        for (int i = 0; i < q.n_rec; i++) s.rec_recv[r].insert(msg_from_flat(&q.rec_recv[i]));
    }
    for (int i = 0; i < f->n_msgs; i++) s.messages[msg_from_flat(&f->msgs[i])] = f->msgs[i].count;
    return s;
}

const char* action_name(int a) {
    static const char* names[VSR_NUM_ACTIONS] = {
        "Initial predicate", "TimerSendSVC", "ReceiveHigherSVC", "ReceiveMatchingSVC", "SendDVC",
        "ReceiveHigherDVC", "ReceiveMatchingDVC", "SendSV", "ReceiveSV", "ReceiveClientRequest",
        "ReceivePrepareMsg", "ReceivePrepareOkMsg", "ExecuteOp", "SendGetState", "ReceiveGetState",
        "ReceiveNewState", "RestartEmpty", "ReceivesRecoveryMsg", "ReceivesRecoveryResponseMsg",
        "CompleteRecovery"};
    return (a >= 0 && a < VSR_NUM_ACTIONS) ? names[a] : "?";
}

} // namespace orc
