/*
 * tlc_text.cpp — TLC "dumpTrace tlc" value text: printer and parser (oracle side; test
 * infrastructure only).  The format is the one of tests/golden/state_transfer_violation_trace.txt.gz:
 * variables alphabetical, functions over 1..n as <<...>>, other functions as (k :> v @@ ...),
 * records [f |-> v, ...] with fields in first-interned order, sets {...}, intervals a..b.
 */
#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sstream>

#include "vsr_oracle.h"

namespace orc {

/* ------------------------------------------------------------------ printer */

static const char* type_name(int t) {
    static const char* n[] = {"RequestMsg", "ReplyMsg", "PrepareMsg", "PrepareOkMsg", "CommitMsg",
                              "StartViewChangeMsg", "DoViewChangeMsg", "StartViewMsg", "GetStateMsg",
                              "NewStateMsg", "RecoveryMsg", "RecoveryResponseMsg"};
    return (t >= 0 && t < 12) ? n[t] : "?";
}
static const char* status_name(int s) {
    static const char* n[] = {"Normal", "ViewChange", "Recovering"};
    return (s >= 0 && s < 3) ? n[s] : "?";
}
static std::string int_or_nil(int v) { return v == NIL ? "Nil" : std::to_string(v); }

static std::string print_entry(const Entry& e) {
    std::ostringstream o;
    o << "[view_number |-> " << e.view << ", operation |-> v" << e.operation << ", client_id |-> " << e.client
      << ", request_number |-> " << e.req << "]";
    return o.str();
}
static std::string print_log_fn(int lo, const std::vector<Entry>& lg) {
    std::ostringstream o;
    if (lg.empty()) return "<<>>";
    if (lo == 1) {
        o << "<<";
        for (size_t i = 0; i < lg.size(); i++) o << (i ? ", " : "") << print_entry(lg[i]);
        o << ">>";
    } else {
        o << "(";
        for (size_t i = 0; i < lg.size(); i++) o << (i ? " @@ " : "") << (lo + (int)i) << " :> " << print_entry(lg[i]);
        o << ")";
    }
    return o.str();
}
static std::string print_msg(const Msg& m) {
    /* fields in first-interned order (see cmp_msg) */
    std::ostringstream o;
    bool first = true;
    auto f = [&](const char* name, const std::string& v) {
        o << (first ? "" : ", ") << name << " |-> " << v;
        first = false;
    };
    o << "[";
    if (m.view != ABSENT) f("view_number", int_or_nil(m.view));
    f("type", type_name(m.type));
    if (m.has_entry) f("message", print_entry(m.entry));
    if (m.op != ABSENT) f("op_number", int_or_nil(m.op));
    if (m.commit != ABSENT) f("commit_number", int_or_nil(m.commit));
    if (m.dest != ABSENT) f("dest", int_or_nil(m.dest));
    if (m.src != ABSENT) f("source", int_or_nil(m.src));
    if (m.has_log == 1) f("log", print_log_fn(m.log_lo, m.log));
    if (m.has_log == 2) f("log", "Nil");
    if (m.lnv != ABSENT) f("last_normal_vn", int_or_nil(m.lnv));
    if (m.x != ABSENT) f("x", int_or_nil(m.x));
    if (m.first_op != ABSENT) f("first_op", int_or_nil(m.first_op));
    o << "]";
    return o.str();
}
static std::string print_set(const MsgSet& s) {
    std::ostringstream o;
    o << "{";
    bool first = true;
    for (const Msg& m : s) { o << (first ? "" : ", ") << print_msg(m); first = false; }
    o << "}";
    return o.str();
}
template <class T, class F> static std::string print_tuple(const std::vector<T>& v, F f) {
    std::ostringstream o;
    o << "<<";
    for (size_t i = 0; i < v.size(); i++) o << (i ? ", " : "") << f(v[i]);
    o << ">>";
    return o.str();
}

static std::string print_vars(const Params& p, const State& s, bool with_rec_vars) {
    std::ostringstream o;
    /* alphabetical variable order, as in the trace file */
    o << "aux_client_acked |-> ";
    if (s.acked.empty()) o << "<<>>";
    else {
        o << "(";
        bool first = true;
        for (const auto& kv : s.acked) { o << (first ? "" : " @@ ") << "v" << kv.first << " :> " << (kv.second ? "TRUE" : "FALSE"); first = false; }
        o << ")";
    }
    o << ",\n";
    if (with_rec_vars) o << "aux_restart |-> " << s.aux_restart << ",\n";
    o << "aux_svc |-> " << s.aux_svc << ",\n";
    o << "clients |-> 1.." << p.C << ",\n";
    o << "messages |-> ";
    if (s.messages.empty()) o << "<<>>";
    else {
        o << "(";
        bool first = true;
        for (const auto& kv : s.messages) { o << (first ? "" : " @@ ") << print_msg(kv.first) << " :> " << kv.second; first = false; }
        o << ")";
    }
    o << ",\n";
    o << "rep_client_table |-> "
      << print_tuple(s.client_table, [&](const std::vector<ClientRow>& rows) {
             return print_tuple(rows, [&](const ClientRow& c) {
                 return "[request_number |-> " + std::to_string(c.req) + ", op_number |-> " + std::to_string(c.op) +
                        ", executed |-> " + (c.executed ? "TRUE" : "FALSE") + "]";
             });
         })
      << ",\n";
    auto itos = [](int v) { return std::to_string(v); };
    auto btos = [](char v) { return std::string(v ? "TRUE" : "FALSE"); };
    o << "rep_commit_number |-> " << print_tuple(s.commit, itos) << ",\n";
    o << "rep_dvc_recv |-> " << print_tuple(s.dvc_recv, print_set) << ",\n";
    o << "rep_last_normal_view |-> " << print_tuple(s.lnv, itos) << ",\n";
    o << "rep_log |-> " << print_tuple(s.log, [&](const std::vector<Entry>& l) { return print_tuple(l, print_entry); }) << ",\n";
    o << "rep_op_number |-> " << print_tuple(s.op, itos) << ",\n";
    o << "rep_peer_op_number |-> " << print_tuple(s.peer_op, [&](const std::vector<int>& v) { return print_tuple(v, itos); }) << ",\n";
    if (with_rec_vars) {
        o << "rep_rec_number |-> " << print_tuple(s.rec_number, itos) << ",\n";
        o << "rep_rec_recv |-> " << print_tuple(s.rec_recv, print_set) << ",\n";
    }
    o << "rep_sent_dvc |-> " << print_tuple(s.sent_dvc, btos) << ",\n";
    o << "rep_sent_sv |-> " << print_tuple(s.sent_sv, btos) << ",\n";
    o << "rep_status |-> " << print_tuple(s.status, [](int v) { return std::string(status_name(v)); }) << ",\n";
    o << "rep_svc_recv |-> " << print_tuple(s.svc_recv, print_set) << ",\n";
    o << "rep_view_number |-> " << print_tuple(s.view, itos) << ",\n";
    o << "replicas |-> 1.." << p.R << "\n";
    return o.str();
}

std::string print_state(const Params& p, const State& s, bool with_rec_vars) { return print_vars(p, s, with_rec_vars); }

std::string print_trace_entry(const Params& p, const State& s, int position, const char* name, const char* location,
                              bool with_rec_vars) {
    std::ostringstream o;
    o << "[\n _TEAction |-> [\n   position |-> " << position << ",\n   name |-> \"" << name << "\",\n   location |-> \""
      << location << "\"\n ],\n"
      << print_vars(p, s, with_rec_vars) << "]";
    return o.str();
}

/* ------------------------------------------------------------------ parser */

namespace {
struct Val {
    enum Kind { INT, BOOL, STR, MV, TUPLE, SET, REC, FCN, INTERVAL } kind = INT;
    int i = 0, hi = 0;
    std::string s;
    std::vector<Val> elems;                          /* TUPLE, SET */
    std::vector<std::pair<std::string, Val>> fields; /* REC */
    std::vector<std::pair<Val, Val>> pairs;          /* FCN */
    const Val* field(const std::string& n) const {
        for (const auto& f : fields)
            if (f.first == n) return &f.second;
        return nullptr;
    }
};

struct Parser {
    const std::string& t;
    size_t i = 0;
    std::string err;
    explicit Parser(const std::string& text) : t(text) {}
    void ws() { while (i < t.size() && isspace((unsigned char)t[i])) i++; }
    bool eat(const char* tok) {
        ws();
        size_t n = strlen(tok);
        if (t.compare(i, n, tok) == 0) { i += n; return true; }
        return false;
    }
    bool peek(const char* tok) {
        ws();
        return t.compare(i, strlen(tok), tok) == 0;
    }
    void fail(const std::string& m) {
        if (err.empty()) err = m + " at offset " + std::to_string(i);
    }
    Val value() {
        Val v;
        ws();
        if (!err.empty() || i >= t.size()) { fail("unexpected end"); return v; }
        if (eat("<<")) {
            v.kind = Val::TUPLE;
            if (eat(">>")) return v;
            do v.elems.push_back(value()); while (err.empty() && eat(","));
            if (!eat(">>")) fail("expected >>");
            return v;
        }
        if (eat("[")) {
            v.kind = Val::REC;
            do {
                ws();
                size_t b = i;
                while (i < t.size() && (isalnum((unsigned char)t[i]) || t[i] == '_')) i++;
                std::string name = t.substr(b, i - b);
                if (name.empty() || !eat("|->")) { fail("expected field |->"); return v; }
                v.fields.emplace_back(name, value());
            } while (err.empty() && eat(","));
            if (!eat("]")) fail("expected ]");
            return v;
        }
        if (eat("{")) {
            v.kind = Val::SET;
            if (eat("}")) return v;
            do v.elems.push_back(value()); while (err.empty() && eat(","));
            if (!eat("}")) fail("expected }");
            return v;
        }
        if (eat("(")) {
            v.kind = Val::FCN;
            do {
                Val k = value();
                if (!eat(":>")) { fail("expected :>"); return v; }
                Val x = value();
                v.pairs.emplace_back(std::move(k), std::move(x));
            } while (err.empty() && eat("@@"));
            if (!eat(")")) fail("expected )");
            return v;
        }
        if (t[i] == '"') {
            v.kind = Val::STR;
            size_t b = ++i;
            while (i < t.size() && t[i] != '"') i++;
            v.s = t.substr(b, i - b);
            i++;
            return v;
        }
        if (isdigit((unsigned char)t[i])) {
            size_t b = i;
            while (i < t.size() && isdigit((unsigned char)t[i])) i++;
            v.kind = Val::INT;
            v.i = atoi(t.substr(b, i - b).c_str());
            if (t.compare(i, 2, "..") == 0) {
                i += 2;
                size_t c = i;
                while (i < t.size() && isdigit((unsigned char)t[i])) i++;
                v.kind = Val::INTERVAL;
                v.hi = atoi(t.substr(c, i - c).c_str());
            }
            return v;
        }
        if (isalpha((unsigned char)t[i]) || t[i] == '_') {
            size_t b = i;
            while (i < t.size() && (isalnum((unsigned char)t[i]) || t[i] == '_')) i++;
            std::string id = t.substr(b, i - b);
            if (id == "TRUE" || id == "FALSE") { v.kind = Val::BOOL; v.i = id == "TRUE"; }
            else { v.kind = Val::MV; v.s = id; }
            return v;
        }
        fail(std::string("unexpected character '") + t[i] + "'");
        return v;
    }
};

int mv_type(const std::string& s) {
    for (int t = 0; t < 12; t++)
        if (s == type_name(t)) return t;
    return -1;
}
int mv_value(const std::string& s) { /* "vN" -> N */
    if (s.size() >= 2 && s[0] == 'v') return atoi(s.c_str() + 1);
    return 0;
}
int as_int(const Val* v) {
    if (!v) return ABSENT;
    if (v->kind == Val::MV && v->s == "Nil") return NIL;
    return v->i;
}
Entry to_entry(const Val& v) {
    Entry e;
    e.view = as_int(v.field("view_number"));
    const Val* o = v.field("operation");
    e.operation = o ? mv_value(o->s) : 0;
    e.client = as_int(v.field("client_id"));
    e.req = as_int(v.field("request_number"));
    return e;
}
Msg to_msg(const Val& v) {
    Msg m;
    const Val* t = v.field("type");
    m.type = t ? mv_type(t->s) : -1;
    m.view = as_int(v.field("view_number"));
    m.src = as_int(v.field("source"));
    m.dest = as_int(v.field("dest"));
    m.op = as_int(v.field("op_number"));
    m.commit = as_int(v.field("commit_number"));
    m.lnv = as_int(v.field("last_normal_vn"));
    m.first_op = as_int(v.field("first_op"));
    m.x = as_int(v.field("x"));
    if (const Val* e = v.field("message")) { m.has_entry = true; m.entry = to_entry(*e); }
    if (const Val* l = v.field("log")) {
        if (l->kind == Val::MV) m.has_log = 2;
        else if (l->kind == Val::TUPLE) {
            m.has_log = 1;
            m.log_lo = 1;
            for (const Val& e : l->elems) m.log.push_back(to_entry(e));
        } else if (l->kind == Val::FCN) {
            m.has_log = 1;
            m.log_lo = l->pairs.empty() ? 1 : l->pairs[0].first.i;
            for (const auto& kv : l->pairs) m.log.push_back(to_entry(kv.second));
        }
    }
    return m;
}
} // namespace

std::string parse_trace_text(const std::string& text, Params& p, std::vector<TraceState>& out) {
    Parser ps(text);
    Val top = ps.value();
    if (!ps.err.empty()) return ps.err;
    if (top.kind != Val::TUPLE) return "trace is not a tuple";
    int maxv = 0, max_svc = 0, max_restart = 0;
    for (const Val& sv : top.elems) {
        if (sv.kind != Val::REC) return "trace element is not a record";
        TraceState ts;
        const Val* act = sv.field("_TEAction");
        if (act) {
            ts.position = as_int(act->field("position"));
            if (const Val* n = act->field("name")) ts.action_name = n->s;
            if (const Val* l = act->field("location")) ts.location = l->s;
        }
        for (const auto& f : sv.fields)
            if (f.first != "_TEAction") ts.var_names.push_back(f.first);
        const Val* reps = sv.field("replicas");
        const Val* cls = sv.field("clients");
        if (!reps || !cls) return "replicas/clients missing";
        p.R = reps->hi;
        p.C = cls->hi;
        State s = init_state(p);
        auto ints = [&](const char* name, std::vector<int>& dst) {
            if (const Val* v = sv.field(name))
                for (size_t r = 0; r < v->elems.size() && r < dst.size(); r++) dst[r] = v->elems[r].i;
        };
        ints("rep_view_number", s.view);
        ints("rep_op_number", s.op);
        ints("rep_commit_number", s.commit);
        ints("rep_last_normal_view", s.lnv);
        ints("rep_rec_number", s.rec_number);
        if (const Val* v = sv.field("rep_status"))
            for (size_t r = 0; r < v->elems.size(); r++)
                s.status[r] = v->elems[r].s == "Normal" ? VSR_NORMAL : (v->elems[r].s == "ViewChange" ? VSR_VIEWCHANGE : VSR_RECOVERING);
        if (const Val* v = sv.field("rep_sent_dvc"))
            for (size_t r = 0; r < v->elems.size(); r++) s.sent_dvc[r] = (char)v->elems[r].i;
        if (const Val* v = sv.field("rep_sent_sv"))
            for (size_t r = 0; r < v->elems.size(); r++) s.sent_sv[r] = (char)v->elems[r].i;
        if (const Val* v = sv.field("rep_log"))
            for (size_t r = 0; r < v->elems.size(); r++)
                for (const Val& e : v->elems[r].elems) s.log[r].push_back(to_entry(e));
        if (const Val* v = sv.field("rep_peer_op_number"))
            for (size_t r = 0; r < v->elems.size(); r++)
                for (size_t k = 0; k < v->elems[r].elems.size(); k++) s.peer_op[r][k] = v->elems[r].elems[k].i;
        if (const Val* v = sv.field("rep_client_table"))
            for (size_t r = 0; r < v->elems.size(); r++)
                for (size_t k = 0; k < v->elems[r].elems.size(); k++) {
                    const Val& row = v->elems[r].elems[k];
                    s.client_table[r][k] = ClientRow{as_int(row.field("request_number")), as_int(row.field("op_number")),
                                                     as_int(row.field("executed")) != 0};
                }
        auto sets = [&](const char* name, std::vector<MsgSet>& dst) {
            if (const Val* v = sv.field(name))
                for (size_t r = 0; r < v->elems.size(); r++)
                    for (const Val& e : v->elems[r].elems) dst[r].insert(to_msg(e));
        };
        sets("rep_svc_recv", s.svc_recv);
        sets("rep_dvc_recv", s.dvc_recv);
        sets("rep_rec_recv", s.rec_recv);
        if (const Val* v = sv.field("messages"))
            for (const auto& kv : v->pairs) s.messages[to_msg(kv.first)] = kv.second.i;
        if (const Val* v = sv.field("aux_svc")) s.aux_svc = v->i;
        if (const Val* v = sv.field("aux_restart")) s.aux_restart = v->i;
        if (const Val* v = sv.field("aux_client_acked"))
            for (const auto& kv : v->pairs) s.acked[mv_value(kv.first.s)] = kv.second.i != 0;
        for (const auto& kv : s.acked) maxv = std::max(maxv, kv.first);
        max_svc = std::max(max_svc, s.aux_svc);
        max_restart = std::max(max_restart, s.aux_restart);
        ts.s = std::move(s);
        out.push_back(std::move(ts));
    }
    p.V = std::max(maxv, 1);
    p.L = max_svc;
    p.restart_limit = max_restart;
    return "";
}

} // namespace orc
