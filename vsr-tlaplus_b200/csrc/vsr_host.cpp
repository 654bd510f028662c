/*
 * vsr_host.cpp — host side of the C ABI (include/vsr_b200.h): TLC-style config loading, identity
 * check of the .tla, single-state operations on packed states, TLC-format state printing.
 * No CUDA in this file; the BFS engine is vsr_gpu.cu.
 */
#include <ctype.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <dlfcn.h>
#include <fcntl.h>
#include <sys/file.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <fstream>
#include <map>
#include <sstream>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "vsr_thunks.h"

namespace vsr {

/* ------------------------------------------------------------------ layout registry */

const ModelOps* find_model_ops(int R, int V, int K) {
#define X(r, v, k) \
    if (R == r && V == v && K == k) return Thunks<Layout<r, v, k>>::get();
    VSR_FOR_EACH_CONFIG(X)
#undef X
    return nullptr;
}

/* ------------------------------------------------------------------ layout plug-ins
 * Constants outside VSR_FOR_EACH_CONFIG: <dir of this library>/layouts/libvsr_layout_R_V_K.so, compiled on first use from
 * <dir>/csrc/vsr_layout_plugin.cu when nvcc is there (VSR_B200_JIT=0 forbids compiling; VSR_B200_NVCC names the compiler).
 * Ranks of one job serialise on a lock file, so one of them compiles and the others load the result. */

struct LayoutPlugin {
    const ModelOps* ops;
    const GpuOps* gpu;
};
static std::mutex g_plugin_mu;
static std::map<std::tuple<int, int, int>, LayoutPlugin> g_plugins;

static std::string library_dir() {
    Dl_info di;
    if (!dladdr((void*)&find_model_ops, &di) || !di.dli_fname) return ".";
    std::string p = di.dli_fname;
    const size_t s = p.rfind('/');
    return s == std::string::npos ? "." : p.substr(0, s);
}
static time_t mtime_of(const std::string& p) {
    struct stat st;
    return stat(p.c_str(), &st) == 0 ? st.st_mtime : 0;
}
static bool try_open_plugin(const std::string& path, int R, int V, int K, LayoutPlugin* out, std::string& why) {
    void* h = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    if (!h) { why = std::string("dlopen failed: ") + dlerror(); return false; }
    typedef int (*abi_fn)(void);
    typedef const ModelOps* (*ops_fn)(void);
    typedef const GpuOps* (*gpu_fn)(void);
    abi_fn abi = (abi_fn)dlsym(h, "vsr_plugin_abi");
    ops_fn ops = (ops_fn)dlsym(h, "vsr_plugin_model_ops");
    gpu_fn gpu = (gpu_fn)dlsym(h, "vsr_plugin_gpu_ops");
    if (!abi || !ops || !gpu || abi() != vsr_gpu_abi()) {
        why = "built against another version of the library";
        dlclose(h);
        return false;
    }
    const ModelOps* o = ops();
    if (o->R != R || o->V != V || o->K != K) { why = "holds another layout"; dlclose(h); return false; }
    out->ops = o;
    out->gpu = gpu();
    return true; /* stays loaded for the life of the process: models point into it */
}
/* A plug-in compile that stopped at one of the layout's compile-time limits (the vsr_limit_* classes of vsr_layout_plugin.cu,
   whose numbers the compiler prints as "vsr_limit_state_bytes<BYTES, MAX> [with BYTES=288, MAX=256]"): one line naming each
   limit it exceeds.  "" when the log shows none of them. */
static std::string plugin_limit_message(const std::string& log) {
    auto nums = [&](const char* cls, long long* a, long long* b) {
        const size_t p = log.find(std::string(cls) + "<"), w = p == std::string::npos ? p : log.find("[with ", p);
        if (w == std::string::npos) return false;
        const char* s = log.c_str() + w;
        const char* e1 = strchr(s, '=');
        const char* e2 = e1 ? strchr(e1 + 1, '=') : nullptr;
        if (!e1 || !e2) return false;
        *a = strtoll(e1 + 1, nullptr, 10);
        *b = strtoll(e2 + 1, nullptr, 10);
        return true;
    };
    std::string out;
    long long a, b;
    auto add = [&](const std::string& m) { out += (out.empty() ? "" : "; ") + m; };
    if (nums("vsr_limit_state_bytes", &a, &b))
        add("the packed state would be " + std::to_string(a) + " bytes, more than " + std::to_string(b) + " (VSR_MAX_STATE_BYTES)");
    if (nums("vsr_limit_smem_bytes", &a, &b))
        add("the expand kernel's shared memory would be " + std::to_string(a) + " bytes, more than the " + std::to_string(b) + " of an SM");
    if (nums("vsr_limit_pool_item", &a, &b))
        add("an action group of " + std::to_string(a) + " bindings does not fit the expand kernel's 16-bit pool items (at most " +
            std::to_string(b) + ")");
    return out;
}
static bool load_layout_plugin(int R, int V, int K, LayoutPlugin* out, std::string& why) {
    std::lock_guard<std::mutex> guard(g_plugin_mu);
    const auto key = std::make_tuple(R, V, K);
    auto it = g_plugins.find(key);
    if (it != g_plugins.end()) { *out = it->second; return true; }
    if (R < 2 || R > VSR_MAX_R || V < 1 || V > VSR_MAX_V || K < 1 || K > 15) {
        why = "outside the packed encoding's range (ReplicaCount 2..7, |Values| 1..7, StartViewOnTimerLimit 0..14)";
        return false;
    }
    const std::string dir = library_dir(), ldir = dir + "/layouts", src = dir + "/csrc/vsr_layout_plugin.cu";
    const std::string name = "libvsr_layout_" + std::to_string(R) + "_" + std::to_string(V) + "_" + std::to_string(K) + ".so";
    const std::string path = ldir + "/" + name;
    time_t newest = 0; /* of the sources the plug-in is made of */
    for (const char* f : {"vsr_layout_plugin.cu", "vsr_gpu_thunks.cuh", "vsr_gpu.cuh", "vsr_spill.cuh", "vsr_thunks.h", "vsr_actions.h", "vsr_layout.h",
                          "vsr_flat_conv.h", "vsr_model.h"})
        newest = std::max(newest, mtime_of(dir + "/csrc/" + f));
    std::string open_why;
    if (mtime_of(path) && mtime_of(path) >= newest && try_open_plugin(path, R, V, K, out, open_why)) {
        g_plugins[key] = *out;
        return true;
    }
    const char* jit = getenv("VSR_B200_JIT");
    if (jit && jit[0] == '0') { why = "not built in, no usable " + path + (open_why.empty() ? "" : " (" + open_why + ")") + ", and VSR_B200_JIT=0"; return false; }
    if (!mtime_of(src)) { why = "not built in, and the plug-in source " + src + " is not installed"; return false; }
    if (dir.find('\'') != std::string::npos) { why = "not built in, and the library path contains a quote character (the compile command cannot name it)"; return false; }
    mkdir(ldir.c_str(), 0755);
    const std::string lock = path + ".lock";
    const int fd = open(lock.c_str(), O_CREAT | O_RDWR, 0644);
    if (fd >= 0) flock(fd, LOCK_EX);
    bool ok = mtime_of(path) >= newest && mtime_of(path) && try_open_plugin(path, R, V, K, out, open_why); /* another rank was faster */
    if (!ok) {
        const char* nv = getenv("VSR_B200_NVCC");
        std::string nvcc = nv ? nv : (access("/usr/local/cuda/bin/nvcc", X_OK) == 0 ? "/usr/local/cuda/bin/nvcc" : "nvcc");
        const std::string tmp = path + ".tmp" + std::to_string((long)getpid()), log = path + ".log";
        const std::string cmd = nvcc + " -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -diag-suppress 128"
                                " -DVSR_ONLY_R=" + std::to_string(R) + " -DVSR_ONLY_V=" + std::to_string(V) + " -DVSR_ONLY_K=" + std::to_string(K) +
                                " -shared -Xlinker -Bsymbolic -o '" + tmp + "' '" + src + "' > '" + log + "' 2>&1";
        const int rc = system(cmd.c_str());
        if (rc == 0 && rename(tmp.c_str(), path.c_str()) == 0) ok = try_open_plugin(path, R, V, K, out, open_why);
        else {
            unlink(tmp.c_str());
            std::ifstream lf(log);
            std::stringstream ss;
            ss << lf.rdbuf();
            std::string t = ss.str();
            const std::string limit = plugin_limit_message(t);
            if (t.size() > 600) t = t.substr(0, 600) + " ...";
            open_why = limit.empty() ? "compiling it failed (" + nvcc + ", log " + log + "): " + t : "the layout cannot be built: " + limit;
        }
    }
    if (fd >= 0) { flock(fd, LOCK_UN); close(fd); }
    if (!ok) { why = "not built in, and " + open_why; return false; }
    g_plugins[key] = *out;
    return true;
}

/* ------------------------------------------------------------------ names */

static const char* const kActionNames[VSR_NUM_ACTIONS] = {
    "Initial predicate", "TimerSendSVC", "ReceiveHigherSVC", "ReceiveMatchingSVC", "SendDVC", "ReceiveHigherDVC",
    "ReceiveMatchingDVC", "SendSV", "ReceiveSV", "ReceiveClientRequest", "ReceivePrepareMsg", "ReceivePrepareOkMsg",
    "ExecuteOp", "SendGetState", "ReceiveGetState", "ReceiveNewState", "RestartEmpty", "ReceivesRecoveryMsg",
    "ReceivesRecoveryResponseMsg", "CompleteRecovery"};
static const char* const kTypeNames[12] = {"RequestMsg", "ReplyMsg", "PrepareMsg", "PrepareOkMsg", "CommitMsg",
                                           "StartViewChangeMsg", "DoViewChangeMsg", "StartViewMsg", "GetStateMsg",
                                           "NewStateMsg", "RecoveryMsg", "RecoveryResponseMsg"};
static const char* const kStatusNames[3] = {"Normal", "ViewChange", "Recovering"};
/* the 20 VARIABLES, VSR.tla:119-138 */
static const char* const kVariables[20] = {
    "replicas", "rep_status", "rep_log", "rep_view_number", "rep_op_number", "rep_commit_number", "rep_peer_op_number",
    "rep_client_table", "rep_last_normal_view", "rep_svc_recv", "rep_dvc_recv", "rep_sent_dvc", "rep_sent_sv",
    "rep_rec_number", "rep_rec_recv", "clients", "messages", "aux_svc", "aux_restart", "aux_client_acked"};
/* model-value constants, VSR.tla:99-117 / VSR.cfg:9-24 */
static const char* const kModelValueConstants[16] = {
    "Normal", "ViewChange", "Recovering", "RequestMsg", "ReplyMsg", "PrepareMsg", "PrepareOkMsg", "CommitMsg",
    "StartViewChangeMsg", "DoViewChangeMsg", "StartViewMsg", "GetStateMsg", "NewStateMsg", "RecoveryMsg",
    "RecoveryResponseMsg", "Nil"};

static void set_err(char* err, size_t cap, const std::string& msg) {
    if (err && cap) {
        snprintf(err, cap, "%s", msg.c_str());
    }
}

/* ------------------------------------------------------------------ .tla identity check */

/* FNV-1a 64 of the spec text without comments ("\\*" to end of line, "(* ... *)" nested), without trailing blanks, without
   empty lines and with LF line ends; leading indentation is kept (junction lists are layout-sensitive in TLA+). */
uint64_t vsr_normalised_spec_hash(const std::string& text) {
    std::string out, line;
    int depth = 0;
    auto flush = [&]() {
        size_t e = line.find_last_not_of(" \t\r");
        if (e != std::string::npos) { out.append(line, 0, e + 1); out.push_back('\n'); }
        line.clear();
    };
    for (size_t i = 0; i < text.size(); i++) {
        const char c = text[i], d = i + 1 < text.size() ? text[i + 1] : 0;
        if (depth == 0 && c == '\\' && d == '*') { while (i < text.size() && text[i] != '\n') i++; flush(); continue; }
        if (c == '(' && d == '*') { depth++; i++; continue; }
        if (depth > 0 && c == '*' && d == ')') { depth--; i++; continue; }
        if (c == '\n') { flush(); continue; }
        if (depth == 0) line.push_back(c);
    }
    flush();
    uint64_t h = 0xcbf29ce484222325ULL;
    for (unsigned char c : out) { h ^= c; h *= 0x100000001b3ULL; }
    return h;
}
/* vsr-revisited/paper/VSR.tla @ 7566e8af (the revision SURVEY.md and every file:line citation in this repo refer to) */
static const uint64_t VSR_TLA_NORMALISED_HASH = 0x2b832f2080e8649cULL;

static int verify_tla(const char* path, VsrModel* m, std::string& why) {
    std::ifstream f(path, std::ios::binary);
    if (!f) { why = std::string("cannot read spec ") + path; return VSR_RC_SPEC_ERROR; }
    std::stringstream ss;
    ss << f.rdbuf();
    const std::string text = ss.str();
    uint64_t h = 0xcbf29ce484222325ULL;
    for (unsigned char c : text) { h ^= c; h *= 0x100000001b3ULL; }
    m->info.spec_hash = h;
    /* The actions and invariants are hand-lowered, so the FILE must be the spec that was lowered: checking the structure
       below is not enough (an edited guard or invariant body would pass it and be "verified" against the built-in
       lowering).  Compare a hash of the text normalised for line ends, trailing blanks, blank lines and comments. */
    const uint64_t nh = vsr_normalised_spec_hash(text);
    const bool pinned = nh == VSR_TLA_NORMALISED_HASH;
    if (!pinned) {
        const char* allow = getenv("VSR_B200_ALLOW_EDITED_SPEC");
        if (!(allow && allow[0] == '1')) {
            char buf[320];
            snprintf(buf, sizeof buf, "%s is not the VSR.tla this checker lowers by hand (normalised text hash %016llx, expected %016llx): Next and the "
                     "invariants are compiled in, so an edited spec would be checked against the ORIGINAL definitions", path, (unsigned long long)nh,
                     (unsigned long long)VSR_TLA_NORMALISED_HASH);
            why = buf;
            return VSR_RC_SPEC_ERROR;
        }
        fprintf(stderr, "WARNING: %s differs from the VSR.tla this checker lowers (VSR_B200_ALLOW_EDITED_SPEC=1): the BUILT-IN Next and invariants are "
                        "checked, NOT the definitions in this file; the spec is reported as unverified\n", path);
    }
    std::vector<std::string> lines;
    {
        std::string cur;
        for (char c : text) {
            if (c == '\n') { lines.push_back(cur); cur.clear(); }
            else if (c != '\r') cur.push_back(c);
        }
        lines.push_back(cur);
    }
    auto strip_comment = [](const std::string& l) {
        size_t p = l.find("\\*");
        return p == std::string::npos ? l : l.substr(0, p);
    };
    /* module header, VSR.tla:1 */
    bool mod = false;
    for (const std::string& l : lines) {
        if (l.find("MODULE") != std::string::npos) {
            std::istringstream is(l);
            std::string a, b, c;
            is >> a >> b >> c;
            mod = (b == "MODULE" && c == "VSR");
            break;
        }
    }
    if (!mod) { why = "spec is not `MODULE VSR` (this checker is hand-lowered for vsr-revisited/paper/VSR.tla only)"; return VSR_RC_SPEC_ERROR; }
    /* VARIABLES, VSR.tla:119-138 */
    std::vector<std::string> vars;
    for (size_t i = 0; i < lines.size(); i++) {
        if (lines[i].compare(0, 9, "VARIABLES") != 0) continue;
        for (size_t j = i; j < lines.size(); j++) {
            std::string l = strip_comment(lines[j]);
            if (j == i) l = l.substr(9);
            bool any = false;
            std::string id;
            for (char c : l + ",") {
                if (isalnum((unsigned char)c) || c == '_') id.push_back(c);
                else { if (!id.empty()) { vars.push_back(id); any = true; id.clear(); } }
            }
            if (!any && j > i) break;
            if (strip_comment(lines[j]).find(',') == std::string::npos && j > i) break;
        }
        break;
    }
    if (vars.size() != 20) { why = "spec declares " + std::to_string(vars.size()) + " VARIABLES, VSR.tla declares 20"; return VSR_RC_SPEC_ERROR; }
    for (int i = 0; i < 20; i++)
        if (vars[i] != kVariables[i]) { why = "VARIABLES differ from VSR.tla at `" + vars[i] + "`"; return VSR_RC_SPEC_ERROR; }
    /* Next, VSR.tla:896-918 */
    std::vector<std::string> disj;
    for (size_t i = 0; i < lines.size(); i++) {
        if (lines[i].compare(0, 7, "Next ==") != 0) continue;
        for (size_t j = i + 1; j < lines.size(); j++) {
            std::string l = strip_comment(lines[j]);
            size_t p = l.find("\\/");
            if (p != std::string::npos) {
                std::istringstream is(l.substr(p + 2));
                std::string name;
                is >> name;
                disj.push_back(name);
            } else if (l.find_first_not_of(" \t") != std::string::npos) break;
            else if (lines[j].find_first_not_of(" \t") == std::string::npos) break;
        }
        break;
    }
    if (disj.size() != 19) { why = "Next has " + std::to_string(disj.size()) + " disjuncts, VSR.tla has 19"; return VSR_RC_SPEC_ERROR; }
    for (int i = 0; i < 19; i++)
        if (disj[i] != kActionNames[i + 1]) { why = "Next disjunct " + std::to_string(i + 1) + " is `" + disj[i] + "`, expected `" + kActionNames[i + 1] + "`"; return VSR_RC_SPEC_ERROR; }
    /* definitions the cfg may name must exist */
    for (const char* d : {"Init ==", "view ==", "symmValues ==", "AcknowledgedWriteNotLost ==", "AcknowledgedWritesExistOnMajority ==", "NoLogDivergence ==", "TestInv =="}) {
        bool found = false;
        for (const std::string& l : lines) found = found || l.compare(0, strlen(d), d) == 0;
        if (!found) { why = std::string("definition `") + d + "` not found in spec"; return VSR_RC_SPEC_ERROR; }
    }
    /* action locations as TLC reports them: extent of the definition body */
    for (int a = 1; a < VSR_NUM_ACTIONS; a++) {
        const std::string head = std::string(kActionNames[a]) + " ==";
        for (size_t i = 0; i < lines.size(); i++) {
            if (lines[i].compare(0, head.size(), head) != 0) continue;
            size_t b = i + 1;
            while (b < lines.size() && lines[b].find_first_not_of(" \t") == std::string::npos) b++;
            size_t e = b;
            while (e + 1 < lines.size() && lines[e + 1].find_first_not_of(" \t") != std::string::npos && isspace((unsigned char)lines[e + 1][0])) e++;
            if (b < lines.size()) {
                const size_t c0 = lines[b].find_first_not_of(" \t") + 1;
                const size_t c1 = lines[e].find_last_not_of(" \t") + 1;
                char buf[128];
                snprintf(buf, sizeof buf, "line %zu, col %zu to line %zu, col %zu of module VSR", b + 1, c0, e + 1, c1);
                m->action_location[a] = buf;
            }
            break;
        }
    }
    m->info.spec_verified = pinned ? 1 : 0;
    return 0;
}

/* ------------------------------------------------------------------ cfg parser (TLC cfg grammar subset, VSR.cfg:1-39) */

struct Tok {
    std::string s;
    int line;
};
static std::vector<Tok> lex_cfg(const std::string& text) {
    std::vector<Tok> out;
    int line = 1;
    size_t i = 0;
    while (i < text.size()) {
        char c = text[i];
        if (c == '\n') { line++; i++; continue; }
        if (isspace((unsigned char)c)) { i++; continue; }
        if (c == '\\' && i + 1 < text.size() && text[i + 1] == '*') { /* \* comment to end of line */
            while (i < text.size() && text[i] != '\n') i++;
            continue;
        }
        if (c == '(' && i + 1 < text.size() && text[i + 1] == '*') { /* (* block comment *) */
            i += 2;
            while (i + 1 < text.size() && !(text[i] == '*' && text[i + 1] == ')')) { if (text[i] == '\n') line++; i++; }
            i += 2;
            continue;
        }
        if (isalnum((unsigned char)c) || c == '_') {
            size_t b = i;
            while (i < text.size() && (isalnum((unsigned char)text[i]) || text[i] == '_')) i++;
            out.push_back({text.substr(b, i - b), line});
            continue;
        }
        if (c == '<' && text.compare(i, 2, "<-") == 0) { out.push_back({"<-", line}); i += 2; continue; }
        out.push_back({std::string(1, c), line});
        i++;
    }
    return out;
}
static bool is_int(const std::string& s) {
    if (s.empty()) return false;
    for (char c : s)
        if (!isdigit((unsigned char)c)) return false;
    return true;
}
static bool is_keyword(const std::string& s) {
    static const char* kw[] = {"CONSTANT", "CONSTANTS", "INIT", "NEXT", "VIEW", "SYMMETRY", "INVARIANT", "INVARIANTS", "SPECIFICATION",
                               "PROPERTY", "PROPERTIES", "CONSTRAINT", "CONSTRAINTS", "ACTION_CONSTRAINT", "ACTION_CONSTRAINTS",
                               "CHECK_DEADLOCK", "POSTCONDITION", "ALIAS", "TYPE", "TYPE_CONSTRAINT"};
    for (const char* k : kw)
        if (s == k) return true;
    return false;
}

static int parse_cfg(const std::string& text, VsrModel* m, std::string& why) {
    std::vector<Tok> t = lex_cfg(text);
    std::map<std::string, int> ints;
    std::map<std::string, std::string> mvs;
    std::vector<std::string> values;
    bool have_values = false;
    std::string init, next, view, symm, spec;
    std::vector<std::string> invs;
    std::vector<Tok> props;
    m->check_deadlock_cfg = -1;
    auto at = [&](size_t i) -> std::string { return i < t.size() ? t[i].s : std::string(); };
    auto where = [&](size_t i) { return " (cfg line " + std::to_string(i < t.size() ? t[i].line : (t.empty() ? 0 : t.back().line)) + ")"; };
    size_t i = 0;
    while (i < t.size()) {
        const std::string k = t[i].s;
        if (k == "CONSTANT" || k == "CONSTANTS") {
            i++;
            while (i < t.size() && !is_keyword(t[i].s)) {
                const std::string name = t[i].s;
                if (at(i + 1) == "<-") { why = "operator substitution `" + name + " <- ...` is not supported" + where(i); return VSR_RC_CONFIG_ERROR; }
                if (at(i + 1) != "=") { why = "expected `=` after constant `" + name + "`" + where(i); return VSR_RC_CONFIG_ERROR; }
                i += 2;
                if (at(i) == "{") {
                    std::vector<std::string> elems;
                    i++;
                    while (i < t.size() && t[i].s != "}") {
                        if (t[i].s != ",") elems.push_back(t[i].s);
                        i++;
                    }
                    if (at(i) != "}") { why = "unterminated set for constant `" + name + "`" + where(i); return VSR_RC_CONFIG_ERROR; }
                    i++;
                    if (name == "Values") { values = elems; have_values = true; }
                    else { why = "constant `" + name + "` is not a set in VSR.tla" + where(i); return VSR_RC_CONFIG_ERROR; }
                } else if (is_int(at(i))) {
                    ints[name] = atoi(t[i].s.c_str());
                    i++;
                } else if (i < t.size()) {
                    mvs[name] = t[i].s;
                    i++;
                } else { why = "missing value for constant `" + name + "`"; return VSR_RC_CONFIG_ERROR; }
            }
        } else if (k == "INIT") { init = at(i + 1); i += 2; }
        else if (k == "NEXT") { next = at(i + 1); i += 2; }
        else if (k == "VIEW") { view = at(i + 1); i += 2; }
        else if (k == "SYMMETRY") { symm = at(i + 1); i += 2; }
        else if (k == "INVARIANT" || k == "INVARIANTS") {
            i++;
            while (i < t.size() && !is_keyword(t[i].s)) invs.push_back(t[i++].s);
        } else if (k == "CHECK_DEADLOCK") {
            m->check_deadlock_cfg = at(i + 1) == "TRUE" ? 1 : 0;
            i += 2;
        } else if (k == "SPECIFICATION") {
            /* Spec == Init /\ [][Next]_vars /\ WF_vars(Next) (VSR.tla:967): for invariant checking TLC explores Init/Next
               exactly as with INIT/NEXT; the fairness conjunct is what PROPERTY ViewChangeCompletes is checked under */
            spec = at(i + 1);
            i += 2;
        } else if (k == "PROPERTY" || k == "PROPERTIES") {
            i++;
            if (i >= t.size() || is_keyword(t[i].s)) { why = "`" + k + "` names no property" + where(i); return VSR_RC_CONFIG_ERROR; }
            while (i < t.size() && !is_keyword(t[i].s)) props.push_back({t[i].s, t[i].line}), i++;
        } else if (k == "CONSTRAINT" || k == "CONSTRAINTS" ||
                   k == "ACTION_CONSTRAINT" || k == "ACTION_CONSTRAINTS" || k == "POSTCONDITION" || k == "ALIAS") {
            why = "`" + k + "` is not supported: this checker runs safety (invariant) checking of VSR.tla only (no temporal "
                  "formulas, liveness or constraints)" + where(i);
            return VSR_RC_CONFIG_ERROR;
        } else { why = "unexpected token `" + k + "`" + where(i); return VSR_RC_CONFIG_ERROR; }
    }
    for (const char* n : {"ReplicaCount", "ClientCount", "StartViewOnTimerLimit", "RestartEmptyLimit"})
        if (!ints.count(n)) { why = std::string("constant `") + n + "` (VSR.tla:92-96) has no integer value in the config"; return VSR_RC_CONFIG_ERROR; }
    if (!have_values || values.empty()) { why = "constant `Values` must be a non-empty set of model values"; return VSR_RC_CONFIG_ERROR; }
    for (const char* n : kModelValueConstants) {
        if (!mvs.count(n)) { why = std::string("model-value constant `") + n + "` (VSR.tla:99-117) is not assigned"; return VSR_RC_CONFIG_ERROR; }
        if (mvs[n] != n) { why = std::string("constant `") + n + "` must be the model value of the same name (`" + n + " = " + n + "`)"; return VSR_RC_CONFIG_ERROR; }
    }
    for (size_t a = 0; a < values.size(); a++)
        for (size_t b = a + 1; b < values.size(); b++)
            if (values[a] == values[b]) { why = "duplicate element `" + values[a] + "` in Values"; return VSR_RC_CONFIG_ERROR; }
    int property = 0;
    for (const Tok& p : props) {
        if (p.s != "ViewChangeCompletes") {
            why = "PROPERTY `" + p.s + "` is not supported: the one temporal property checked is ViewChangeCompletes (VSR.tla:964-965)" +
                  (p.s == "AllReplicasMoveToSameView" ? std::string("; AllReplicasMoveToSameView is its state predicate, not a temporal formula") : std::string()) +
                  " (cfg line " + std::to_string(p.line) + ")";
            return VSR_RC_CONFIG_ERROR;
        }
        property |= 1;
    }
    if (property && spec.empty()) {
        /* under [][Next]_vars alone stuttering at the first not-P state violates []<>P trivially: the property is only
           meaningful with the fairness conjunct of Spec */
        why = "PROPERTY ViewChangeCompletes needs `SPECIFICATION Spec` (VSR.tla:967: Spec's WF_vars(Next) is what makes it "
              "meaningful); with INIT/NEXT and no fairness it is refused";
        return VSR_RC_CONFIG_ERROR;
    }
    if (!spec.empty()) {
        if (!init.empty() || !next.empty()) { why = "the config names both SPECIFICATION and INIT/NEXT (TLC refuses that too)"; return VSR_RC_CONFIG_ERROR; }
        if (spec != "Spec") { why = "SPECIFICATION `" + spec + "` unknown; VSR.tla defines `Spec` (:966)"; return VSR_RC_CONFIG_ERROR; }
        init = "Init";
        next = "Next";
    }
    if (init != "Init") { why = "INIT must be `Init` (VSR.tla:323)"; return VSR_RC_CONFIG_ERROR; }
    if (next != "Next") { why = "NEXT must be `Next` (VSR.tla:896)"; return VSR_RC_CONFIG_ERROR; }
    if (!view.empty() && view != "view") { why = "VIEW `" + view + "` unknown; VSR.tla defines `view` (:149)"; return VSR_RC_CONFIG_ERROR; }
    if (!symm.empty() && symm != "symmValues") { why = "SYMMETRY `" + symm + "` unknown; VSR.tla defines `symmValues` (:151)"; return VSR_RC_CONFIG_ERROR; }
    int mask = 0;
    m->inv_order.clear();
    for (const std::string& s : invs) {
        int bit = 0;
        for (int b = 0; b < 4; b++)
            if (s == INVARIANT_NAMES[b]) bit = 1 << b;
        if (!bit) { why = "INVARIANT `" + s + "` is not defined in VSR.tla (:926-952)"; return VSR_RC_CONFIG_ERROR; }
        if (!(mask & bit)) m->inv_order.push_back(bit);
        mask |= bit;
    }
    VsrModelInfo& I = m->info;
    I.replica_count = ints["ReplicaCount"];
    I.client_count = ints["ClientCount"];
    I.value_count = (int)values.size();
    I.start_view_on_timer_limit = ints["StartViewOnTimerLimit"];
    I.restart_empty_limit = ints["RestartEmptyLimit"];
    I.symmetry = symm.empty() ? 0 : 1;
    I.view = view.empty() ? 0 : 1;
    I.invariant = mask;
    I.property = property;
    for (size_t v = 0; v < values.size() && v < VSR_MAX_V; v++) snprintf(I.value_names[v], sizeof I.value_names[v], "%s", values[v].c_str());
    return 0;
}

static int bind_model(VsrModel* m, std::string& why) {
    VsrModelInfo& I = m->info;
    if (I.replica_count < 2) { why = "ReplicaCount must be >= 2"; return VSR_RC_CONFIG_ERROR; }
    if (I.client_count != 1) {
        why = "ClientCount = " + std::to_string(I.client_count) + ": ReceivePrepareMsg reads the non-existent field m.commit "
              "(VSR.tla:421) as soon as there are two clients — TLC aborts there too; only ClientCount = 1 is checkable";
        return VSR_RC_CONFIG_ERROR;
    }
    if (I.restart_empty_limit != 0) {
        why = "RestartEmptyLimit = " + std::to_string(I.restart_empty_limit) + ": the recovery actions (VSR.tla:813-894) are not "
              "lowered yet; every config of the reference sets it to 0 (VSR.cfg:8)";
        return VSR_RC_CONFIG_ERROR;
    }
    if (I.start_view_on_timer_limit < 0) { why = "StartViewOnTimerLimit must be >= 0"; return VSR_RC_CONFIG_ERROR; }
    const int K = 1 + I.start_view_on_timer_limit;
    m->ops = find_model_ops(I.replica_count, I.value_count, K);
    m->gpu = find_gpu_ops(I.replica_count, I.value_count, K);
    if (!m->ops) {
        LayoutPlugin pl;
        std::string pwhy;
        if (!load_layout_plugin(I.replica_count, I.value_count, K, &pl, pwhy)) {
            why = "packed layout for ReplicaCount=" + std::to_string(I.replica_count) + " |Values|=" + std::to_string(I.value_count) +
                  " StartViewOnTimerLimit=" + std::to_string(I.start_view_on_timer_limit) + ": " + pwhy;
            return VSR_RC_CONFIG_ERROR;
        }
        m->ops = pl.ops;
        m->gpu = pl.gpu;
    }
    if (I.value_count == 1) I.symmetry = 0; /* Permutations of a singleton: identity */
    m->run.symmetry = I.symmetry;
    m->run.use_view = I.view;
    m->run.invariant = I.invariant;
    I.state_bytes = m->ops->bytes;
    I.state_bits = m->ops->bits;
    I.num_candidates = m->ops->ncand;
    for (int a = 0; a < VSR_NUM_ACTIONS; a++)
        if (m->action_location[a].empty()) m->action_location[a] = "Unknown location";
    return 0;
}

} // namespace vsr

using namespace vsr;

/* ------------------------------------------------------------------ TLC-format printing of a flat state */

namespace {

struct Printer {
    const VsrModel* m;
    std::string o;
    explicit Printer(const VsrModel* mm) : m(mm) {}
    void num(int v) {
        if (v == VSR_NIL) o += "Nil";
        else o += std::to_string(v);
    }
    void value_name(int x) {
        if (x >= 1 && x <= m->info.value_count && m->info.value_names[x - 1][0]) o += m->info.value_names[x - 1];
        else { o += "v"; o += std::to_string(x); }
    }
    void entry(const VsrEntry& e) {
        o += "[view_number |-> "; num(e.view);
        o += ", operation |-> "; value_name(e.operation);
        o += ", client_id |-> "; num(e.client);
        o += ", request_number |-> "; num(e.req);
        o += "]";
    }
    void logfn(const VsrMsg& k) {
        if (k.has_log == 2) { o += "Nil"; return; }
        if (k.log_n == 0) { o += "<<>>"; return; }
        if (k.log_lo == 1) {
            o += "<<";
            for (int i = 0; i < k.log_n; i++) { if (i) o += ", "; entry(k.log[i]); }
            o += ">>";
        } else { /* a function whose domain does not start at 1 (NewState, VSR.tla:535-536) */
            o += "(";
            for (int i = 0; i < k.log_n; i++) { if (i) o += " @@ "; num(k.log_lo + i); o += " :> "; entry(k.log[i]); }
            o += ")";
        }
    }
    /* fields in TLC's first-interned order (evidenced by state_transfer_violation_trace.txt:563) */
    void msg(const VsrMsg& k) {
        bool first = true;
        auto f = [&](const char* name) { o += first ? "" : ", "; o += name; o += " |-> "; first = false; };
        o += "[";
        if (k.view != VSR_ABSENT) { f("view_number"); num(k.view); }
        f("type"); o += kTypeNames[k.type < 12 ? k.type : 0];
        if (k.has_entry) { f("message"); entry(k.entry); }
        if (k.op != VSR_ABSENT) { f("op_number"); num(k.op); }
        if (k.commit != VSR_ABSENT) { f("commit_number"); num(k.commit); }
        if (k.dest != VSR_ABSENT) { f("dest"); num(k.dest); }
        if (k.src != VSR_ABSENT) { f("source"); num(k.src); }
        if (k.has_log) { f("log"); logfn(k); }
        if (k.lnv != VSR_ABSENT) { f("last_normal_vn"); num(k.lnv); }
        if (k.x != VSR_ABSENT) { f("x"); num(k.x); }
        if (k.first_op != VSR_ABSENT) { f("first_op"); num(k.first_op); }
        o += "]";
    }
};

/* TLC's RecordValue order on message records: number of fields, then field by field (name index in
   intern order, then value) — SURVEY App. B.3.  Independent of the oracle's implementation. */
struct FieldList {
    int n = 0;
    int name[12];
    long val[12]; /* scalar fields; entries/logs compared separately */
};
static const int kFieldRank[] = {/*view*/ 0, /*type*/ 4, /*message*/ 5, /*op*/ 6, /*commit*/ 7, /*dest*/ 8, /*source*/ 9, /*log*/ 10, /*lnv*/ 11, /*x*/ 12, /*first_op*/ 14};
static int cmp_u8_nil(int a, int b) {
    if (a == b) return 0;
    if (a == VSR_NIL) return -1;
    if (b == VSR_NIL) return 1;
    return a < b ? -1 : 1;
}
static int cmp_flat_entry(const VsrEntry& a, const VsrEntry& b) {
    if (a.view != b.view) return a.view < b.view ? -1 : 1;
    if (a.operation != b.operation) return a.operation < b.operation ? -1 : 1;
    if (a.client != b.client) return a.client < b.client ? -1 : 1;
    if (a.req != b.req) return a.req < b.req ? -1 : 1;
    return 0;
}
static int cmp_flat_msg(const VsrMsg& a, const VsrMsg& b) {
    auto present = [](const VsrMsg& k, bool p[11]) {
        p[0] = k.view != VSR_ABSENT; p[1] = true; p[2] = k.has_entry != 0; p[3] = k.op != VSR_ABSENT; p[4] = k.commit != VSR_ABSENT;
        p[5] = k.dest != VSR_ABSENT; p[6] = k.src != VSR_ABSENT; p[7] = k.has_log != 0; p[8] = k.lnv != VSR_ABSENT; p[9] = k.x != VSR_ABSENT;
        p[10] = k.first_op != VSR_ABSENT;
    };
    bool pa[11], pb[11];
    present(a, pa); present(b, pb);
    int na = 0, nb = 0;
    for (int i = 0; i < 11; i++) { na += pa[i]; nb += pb[i]; }
    if (na != nb) return na < nb ? -1 : 1;
    int ia = 0, ib = 0;
    for (;;) {
        while (ia < 11 && !pa[ia]) ia++;
        while (ib < 11 && !pb[ib]) ib++;
        if (ia >= 11 || ib >= 11) return 0;
        if (kFieldRank[ia] != kFieldRank[ib]) return kFieldRank[ia] < kFieldRank[ib] ? -1 : 1;
        int c = 0;
        switch (ia) {
        case 0: c = cmp_u8_nil(a.view, b.view); break;
        case 1: c = cmp_u8_nil(a.type, b.type); break;
        case 2: c = cmp_flat_entry(a.entry, b.entry); break;
        case 3: c = cmp_u8_nil(a.op, b.op); break;
        case 4: c = cmp_u8_nil(a.commit, b.commit); break;
        case 5: c = cmp_u8_nil(a.dest, b.dest); break;
        case 6: c = cmp_u8_nil(a.src, b.src); break;
        case 7:
            if (a.has_log != b.has_log) c = a.has_log == 2 ? -1 : 1;
            else if (a.has_log == 1) {
                if (a.log_n != b.log_n) c = a.log_n < b.log_n ? -1 : 1;
                for (int i = 0; !c && i < a.log_n; i++) {
                    if (a.log_lo != b.log_lo) c = a.log_lo < b.log_lo ? -1 : 1;
                    else c = cmp_flat_entry(a.log[i], b.log[i]);
                }
            }
            break;
        case 8: c = cmp_u8_nil(a.lnv, b.lnv); break;
        case 9: c = cmp_u8_nil(a.x, b.x); break;
        case 10: c = cmp_u8_nil(a.first_op, b.first_op); break;
        }
        if (c) return c;
        ia++; ib++;
    }
}

static std::string flat_to_tla(const VsrModel* m, const VsrFlatState* f) {
    Printer p(m);
    std::string& o = p.o;
    const int R = f->R, C = f->C, V = f->V;
    auto sorted = [](const VsrMsg* a, int n) {
        std::vector<const VsrMsg*> v;
        for (int i = 0; i < n; i++) v.push_back(&a[i]);
        std::sort(v.begin(), v.end(), [](const VsrMsg* x, const VsrMsg* y) { return cmp_flat_msg(*x, *y) < 0; });
        return v;
    };
    auto set_of = [&](const VsrMsg* a, int n) {
        o += "{";
        bool first = true;
        for (const VsrMsg* k : sorted(a, n)) { if (!first) o += ", "; p.msg(*k); first = false; }
        o += "}";
    };
    auto tuple_int = [&](const char* name, auto get) {
        o += name; o += " |-> <<";
        for (int r = 0; r < R; r++) { if (r) o += ", "; o += get(r); }
        o += ">>,\n";
    };
    /* variables alphabetical, as TLC prints them (trace:8-24) */
    o += "aux_client_acked |-> ";
    {
        int n = 0;
        for (int x = 0; x < V; x++) n += f->acked[x] != 0;
        if (!n) o += "<<>>";
        else {
            o += "(";
            bool first = true;
            for (int x = 0; x < V; x++) {
                if (!f->acked[x]) continue;
                if (!first) o += " @@ ";
                p.value_name(x + 1);
                o += f->acked[x] == 2 ? " :> TRUE" : " :> FALSE";
                first = false;
            }
            o += ")";
        }
    }
    o += ",\n";
    o += "aux_restart |-> " + std::to_string(f->aux_restart) + ",\n";
    o += "aux_svc |-> " + std::to_string(f->aux_svc) + ",\n";
    o += "clients |-> 1.." + std::to_string(C) + ",\n";
    o += "messages |-> ";
    if (!f->n_msgs) o += "<<>>";
    else {
        o += "(";
        bool first = true;
        for (const VsrMsg* k : sorted(f->msgs, f->n_msgs)) {
            if (!first) o += " @@ ";
            p.msg(*k);
            o += " :> " + std::to_string(k->count);
            first = false;
        }
        o += ")";
    }
    o += ",\n";
    o += "rep_client_table |-> <<";
    for (int r = 0; r < R; r++) {
        if (r) o += ", ";
        o += "<<";
        for (int c = 0; c < C; c++) {
            if (c) o += ", ";
            const VsrClientRow& row = f->rep[r].client_table[c];
            o += "[request_number |-> " + std::to_string(row.req) + ", op_number |-> " + std::to_string(row.op) + ", executed |-> " +
                 (row.executed ? "TRUE" : "FALSE") + "]";
        }
        o += ">>";
    }
    o += ">>,\n";
    tuple_int("rep_commit_number", [&](int r) { return std::to_string(f->rep[r].commit); });
    o += "rep_dvc_recv |-> <<";
    for (int r = 0; r < R; r++) { if (r) o += ", "; set_of(f->rep[r].dvc_recv, f->rep[r].n_dvc); }
    o += ">>,\n";
    tuple_int("rep_last_normal_view", [&](int r) { return std::to_string(f->rep[r].lnv); });
    o += "rep_log |-> <<";
    for (int r = 0; r < R; r++) {
        if (r) o += ", ";
        o += "<<";
        for (int i = 0; i < f->rep[r].log_n; i++) { if (i) o += ", "; p.entry(f->rep[r].log[i]); }
        o += ">>";
    }
    o += ">>,\n";
    tuple_int("rep_op_number", [&](int r) { return std::to_string(f->rep[r].op); });
    o += "rep_peer_op_number |-> <<";
    for (int r = 0; r < R; r++) {
        if (r) o += ", ";
        o += "<<";
        for (int q = 0; q < R; q++) { if (q) o += ", "; o += std::to_string(f->rep[r].peer_op[q]); }
        o += ">>";
    }
    o += ">>,\n";
    tuple_int("rep_rec_number", [&](int r) { return std::to_string(f->rep[r].rec_number); });
    o += "rep_rec_recv |-> <<";
    for (int r = 0; r < R; r++) { if (r) o += ", "; set_of(f->rep[r].rec_recv, f->rep[r].n_rec); }
    o += ">>,\n";
    tuple_int("rep_sent_dvc", [&](int r) { return std::string(f->rep[r].sent_dvc ? "TRUE" : "FALSE"); });
    tuple_int("rep_sent_sv", [&](int r) { return std::string(f->rep[r].sent_sv ? "TRUE" : "FALSE"); });
    tuple_int("rep_status", [&](int r) { return std::string(kStatusNames[f->rep[r].status < 3 ? f->rep[r].status : 0]); });
    o += "rep_svc_recv |-> <<";
    for (int r = 0; r < R; r++) { if (r) o += ", "; set_of(f->rep[r].svc_recv, f->rep[r].n_svc); }
    o += ">>,\n";
    tuple_int("rep_view_number", [&](int r) { return std::to_string(f->rep[r].view); });
    o += "replicas |-> 1.." + std::to_string(R) + "\n";
    return o;
}

int copy_out(const std::string& s, char* buf, size_t cap) {
    if (s.size() + 1 > cap) return -(int)(s.size() + 1);
    memcpy(buf, s.c_str(), s.size() + 1);
    return (int)s.size();
}

} // namespace

/* ------------------------------------------------------------------ C ABI */

extern "C" {

const char* vsr_version(void) { return "vsr-b200-mc 0.1 (round 1)"; }
const char* vsr_action_name(int a) { return (a >= 0 && a < VSR_NUM_ACTIONS) ? kActionNames[a] : "?"; }

static int finish_load(VsrModel* m, const char* tla_path, VsrModel** out, char* err, size_t errcap) {
    std::string why;
    int rc = 0;
    if (tla_path && tla_path[0]) rc = verify_tla(tla_path, m, why);
    if (!rc) rc = bind_model(m, why);
    if (rc) {
        set_err(err, errcap, why);
        delete m;
        return rc;
    }
    *out = m;
    return 0;
}

int vsr_load_cfg_text(const char* cfg_text, const char* tla_path, VsrModel** out, char* err, size_t errcap) {
    if (!cfg_text || !out) return VSR_RC_ERROR;
    VsrModel* m = new VsrModel();
    memset(&m->info, 0, sizeof m->info);
    std::string why;
    int rc = parse_cfg(cfg_text, m, why);
    if (rc) {
        set_err(err, errcap, why);
        delete m;
        return rc;
    }
    return finish_load(m, tla_path, out, err, errcap);
}

int vsr_load(const char* cfg_path, const char* tla_path, VsrModel** out, char* err, size_t errcap) {
    if (!cfg_path) return VSR_RC_ERROR;
    std::ifstream f(cfg_path, std::ios::binary);
    if (!f) { set_err(err, errcap, std::string("cannot read config ") + cfg_path); return VSR_RC_CONFIG_ERROR; }
    std::stringstream ss;
    ss << f.rdbuf();
    return vsr_load_cfg_text(ss.str().c_str(), tla_path, out, err, errcap);
}

int vsr_model_create(int R, int C, int V, int L, int restart, int symmetry, int view, int invariant, VsrModel** out, char* err, size_t errcap) {
    if (!out) return VSR_RC_ERROR;
    VsrModel* m = new VsrModel();
    memset(&m->info, 0, sizeof m->info);
    m->check_deadlock_cfg = -1;
    VsrModelInfo& I = m->info;
    I.replica_count = R; I.client_count = C; I.value_count = V; I.start_view_on_timer_limit = L; I.restart_empty_limit = restart;
    I.symmetry = symmetry ? 1 : 0; I.view = view ? 1 : 0;
    I.invariant = invariant & ~(MODEL_PROPERTY_BIT | MODEL_HOOK_Q_BIT | MODEL_HOOK_INIT_EDGE_BIT | MODEL_MAJORITY_FIRST_BIT);
    I.property = (invariant & MODEL_PROPERTY_BIT) ? 1 : 0;
    static const int order[2][4] = {{1, 2, 4, 8}, {2, 1, 4, 8}};
    for (int b : order[(invariant & MODEL_MAJORITY_FIRST_BIT) ? 1 : 0])
        if (I.invariant & b) m->inv_order.push_back(b);
    m->live_hooks = ((invariant & MODEL_HOOK_Q_BIT) ? LIVE_HOOK_Q : 0) | ((invariant & MODEL_HOOK_INIT_EDGE_BIT) ? LIVE_HOOK_INIT_EDGE : 0);
    if (V < 1 || V > VSR_MAX_V) { set_err(err, errcap, "|Values| out of range"); delete m; return VSR_RC_CONFIG_ERROR; }
    for (int v = 0; v < V; v++) snprintf(I.value_names[v], sizeof I.value_names[v], "v%d", v + 1);
    return finish_load(m, nullptr, out, err, errcap);
}

void vsr_model_free(VsrModel* m) { delete m; }

int vsr_model_info(const VsrModel* m, VsrModelInfo* out) {
    if (!m || !out) return VSR_RC_ERROR;
    *out = m->info;
    out->check_deadlock = m->check_deadlock_cfg;
    return 0;
}

int vsr_init(const VsrModel* m, void* s) {
    m->ops->init((uint32_t*)s);
    return 0;
}

int vsr_successors(const VsrModel* m, const void* state, void* out, size_t cap, uint8_t* action_ids, uint32_t* mult) {
    const ModelOps* ops = m->ops;
    uint32_t tmp[VSR_MAX_STATE_BYTES / 4];
    int n = 0;
    for (int c = 0; c < ops->ncand; c++) {
        if (!ops->guard(&m->run, (const uint32_t*)state, c)) continue;
        int r = ops->step(&m->run, (const uint32_t*)state, c, tmp);
        if (r < 0) return r;
        if (r == 0) continue;
        if ((size_t)n < cap) {
            memcpy((char*)out + (size_t)n * ops->bytes, tmp, ops->bytes);
            if (action_ids) action_ids[n] = (uint8_t)ops->action_of(c);
            if (mult) mult[n] = (uint32_t)r;
        }
        n++;
    }
    return n;
}

int vsr_enabled_candidates(const VsrModel* m, const void* state, uint32_t* out, size_t cap) {
    /* Two forms of the same guards: one candidate at a time on the packed words (what vsr_successors and the kernel's
       apply step use), and all candidates of a group at once on a register copy of the state (what the kernel's scan
       uses).  Both are evaluated here and must agree; -100 says they do not (a bug in the lowering, never expected). */
    std::vector<uint32_t> fast((size_t)m->ops->ncand);
    const int nf = m->ops->enabled_list(&m->run, (const uint32_t*)state, fast.data());
    int n = 0;
    for (int c = 0; c < m->ops->ncand; c++) {
        if (!m->ops->guard(&m->run, (const uint32_t*)state, c)) continue;
        if (n >= nf || fast[(size_t)n] != (uint32_t)c) return -100;
        if ((size_t)n < cap) out[n] = (uint32_t)c;
        n++;
    }
    return n == nf ? n : -100;
}

int vsr_canon(const VsrModel* m, void* s) { return m->run.symmetry ? m->ops->canon((uint32_t*)s) : 0; }
uint64_t vsr_fingerprint(const VsrModel* m, const void* s) { return m->ops->fingerprint((const uint32_t*)s, m->run.use_view); }
uint64_t vsr_fingerprint_bytewise(const VsrModel* m, const void* s) { return m->ops->fingerprint_bytewise((const uint32_t*)s, m->run.use_view); }
uint32_t vsr_aux_key(const VsrModel* m, const void* s) { return m->ops->aux_key((const uint32_t*)s); }
int vsr_owner_rank(uint64_t fingerprint, int world) {
    if (world < 1 || world > 8 || (world & (world - 1))) return -1;
    int lg = 0;
    while ((1 << lg) < world) lg++;
    return vsr::owner_of(fingerprint ? fingerprint : 1, 64 - lg);
}
int vsr_invariant(const VsrModel* m, const void* s) { return m->ops->invariant(&m->run, (const uint32_t*)s); }
const char* vsr_reported_invariant(const VsrModel* m, const void* s) {
    const int bad = vsr_invariant(m, s);
    for (int b : m->inv_order)
        if (bad & b) return INVARIANT_NAMES[__builtin_ctz((unsigned)b)];
    return nullptr;
}
int vsr_property(const VsrModel* m, const void* s) { return m->ops->property(&m->run, (const uint32_t*)s, m->live_hooks); }
int vsr_unpack(const VsrModel* m, const void* s, VsrFlatState* out) { return m->ops->unpack((const uint32_t*)s, out); }
int vsr_pack(const VsrModel* m, const VsrFlatState* in, void* s) { return m->ops->pack(in, (uint32_t*)s, m->run.symmetry); }

int vsr_flat_to_tla(const VsrModel* m, const VsrFlatState* f, char* buf, size_t cap) { return copy_out(flat_to_tla(m, f), buf, cap); }

int vsr_state_to_tla(const VsrModel* m, const void* s, char* buf, size_t cap) {
    VsrFlatState* f = new VsrFlatState;
    int rc = m->ops->unpack((const uint32_t*)s, f);
    int n = rc < 0 ? rc : copy_out(flat_to_tla(m, f), buf, cap);
    delete f;
    return n;
}

int vsr_action_location(const VsrModel* m, int a, char* buf, size_t cap) {
    if (a < 0 || a >= VSR_NUM_ACTIONS) return VSR_RC_ERROR;
    return copy_out(m->action_location[a], buf, cap);
}

/* one random walk of simulation mode on the host: the walk `walk` of vsr_simulate(seed) exactly (same generator, same
   step function).  cands_out receives the chosen candidate indices; returns the number of transitions taken;
   *violated_at = depth (Init = 1) of the first state violating the invariant, 0 if none. */
int vsr_walk(const VsrModel* m, uint64_t seed, uint64_t walk, int depth, uint32_t* cands_out, int* violated_at) {
    const ModelOps* ops = m->ops;
    uint32_t cur[VSR_MAX_STATE_BYTES / 4], nxt[VSR_MAX_STATE_BYTES / 4];
    ops->init(cur);
    uint64_t rng = seed ^ (walk * 0xD1B54A32D192ED03ULL);
    int n = 0;
    if (violated_at) *violated_at = 0;
    for (int d = 2; d <= depth; d++) {
        const int c = ops->random_enabled(&m->run, cur, &rng);
        if (c < 0 || ops->step(&m->run, cur, c, nxt) <= 0) break;
        memcpy(cur, nxt, ops->bytes);
        if (cands_out) cands_out[n] = (uint32_t)c;
        n++;
        if (ops->invariant(&m->run, cur)) {
            if (violated_at) *violated_at = d;
            break;
        }
    }
    return n;
}

int vsr_replay_candidates(const VsrModel* m, const uint32_t* cands, int n, void* trace_out, uint8_t* trace_actions, size_t trace_cap) {
    /* The engine explores canonical representatives; like TLC, the reported trace is re-executed from
       Init so that consecutive states are literal steps of Next with fixed value names. */
    const ModelOps* ops = m->ops;
    RunCfg lit = m->run;
    lit.symmetry = 0;
    uint32_t cur[VSR_MAX_STATE_BYTES / 4], nxt[VSR_MAX_STATE_BYTES / 4];
    ops->init(cur);
    if (trace_cap >= 1) {
        memcpy(trace_out, cur, ops->bytes);
        trace_actions[0] = VSR_ACT_INIT;
    }
    for (int i = 0; i < n; i++) {
        const int c = m->run.symmetry ? ops->literal_cand(cur, (int)cands[i]) : (int)cands[i];
        if (c < 0) return -VSR_RC_ERROR;
        int r = ops->step(&lit, cur, c, nxt);
        if (r <= 0) return -VSR_RC_ERROR;
        memcpy(cur, nxt, ops->bytes);
        if ((size_t)(i + 1) < trace_cap) {
            memcpy((char*)trace_out + (size_t)(i + 1) * ops->bytes, cur, ops->bytes);
            trace_actions[i + 1] = (uint8_t)ops->action_of(c);
        }
    }
    return n + 1;
}

} /* extern "C" */
