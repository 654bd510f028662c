/*
 * vsr_oracle.h — CPU restatement of vsr-revisited/paper/VSR.tla (reference @ 7566e8af).
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may build, link
 * or run it, and there only as the checker or as the reported CPU baseline.
 *
 * PARITY STATUS: the algorithm on this path lives in TLC (tla2tools.jar), an external tool that
 * is neither vendored nor version-pinned by the reference and cannot run here (no JVM).  The only
 * golden vector the reference holds is state_transfer_violation_trace.txt (24 states): this oracle
 * is pinned to it (every transition replays through Next below, the final state violates
 * AcknowledgedWriteNotLost, and print_state() reproduces the file's text byte for byte apart from
 * `location` strings and three variables the file predates).
 * Second pin: the reference's own SOURCE TEXT.  oracle/tla_eval.py parses VSR.tla as it lies under
 * the reference (Vanlightly/vsr-tlaplus) and enumerates Init/Next the way TLC does; tests/test_spec_text.py compares it with
 * this file — complete state spaces level by level (cfg1 = BASELINE configs[0]: 76 distinct / 100
 * generated / depth 14, and eight more up to 697,364 states), successor sets state by state along the golden trace,
 * random walks on cfg2/cfg3/cfg4 constants, the recovery actions with RestartEmptyLimit 1 and 2, both
 * safety invariants, orbit counts under SYMMETRY: 0 differences (tests/golden/spec_text_results.json).
 * Still "parity unpinned": TLC's FINGERPRINT values (its value serialisation and model-value intern
 * order are TLC internals) and, for configurations too large for the text evaluator (cfg2's complete
 * 1.17e9-state space, cfg3), the totals — there this oracle is the reference, with that caveat.
 *
 * Value model: records are C++ structs spelled out field by field, sets are ordered std::set,
 * the message bag is an ordered std::map record -> pending count — no bit packing, no slot
 * assumptions, so that it is an independent check of the packed product encoding.
 */
#ifndef VSR_ORACLE_H
#define VSR_ORACLE_H

#include <cstdint>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../include/vsr_flat.h"

namespace orc {

constexpr int ABSENT = -1; /* field not in this record shape */
constexpr int NIL = -2;    /* the model value Nil */

struct Params {
    int R = 3, C = 1, V = 2, L = 2, restart_limit = 0; /* VSR.cfg:4-8 */
    bool symmetry = true;                              /* SYMMETRY symmValues, VSR.cfg:31 */
    bool use_view = true;                              /* VIEW view, VSR.cfg:29 */
    int invariant = 1; /* 1 AcknowledgedWriteNotLost, 2 AcknowledgedWritesExistOnMajority,
                          3 NoLogDivergence, 4 TestInv, 0 none (VSR.tla:926-952) */
};

/* LogEntryType, VSR.tla:157-161 */
struct Entry {
    int view = 0, operation = 0, client = 0, req = 0;
};
int cmp_entry(const Entry& a, const Entry& b);

/* any message record; shapes at VSR.tla:163-225, GetState :510-514, NewState :533-541 */
struct Msg {
    int type = 0;
    int view = ABSENT, src = ABSENT, dest = ABSENT, op = ABSENT, commit = ABSENT, lnv = ABSENT,
        first_op = ABSENT, x = ABSENT;
    bool has_entry = false;
    Entry entry;
    int has_log = 0; /* 0 none, 1 function on log_lo.., 2 Nil */
    int log_lo = 1;
    std::vector<Entry> log;
};
int cmp_msg(const Msg& a, const Msg& b); /* TLC RecordValue order (SURVEY App. B.3) */
struct MsgLess {
    bool operator()(const Msg& a, const Msg& b) const { return cmp_msg(a, b) < 0; }
};
typedef std::set<Msg, MsgLess> MsgSet;
typedef std::map<Msg, int, MsgLess> MsgBag;

struct ClientRow {
    int req = 0, op = 0;
    bool executed = true;
};

/* the 20 VARIABLES of VSR.tla:119-138 (replicas = 1..R and clients = 1..C are implicit) */
struct State {
    std::vector<int> status, view, op, commit, lnv, rec_number; /* index r-1 */
    std::vector<char> sent_dvc, sent_sv;
    std::vector<std::vector<Entry>> log;
    std::vector<std::vector<int>> peer_op;
    std::vector<std::vector<ClientRow>> client_table;
    std::vector<MsgSet> svc_recv, dvc_recv, rec_recv;
    MsgBag messages;
    int aux_svc = 0, aux_restart = 0;
    std::map<int, bool> acked; /* aux_client_acked */
};

struct Succ {
    State s;
    int action; /* VSR_ACT_* */
};

/* counters for reasoning the product relies on; all must stay 0 on the explored space */
struct Assumptions {
    uint64_t bag_count_gt1 = 0;         /* some messages[m] > 1 */
    uint64_t op_ne_loglen = 0;          /* rep_op_number[r] # Len(rep_log[r]) */
    uint64_t recv_view_mismatch = 0;    /* element of rep_svc_recv/rep_dvc_recv[r] with view # View(r) */
    uint64_t dup_value_in_log = 0;      /* a value twice in one log / log longer than |Values| */
    uint64_t entry_not_unique = 0;      /* two different LogEntry records for one value anywhere */
    uint64_t choose_tie_diff_logs = 0;  /* HighestLog CHOOSE tie between DVCs with different logs */
    uint64_t prepare_key_clash = 0;     /* two created values share (view, op_number) of their Prepare */
    uint64_t slot_clash = 0;            /* two messages the slot encoding would put in one slot */
    uint64_t view_gt_max = 0;           /* a view number above 1 + StartViewOnTimerLimit */
};

State init_state(const Params& p);                                           /* VSR.tla:323-348 */
void successors(const Params& p, const State& s, std::vector<Succ>& out,
                Assumptions* as = nullptr);                                  /* Next, VSR.tla:896-918 */
bool invariant_holds(const Params& p, const State& s);                       /* VSR.tla:926-952 */
void check_assumptions(const Params& p, const State& s, Assumptions& as);

int cmp_state(const State& a, const State& b, bool with_aux);   /* declaration order, VSR.tla:119-138 */
State permute(const State& s, const std::vector<int>& perm);    /* perm[v-1] = image of value v */
State canonical(const Params& p, const State& s);               /* min over symmValues (VSR.tla:151) */

/* label-independent key of the three aux variables used to break same-level VIEW ties (DESIGN.md §H2) */
uint32_t aux_key(const Params& p, const State& s);

/* byte serialisation (exact, self-delimiting) and a 128-bit digest of it */
void serialize(const State& s, bool with_aux, std::string& out);
State deserialize(const Params& p, const std::string& in);
void digest128(const std::string& bytes, uint64_t out[2]);

void to_flat(const Params& p, const State& s, VsrFlatState* f);
State from_flat(const VsrFlatState* f);

/* TLC "dumpTrace tlc" text (format of state_transfer_violation_trace.txt) */
std::string print_state(const Params& p, const State& s, bool with_rec_vars = true);
std::string print_trace_entry(const Params& p, const State& s, int position, const char* action_name,
                              const char* location, bool with_rec_vars);
struct TraceState {
    int position;
    std::string action_name, location;
    State s;
    std::vector<std::string> var_names; /* as listed in the file */
};
/* returns "" on success, else an error message */
std::string parse_trace_text(const std::string& text, Params& p_out, std::vector<TraceState>& out);

const char* action_name(int a);

struct BfsOptions {
    int workers = 1;
    int max_depth = 0;          /* 0 = unbounded; TLC depth counting: Init is depth 1 */
    uint64_t max_states = 0;    /* stop after the level that crosses this many distinct states */
    double max_seconds = 0;     /* stop after the level that crosses this much wall time */
    bool stop_on_violation = true;
    bool check_deadlock = false; /* TLC's default is true; VSR has reachable terminal states (SURVEY §5) */
    std::string level_digest_path; /* if set: binary file of per-level sorted 16-byte digests */
    bool keep_trace = true;
    bool check_assumptions = true;
};
struct BfsResult {
    uint64_t generated = 0, distinct = 0, queue = 0;
    int depth = 0;              /* TLC convention: Init = 1 */
    int rc = 0;                 /* 0 ok, 12 invariant violated, 11 deadlock */
    bool complete = false;
    std::vector<uint64_t> level_sizes;     /* distinct states first seen at depth i+1 */
    std::vector<uint64_t> level_generated; /* successors generated while expanding depth i+1 */
    uint64_t h2_ties = 0;       /* same level, same view key, different aux */
    Assumptions as;
    double seconds = 0;
    std::vector<std::pair<int, State>> trace; /* (action, state) from Init to the violating state */
};
BfsResult bfs(const Params& p, const BfsOptions& o);

} // namespace orc
#endif
