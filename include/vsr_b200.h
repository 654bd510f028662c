/*
 * vsr_b200.h — C ABI of the H100-native explicit-state model checker for
 * vsr-revisited/paper/VSR.tla (reference: Vanlightly/vsr-tlaplus @ 7566e8af).
 *
 * What this replaces.  The reference has no plugin/operator ABI: TLA+ has no FFI and the path
 * "model-check VSR.tla under VSR.cfg" is executed by the external TLC tool
 *     java -cp tla2tools.jar tlc2.TLC [-deadlock] [-workers N] [-fp N] [-dumpTrace tlc F] -config VSR.cfg VSR.tla
 * so the drop-in boundary is TLC's file + CLI surface (SURVEY §8b).  Each entry point below cites
 * the part of the reference it stands in for.  Plain pointers and sizes; caller owns every buffer;
 * no torch / C++ types.  Return codes follow TLC's exit statuses where one exists:
 *     0 ok, 11 deadlock, 12 safety (invariant) violation, 13 temporal property violated, 150 spec error, 151 config error,
 *     152 state space too large for the configured capacity, 153 system (CUDA) error, 255 other.
 */
#ifndef VSR_B200_H
#define VSR_B200_H

#include <stddef.h>
#include <stdint.h>

#include "vsr_flat.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VSR_RC_OK 0
#define VSR_RC_DEADLOCK 11
#define VSR_RC_VIOLATION 12
#define VSR_RC_LIVENESS 13
#define VSR_RC_SPEC_ERROR 150
#define VSR_RC_CONFIG_ERROR 151
#define VSR_RC_TOO_LARGE 152
#define VSR_RC_SYSTEM 153
#define VSR_RC_ERROR 255

#define VSR_MAX_STATE_BYTES 256

typedef struct VsrModel VsrModel; /* opaque: parsed config + selected packed layout */

typedef struct VsrModelInfo {
    int32_t replica_count, client_count, value_count;   /* VSR.cfg:4-6 */
    int32_t start_view_on_timer_limit, restart_empty_limit; /* VSR.cfg:7-8 */
    int32_t symmetry, view;                             /* SYMMETRY symmValues / VIEW view present (VSR.cfg:29,31) */
    int32_t invariant;                                  /* bitmask of INVARIANT names (VSR.cfg:36-39): 1 AcknowledgedWriteNotLost
                                                           2 AcknowledgedWritesExistOnMajority 4 NoLogDivergence 8 TestInv */
    int32_t state_bytes;                                /* size of one packed state */
    int32_t state_bits;                                 /* bits in use */
    int32_t num_candidates;                             /* (action, binding) pairs tried per state */
    int32_t spec_verified;                              /* 1 if a .tla was given and matched VSR.tla's structure */
    uint64_t spec_hash;                                 /* FNV-1a 64 of the .tla bytes (0 if none) */
    char value_names[VSR_MAX_V][32];                    /* model values of Values, cfg order */
    int32_t check_deadlock;                             /* CHECK_DEADLOCK in the cfg: 1 TRUE, 0 FALSE, -1 absent (TLC's default: check) */
    int32_t property;                                   /* bitmask of PROPERTY names: 1 ViewChangeCompletes (VSR.tla:964-965; needs
                                                           SPECIFICATION Spec, whose WF_vars(Next) makes it meaningful) */
} VsrModelInfo;

/* ---- loading: TLC's `-config VSR.cfg VSR.tla` (SURVEY §8b; grammar of vsr-revisited/paper/VSR.cfg:1-39).
 * tla_path may be NULL (the spec is hand-lowered; when given, it is verified to BE VSR.tla: module
 * name :1, the 20 VARIABLES :119-138, the 19 disjuncts of Next :896-918).  On failure returns
 * 150/151 and writes a message to err.
 * Constants: ReplicaCount 2..7, |Values| 1..7, StartViewOnTimerLimit 0..14, ClientCount 1, RestartEmptyLimit 0.  The
 * packed layouts of the reference's configurations and their neighbours are built in; any other combination is
 * compiled on first use into <library dir>/layouts/ (needs nvcc, 20 s to a minute; VSR_B200_JIT=0 turns that into a
 * 151).  Only StartViewOnTimerLimit up to the value in this table builds; a larger one is a 151 naming the limit it
 * exceeds (packed state over VSR_MAX_STATE_BYTES, or an action group over the expand kernel's 16-bit pool item):
 * | ReplicaCount | \|Values\| = 1 | 2 | 3 | 4 | 5 | 6 | 7 |
 * |---|---|---|---|---|---|---|---|
 * | 2 | 14 | 14 | 14 | 14 | 14 | 14 | 12 |
 * | 3 | 10 | 10 | 10 | 10 | 8 | 7 | 6 |
 * | 4 | 5 | 5 | 5 | 5 | 5 | 4 | 4 |
 * | 5 | 3 | 3 | 3 | 3 | 3 | 3 | 2 |
 * | 6 | 2 | 2 | 2 | 2 | 2 | - | - |
 * | 7 | 1 | 1 | 1 | - | - | - | - |
 */
int vsr_load(const char* cfg_path, const char* tla_path, VsrModel** out, char* err, size_t errcap);
/* same, from the text of a cfg file */
int vsr_load_cfg_text(const char* cfg_text, const char* tla_path, VsrModel** out, char* err, size_t errcap);
/* same, straight from constants (CONSTANTS of VSR.tla:92-96).  `invariant` is the INVARIANT bitmask of VsrModelInfo, plus
 * bits only this entry point knows: 512 = check PROPERTY ViewChangeCompletes (as a cfg with SPECIFICATION Spec does); test
 * hooks of the liveness pass, which leave the BFS as it is: 1024 = the pass checks []<>Q with Q = "some replica's
 * rep_commit_number >= 1" instead (reachable not-Q states without successors exist), 2048 = in the pass every state
 * without successors gets one extra successor, Init (with 1024: cycles through Init); 4096 = the INVARIANT list names
 * AcknowledgedWritesExistOnMajority before AcknowledgedWriteNotLost (otherwise the list is in bit order), which decides
 * the name vsr_reported_invariant gives a state that violates both.  Test hook 256: the invariant "no replica has
 * committed every value", reported in the masks as 256 (vsr_reported_invariant does not name it) */
int vsr_model_create(int replica_count, int client_count, int value_count, int start_view_on_timer_limit,
                     int restart_empty_limit, int symmetry, int view, int invariant, VsrModel** out, char* err,
                     size_t errcap);
void vsr_model_free(VsrModel* m);
int vsr_model_info(const VsrModel* m, VsrModelInfo* out);

/* ---- single-state operations on packed states (host; re-entrant).  A packed state is
 * info.state_bytes bytes, 16-byte aligned. */
int vsr_init(const VsrModel* m, void* state_out);                        /* Init, VSR.tla:323-348 */
/* Next, VSR.tla:896-918: writes up to cap successors (state_bytes apart) in TLC's binding order,
 * action_ids[i] = VSR_ACT_*, mult[i] = TLC bindings that successor stands for; returns the number
 * of successors, or a negative E_* code if one cannot be represented. */
int vsr_successors(const VsrModel* m, const void* state, void* out, size_t cap, uint8_t* action_ids, uint32_t* mult);
/* candidate (action, binding) indices whose guard holds in `state`, in the order vsr_successors emits them.  Evaluates the
 * guards in both of their forms (one candidate at a time, and the register-mask form of the GPU scan); -100 if they
 * ever disagree */
int vsr_enabled_candidates(const VsrModel* m, const void* state, uint32_t* out, size_t cap);
int vsr_canon(const VsrModel* m, void* state);                           /* SYMMETRY representative, VSR.tla:151 */
uint64_t vsr_fingerprint(const VsrModel* m, const void* state);          /* FP64 of the VIEW projection, VSR.tla:149-150 */
/* the same fingerprint by its byte-at-a-time definition (vsr_fingerprint and the GPU use the slicing-by-8 form) */
uint64_t vsr_fingerprint_bytewise(const VsrModel* m, const void* state);
uint32_t vsr_aux_key(const VsrModel* m, const void* state);
/* rank (GPU) that owns a fingerprint when the state space is sharded over `world` = 1, 2, 4 or 8 ranks: the high bits of
 * fingerprint x an odd constant (FP64 is GF(2)-linear: its own high bits would route a rank's successors to a few peers only) */
int vsr_owner_rank(uint64_t fingerprint, int world);
/* invariants, VSR.tla:926-952: the mask of the configured INVARIANT bits the state violates (0 = all hold), all of them */
int vsr_invariant(const VsrModel* m, const void* state);
/* the invariant TLC names for the state ("Error: Invariant X is violated."): the first of the config's INVARIANT list, in
 * its order, that the state violates; NULL if it violates none */
const char* vsr_reported_invariant(const VsrModel* m, const void* state);
/* 1 if the state predicate the liveness pass checks holds in `state`: AllReplicasMoveToSameView (VSR.tla:958-962), or the
 * test hook's Q (vsr_model_create bit 1024); 0 if not */
int vsr_property(const VsrModel* m, const void* state);
int vsr_unpack(const VsrModel* m, const void* state, VsrFlatState* out);
int vsr_pack(const VsrModel* m, const VsrFlatState* in, void* state_out);
/* TLC value text of one state, format of state_transfer_violation_trace.txt (variables
 * alphabetical, records in first-interned field order); returns length or -needed. */
int vsr_state_to_tla(const VsrModel* m, const void* state, char* buf, size_t cap);
int vsr_flat_to_tla(const VsrModel* m, const VsrFlatState* f, char* buf, size_t cap);
const char* vsr_action_name(int action_id);
/* "line A, col B to line C, col D of module VSR" for an action when a .tla was loaded, else "Unknown location" */
int vsr_action_location(const VsrModel* m, int action_id, char* buf, size_t cap);

/* ---- the BFS (TLC's worker loop; SURVEY §3.1, stages E1-E9) on the GPU */
#define VSR_MAX_LEVELS 512
/* Action coverage, TLC's `-coverage`: per action of Next (VSR_ACT_*; 0 = the initial predicate) and per BFS level d
 * (depth of the SUCCESSOR, Init = 1; row d - 1):
 *   generated  sum of mult over the successors produced by a binding of that action: TLC's "states generated", one per
 *              binding.  Deterministic, and the same for every number of GPUs.
 *   distinct   states whose first arrival in the seen-set came through that action (after a same-level VIEW tie was
 *              resolved with parent records kept: the surviving arrival's action, as in the trace).  A state reachable
 *              in one level through two actions goes to whichever insert won, so the split over actions may differ
 *              from run to run; its sum per level is the level's size.
 * num_levels = rows in use: a complete run whose deepest level has successors has depth + 1, the last one holding those
 * successors, all of them seen before.  Counted by the expand kernel where a state is inserted, on the GPU that owns it. */
typedef struct VsrCoverage {
    uint64_t generated[VSR_NUM_ACTIONS], distinct[VSR_NUM_ACTIONS];
    int32_t num_levels, _pad;
    uint64_t level_generated[VSR_MAX_LEVELS][VSR_NUM_ACTIONS], level_distinct[VSR_MAX_LEVELS][VSR_NUM_ACTIONS];
} VsrCoverage;

typedef struct VsrRunOpts {
    int32_t device;              /* CUDA device ordinal */
    int32_t check_deadlock;      /* TLC default is on; `-deadlock` turns it off.  Here default 0 (VSR has terminal states) */
    int32_t max_depth;           /* TLC `-depth`-like bound for BFS (0 = none) */
    int32_t stop_on_violation;   /* 1: stop at the first violating level (TLC behaviour) */
    int32_t keep_trace;          /* 1: keep (parent, binding) per distinct state so a counterexample can be rebuilt */
    int32_t verbose;
    uint64_t table_capacity;     /* seen-set slots (any number, rounded up to 64; 0 = auto from free memory) */
    uint64_t frontier_capacity;  /* states per frontier buffer (0 = auto) */
    uint64_t max_states;         /* stop after the level that crosses this many distinct states (0 = none) */
    double max_seconds;          /* stop after the level that crosses this much time (0 = none) */
    int32_t collect_levels;      /* 1: keep every level's states on the host (tests) */
    int32_t _reserved0;
    /* frontier spill (BASELINE configs[3], "spill to pinned host DRAM"): each of the two frontier buffers continues, after
       its frontier_capacity states in HBM, with this many states in pinned host memory mapped into the device; the kernels
       write and read that part over PCIe / C2C.  0 = no spill: a level that does not fit is a 152. */
    uint64_t frontier_host_capacity;
    /* checkpoint / recover: TLC's `-checkpoint <minutes>` and `-recover <dir>` (the reference's .gitignore:1 ignores TLC's
       states/ metadir, i.e. its users run with checkpoints).  checkpoint_path: file written at the first level boundary after
       checkpoint_seconds since the last one (0 = after every level; written to <path>.tmp and renamed, so an interrupted write
       leaves the previous checkpoint intact); recover_path: continue the BFS from the checkpoint at that base path instead of
       Init (vsr_engine_recover).  With several ranks every rank writes <path>.rank<r>.  NULL = off. */
    const char* checkpoint_path;
    const char* recover_path;
    double checkpoint_seconds;
    /* seen-set host tier (delayed duplicate detection): at a level boundary where the HBM seen-set's resident entries pass a
       load threshold, the entries of levels older than the current frontier move, unchanged, to an append-only array of up
       to this many 16-byte entries in pinned host memory, and the table is rebuilt from the rest.  A successor equal to a
       moved state is first inserted as new; after the level, one pass streams the tier against the table and the level's
       rows are compacted, so totals, levels, traces and verdicts are those of a run with the whole seen-set in HBM.  Each
       rank has its own tier.  0 = off: the seen-set is the HBM table alone.  Refused (151) together with checkpoint_path /
       recover_path: the tier is not part of a checkpoint. */
    uint64_t table_host_capacity;
    /* action coverage: NULL = off (the kernels are launched without the counters).  Else the BFS counts, and
       vsr_bfs_sharded (vsr_bfs, vsr_bfs_multi) writes the job's totals here when it returns, however the run ended; an
       engine created with it set counts in the stepwise interface too (vsr_engine_coverage).  Refused (151) together
       with checkpoint_path / recover_path: the counters are not in the checkpoint file. */
    VsrCoverage* coverage;
} VsrRunOpts;

typedef struct VsrStats {
    uint64_t generated, distinct, queue;  /* TLC's "N states generated, M distinct states found, Q left on queue" */
    int32_t depth;                        /* TLC's "depth of the complete state graph search" (Init = 1) */
    int32_t rc;
    int32_t complete;
    int32_t num_levels;
    uint64_t level_sizes[VSR_MAX_LEVELS];
    uint64_t level_generated[VSR_MAX_LEVELS];
    double level_ms[VSR_MAX_LEVELS];      /* device time of each level's kernels (CUDA events) */
    uint64_t h2_ties;                     /* same-level VIEW ties with different aux variables */
    uint64_t fp_collisions;               /* equal 64-bit fingerprints told apart by the check hash */
    uint64_t probe_total;                 /* table slots inspected */
    uint64_t kernel_launches;
    double seconds_total, seconds_kernels;
    int32_t violation_level;              /* depth of the violating state */
    int32_t trace_len;
    int32_t error_code;                   /* first E_* raised on the device (0 = none) */
    int32_t violation_mask;               /* every INVARIANT bit the reported state violates (vsr_invariant; 0 = none reported) */
    uint64_t violation_id;
    uint64_t table_capacity, frontier_capacity;
    uint64_t bytes_table, bytes_frontier;
    uint64_t bytes_h2d, bytes_d2h;         /* host<->device bytes moved by the engine (inputs, per-level counters, trace reads) */
    double seconds_setup;                 /* engine creation: allocation + clearing the seen-set */
    uint64_t records_sent, records_received; /* several GPUs: records this rank pushed to / drained from peers */
    double seconds_insert;                /* several GPUs: part of seconds_kernels spent in drain-only launches */
    int32_t levels_expanded;              /* frontiers expanded = valid entries of level_generated / level_ms */
    int32_t trace_loop;                   /* rc 13: the lasso's "Back to state K" (1-based; 0 = it ends in stuttering) */
    /* seen-set host tier (table_host_capacity > 0; summed over the ranks, times of the slowest rank per level) */
    uint64_t host_entries;                /* seen-set entries moved to pinned host memory (each moves once, at one boundary) */
    uint64_t host_false_new;              /* states first inserted as new that the tier pass found in host memory, removed */
    double seconds_host_pass, seconds_host_compact, seconds_host_evict; /* tier passes, level compactions, evictions */
} VsrStats;

typedef struct VsrEngine VsrEngine;

/* One-call BFS on one GPU: engine creation (stats.seconds_setup), vsr_bfs_sharded on that world-1 engine, then, when the
 * model has a property and the BFS completed, vsr_engine_liveness (rc 13: the trace is the lasso, stats.trace_loop its
 * back edge), teardown.
 * Fails loudly (153) when no CUDA device is usable — there is no CPU fallback.  If trace_out != NULL and a
 * violation/deadlock is found, writes the counterexample (packed states, trace_cap capacity) with its action ids;
 * stats.trace_len is its length, stats.violation_mask the invariants its last state violates (all of them: the one TLC
 * names is vsr_reported_invariant of that state). */
int vsr_bfs(const VsrModel* m, const VsrRunOpts* opts, VsrStats* stats, void* trace_out, uint8_t* trace_actions,
            size_t trace_cap);

/* Stepwise engine (what vsr_bfs_sharded, and through it vsr_bfs and vsr_bfs_multi, is made of).
 * rank/world: this engine owns the fingerprints f with owner(f) == rank (world = 1, 2, 4 or 8: the high bits of f). */
int vsr_engine_create(const VsrModel* m, const VsrRunOpts* opts, int rank, int world, VsrEngine** out, char* err,
                      size_t errcap);
void vsr_engine_destroy(VsrEngine* e);
/* bytes of one record that travels between ranks or into vsr_engine_insert_records: the packed state, then
 * { uint64 fingerprint; uint64 parent global id << 12 | candidate index | mult << 56 } */
int vsr_engine_record_bytes(const VsrEngine* e);
int vsr_engine_seed_init(VsrEngine* e);                       /* inserts Init if this rank owns it */
/* one launch of the wavefront kernel over the whole current frontier (world = 1: that is the level) */
int vsr_engine_expand(VsrEngine* e);
/* same for frontier states [first, first + count) only */
int vsr_engine_expand_part(VsrEngine* e, uint64_t first, uint64_t count);
/* world > 1, one step = one launch: expand frontier states [first, first + count) — successors owned here are inserted,
 * the others are stored into their owners' inboxes (half `parity` of the double buffer) by the kernel itself — then insert
 * the records the peers stored HERE in the previous step: drain_counts[s] from rank s (NULL = none).  sent_out[d] = records
 * this launch pushed to rank d (tell rank d: it is its drain_counts[this rank] of the next step).  Returns after the
 * kernel has completed, i.e. after the pushed records have landed. */
int vsr_engine_step(VsrEngine* e, uint64_t first, uint64_t count, int parity, const uint32_t* drain_counts, uint32_t* sent_out);
/* inserts n records (device pointer, 16-byte aligned, layout above; n <= UINT32_MAX) as states of the level being
 * generated: one launch of the wavefront kernel with no frontier share that drains them, i.e. the insert every successor
 * of the BFS goes through (vsr_engine_seed_init inserts Init the same way).  Tests inject records here. */
int vsr_engine_insert_records(VsrEngine* e, const void* dev_records, uint64_t n);
/* finishes the level: resolves ties, swaps frontiers; writes this rank's level numbers */
typedef struct VsrLevelInfo {
    uint64_t new_states, generated, frontier_in, ties, collisions;
    int32_t violation, deadlock, error_code, overflow;
    uint64_t violation_id, deadlock_id;
    double ms;        /* kernel time of the level on this rank (expand + insert), CUDA events on the launch stream */
    double ms_insert; /* of which launches that only inserted records received from peers */
    int32_t violation_mask, _pad; /* OR over the level's new states of the INVARIANT bits each violates (vsr_invariant) */
    /* seen-set host tier (table_host_capacity > 0): entries held after this boundary, this level's states removed because
       the tier already held them (new_states excludes them), entries moved at this boundary, and the host clock of the
       tier pass, the level's compaction and the eviction (each ends in a stream synchronise) */
    uint64_t host_entries, false_new, evicted;
    double ms_host_pass, ms_host_compact, ms_host_evict;
} VsrLevelInfo;
int vsr_engine_finish_level(VsrEngine* e, VsrLevelInfo* out);
uint64_t vsr_engine_frontier_size(const VsrEngine* e);
/* copies `n` states of the current frontier starting at `first` to a host buffer */
int vsr_engine_read_frontier(VsrEngine* e, uint64_t first, uint64_t n, void* host_out);
/* trace record of a locally owned state id: parent global id (rank << 40 | local id; 2^44 - 1 = none: Init) and candidate index */
int vsr_engine_trace_record(VsrEngine* e, uint64_t local_id, uint64_t* parent_out, uint32_t* cand_out);
int vsr_engine_stats(const VsrEngine* e, VsrStats* out);
/* membership query: *level_out = BFS depth at which `state` (a canonical packed state) was first seen, 0 if it is not
 * in this rank's shard of the seen-set (the HBM table, then the host tier); *owner_out = the rank owning its fingerprint */
int vsr_engine_lookup(VsrEngine* e, const void* state, int* level_out, int* owner_out);
/* Checkpoint of this rank's shard at a level boundary (after vsr_engine_finish_level, before the next expansion): the
 * current frontier, every seen-set entry {fingerprint, meta}, the trace records and the run's statistics, to one file.
 * vsr_engine_recover loads this rank's share of the checkpoint at base path `path` into a fresh (or reset) engine of the
 * same model: <path> when one rank wrote it, <path>.rank0 ... <path>.rank<W_old - 1> when W_old ranks did (both present:
 * the one of this engine's world; 151 when neither is).  W_old and the engine's world may differ (1, 2, 4 or 8): the rank
 * checks the header of every old file and reads the bulk of only those that hold its share — its own file in the same world,
 * so a world-1 engine loads <path> as it always has.  The seen-set is re-inserted entry by entry, so its capacity may
 * differ from the one the checkpoint was written with.  `totals` (may be NULL) travels with the file: vsr_bfs_sharded
 * stores the job's running totals there.  150 = not a checkpoint of this model, or files that are not one checkpoint;
 * 152 = this rank's share does not fit; 153 = a file cannot be opened. */
int vsr_engine_checkpoint(VsrEngine* e, const char* path, const VsrStats* totals);
int vsr_engine_recover(VsrEngine* e, const char* path, VsrStats* totals_out);
/* forget everything explored (clears the seen-set, keeps the allocations): ready for seed_init again */
int vsr_engine_reset(VsrEngine* e);
const char* vsr_engine_last_error(const VsrEngine* e);
/* THIS rank's action coverage of the levels finished so far (engines created with opts.coverage set; else 151) */
int vsr_engine_coverage(const VsrEngine* e, VsrCoverage* out);
/* with opts.collect_levels: number of states first seen at depth `level` (1-based) and, if host_out has room, a copy */
uint64_t vsr_engine_collected(const VsrEngine* e, int level, void* host_out, uint64_t cap_states);
/* Audit of the level just finished (tests): one device pass over this rank's seen-set and current frontier.
 * tagged = seen-set entries whose level tag is `level`; found = frontier states whose (VIEW fingerprint, check hash) is in
 * the seen-set with that tag; the digests are order-independent: sum and xor of mix64(VIEW fingerprint), and of a hash
 * of all the state's words; tagged_fp_* are the same fingerprint digests over the tagged seen-set entries.  A correct level
 * has found == tagged == size and equal fingerprint digests on both sides (a state written twice and another not at all
 * keep the counts but not the digests). */
typedef struct VsrLevelAudit {
    uint64_t size, tagged, found;
    uint64_t fp_sum, fp_xor, words_sum, words_xor;
    uint64_t tagged_fp_sum, tagged_fp_xor;
    int32_t level, _pad;
} VsrLevelAudit;
int vsr_engine_audit_level(VsrEngine* e, VsrLevelAudit* out);
/* the expand kernel's shape for this model's layout (no GPU needed): warps per block, blocks per SM, scan passes per
 * round, staging rows per warp */
int vsr_expand_shape(const VsrModel* m, int* warps, int* blocks, int* passes, int* stage_rows);
/* Rebuild the behaviour from Init to local state id (world-1 engines; tests): the parent-chain walk of vsr_bfs_sharded,
 * replayed with vsr_replay_candidates.  Returns the number of states, or a negative status. */
int vsr_engine_build_trace(VsrEngine* e, uint64_t local_id, void* trace_out, uint8_t* trace_actions, size_t trace_cap);

/* ---- liveness: PROPERTY ViewChangeCompletes == []<>P under Spec's WF_vars(Next), P = AllReplicasMoveToSameView (DESIGN
 * "Liveness").  When the model has the property, every finished level appends its not-P states to a store (words in HBM,
 * continued in pinned host memory) and to a live index {fingerprint, check} -> store index.  After a COMPLETE BFS,
 * vsr_engine_liveness sweeps the store deepest level first, keeping a state alive while some not-P successor other than
 * itself is alive, until a sweep removes nothing.  The property is violated iff a not-P state has no successor but itself
 * (stuttering forever is fair there) or some state stays alive (a not-P cycle).  One GPU (world 1) only. */
#define VSR_MAX_SWEEPS 64
typedef struct VsrLiveStats {
    uint64_t stored;               /* not-P states in the store (all levels) */
    uint64_t capacity;             /* states the store holds */
    uint64_t bytes_hbm, bytes_host; /* store, live index and alive bits in HBM; the store's continuation in host memory */
    uint64_t sinks;                /* not-P states without a successor other than themselves (first sweep) */
    uint64_t survivors;            /* states alive after the last sweep */
    uint64_t violation_index;      /* store index of the reported state (the smallest sink, else the smallest survivor) */
    int32_t sweeps;                /* full passes over the store, the last of which removed nothing (or found sinks) */
    int32_t rc;                    /* 0 holds, 13 violated, else an error status */
    int32_t violation_level;       /* BFS depth of the reported state */
    int32_t trace_loop;            /* "Back to state K" of the lasso (1-based); 0 = the lasso ends in stuttering */
    int32_t trace_loop_action;     /* VSR_ACT_* of the step back to state K (0 = the test hook's edge to Init) */
    int32_t trace_len;             /* candidates written to cands_out (the lasso has trace_len + 1 states; 0 = none kept) */
    int32_t error_code;            /* E_* raised by a sweep (0 = none) */
    int32_t _pad;
    double seconds_total;          /* the whole liveness phase (sweeps and the lasso walk) */
    double ms_sweep[VSR_MAX_SWEEPS]; /* device time of each sweep (CUDA events) */
} VsrLiveStats;
/* After vsr_bfs_sharded returned 0 with stats.complete on a world-1 engine of a model with a property: the sweeps and, on a
 * violation, the lasso as a candidate chain from Init (cands_out[0 .. trace_len), replay with vsr_replay_candidates) whose
 * last state steps back to state trace_loop (or stutters).  Returns 0 (holds), 13 (violated), 255 (the store disagrees with
 * the BFS: stats.error_code), 151 (no property / not a complete one-GPU run) or 153. */
int vsr_engine_liveness(VsrEngine* e, VsrLiveStats* stats, uint32_t* cands_out, size_t cands_cap);

/* ---- several GPUs of one node (SURVEY §8e: TLC's `-workers` / distributed mode).  One rank per GPU — processes
 * (torchrun) or threads of one process — fingerprint space split by its high bits.  The ranks coordinate through a
 * VsrGroup: a block of shared memory with a barrier and an all-gather of one small message per rank (a few per wavefront,
 * about a microsecond each).  The states do not pass through it: expand_kernel stores a successor owned by a peer straight
 * into that peer's inbox over NVLink (CUDA IPC mapping / peer access) and the peer inserts it in its next launch. */
typedef struct VsrGroup VsrGroup;
#define VSR_GROUP_MSG_BYTES 256
/* processes: `name` is a POSIX shared-memory name ("/vsr-<job>") every rank of the job passes and nobody else uses; rank 0
 * creates it, the others wait for it up to timeout_s; the name is unlinked once all have attached */
int vsr_group_open(const char* name, int rank, int world, double timeout_s, VsrGroup** out, char* err, size_t errcap);
/* threads of one process: `world` handles on one heap block */
int vsr_group_open_local(int world, VsrGroup** out_handles);
void vsr_group_close(VsrGroup* g);
int vsr_group_barrier(VsrGroup* g);                                  /* 0, or 153 when a rank aborted / timed out */
int vsr_group_allgather(VsrGroup* g, const void* mine, size_t bytes, void* all_out); /* bytes <= VSR_GROUP_MSG_BYTES */
void vsr_group_abort(VsrGroup* g);                                   /* make every pending and future wait fail */
void vsr_group_set_timeout(VsrGroup* g, double seconds);
int vsr_group_rank(const VsrGroup* g);
int vsr_group_world(const VsrGroup* g);
const char* vsr_group_last_error(const VsrGroup* g);
/* collective over the group: allocate this rank's inbox (2 halves x world segments x inbox_records records; 0 = default
 * from the frontier capacity) and map every peer's.  153 with a message if peer memory is unavailable. */
int vsr_engine_attach_group(VsrEngine* e, VsrGroup* g, uint64_t inbox_records);
/* the same kernels with the outgoing records in a LOCAL staging buffer (world segments of inbox_records records, destination
 * major) for a host that moves them with its own collective: segment d of *stage_out goes to segment <this rank> of half
 * `parity` of rank d's *inbox_out (2 halves x world segments).  Used by dist.ShardedBfs (torch.distributed all-to-all). */
int vsr_engine_attach_staged(VsrEngine* e, uint64_t inbox_records, void** stage_out, void** inbox_out, uint64_t* cap_out);
int vsr_engine_detach(VsrEngine* e);                                 /* collective when attached to a group */
uint64_t vsr_engine_default_inbox_records(const VsrEngine* e);
/* The whole BFS, called by every rank of the group with the same opts (world 1: one call, no group); it starts from Init,
 * or from opts.recover_path — a checkpoint of any world (1, 2, 4 or 8 ranks) — whatever the engine explored before.  All ranks return the same rc and the same totals
 * (records_sent / received, bytes_* and kernel_launches are this rank's).  part_states = frontier states per rank and step
 * (0 = from the inbox size).  On a violation / deadlock trace_cands[0 .. *trace_len) is the candidate chain from Init,
 * walked across ranks: vsr_replay_candidates turns it into the literal behaviour. */
int vsr_bfs_sharded(VsrEngine* e, const VsrRunOpts* opts, uint64_t part_states, VsrStats* stats, uint32_t* trace_cands, int* trace_len,
                    size_t trace_cap);
/* `vsrmc -gpus N`: the same from ONE process, one thread per GPU (devices opts->device ... + ngpus - 1); opts.recover_path
 * may have been written by any number of GPUs */
int vsr_bfs_multi(const VsrModel* m, const VsrRunOpts* opts, int ngpus, uint64_t inbox_records, uint64_t part_states, VsrStats* stats,
                  void* trace_out, uint8_t* trace_actions, size_t trace_cap, char* err, size_t errcap);

/* Host replay helper for multi-rank traces: given a chain of candidate indices from Init, re-executes
 * them (canonicalising as the engine does) and writes the literal states. */
int vsr_replay_candidates(const VsrModel* m, const uint32_t* cands, int n, void* trace_out, uint8_t* trace_actions,
                          size_t trace_cap);

/* ---- simulation mode: TLC `-simulate [-depth N]` (the reference's README.md:22 recommends it for the defect).
 * num_walks random behaviours from Init of at most `depth` states (TLC's default 100), one GPU thread per walk.  Each step
 * is drawn uniformly among the enabled candidates of the current state: one per (action, binding) pair, except that under
 * SYMMETRY one ReceiveClientRequest candidate stands for every value not yet requested.  The invariant is checked on
 * every state after Init.  The reported walk is the smallest walk index that violates the invariant (returns 12) or, with
 * check_deadlock, reaches a state without successors before the depth bound (returns 11, TLC's "Deadlock reached"); it is
 * re-walked on the host and returned as a literal behaviour (literal value names).  Walks ending in a state without
 * successors are counted in dead_ends either way. */
typedef struct VsrSimOpts {
    int32_t device, depth;
    uint64_t num_walks, seed;
    uint64_t probe_walks;   /* optional cross-check: for walks 0 .. min(probe_walks, num_walks)-1 the device reports ... */
    uint64_t* probe_out;    /* ... [2w] = bytewise FP64 of the walk's last state (all words), [2w+1] = transitions taken; NULL = off */
    int32_t check_deadlock; /* TLC checks deadlock unless -deadlock is given; 0 = only count walks without successors */
    int32_t _pad;
} VsrSimOpts;
typedef struct VsrSimStats {
    uint64_t walks, steps, dead_ends;
    uint64_t violating_walk;          /* the reported walk: its index ... */
    int32_t rc, violation_depth;      /* ... and the depth (Init = 1) of its violating / successor-less last state */
    int32_t trace_len, _pad;
    double kernel_ms, seconds_total;
} VsrSimStats;
int vsr_simulate(const VsrModel* m, const VsrSimOpts* opts, VsrSimStats* out, void* trace_out, uint8_t* trace_actions,
                 size_t trace_cap);

/* the same walk on the host (walk index `walk` of vsr_simulate with this seed): chosen candidate indices, number of
 * transitions, and the depth of the first violating state (0 = none) */
int vsr_walk(const VsrModel* m, uint64_t seed, uint64_t walk, int depth, uint32_t* cands_out, int* violated_at);

/* seen-set micro-benchmark (SURVEY §8d): inserts n splitmix64 keys (a fraction dup_frac of them repeats) into a fresh
 * table of `capacity` slots (power of two) with the BFS's own insert routine; best of `iters` launches.
 * out[0] = device ms per launch, out[1] = keys found new (must equal the number of distinct keys), out[2] = slots probed. */
int vsr_probe_bench(int device, uint64_t capacity, uint64_t n, double dup_frac, int iters, double* out);

const char* vsr_version(void);
/* sizeof of an ABI struct by name ("VsrRunOpts", "VsrCoverage", "VsrStats", "VsrLevelInfo"; 0 = unknown), for bindings that
 * mirror the structs to check themselves against */
size_t vsr_sizeof(const char* struct_name);

#ifdef __cplusplus
}
#endif
#endif /* VSR_B200_H */
