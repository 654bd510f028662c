/*
 * vsr_cli.cpp — `vsrmc`: TLC's command line for the one path this repo replaces,
 *     java -cp tla2tools.jar tlc2.TLC [-deadlock] [-depth N] [-fp N] [-dumpTrace tlc FILE] -config VSR.cfg VSR.tla
 * becomes
 *     vsrmc [-deadlock] [-depth N] [-fp 0] [-dumpTrace tlc FILE] [-gpu N] -config VSR.cfg [VSR.tla]
 * with TLC's summary lines and exit statuses (0, 11 deadlock, 12 invariant, 150/151 parse errors).
 * Thin: all work is behind the C ABI (include/vsr_b200.h).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <sys/types.h>

#include <time.h>

#include <chrono>
#include <string>
#include <vector>

#include "../../include/vsr_b200.h"

static double vsr_now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
static std::string vsr_clock_text() { /* TLC's "(2024-01-01 12:00:00)" time stamps */
    char b[64];
    const time_t t = time(nullptr);
    strftime(b, sizeof b, "%Y-%m-%d %H:%M:%S", localtime(&t));
    return b;
}

static void usage() {
    fprintf(stderr,
            "usage: vsrmc -config FILE.cfg [SPEC.tla] [options]\n"
            "  -deadlock            do NOT check for deadlock (TLC's flag; TLC checks by default, and so does vsrmc)\n"
            "  -depth N             stop after BFS depth N\n"
            "  -dumpTrace tlc FILE  write a counterexample in TLC's `dumpTrace tlc` format\n"
            "  -fp N                fingerprint polynomial index; only 0 (TLC's Polys[0]) is available\n"
            "  -checkpoint MIN      write a checkpoint at the first level boundary after MIN minutes since the last one (0 = after every\n"
            "                       level) to <metadir>/vsr.ckpt; a run stopped by -depth also leaves one\n"
            "  -metadir DIR         where checkpoints go (default: states/, as in TLC)\n"
            "  -recover DIR         continue from the checkpoint in DIR (or from that file) instead of Init\n"
            "  -workers N           accepted for compatibility; the BFS runs on the GPU (likewise -coverage, -fpmem, -fpbits, -cleanup,\n"
            "                       -nowarning, -tool, ...); -dfid is refused\n"
            "  -gpu N               CUDA device ordinal (default 0; with -gpus: the first of N consecutive devices)\n"
            "  -gpus N              shard the state space over N = 1, 2, 4 or 8 GPUs of this node (by fingerprint; the kernel stores\n"
            "                       a successor owned by another GPU straight into that GPU's inbox over NVLink)\n"
            "  -inbox N / -part N   -gpus > 1: records per inbox segment / frontier states per GPU and step (default: from -frontier)\n"
            "  -table N / -frontier N   seen-set slots / states per frontier buffer (default: from free memory)\n"
            "  -spill N             let each frontier buffer continue with N states in pinned host memory once its HBM part is full\n"
            "  -continue            keep exploring after the first violation\n"
            "  -simulate [-num W] [-seed S]   TLC's simulation mode: W random behaviours of at most -depth (default 100) states\n"
            "  -notrace             do not keep parent records (no counterexample)\n");
}

int main(int argc, char** argv) {
    const char *cfg = nullptr, *tla = nullptr, *dump = nullptr;
    bool simulate = false, deadlock_flag = false;
    std::string metadir = "states", ckpt_file, recover_file;
    double ckpt_minutes = -1;
    int gpus = 1;
    unsigned long long inbox_records = 0, part_states = 0;
    unsigned long long sim_walks = 1ull << 22, sim_seed = 1;
    VsrRunOpts o;
    memset(&o, 0, sizeof o);
    o.check_deadlock = 1; /* TLC's default */
    o.stop_on_violation = 1;
    o.keep_trace = 1;
    o.verbose = 1;
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        if (a == "-config" && i + 1 < argc) cfg = argv[++i];
        else if (a == "-deadlock") { o.check_deadlock = 0; deadlock_flag = true; }
        else if (a == "-gpus" && i + 1 < argc) gpus = atoi(argv[++i]);
        else if (a == "-inbox" && i + 1 < argc) inbox_records = strtoull(argv[++i], 0, 10);
        else if (a == "-part" && i + 1 < argc) part_states = strtoull(argv[++i], 0, 10);
        else if (a == "-depth" && i + 1 < argc) o.max_depth = atoi(argv[++i]);
        else if (a == "-dumpTrace" && i + 2 < argc) {
            if (strcmp(argv[i + 1], "tlc") != 0) { fprintf(stderr, "Error: only `-dumpTrace tlc FILE` is supported\n"); return 255; }
            dump = argv[i + 2];
            i += 2;
        } else if (a == "-fp" && i + 1 < argc) {
            if (atoi(argv[++i]) != 0) { fprintf(stderr, "Error: only -fp 0 is available\n"); return 255; }
        } else if (a == "-checkpoint" && i + 1 < argc) ckpt_minutes = atof(argv[++i]);
        else if (a == "-metadir" && i + 1 < argc) metadir = argv[++i];
        else if (a == "-recover" && i + 1 < argc) recover_file = argv[++i];
        else if ((a == "-workers" || a == "-coverage" || a == "-userFile" || a == "-fpmem" ||
                    a == "-fpbits" || a == "-maxSetSize" || a == "-lncheck") && i + 1 < argc) {
            i++; /* TLC tuning / housekeeping flags that have no counterpart here: accepted so existing command lines keep working */
        } else if (a == "-cleanup" || a == "-nowarning" || a == "-tool" || a == "-terse" || a == "-gzip" || a == "-debug") {
        } else if (a == "-dfid" || a == "-generateSpecTE" || a == "-continue-from") {
            fprintf(stderr, "Error: %s is not available (no depth-first iterative deepening, no trace-expression specs)\n", a.c_str());
            return 255;
        } else if (a == "-gpu" && i + 1 < argc) o.device = atoi(argv[++i]);
        else if (a == "-table" && i + 1 < argc) o.table_capacity = strtoull(argv[++i], 0, 10);
        else if (a == "-frontier" && i + 1 < argc) o.frontier_capacity = strtoull(argv[++i], 0, 10);
        else if (a == "-spill" && i + 1 < argc) o.frontier_host_capacity = strtoull(argv[++i], 0, 10);
        else if (a == "-continue") o.stop_on_violation = 0;
        else if (a == "-simulate") simulate = true;
        else if (a == "-num" && i + 1 < argc) sim_walks = strtoull(argv[++i], 0, 10);
        else if (a == "-seed" && i + 1 < argc) sim_seed = strtoull(argv[++i], 0, 10);
        else if (a == "-notrace") o.keep_trace = 0;
        else if (a == "-h" || a == "-help" || a == "--help") { usage(); return 0; }
        else if (a[0] != '-') tla = argv[i];
        else { fprintf(stderr, "Error: unrecognized option %s\n", a.c_str()); usage(); return 255; }
    }
    if (!cfg) { usage(); return 255; }
    if (ckpt_minutes >= 0) {
        mkdir(metadir.c_str(), 0777); /* may exist */
        ckpt_file = metadir + "/vsr.ckpt";
        o.checkpoint_path = ckpt_file.c_str();
        o.checkpoint_seconds = ckpt_minutes * 60.0;
    }
    if (!recover_file.empty()) {
        struct stat sb;
        if (stat(recover_file.c_str(), &sb) == 0 && S_ISDIR(sb.st_mode)) recover_file += "/vsr.ckpt";
        o.recover_path = recover_file.c_str();
    }
    char err[1024];
    VsrModel* m = nullptr;
    int rc = vsr_load(cfg, tla, &m, err, sizeof err);
    if (rc) { fprintf(stderr, "Error: %s\n", err); return rc; }
    VsrModelInfo info;
    vsr_model_info(m, &info);
    printf("%s\n", vsr_version());
    printf("Model: ReplicaCount=%d ClientCount=%d |Values|=%d StartViewOnTimerLimit=%d RestartEmptyLimit=%d%s%s; packed state %d bytes (%d bits), %d candidate bindings per state\n",
           info.replica_count, info.client_count, info.value_count, info.start_view_on_timer_limit, info.restart_empty_limit,
           info.view ? " VIEW view" : "", info.symmetry ? " SYMMETRY symmValues" : "", info.state_bytes, info.state_bits, info.num_candidates);
    if (tla && info.spec_verified) printf("Spec %s verified as MODULE VSR (hash %016llx)\n", tla, (unsigned long long)info.spec_hash);
    else if (tla) printf("Spec %s is NOT the VSR.tla this checker lowers: checking the built-in definitions, not the file's\n", tla);
    if (!deadlock_flag && info.check_deadlock == 0) o.check_deadlock = 0; /* CHECK_DEADLOCK FALSE in the cfg, as in TLC */
    VsrStats st;
    memset(&st, 0, sizeof st);
    const size_t tcap = 4096;
    std::vector<unsigned char> trace(tcap * (size_t)info.state_bytes);
    std::vector<uint8_t> acts(tcap);
    VsrSimStats sim;
    memset(&sim, 0, sizeof sim);
    VsrLiveStats live;
    memset(&live, 0, sizeof live);
    const char* refused = !info.property ? nullptr
                          : simulate ? "-simulate with PROPERTY ViewChangeCompletes: temporal properties are checked on the complete state graph only"
                          : gpus > 1 ? "-gpus > 1 with PROPERTY ViewChangeCompletes: liveness on several GPUs is not supported"
                          : (o.checkpoint_path || o.recover_path) ? "-checkpoint / -recover with PROPERTY ViewChangeCompletes: checkpointing the liveness store is not supported"
                          : nullptr;
    if (refused) {
        fprintf(stderr, "Error: %s\n", refused);
        vsr_model_free(m);
        return VSR_RC_CONFIG_ERROR;
    }
    if (info.property && gpus == 1) {
        /* one GPU: the BFS, then the liveness pass on the same engine (it keeps the store of not-P states) */
        printf("Running breadth-first search Model-Checking with fp 0 on GPU %d.\n", o.device);
        const double t0 = vsr_now_s();
        VsrEngine* e = nullptr;
        rc = vsr_engine_create(m, &o, 0, 1, &e, err, sizeof err);
        if (rc) { fprintf(stderr, "Error: %s\n", err); vsr_model_free(m); return rc; }
        std::vector<uint32_t> cands(tcap);
        int n = 0;
        rc = vsr_bfs_sharded(e, &o, 0, &st, cands.data(), &n, cands.size());
        if (rc == VSR_RC_OK && st.complete) {
            printf("Checking temporal properties for the complete state space with %llu total distinct states at (%s)\n", (unsigned long long)st.distinct,
                   vsr_clock_text().c_str());
            rc = vsr_engine_liveness(e, &live, cands.data(), cands.size());
            n = live.trace_len;
            if (rc == VSR_RC_LIVENESS) st.trace_len = o.keep_trace ? n + 1 : 0;
            double sweep_ms = 0;
            for (int i = 0; i < live.sweeps && i < VSR_MAX_SWEEPS; i++) sweep_ms += live.ms_sweep[i];
            if (rc == VSR_RC_OK || rc == VSR_RC_LIVENESS)
                printf("Liveness: %llu states where AllReplicasMoveToSameView is false stored (%.1f %% of %llu; %.2f GB in HBM, %.2f GB in host memory), "
                       "%d sweeps in %.3f s of kernel time, %llu without successors, %llu on cycles\n",
                       (unsigned long long)live.stored, st.distinct ? 100.0 * live.stored / st.distinct : 0.0, (unsigned long long)st.distinct,
                       live.bytes_hbm / 1e9, live.bytes_host / 1e9, live.sweeps, sweep_ms * 1e-3, (unsigned long long)live.sinks,
                       (unsigned long long)live.survivors);
            if (rc == VSR_RC_OK) printf("Finished checking temporal properties in %.3f s at %s\n", live.seconds_total, vsr_clock_text().c_str());
        } else if (rc == VSR_RC_OK) {
            printf("Temporal properties were not checked: the search stopped before the state graph was complete "
                   "(they are checked on the complete graph only).\n");
        }
        if ((rc == VSR_RC_VIOLATION || rc == VSR_RC_DEADLOCK || rc == VSR_RC_LIVENESS) && st.trace_len > 0) {
            const int k = vsr_replay_candidates(m, cands.data(), n, trace.data(), acts.data(), tcap);
            st.trace_len = k > 0 ? (k < (int)tcap ? k : (int)tcap) : 0;
        }
        if (rc && rc != VSR_RC_VIOLATION && rc != VSR_RC_DEADLOCK && rc != VSR_RC_LIVENESS) fprintf(stderr, "Error: %s\n", vsr_engine_last_error(e));
        vsr_engine_destroy(e);
        st.seconds_total = vsr_now_s() - t0;
    } else if (simulate) {
        VsrSimOpts so;
        so.device = o.device;
        so.depth = o.max_depth > 0 ? o.max_depth : 100;
        so.num_walks = sim_walks;
        so.seed = sim_seed;
        printf("Running Random Simulation with seed %llu: %llu behaviours of at most %d states on GPU %d.\n", sim_seed, sim_walks, so.depth, o.device);
        rc = vsr_simulate(m, &so, &sim, trace.data(), acts.data(), tcap);
        st.trace_len = sim.trace_len;
    } else {
        if (gpus > 1) printf("Running breadth-first search Model-Checking with fp 0 on GPUs %d..%d (state space sharded by fingerprint).\n", o.device, o.device + gpus - 1);
        else printf("Running breadth-first search Model-Checking with fp 0 on GPU %d.\n", o.device);
        err[0] = 0;
        rc = vsr_bfs_multi(m, &o, gpus, inbox_records, part_states, &st, trace.data(), acts.data(), tcap, err, sizeof err);
        if (err[0]) fprintf(stderr, "Error: %s\n", err);
    }
    if (rc == VSR_RC_VIOLATION || rc == VSR_RC_DEADLOCK || rc == VSR_RC_LIVENESS) {
        if (rc == VSR_RC_LIVENESS) {
            printf("Error: Temporal properties were violated.\n");
        } else if (rc == VSR_RC_VIOLATION) {
            /* which of the configured invariants the reported state violates: evaluated on that state (several may be configured) */
            int mask = st.violation_mask;
            if (!mask && st.trace_len > 0) mask = vsr_invariant(m, trace.data() + (size_t)(st.trace_len - 1) * info.state_bytes);
            static const char* names[4] = {"AcknowledgedWriteNotLost", "AcknowledgedWritesExistOnMajority", "NoLogDivergence", "TestInv"};
            bool any = false;
            for (int b = 0; b < 4; b++)
                if (mask & (1 << b)) { printf("Error: Invariant %s is violated.\n", names[b]); any = true; }
            if (!any) printf("Error: Invariant is violated.\n");
        }
        else if (rc == VSR_RC_DEADLOCK) printf("Error: Deadlock reached.\n");
        if (rc == VSR_RC_LIVENESS) printf("Error: The following behavior constitutes a counter-example:\n");
        else printf("Error: The behavior up to this point is:\n");
        std::vector<char> buf(1 << 18);
        std::string dumptext = "<<\n";
        for (int i = 0; i < st.trace_len; i++) {
            const unsigned char* s = trace.data() + (size_t)i * info.state_bytes;
            char loc[128];
            vsr_action_location(m, acts[i], loc, sizeof loc);
            vsr_state_to_tla(m, s, buf.data(), buf.size());
            if (i == 0) printf("State 1: <Initial predicate>\n%s\n", buf.data());
            else printf("State %d: <%s %s>\n%s\n", i + 1, vsr_action_name(acts[i]), loc, buf.data());
            dumptext += "[\n _TEAction |-> [\n   position |-> " + std::to_string(i + 1) + ",\n   name |-> \"" + vsr_action_name(acts[i]) +
                        "\",\n   location |-> \"" + loc + "\"\n ],\n" + buf.data() + "]" + (i + 1 < st.trace_len ? ",\n" : "\n");
        }
        dumptext += ">>";
        if (rc == VSR_RC_LIVENESS && st.trace_len > 0) { /* the lasso's end: a step back into the behaviour, or stuttering forever */
            std::string tail;
            if (live.trace_loop > 0) {
                char loc[128];
                vsr_action_location(m, live.trace_loop_action, loc, sizeof loc);
                tail = std::to_string(st.trace_len + 1) + ": Back to state " + std::to_string(live.trace_loop) + ": <" +
                       vsr_action_name(live.trace_loop_action) + " " + loc + ">";
            } else {
                tail = std::to_string(st.trace_len + 1) + ": Stuttering";
            }
            printf("%s\n", tail.c_str());
            dumptext += "\n\\* " + tail + "\n";
        }
        if (dump) {
            FILE* f = fopen(dump, "w");
            if (f) { fputs(dumptext.c_str(), f); fclose(f); printf("Trace written to %s\n", dump); }
        }
    } else if (rc) {
        fprintf(stderr, "Error: run failed with status %d (device error code %d)\n", rc, st.error_code);
    } else if (st.complete) {
        printf("Model checking completed. No error has been found.\n");
    }
    if (simulate) {
        printf("%llu behaviours, %llu states checked (%llu ended in a state without successors); %.3f s, %.0f states/s.\n",
               (unsigned long long)sim.walks, (unsigned long long)(sim.steps + sim.walks), (unsigned long long)sim.dead_ends, sim.seconds_total,
               (sim.steps + sim.walks) / (sim.kernel_ms > 0 ? sim.kernel_ms / 1e3 : 1));
        vsr_model_free(m);
        return rc;
    }
    printf("%llu states generated, %llu distinct states found, %llu states left on queue.\n", (unsigned long long)st.generated,
           (unsigned long long)st.distinct, (unsigned long long)st.queue);
    if (st.complete) printf("The depth of the complete state graph search is %d.\n", st.depth);
    else printf("The depth of the state graph search so far is %d.\n", st.depth);
    printf("Finished in %.3f s (kernels %.3f s): %.0f distinct states/s; same-level VIEW ties %llu, fingerprint collisions detected %llu\n",
           st.seconds_total, st.seconds_kernels, st.distinct / (st.seconds_total > 0 ? st.seconds_total : 1), (unsigned long long)st.h2_ties,
           (unsigned long long)st.fp_collisions);
    vsr_model_free(m);
    return rc;
}
