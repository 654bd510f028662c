#!/usr/bin/env python
"""live_bench.py — PROPERTY ViewChangeCompletes on the shipped VSR.cfg (SPECIFICATION Spec): the BFS, then the liveness pass.

The config's INVARIANT is dropped (it is violated at depth 28 and would end the run first).  Prints one JSON line: the card's name and power limit (read in the same run), the verdict, the share of states where
AllReplicasMoveToSameView is false, the store's bytes in HBM and in host memory, the sweeps with their device time (CUDA
events, stream synchronised), and the BFS's kernel seconds beside them.  A store that does not fit is reported as rc 152
with the sizes tried.  With --out DIR a lasso (rc 13) is written there in TLC's -dumpTrace format.

    python tools/live_bench.py [--table N] [--frontier N] [--live-states N] [--trace] [--out DIR]

Sizes (defaults): 1.35e9 seen-set slots (1,173,992,337 distinct states at load 0.87), 2 x 121e6 frontier states (widest
level 120,193,500), a store of --live-states not-P states whose words continue in pinned host memory past what HBM holds.
Without --trace no parent records are kept (8 B per slot): a violation is then reported without its lasso.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # the measurement still stands; the card is then unknown
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--table", type=int, default=1_350_000_000)
    ap.add_argument("--frontier", type=int, default=121_000_000)
    ap.add_argument("--live-states", type=int, default=930_000_000)
    ap.add_argument("--trace", action="store_true")
    ap.add_argument("--cfg", default=os.path.join(ROOT, "tests", "golden", "VSR.cfg"))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    os.environ["VSR_B200_LIVE_STATES"] = str(a.live_states)
    import _pkg
    pkg = _pkg.load()
    # the property alone: AcknowledgedWriteNotLost is violated at depth 28 (DESIGN §5), and TLC, like this checker, checks
    # temporal properties only when the search found no other error
    text = open(a.cfg).read().replace("INIT Init\nNEXT Next\n", "SPECIFICATION Spec\n").replace("\\* PROPERTY\n", "PROPERTY ViewChangeCompletes\n")
    text = text.replace("INVARIANT\nAcknowledgedWriteNotLost\n", "")
    mc = pkg.ModelChecker.from_cfg_text(text)
    assert mc.info.property == 1
    card = gpu_info()
    t0 = time.time()
    res = mc.check(deadlock=False, stop_on_violation=False, keep_trace=a.trace, table_capacity=a.table, frontier_capacity=a.frontier,
                   frontier_host_capacity=1024)
    wall = time.time() - t0
    live = res.liveness
    out = {"card": card, "rc": res.rc, "verdict": {0: "holds", 13: "violated"}.get(res.rc, "not decided"), "complete": res.complete,
           "distinct": res.distinct, "generated": res.generated, "depth": res.depth, "bfs_kernel_seconds": res.seconds_kernels,
           "seconds_total": wall, "table_capacity": a.table, "frontier_capacity": a.frontier, "live_states_capacity": a.live_states}
    if live:
        sweep_ms = live["ms_sweep"]
        out.update({"not_p_states": live["stored"], "not_p_share": live["stored"] / max(res.distinct, 1), "store_bytes_hbm": live["bytes_hbm"],
                    "store_bytes_host": live["bytes_host"], "sweeps": live["sweeps"], "ms_per_sweep": sweep_ms,
                    "liveness_kernel_seconds": sum(sweep_ms) * 1e-3, "liveness_seconds": live["seconds_total"], "sinks": live["sinks"],
                    "survivors": live["survivors"], "violation_level": live["violation_level"], "trace_loop": res.trace_loop})
    if res.rc == 13 and res.trace and a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "lasso.tla"), "w") as f:
            f.write(mc.dump_trace_tlc(res.trace) + "\n\\* %d: %s\n" % (len(res.trace) + 1, "Back to state %d" % res.trace_loop if res.trace_loop else "Stuttering"))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
