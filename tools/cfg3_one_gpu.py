"""The README constants (ReplicaCount 3, Values {v1, v2, v3}, StartViewOnTimerLimit 3) on ONE GPU, to the first
AcknowledgedWriteNotLost violation, with the trace kept.  The seen-set and the frontier buffers' HBM parts fill an 80 GB
card; each frontier buffer continues in pinned host memory (level 24 alone is 1.345e9 states of 64 B, and the one-GPU loop
generates the whole level before it reports the violation), and the trace, which no longer fits in HBM beside them, goes
to pinned host memory as a whole (csrc/vsr_gpu.cu trace_alloc).  About 180 GB are pinned, so the run refuses to start
unless the host has about 300 GB available (bench.py's pinning_fits).

    python tools/cfg3_one_gpu.py [--out FILE.json]

Prints one JSON line: the verdict and counts, the level sizes, the times, the bytes pinned, the depths at which the
reference's published 24-state counterexample lies in the explored set, and the checks of the checker's own
counterexample (every step a Next step of the literal model, the violation only at its end)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (host_memory_available, pinning_fits, golden_depths: the multi-GPU block's own checks)

TABLE = 3_750_000_000       # seen-set slots: 60.0 GB, load 0.845 at the violation
FRONTIER = 160_000_000      # per frontier buffer in HBM: 2 x 10.2 GB
FRONTIER_HOST = 1_200_000_000  # per frontier buffer in pinned host memory: 2 x 76.8 GB


def gpu_name_and_power():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except (OSError, ValueError, subprocess.SubprocessError):
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    import _pkg
    pkg = _pkg.load()
    from vsr_tlaplus_b200 import dist as vdist
    name, power = gpu_name_and_power()
    mc = pkg.ModelChecker.from_constants(3, 3, 3)
    trace_records = TABLE - TABLE // 8 + 64
    pinned = 2 * FRONTIER_HOST * mc.state_bytes + trace_records * 8
    avail = bench.host_memory_available()
    out = {"workload": "VSR.tla ReplicaCount=3 Values={v1,v2,v3} StartViewOnTimerLimit=3 to the first AcknowledgedWriteNotLost violation, one GPU",
           "gpu": name, "power_limit": power, "table_capacity": TABLE, "frontier_capacity": FRONTIER, "frontier_host_capacity": FRONTIER_HOST,
           "bytes_pinned_planned": pinned, "host_bytes_available": avail}
    if not bench.pinning_fits(pinned, 1, avail):
        out["refused"] = "needs %.0f GB of pinned host memory; %s available, and 40 %% of it stays free" % (
            pinned / 1e9, "unknown" if avail is None else "%.0f GB" % (avail / 1e9))
    else:
        t0 = time.time()
        eng = vdist.GpuEngine(mc, 0, 1, table_capacity=TABLE, frontier_capacity=FRONTIER, keep_trace=True, frontier_host_capacity=FRONTIER_HOST)
        t1 = time.time()
        try:
            res = eng.run(stop_on_violation=True, want_trace=True)
            t2 = time.time()
            gold = bench.golden_depths(pkg, mc, eng, torch, None, 1, torch.device("cuda", 0), 0)
        finally:
            eng.close()
        trace = vdist.replay_trace(mc, res.trace_cands) if res.rc == 12 else []
        lit = pkg.ModelChecker.from_constants(3, 3, 3, symmetry=False)
        steps_ok = bool(trace) and all(trace[i + 1][1] in [t for t, _, _ in lit.successors(trace[i][1])] for i in range(len(trace) - 1))
        viol_ok = bool(trace) and lit.invariant(trace[-1][1]) != 0 and all(lit.invariant(s) == 0 for _, s in trace[:-1])
        out.update({"rc": res.rc, "violation_depth": res.violation_level, "distinct_states": res.distinct, "states_generated": res.generated,
                    "level_sizes": res.level_sizes, "seconds_setup": t1 - t0, "seconds_bfs": t2 - t1, "kernel_seconds": res.kernel_ms_max / 1e3,
                    "golden_state_depths": gold, "golden_state_depths_ok": gold == list(range(1, 25)),
                    "counterexample_len": len(trace), "counterexample_steps_are_next_steps": steps_ok, "counterexample_violates_only_at_end": viol_ok,
                    "matches_expected": (res.rc, res.violation_level, res.distinct, res.generated) == (12, 24, 3_166_753_191, 8_944_515_179)})
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
