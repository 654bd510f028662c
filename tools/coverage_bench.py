#!/usr/bin/env python
"""coverage_bench.py — what TLC's action coverage (-coverage) costs, and the action table of a configuration.

Runs the BFS of a cfg without and with coverage in ONE process, alternating the two arms after a warm-up run of each, and
prints one JSON line: the card's name and power limit (read in the same run), every run's kernel seconds (CUDA events) per
arm, and the action table (distinct, generated per action of Next).  The config's INVARIANT is dropped so that the search
covers the whole state space.  With --out DIR the per-level matrices are written there: coverage_distinct.npy,
coverage_generated.npy ([rows, 20], row d - 1 = successors of depth d) and coverage.json.

    python tools/coverage_bench.py [--cfg FILE] [--gpus N] [--reps K] [--table N] [--frontier N] [--out DIR]

Default sizes fit the shipped VSR.cfg (1,173,992,337 distinct states) on one 80 GB card without parent records.
"""
import argparse
import json
import os
import subprocess
import sys

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
    ap.add_argument("--cfg", default=os.path.join(ROOT, "tests", "golden", "VSR.cfg"))
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--table", type=int, default=1_350_000_000)
    ap.add_argument("--frontier", type=int, default=121_000_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import _pkg
    pkg = _pkg.load()
    mc = pkg.ModelChecker.from_cfg_text(open(a.cfg).read().replace("INVARIANT\nAcknowledgedWriteNotLost\n", ""))
    kw = dict(deadlock=False, keep_trace=False, table_capacity=a.table // a.gpus, frontier_capacity=a.frontier // a.gpus)

    def run(coverage):
        res = mc.check(coverage=coverage, **kw) if a.gpus == 1 else mc.check_multi(a.gpus, coverage=coverage, **kw)
        if res.rc != 0 or not res.complete:
            raise SystemExit("run failed: rc %d, complete %s" % (res.rc, res.complete))
        return res

    card = gpu_info()
    arms = {"off": [], "on": []}
    last = {}
    for rep in range(a.reps + 1):  # rep 0 warms both arms up (module load, the memory pool's first mapping)
        for name in ("off", "on"):
            res = run(name == "on")
            last[name] = res
            if rep:
                arms[name].append(res.seconds_kernels)
    off, on = last["off"], last["on"]
    assert (on.generated, on.distinct, on.level_sizes) == (off.generated, off.distinct, off.level_sizes)
    cov = on.coverage
    dis, gen = cov.levels
    assert int(gen.sum()) == on.generated and int(dis.sum()) == on.distinct
    out = {"card": card, "cfg": os.path.relpath(a.cfg, ROOT), "gpus": a.gpus, "distinct": on.distinct, "generated": on.generated, "depth": on.depth,
           "kernel_seconds_off": arms["off"], "kernel_seconds_on": arms["on"],
           "overhead": min(arms["on"]) / min(arms["off"]) - 1.0 if arms["off"] else None,
           "kernel_launches": {"off": off.kernel_launches, "on": on.kernel_launches},
           "by_action": {k: list(v) for k, v in cov.by_action.items()}, "never_enabled": cov.never_enabled}
    if a.out:
        import numpy as np
        os.makedirs(a.out, exist_ok=True)
        np.save(os.path.join(a.out, "coverage_distinct.npy"), dis)
        np.save(os.path.join(a.out, "coverage_generated.npy"), gen)
        with open(os.path.join(a.out, "coverage.json"), "w") as f:
            json.dump(dict(out, level_distinct=dis.tolist(), level_generated=gen.tolist()), f)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
