#!/usr/bin/env python
"""reshard_bench.py — what recovering a checkpoint on another number of GPUs costs, on the shipped VSR.cfg.

One GPU checkpoints the BFS at --depth (its INVARIANT dropped, so that the search goes on past depth 28), then the checkpoint
is recovered twice through the one loader: on one rank (the same world: the rank reads its file and keeps every id
where it was) and on two ranks (the world grows: each rank reads the one old file and keeps its share).  Two GPUs are used when the machine has them, else two ranks
share device 0 through VSR_B200_MULTI_ONE_DEVICE; the JSON says which.  The two-rank run continues to the end of the
search and its totals are compared with 1,173,992,337 distinct / 3,129,587,684 generated / depth 47.

Prints one JSON line: the card's name and power limit (read in the same run), the checkpoint's size and how long writing
it took, and per recovery its wall seconds.  For the two-rank recovery the engine's own split is reported per rank
(reading the files, seen-set insert, frontier kernel, trace) with the files and bytes each rank read.

    python tools/reshard_bench.py [--depth 30] [--trace] [--dir DIR]

Sizes: one rank 1.35e9 seen-set slots and 2 x 121e6 frontier states; each of the two ranks 0.7e9 slots and 2 x 62e6 states.
The checkpoint goes to a temporary directory (or --dir) and is removed afterwards.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EXPECTED = (1_173_992_337, 3_129_587_684, 47)
SPLIT = re.compile(r"recover: rank (\d+) of (\d+) took its share of (\d+) checkpoint files \((\d+) bytes read\) in ([\d.]+) s: ([\d.]+) s reading, "
                   r"([\d.]+) s seen-set insert, ([\d.]+) s frontier, ([\d.]+) s trace; (\d+) seen-set entries, (\d+) frontier states")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out
    except Exception as e:  # the measurement still stands; the card is then unknown
        return ["unknown (%s)" % e]


def with_stderr(fn):
    """fn() with the process's stderr (the library's verbose lines) captured: (result, text)"""
    with tempfile.TemporaryFile(mode="w+") as tmp:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            res = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        return res, tmp.read()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=30)
    ap.add_argument("--trace", action="store_true", help="keep parent records (8 B per state more in the checkpoint)")
    ap.add_argument("--cfg", default=os.path.join(ROOT, "tests", "golden", "VSR.cfg"))
    ap.add_argument("--dir", default=None)
    ap.add_argument("--table", type=int, default=1_350_000_000)
    ap.add_argument("--frontier", type=int, default=121_000_000)
    ap.add_argument("--table2", type=int, default=700_000_000)
    ap.add_argument("--frontier2", type=int, default=62_000_000)
    a = ap.parse_args()
    import _pkg
    pkg = _pkg.load()
    text = open(a.cfg).read().replace("INVARIANT\nAcknowledgedWriteNotLost\n", "")
    mc = pkg.ModelChecker.from_cfg_text(text)
    cards = gpu_info()
    import torch
    two_devices = torch.cuda.device_count() >= 2
    if not two_devices:
        os.environ["VSR_B200_MULTI_ONE_DEVICE"] = "1"
    d = a.dir or tempfile.mkdtemp(prefix="vsr-reshard-")
    os.makedirs(d, exist_ok=True)
    ck = os.path.join(d, "vsr.ckpt")
    out = {"card": cards, "depth": a.depth, "keep_trace": a.trace,
           "two_ranks_on": "two GPUs" if two_devices else "one GPU shared by both ranks (VSR_B200_MULTI_ONE_DEVICE=1)"}
    try:
        one = dict(stop_on_violation=False, keep_trace=a.trace, table_capacity=a.table, frontier_capacity=a.frontier)
        t0 = time.time()
        part = mc.check(max_depth=a.depth, checkpoint_path=ck, checkpoint_seconds=1e9, **one)
        out["checkpoint"] = {"rc": part.rc, "depth": part.depth, "distinct": part.distinct, "bytes": os.path.getsize(ck),
                             "frontier_states": part.level_sizes[-1], "bfs_and_write_seconds": time.time() - t0}
        # the same world: one rank reads its own file, and stops at the boundary it recovered
        t0 = time.time()
        same = mc.check(recover_path=ck, max_depth=a.depth, **one)
        out["recover_world1"] = {"rc": same.rc, "wall_seconds": time.time() - t0, "seconds_setup": same.seconds_setup,
                                 "seconds_after_setup": same.seconds_total - same.seconds_setup, "bytes_read": os.path.getsize(ck)}
        # re-sharded onto two ranks, continued to the end of the search
        t0 = time.time()
        two, err = with_stderr(lambda: mc.check_multi(2, stop_on_violation=False, keep_trace=a.trace, recover_path=ck, verbose=True,
                                                      table_capacity=a.table2, frontier_capacity=a.frontier2))
        wall = time.time() - t0
        ranks = []
        for m in SPLIT.finditer(err):
            g = m.groups()
            ranks.append({"rank": int(g[0]), "files": int(g[2]), "bytes_read": int(g[3]), "seconds": float(g[4]), "reading": float(g[5]),
                          "seen_set_insert": float(g[6]), "frontier_kernel": float(g[7]), "trace": float(g[8]), "entries": int(g[9]),
                          "frontier_states": int(g[10])})
        out["recover_world2"] = {"rc": two.rc, "ranks": ranks, "whole_run_wall_seconds": wall, "complete": two.complete,
                                 "distinct": two.distinct, "generated": two.generated, "depth": two.depth,
                                 "expected": EXPECTED, "equal": (two.distinct, two.generated, two.depth) == EXPECTED}
        if not ranks:
            out["recover_world2"]["stderr_tail"] = err[-2000:]
    finally:
        if not a.dir:
            shutil.rmtree(d, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
