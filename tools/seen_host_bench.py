"""The shipped VSR.cfg to completion (continued past the AcknowledgedWriteNotLost violation, as bench.py runs it) on ONE GPU
with the HBM seen-set capped well below the space and the seen-set's host tier taking the older levels (DESIGN §2
"Seen-set host tier"), beside the same run with the whole seen-set in HBM.  Both runs pump the engine level by level
(vsr_engine_expand / vsr_engine_finish_level, what vsr_bfs_sharded does on one GPU), so every level's tier figures are read.

    python tools/seen_host_bench.py [--table-log2 29] [--out FILE.json]

Prints one JSON line: the card's name and power limit, both runs' totals, level sizes and time, and per level of the tier
run: false new states removed, tier entries read by the pass and its host GB/s, eviction / tier-pass / compaction time
beside the expand kernel's; the tier's peak size; and the counterexample of the violation replayed by the oracle."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (EXPECT, TABLE_CAP, FRONTIER_CAP: the flagship workload's numbers and its HBM-only sizes)
from cfg3_one_gpu import gpu_name_and_power  # noqa: E402

TIER = 1_200_000_000     # host tier entries: 19.2 GB pinned, the whole space (1,173,992,337 states) with room to spare
FRONTIER = 300_000_000   # per frontier buffer: the widest level (120,193,500) and its false new states before compaction


def run(pkg, mc, table, frontier, tier):
    """the BFS pumped level by level; per level the VsrLevelInfo fields this tool reports"""
    from vsr_tlaplus_b200 import dist as vdist
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=table, frontier_capacity=frontier, keep_trace=True, table_host_capacity=tier)
    try:
        t0 = time.time()
        eng.reset()
        eng.seed()
        li = eng.finish()
        levels, viol = [], None
        held_before = 0
        while True:
            assert li.error_code == 0 and li.overflow == 0, (len(levels) + 1, li.error_code, li.overflow,
                                                            eng.lib.vsr_engine_last_error(eng._e).decode())
            if li.new_states == 0:
                break
            levels.append(dict(depth=len(levels) + 1, new=int(li.new_states), generated=int(li.generated), expand_ms=float(li.ms),
                               false_new=int(li.false_new), tier_read=held_before, pass_ms=float(li.ms_host_pass),
                               compact_ms=float(li.ms_host_compact), evict_ms=float(li.ms_host_evict), evicted=int(li.evicted),
                               held=int(li.host_entries)))
            held_before = int(li.host_entries)
            if li.violation and viol is None:
                viol = (len(levels), int(li.violation_id))
            eng.expand()
            li = eng.finish()
        seconds = time.time() - t0
        st = eng.stats()
        out = dict(distinct=sum(lv["new"] for lv in levels), generated=int(st.generated), depth=len(levels), seconds=seconds,
                   seconds_kernels=float(st.seconds_kernels), violation_level=viol[0] if viol else 0, levels=levels,
                   host_entries=int(st.host_entries), host_false_new=int(st.host_false_new),
                   seconds_host={"pass": float(st.seconds_host_pass), "compact": float(st.seconds_host_compact), "evict": float(st.seconds_host_evict)})
        if viol:
            cap = viol[0] + 2
            tr, acts = mc._buf(cap), (C.c_uint8 * cap)()
            n = mc._lib.vsr_engine_build_trace(eng._e, viol[1], tr, acts, cap)
            raw, sb = bytes(tr), mc.state_bytes
            trace = [(pkg.ACTION_NAMES[acts[i]], raw[i * sb:(i + 1) * sb]) for i in range(max(n, 0))]
            out["trace_len"] = len(trace)
            out["reported_invariant"] = mc.reported_invariant(trace[-1][1]) if trace else None
            with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
                f.write(mc.dump_trace_tlc(trace))
            rep = subprocess.run([os.path.join(ROOT, "oracle", "_build", "vsr_oracle"), "replay", f.name], capture_output=True, text=True)
            os.unlink(f.name)
            out["oracle_replay_ok_steps"] = rep.stdout.count(" ok (")
            out["oracle_replay_not_a_step"] = "NOT A STEP" in rep.stdout
        return out
    finally:
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--table-log2", type=int, default=29)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import _pkg
    pkg = _pkg.load()
    name, power = gpu_name_and_power()
    mc = pkg.ModelChecker.from_cfg(os.path.join(ROOT, "tests", "golden", "VSR.cfg"))
    hbm = run(pkg, mc, bench.TABLE_CAP, bench.FRONTIER_CAP, 0)
    tier = run(pkg, mc, 1 << a.table_log2, FRONTIER, TIER)
    for r in (hbm, tier):
        r["expect_ok"] = (r["distinct"], r["generated"], r["depth"], r["violation_level"]) == tuple(bench.EXPECT[k] for k in
                                                                                                   ("distinct", "generated", "depth", "violation_level"))
    same_levels = [lv["new"] for lv in hbm["levels"]] == [lv["new"] for lv in tier["levels"]] and \
                  [lv["generated"] for lv in hbm["levels"]] == [lv["generated"] for lv in tier["levels"]]
    passes = [lv for lv in tier["levels"] if lv["tier_read"]]
    rec = dict(gpu=name, power_limit=power, table_slots=1 << a.table_log2, tier_capacity=TIER, frontier=FRONTIER, same_levels=same_levels,
               tier_peak_entries=max(lv["held"] for lv in tier["levels"]), tier_peak_gb=max(lv["held"] for lv in tier["levels"]) * 16e-9,
               pass_gbs=[round(lv["tier_read"] * 16e-9 / (lv["pass_ms"] * 1e-3), 2) for lv in passes if lv["pass_ms"] > 0],
               hbm=hbm, tier=tier)
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
