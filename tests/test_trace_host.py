"""The trace in pinned host memory: a run that allows host memory (frontier_host_capacity > 0) keeps the trace records that
HBM has no room for in pinned, device-mapped host memory (csrc/vsr_gpu.cu trace_alloc).  The test hook
VSR_B200_TRACE_HBM_RECORDS=k puts the boundary after record k (0: the whole trace in host memory), so every writer of a
record — the flush, the VIEW-tie patch, the re-shard, the checkpoint loaders — and every reader — counterexamples, lassos,
checkpoints — is exercised on both sides of it.  Every run must equal the run with the trace in HBM, and every
counterexample must be a behaviour of Next that violates only at its end."""
import os
import random
import subprocess
import struct
import sys

import pytest

import orc
import test_kernel_shapes as tks
import test_liveness as tl
from conftest import ROOT
from test_checkpoint import same_exploration
from test_reshard import INV, assert_behaviour

pytestmark = pytest.mark.gpu

HOOK = "VSR_B200_TRACE_HBM_RECORDS"
HOST = 1 << 16  # frontier_host_capacity: the run allows host memory
CAPS = dict(table_capacity=1 << 20, frontier_capacity=1 << 17)
VSRMC = os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc")


@pytest.fixture(scope="module")
def viol_depth():
    o = orc.bfs(orc.params(3, 2, 1, invariant=2), workers=8, keep_trace=False, check_assumptions=False)
    assert o.rc == 12 and o.depth > 8
    return o.depth


# -------------------------------------------------------------------------------------------------- 1. every record
@pytest.mark.parametrize("k", [0, 5_000])
def test_every_record_is_a_step_on_both_sides_of_the_boundary(pkg, monkeypatch, k):
    import ctypes as C
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    hbm, hbm_rows = tks.engine_bfs(pkg, mc, table=1 << 21, frontier=1 << 18, keep_trace=True, frontier_host_capacity=HOST, collect=False)
    monkeypatch.setenv(HOOK, str(k))
    res, rows = tks.engine_bfs(pkg, mc, table=1 << 21, frontier=1 << 18, keep_trace=True, frontier_host_capacity=HOST, keep=True)
    eng = res.engine
    try:
        assert res.distinct == 697_364 and res.complete
        assert (res.level_sizes, res.level_generated, res.generated, rows) == (hbm.level_sizes, hbm.level_generated, hbm.generated, hbm_rows)
        starts = [0]
        for n in res.level_sizes:
            starts.append(starts[-1] + n)
        near = set(range(max(0, k - 10_000), min(res.distinct, k + 10_000)))
        rng = random.Random(1234)
        others = set(rng.sample([i for i in range(res.distinct) if i not in near], 20_000))
        sb = mc.state_bytes
        cap = len(res.level_sizes) + 2
        tr, acts = mc._buf(cap), (C.c_uint8 * cap)()
        for i in sorted(near | others):
            d = next(j for j in range(len(res.level_sizes)) if i < starts[j + 1]) + 1  # depth of local id i
            parent, _ = eng.trace_record(i)
            if d == 1:
                assert parent == vdist.ROOT_PARENT, i
            else:
                assert starts[d - 2] <= parent < starts[d - 1], (i, d, parent)
            # the chain replayed from Init: its last step is this record's candidate applied to the parent's state
            m = mc._lib.vsr_engine_build_trace(eng._e, i, tr, acts, cap)
            j = i - starts[d - 1]
            assert m == d and bytes(tr)[(m - 1) * sb:m * sb] == res.levels[d - 1][j * sb:(j + 1) * sb], (i, d, m)
    finally:
        eng.close()


# -------------------------------------------------------------------------------------------------- 2. counterexamples
def test_counterexamples_with_the_trace_in_host_memory(pkg, monkeypatch, viol_depth):
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    ref = mc.check(**CAPS)
    assert_behaviour(pkg, ref, viol_depth)
    for k in (0, 1, 5_000):
        monkeypatch.setenv(HOOK, str(k))
        res = mc.check(frontier_host_capacity=HOST, **CAPS)
        assert (res.rc, res.violation_level, len(res.trace), res.distinct, res.level_sizes) == (12, ref.violation_level, len(ref.trace), ref.distinct,
                                                                                             ref.level_sizes), k
        assert_behaviour(pkg, res, viol_depth)


# -------------------------------------------------------------------------------------------------- 3. VIEW ties
def test_view_tie_patch_rewrites_a_host_record_and_moves_coverage(pkg, monkeypatch):
    """test_view_ties_resolve_to_smallest_aux_key's injected tie, with the whole trace in host memory and -coverage on: the
    winner's record is rewritten there, and the count moves from the first arrival's action to the winner's"""
    import torch
    from test_coverage import NA, host_walk
    from vsr_tlaplus_b200 import dist as vdist
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(3, 2, 2)
    _, cand_action, _ = host_walk(mc, max_states=2000)
    by_action = {}
    for c, a in sorted(cand_action.items()):
        by_action.setdefault(a, c)
    (a_first, c_first), (a_win, c_win) = sorted(by_action.items())[:2]
    eng = vdist.GpuEngine(mc, 0, 1, coverage=True, table_capacity=1 << 12, frontier_capacity=1 << 10, frontier_host_capacity=1 << 10)
    try:
        eng.reset()
        eng.seed()
        assert eng.finish().new_states == 1
        base = [t for t, a, _ in mc.successors(mc.init_state()) if pkg.ACTION_NAMES[a] == "TimerSendSVC"][0]
        variants = {}
        for aux in (2, 0, 1):
            f = mc.unpack(base)
            f.aux_svc = aux
            variants[aux] = mc.pack(f)

        def rec(aux, cand, mult):
            v = variants[aux]
            return v + struct.pack("<QQ", mc.fingerprint(v), (0 << 12) | cand | (mult << 56))  # vsr_gpu.cuh RecHdr

        for blob, n in ((rec(2, c_first, 2), 1), (rec(0, c_win, 1) + rec(1, c_first, 3), 2)):
            eng.insert(torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda(), n)
        li = eng.finish()
        assert (li.new_states, li.ties, li.generated) == (1, 2, 6)
        assert eng.trace_record(0) == (vdist.ROOT_PARENT, 0) and eng.trace_record(1) == (0, c_win)
        dis, gen = eng.coverage().levels
        want_gen, want_dis = [0] * NA, [0] * NA
        want_gen[a_first], want_gen[a_win], want_dis[a_win] = 5, 1, 1
        assert gen[1].tolist() == want_gen and dis[1].tolist() == want_dis
    finally:
        eng.close()


# -------------------------------------------------------------------------------------------------- 4. checkpoints
def test_checkpoints_across_the_boundary(pkg, monkeypatch, tmp_path, viol_depth):
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    whole = mc.check(stop_on_violation=False, **CAPS)
    ck = str(tmp_path / "host.ckpt")
    monkeypatch.setenv(HOOK, "5000")
    part = mc.check(stop_on_violation=False, max_depth=viol_depth - 6, checkpoint_path=ck, checkpoint_seconds=1e9, frontier_host_capacity=HOST, **CAPS)
    assert part.depth == viol_depth - 6 and part.distinct > 5_000
    for k in ("5000", "0", None):  # recovered with the same boundary, with all of it in host memory, with all of it in HBM
        if k is None:
            monkeypatch.delenv(HOOK)
        else:
            monkeypatch.setenv(HOOK, k)
        host = 0 if k is None else HOST
        same_exploration(mc.check(stop_on_violation=False, recover_path=ck, frontier_host_capacity=host, **CAPS), whole)
        assert_behaviour(pkg, mc.check(recover_path=ck, frontier_host_capacity=host, **CAPS), viol_depth)
    # re-sharded: the one-rank host-trace checkpoint onto 2 ranks, and a 2-rank one onto 1, with the trace in host memory
    monkeypatch.setenv(HOOK, "0")
    for kw in (dict(stop_on_violation=False), {}):
        res = mc.check_multi(2, recover_path=ck, frontier_host_capacity=HOST, **kw, **CAPS)
        if kw:
            same_exploration(res, whole)
        else:
            assert_behaviour(pkg, res, viol_depth)
    ck2 = str(tmp_path / "two.ckpt")
    part2 = mc.check_multi(2, stop_on_violation=False, max_depth=viol_depth - 6, checkpoint_path=ck2, checkpoint_seconds=1e9, frontier_host_capacity=HOST, **CAPS)
    assert part2.depth == viol_depth - 6
    same_exploration(mc.check(stop_on_violation=False, recover_path=ck2, frontier_host_capacity=HOST, **CAPS), whole)
    assert_behaviour(pkg, mc.check(recover_path=ck2, frontier_host_capacity=HOST, **CAPS), viol_depth)


# -------------------------------------------------------------------------------------------------- 5. sharded runs
def _sharded_worker(rank, world, name, q):
    import _pkg
    pkg = _pkg.load()
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    g = vdist.Group(name, rank, world, timeout_s=120)
    try:
        eng = vdist.GpuEngine(mc, rank, world, group=g, frontier_host_capacity=HOST, **CAPS)
        try:
            res = eng.run(stop_on_violation=True)
        finally:
            eng.close()
        q.put((rank, res.rc, res.violation_level, res.distinct, res.generated, res.level_sizes, list(res.trace_cands)))
    finally:
        g.close()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_runs_with_the_trace_in_host_memory(pkg, monkeypatch, viol_depth, world):
    import torch.multiprocessing as mp
    from vsr_tlaplus_b200 import dist as vdist
    monkeypatch.setenv(HOOK, "0")
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    one = mc.check(**CAPS)
    # threads of one process, inboxes through peer pointers
    res = mc.check_multi(world, frontier_host_capacity=HOST, **CAPS)
    assert (res.rc, res.violation_level, res.distinct, res.generated, res.level_sizes) == (12, one.violation_level, one.distinct, one.generated, one.level_sizes)
    assert_behaviour(pkg, res, viol_depth)
    # processes, inboxes through CUDA IPC
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    name = "/vsr-trace-host-%d-%d" % (os.getpid(), world)
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, name, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = sorted(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    _, rc, level, distinct, generated, sizes, cands = got[0]
    assert (rc, level, distinct, generated, sizes) == (12, one.violation_level, one.distinct, one.generated, one.level_sizes)
    res.trace = vdist.replay_trace(mc, cands)
    assert_behaviour(pkg, res, viol_depth)


# -------------------------------------------------------------------------------------------------- 6. liveness
def test_liveness_lassos_with_the_trace_in_host_memory(pkg, monkeypatch):
    monkeypatch.setenv(HOOK, "0")
    got = tl.run_case(pkg, 3, 1, 1, hooks=1, frontier_host_capacity=1 << 10)
    assert got["rc"] == 13 and got["trace_len"] > 1 and got["lasso_errors"] == [], got
    got = tl.run_case(pkg, 3, 1, 1, hooks=3, frontier_host_capacity=1 << 10)
    assert got["rc"] == 13 and got["trace_loop"] >= 1 and got["lasso_errors"] == [], got


# -------------------------------------------------------------------------------------------------- 7. the production rule
_PRODUCTION = r"""
import torch, _pkg
import test_kernel_shapes as tks
pkg = _pkg.load()
mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
table, frontier = 1 << 24, 1 << 18
trace = (table - table // 8 + 64) * 8
need = table * 16 + 2 * frontier * mc.state_bytes + (32 << 20)  # seen-set, frontiers, the small buffers and some slack
free = tks.release_device_memory()
assert trace > (64 << 20) and free > need + trace, (free, need, trace)
hold = torch.empty(free - need, dtype=torch.uint8, device="cuda")  # what is left holds all but the trace
try:
    res = mc.check(stop_on_violation=False, table_capacity=table, frontier_capacity=frontier, frontier_host_capacity=%d, verbose=True)
    print("RESULT", res.rc, res.distinct, res.generated, res.depth)
except pkg.VsrError as ex:
    print("RESULT", ex.rc, 0, 0, 0)
print("CHILD-OK")
"""


@pytest.mark.parametrize("host", [HOST, 0])
def test_trace_goes_to_host_memory_only_when_hbm_has_no_room(pkg, host):
    tks.release_device_memory()
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path[:0] = [%r, %r]\n" % (ROOT, os.path.join(ROOT, "tests")) + _PRODUCTION % host],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, (r.stdout[-2000:], r.stderr[-3000:])
    rc, distinct, generated, depth = map(int, [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT")][0].split()[1:])
    if host:
        assert (rc, distinct, generated, depth) == (0, 697_364, 1_831_657, 30)
        assert "in pinned host memory" in r.stderr, r.stderr[-2000:]
    else:
        assert rc == 153 and "cudaMalloc(trace)" in r.stderr, (rc, r.stderr[-2000:])  # as before: the engine cannot be created
        assert "in pinned host memory" not in r.stderr


# -------------------------------------------------------------------------------------------------- 8. the command line
def _vsrmc(tmp_path, cfg, name, args, env):
    dump = tmp_path / (name + ".txt")
    r = subprocess.run([VSRMC, "-config", str(cfg), "-deadlock", "-table", "1048576", "-frontier", "200000", "-dumpTrace", "tlc", str(dump)] + args,
                       capture_output=True, text=True, timeout=300, env=dict(os.environ, **env))
    out = r.stdout + r.stderr
    states = [ln for ln in out.splitlines() if "distinct states found" in ln]
    rep = subprocess.run([os.path.join(ROOT, "oracle", "_build", "vsr_oracle"), "replay", str(dump)], capture_output=True, text=True)
    return r.returncode, states, dump.read_text().count("position |->"), rep.stdout


def test_cli_spill_and_gpus_with_the_trace_in_host_memory(pkg, tmp_path, viol_depth):
    cfg = tmp_path / "m.cfg"
    cfg.write_text(pkg.cfg_text(3, ["v1", "v2"], 1, invariants=list(INV)))
    rc, states, steps, rep = _vsrmc(tmp_path, cfg, "hbm", [], {})
    assert rc == 12 and states and steps == viol_depth
    for name, args, env in (("spill", ["-spill", "65536"], {HOOK: "0"}),
                            ("gpus", ["-spill", "65536", "-gpus", "2"], {HOOK: "0", "VSR_B200_MULTI_ONE_DEVICE": "1"})):
        rc2, states2, steps2, rep2 = _vsrmc(tmp_path, cfg, name, args, env)
        assert (rc2, states2, steps2) == (12, states, steps), name
        assert "NOT A STEP" not in rep2 and rep2.count(" ok (") == viol_depth - 1, (name, rep2[-2000:])
