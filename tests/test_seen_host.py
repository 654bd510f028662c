"""The seen-set's host tier (table_host_capacity > 0, vsrmc -tablehost; csrc/vsr_seen_host.cu): at level boundaries the
entries of older levels move to pinned host memory, successors equal to them are first inserted as new, and after each
level a tier pass marks those states and a compaction drops them from the level.  The test hook VSR_B200_EVICT_LOAD=0
moves them at every boundary, so every level runs the tier pass.  Every run must equal the run with the whole seen-set in
HBM: totals, level tables, per-depth state sets, trace records, verdicts, coverage and liveness.

VSR's successors never lie two levels back, so its own runs find no state of the tier again (host_false_new is 0 on every
space here, and on the shipped VSR.cfg to completion): the false new states, their removal and the repairs after it are
made by records injected through the engine's record interface (section 2)."""
import os
import random
import struct
import subprocess

import pytest

import test_kernel_shapes as tks
import test_gpu_parity as tgp
import test_liveness as tl
from conftest import ROOT
from test_coverage import host_walk, identities, reference
from test_reshard import INV, assert_behaviour

HOOK = "VSR_B200_EVICT_LOAD"
TIER = 1 << 20                       # table_host_capacity: room for every (3, 2, 1) state
FULL_321 = (697_364, 1_831_657, 30)  # (3, 2, 1) without SYMMETRY, complete: distinct, generated, depth
VSRMC = os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc")
CAPS = dict(table_capacity=1 << 20, frontier_capacity=1 << 17)


def _tier_seen(eng):
    st = eng.stats()
    return int(st.host_entries), int(st.host_false_new)


def _same_levels(a, b):
    assert (a.distinct, a.generated, a.depth, a.complete) == (b.distinct, b.generated, b.depth, b.complete)
    assert (a.level_sizes, a.level_generated) == (b.level_sizes, b.level_generated)


@pytest.fixture(scope="module")
def viol_depth():
    import orc
    o = orc.bfs(orc.params(3, 2, 1, invariant=2), workers=8, keep_trace=False, check_assumptions=False)
    assert o.rc == 12 and o.depth > 8
    return o.depth


# -------------------------------------------------------------------------------------------------- 1. a table smaller than the space
@pytest.mark.gpu
def test_small_table_holds_the_complete_space_with_the_tier(pkg):
    """2^18 slots for 697,364 states: the run continues where the HBM-only table stops, with the oracle's state sets"""
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    hbm, _ = tks.engine_bfs(pkg, mc, table=1 << 21, frontier=1 << 18, collect=False)
    assert hbm.distinct > (1 << 18)
    res, _ = tks.engine_bfs(pkg, mc, table=1 << 18, frontier=1 << 18, table_host_capacity=TIER, keep=True)
    try:
        held, false_new = _tier_seen(res.engine)
    finally:
        res.engine.close()
    assert (res.distinct, res.generated, res.depth) == FULL_321
    _same_levels(res, hbm)
    assert 0 < held < res.distinct and false_new == 0, (held, false_new)
    q, o = tks.oracle(3, 2, 1, 0, symmetry=False)
    tgp.assert_same_exploration(pkg, mc, res, q, o, complete=True)


# -------------------------------------------------------------------------------------------------- 2. false new states
@pytest.mark.gpu
def test_states_of_evicted_levels_are_removed_from_the_level(pkg, monkeypatch, viol_depth):
    """Init, states of depth 2 and the violating states of the first violating depth V, evicted, injected again as records BEFORE depth V + 3
    is expanded: they are inserted as new, get the level's first ids, violate, are counted and traced.  The tier pass
    finds them, the compaction moves the level's last states into their rows, and the level ends as in the HBM-only run:
    its size, its state set, a violating id that is a kept state, its trace records and its coverage counts"""
    import torch
    from vsr_tlaplus_b200 import dist as vdist
    _, cand_action, _ = host_walk(pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV), max_states=4000)
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    D = viol_depth + 3
    ref, _ = tks.engine_bfs(pkg, mc, max_depth=D, table=1 << 20, frontier=1 << 17)
    sb = mc.state_bytes
    split = lambda lv: [lv[i:i + sb] for i in range(0, len(lv), sb)]
    want_mask = 0
    for s in split(ref.levels[D - 1]):
        want_mask |= mc.invariant(s)
    bad = [s for s in split(ref.levels[viol_depth - 1]) if mc.invariant(s)][:40]
    inject = [mc.init_state()] + bad + split(ref.levels[1])[:3]
    assert bad and want_mask
    cand = next(iter(cand_action))
    blob = b"".join(s + struct.pack("<QQ", mc.fingerprint(s), (0 << 12) | cand | (1 << 56)) for s in inject)  # vsr_gpu.cuh RecHdr
    monkeypatch.setenv(HOOK, "0")
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=1 << 20, frontier_capacity=1 << 17, keep_trace=True, collect_levels=True, coverage=True,
                          table_host_capacity=TIER)
    try:
        eng.reset()
        eng.seed()
        li = eng.finish()
        for d in range(2, D):
            eng.expand()
            li = eng.finish()
            assert li.new_states == ref.level_sizes[d - 1] and li.false_new == 0, d
        assert _tier_seen(eng)[0] == sum(ref.level_sizes[:D - 2])  # the boundary of depth D - 1 moved the levels before it
        eng.insert(torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda(), len(inject))
        eng.expand()
        li = eng.finish()
        assert (li.false_new, li.new_states, li.generated) == (len(inject), ref.level_sizes[D - 1], ref.level_generated[D - 2] + len(inject))
        assert li.violation and li.violation_mask == want_mask
        rows = eng.read_frontier()
        first = sum(ref.level_sizes[:D - 1])
        v = rows[(li.violation_id - first) * sb:(li.violation_id - first + 1) * sb]
        assert mc.invariant(v) and v not in inject
        assert sorted(split(rows)) == sorted(split(ref.levels[D - 1])) and sorted(split(eng.collected(D))) == sorted(split(rows))
        tks.check_audit(eng.audit(), D, li.new_states)
        start = first - ref.level_sizes[D - 2]
        for i in range(first, first + li.new_states):
            parent, c = eng.trace_record(i)
            assert start <= parent < first, (i, parent)
        dis, _ = eng.coverage().levels
        assert int(dis[D - 1].sum()) == li.new_states
        assert [eng.lookup(s)[0] for s in inject] == [1] + [viol_depth] * len(bad) + [2] * (len(inject) - 1 - len(bad))
    finally:
        eng.close()


# -------------------------------------------------------------------------------------------------- 3. eviction at every boundary
FORCED = [(2, 1, 1, 0, True), (2, 2, 2, 0, True), (2, 2, 2, 0, False), (3, 1, 1, 0, True), (2, 2, 1, 0, True), (2, 3, 2, 0, True),
          (3, 2, 2, 12, True), (3, 3, 3, 10, True), (5, 2, 2, 7, True),  # cfg2 (two-pass), cfg3 (one-pass), cfg4 (two blocks per SM)
          (2, 4, 2, 12, True)]                                            # a layout compiled as a plug-in


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth,sym", FORCED)
def test_eviction_at_every_boundary_equals_the_hbm_run(pkg, monkeypatch, R, V, L, depth, sym):
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=sym)
    hbm, hbm_rows = tks.engine_bfs(pkg, mc, max_depth=depth, table=1 << 22, frontier=1 << 20, collect=False)
    monkeypatch.setenv(HOOK, "0")
    res, rows = tks.engine_bfs(pkg, mc, max_depth=depth, table=1 << 22, frontier=1 << 20, collect=False, table_host_capacity=TIER, keep=True)
    try:
        held, false_new = _tier_seen(res.engine)
    finally:
        res.engine.close()
    _same_levels(res, hbm)
    assert rows == hbm_rows  # per level: size, generated and the order-independent digests of its states
    assert held == (hbm.distinct if hbm.complete else sum(hbm.level_sizes[:-1])), (held, false_new)


# -------------------------------------------------------------------------------------------------- 4. trace records
@pytest.mark.gpu
def test_trace_records_and_audit_after_compaction(pkg, monkeypatch):
    import ctypes as C
    from vsr_tlaplus_b200 import dist as vdist
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    res, _ = tks.engine_bfs(pkg, mc, table=1 << 20, frontier=1 << 18, keep_trace=True, table_host_capacity=TIER, keep=True)
    eng = res.engine
    try:
        assert (res.distinct, res.generated, res.depth) == FULL_321
        starts = [0]
        for n in res.level_sizes:
            starts.append(starts[-1] + n)
        sb = mc.state_bytes
        cap = len(res.level_sizes) + 2
        tr, acts = mc._buf(cap), (C.c_uint8 * cap)()
        rng = random.Random(7)
        for d in range(1, len(res.level_sizes) + 1):
            n = res.level_sizes[d - 1]
            for j in sorted(set(rng.sample(range(n), min(n, 150))) | {0, n - 1}):
                i = starts[d - 1] + j
                parent, _ = eng.trace_record(i)
                if d == 1:
                    assert parent == vdist.ROOT_PARENT
                else:
                    assert starts[d - 2] <= parent < starts[d - 1], (i, d, parent)
                m = mc._lib.vsr_engine_build_trace(eng._e, i, tr, acts, cap)
                assert m == d and bytes(tr)[(m - 1) * sb:m * sb] == res.levels[d - 1][j * sb:(j + 1) * sb], (i, d, m)
    finally:
        eng.close()


# -------------------------------------------------------------------------------------------------- 5. counterexample
@pytest.mark.gpu
def test_counterexample_with_the_tier(pkg, monkeypatch, viol_depth):
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    ref = mc.check(**CAPS)
    monkeypatch.setenv(HOOK, "0")
    res = mc.check(table_host_capacity=TIER, **CAPS)
    assert (res.rc, res.violation_level, res.distinct, res.level_sizes) == (12, ref.violation_level, ref.distinct, ref.level_sizes)
    assert res.host_entries > 0
    assert_behaviour(pkg, res, viol_depth)
    go_on = mc.check(table_host_capacity=TIER, stop_on_violation=False, **CAPS)
    whole = mc.check(stop_on_violation=False, **CAPS)
    assert (go_on.rc, go_on.violation_level, go_on.distinct, go_on.generated, go_on.level_sizes) == (12, whole.violation_level, whole.distinct,
                                                                                                  whole.generated, whole.level_sizes)


# -------------------------------------------------------------------------------------------------- 6. weak fingerprints
@pytest.mark.gpu
def test_weak_fingerprints_keep_states_apart_in_the_tier(monkeypatch, tmp_path):
    """a -DVSR_WEAK_FP_BITS=16 build: equal fingerprints are common, and the tier pass and the compaction compare the check
    hash, so the per-depth state sets stay the oracle's"""
    so = tks.build_variants(str(tmp_path), {"weak16": ("-DVSR_WEAK_FP_BITS=16", [(3, 2, 1)])})[("weak16", 3, 2, 1)]
    monkeypatch.setenv(HOOK, "0")
    res, _, sets = tks.run_in_child(so, 3, 2, 1, 0, str(tmp_path / "out.pkl"), table_host_capacity=TIER)
    tks.assert_child_parity(3, 2, 1, 0, res, sets)
    assert sum(res.level_collisions) > 0


# -------------------------------------------------------------------------------------------------- 7. several ranks
def _sharded_worker(rank, world, name, q):
    import _pkg
    os.environ[HOOK] = "0"
    pkg = _pkg.load()
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    g = vdist.Group(name, rank, world, timeout_s=120)
    try:
        res = vdist.check_sharded(mc, g, table_host_capacity=TIER, **CAPS)
        q.put((rank, res.rc, res.distinct, res.generated, res.depth, res.level_sizes, res.host_entries, res.host_false_new))
    finally:
        g.close()


@pytest.mark.gpu
def test_ranks_filter_their_own_tier(pkg, monkeypatch):
    import torch.multiprocessing as mp
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    one = mc.check(**CAPS)
    assert (one.distinct, one.generated, one.depth) == FULL_321
    monkeypatch.setenv(HOOK, "0")
    for world in (2, 4):
        res = mc.check_multi(world, table_host_capacity=TIER, **CAPS)
        assert (res.rc, res.distinct, res.generated, res.depth, res.level_sizes) == (0, one.distinct, one.generated, one.depth, one.level_sizes), world
        assert res.host_entries == one.distinct, world
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    name = "/vsr-seen-host-%d" % os.getpid()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, name, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = sorted(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for _, rc, distinct, generated, depth, sizes, held, false_new in got:
        assert (rc, distinct, generated, depth, sizes) == (0, one.distinct, one.generated, one.depth, one.level_sizes)
        assert held == one.distinct


# -------------------------------------------------------------------------------------------------- 8. coverage
@pytest.mark.gpu
def test_coverage_with_the_tier(pkg, monkeypatch):
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 1, 1)
    hbm = mc.check(coverage=True, **CAPS)
    monkeypatch.setenv(HOOK, "0")
    res = mc.check(coverage=True, table_host_capacity=TIER, **CAPS)
    assert (res.rc, res.distinct, res.generated, res.level_sizes) == (0, hbm.distinct, hbm.generated, hbm.level_sizes)
    assert res.host_entries == res.distinct
    identities(res, res.coverage, reference(3, 1, 1))
    assert res.coverage.levels[1].tolist() == hbm.coverage.levels[1].tolist()              # generated per level and action
    assert res.coverage.levels[0].sum(1).tolist() == hbm.coverage.levels[0].sum(1).tolist()  # distinct per level
    # distinct is still the histogram of the trace records' actions
    import numpy as np
    _, cand_action, _ = host_walk(mc)
    eng = vdist.GpuEngine(mc, 0, 1, coverage=True, table_host_capacity=TIER, **CAPS)
    try:
        run = eng.run()
        assert run.rc == 0 and run.complete and run.host_entries == run.distinct
        hist = np.zeros_like(run.coverage.levels[0])
        gid = 0
        for d, n in enumerate(run.level_sizes):
            for _ in range(n):
                parent, cand = eng.trace_record(gid)
                hist[d][0 if parent == vdist.ROOT_PARENT else cand_action[cand]] += 1
                gid += 1
        assert hist.tolist() == run.coverage.levels[0].tolist()
    finally:
        eng.close()


# -------------------------------------------------------------------------------------------------- 9. liveness
@pytest.mark.gpu
def test_liveness_with_the_tier(pkg, monkeypatch):
    monkeypatch.setenv(HOOK, "0")
    got = tl.run_case(pkg, 3, 1, 1, table_host_capacity=TIER)
    assert got["rc"] == 0 and got["live"]["stored"] == tl.TABLE[(3, 1, 1)][1], got
    got = tl.run_case(pkg, 3, 1, 1, hooks=1, table_host_capacity=TIER)
    assert got["rc"] == 13 and got["live"]["sinks"] == tl.Q_SINKS_311 == 55 and got["lasso_errors"] == [], got


# -------------------------------------------------------------------------------------------------- 10. lookup, refusals, capacity
@pytest.mark.gpu
def test_lookup_finds_evicted_states(pkg, monkeypatch):
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    res, _ = tks.engine_bfs(pkg, mc, max_depth=12, table=1 << 20, frontier=1 << 18, table_host_capacity=TIER, keep=True)
    eng = res.engine
    try:
        assert _tier_seen(eng)[0] == sum(res.level_sizes[:-1])
        sb = mc.state_bytes
        for d in (1, 2, 5, 11, 12):  # in the tier, except the frontier's depth
            lv = res.levels[d - 1]
            for j in range(0, len(lv) // sb, max(1, len(lv) // sb // 20)):
                assert eng.lookup(lv[j * sb:(j + 1) * sb]) == (d, 0), (d, j)
        succ = [t for t, _, _ in mc.successors(res.levels[11][:sb])]
        assert all(eng.lookup(t)[0] in (0, 11, 12, 13) for t in succ)
    finally:
        eng.close()


@pytest.mark.gpu
def test_checkpoint_with_the_tier_is_refused(pkg, monkeypatch, tmp_path):
    from vsr_tlaplus_b200 import dist as vdist
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(2, 1, 1)
    ck = str(tmp_path / "t.ckpt")
    assert mc.check(checkpoint_path=ck, table_host_capacity=1 << 10, **CAPS).rc == 151
    assert mc.check(recover_path=ck, table_host_capacity=1 << 10, **CAPS).rc == 151
    with pytest.raises(pkg.VsrError) as e:
        mc.check_multi(2, checkpoint_path=ck, table_host_capacity=1 << 10, **CAPS)
    assert e.value.rc == 151 and "host tier" in str(e.value)
    eng = vdist.GpuEngine(mc, 0, 1, table_host_capacity=1 << 10, **CAPS)
    try:
        with pytest.raises(pkg.VsrError) as e:
            eng.run(checkpoint_path=ck)
        assert e.value.rc == 151 and "host tier" in str(e.value)
        assert eng.run().rc == 0  # the same engine without the checkpoint
        assert mc._lib.vsr_engine_checkpoint(eng._e, ck.encode(), None) == 151 and not os.path.exists(ck)
    finally:
        eng.close()
    assert mc.check(checkpoint_path=ck, **CAPS).rc == 0 and os.path.exists(ck)  # without the tier, as before


@pytest.mark.gpu
def test_both_capacity_limits_stop_the_run_with_152(pkg, monkeypatch):
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    """(3, 2, 1)'s two largest neighbouring levels hold 173,054 states: with 196,608 slots they pass the 7/8 limit without
    filling the table; a tier of 5,000 entries fills at an early boundary"""
    monkeypatch.setenv(HOOK, "0")
    for caps, tier, words in ((dict(table_capacity=196_608, frontier_capacity=1 << 17), TIER, ("capacity exceeded (seen-set)", "host tier", "false ones included")),
                              (dict(table_capacity=1 << 20, frontier_capacity=1 << 17), 5_000, ("capacity exceeded (seen-set host tier)", "move to host memory"))):
        eng = vdist.GpuEngine(mc, 0, 1, table_host_capacity=tier, **caps)
        try:
            res = eng.run()
            msg = eng.lib.vsr_engine_last_error(eng._e).decode()
        finally:
            eng.close()
        assert res.rc == 152 and not res.complete, (res.rc, msg)
        assert all(w in msg for w in words), msg


def _vsrmc(cfg, args, env):
    r = subprocess.run([VSRMC, "-config", str(cfg), "-deadlock", "-frontier", "200000"] + args, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, **env))
    return r.returncode, r.stdout + r.stderr


@pytest.mark.gpu
def test_cli_tablehost(pkg, tmp_path):
    cfg = tmp_path / "m.cfg"
    cfg.write_text(pkg.cfg_text(3, ["v1", "v2"], 1, symmetry=False))
    rc, out = _vsrmc(cfg, ["-table", "2097152"], {})
    states = [ln for ln in out.splitlines() if "distinct states found" in ln]
    assert rc == 0 and states and "%d distinct states found" % FULL_321[0] in states[0], out[-2000:]
    assert "host tier" not in out
    rc2, out2 = _vsrmc(cfg, ["-table", "262144", "-tablehost", str(TIER)], {HOOK: "0"})
    assert rc2 == 0 and [ln for ln in out2.splitlines() if "distinct states found" in ln] == states, out2[-2000:]
    tier = [ln for ln in out2.splitlines() if ln.startswith("Seen-set host tier: ")]
    assert tier and int(tier[0].split()[3]) == FULL_321[0], out2[-2000:]  # the last boundary moved the deepest level too


def test_cli_tablehost_with_checkpoint_is_refused(pkg, tmp_path):
    cfg = tmp_path / "m.cfg"
    cfg.write_text(pkg.cfg_text(2, ["v1"], 1))
    for args in (["-checkpoint", "0", "-metadir", str(tmp_path / "states")], ["-recover", str(tmp_path)]):
        r = subprocess.run([VSRMC, "-config", str(cfg), "-tablehost", "1024"] + args, capture_output=True, text=True)
        assert r.returncode == 151 and "-tablehost" in r.stderr and "checkpoint" in r.stderr, r.stdout + r.stderr
    assert "-tablehost N" in subprocess.run([VSRMC, "-help"], capture_output=True, text=True).stderr
