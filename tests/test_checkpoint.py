"""Checkpoint / recover (TLC's -checkpoint / -recover; SURVEY §8f item 4): a BFS stopped at a level boundary and continued
from its checkpoint file must report exactly what the uninterrupted BFS reports — the four TLC scalars, every level's size
and successor count, the violation depth — whatever the capacity of the seen-set it continues with, on one GPU and with the
state space sharded over several ranks; and the oracle agrees with both."""
import os
import subprocess

import pytest

import orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def same_exploration(a, b):
    assert (a.rc, a.complete, a.generated, a.distinct, a.queue, a.depth) == (b.rc, b.complete, b.generated, b.distinct, b.queue, b.depth)
    assert a.level_sizes == b.level_sizes
    assert a.level_generated[:a.depth - 1] == b.level_generated[:b.depth - 1]
    assert a.violation_level == b.violation_level


def test_recovered_run_equals_uninterrupted_run(pkg, tmp_path):
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    ck = str(tmp_path / "vsr.ckpt")
    whole = mc.check(stop_on_violation=False, table_capacity=1 << 21, frontier_capacity=1 << 18)
    assert (whole.complete, whole.distinct, whole.generated, whole.depth) == (True, 697364, 1831657, 30)  # pinned to the spec's text
    part = mc.check(stop_on_violation=False, max_depth=17, checkpoint_path=ck, checkpoint_seconds=1e9, table_capacity=1 << 21, frontier_capacity=1 << 18)
    assert not part.complete and part.depth == 17 and os.path.getsize(ck) > part.distinct * 16
    # continue in a seen-set of another (odd) capacity: the entries are re-inserted, not copied
    rest = mc.check(stop_on_violation=False, recover_path=ck, table_capacity=(1 << 20) + 8192 + 64, frontier_capacity=1 << 18)
    same_exploration(rest, whole)
    # ... and a second generation: checkpoint again after every level, stop, continue
    ck2 = str(tmp_path / "second.ckpt")
    mid = mc.check(stop_on_violation=False, recover_path=ck, max_depth=23, checkpoint_path=ck2, checkpoint_seconds=0, table_capacity=1 << 21, frontier_capacity=1 << 18)
    assert mid.depth == 23 and mid.level_sizes == whole.level_sizes[:23]
    same_exploration(mc.check(stop_on_violation=False, recover_path=ck2, table_capacity=1 << 21, frontier_capacity=1 << 18), whole)


def test_collecting_check_and_one_rank_engine_checkpoint_to_the_given_path(pkg, tmp_path):
    """check(collect_levels=True) writes and continues from checkpoints as check() does, and one rank writes <path> itself,
    not <path>.rank0"""
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    caps = dict(table_capacity=1 << 21, frontier_capacity=1 << 18)
    whole = mc.check(stop_on_violation=False, **caps)
    ck = str(tmp_path / "collect.ckpt")
    part = mc.check(collect_levels=True, stop_on_violation=False, max_depth=17, checkpoint_path=ck, checkpoint_seconds=1e9, **caps)
    assert part.depth == 17 and os.path.exists(ck)
    rest = mc.check(collect_levels=True, stop_on_violation=False, recover_path=ck, **caps)
    same_exploration(rest, whole)
    assert [len(lv) // mc.state_bytes for lv in rest.levels] == [0] * 17 + whole.level_sizes[17:]
    eng = vdist.GpuEngine(mc, 0, 1, **caps)
    ck1 = str(tmp_path / "engine.ckpt")
    try:
        assert eng.run(stop_on_violation=False, max_depth=17, checkpoint_path=ck1, checkpoint_seconds=1e9).depth == 17
    finally:
        eng.close()
    assert os.path.exists(ck1) and not os.path.exists(ck1 + ".rank0")
    same_exploration(mc.check(stop_on_violation=False, recover_path=ck1, **caps), whole)


def test_counterexample_after_recovery_is_a_behaviour(pkg, tmp_path):
    """The trace records travel with the checkpoint: a violation found after recovery is traced back to Init through states
    explored before it.  Every step must be a step of Next, the last state (only) violates the invariant; the oracle finds the
    violation at the same depth."""
    inv = ("AcknowledgedWritesExistOnMajority",)
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=inv)
    ck = str(tmp_path / "vsr.ckpt")
    o = orc.bfs(orc.params(3, 2, 1, invariant=2), workers=8, keep_trace=False, check_assumptions=False)
    assert o.rc == 12 and o.depth > 8
    part = mc.check(max_depth=o.depth - 6, checkpoint_path=ck, checkpoint_seconds=1e9, table_capacity=1 << 20, frontier_capacity=1 << 18)
    assert part.rc == 0 and not part.trace
    res = mc.check(recover_path=ck, table_capacity=1 << 21, frontier_capacity=1 << 18)
    assert res.rc == 12 and res.violation_level == o.depth and len(res.trace) == o.depth
    assert res.level_sizes == o.level_sizes
    lit = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False, invariants=inv)
    assert res.trace[0][1] == lit.init_state()
    for (_, a), (_, b) in zip(res.trace, res.trace[1:]):
        assert b in [t for t, _, _ in lit.successors(a)]
    assert lit.invariant(res.trace[-1][1]) != 0 and all(lit.invariant(s) == 0 for _, s in res.trace[:-1])


def test_sharded_checkpoint(pkg, tmp_path, monkeypatch):
    """Several ranks (threads of one process, all on device 0 through the test hook): every rank writes <path>.rank<r> at the
    same level boundary and continues from it."""
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    for world in (2, 4):
        ck = str(tmp_path / ("w%d.ckpt" % world))
        part = mc.check_multi(world, stop_on_violation=False, max_depth=16, checkpoint_path=ck, checkpoint_seconds=0, table_capacity=1 << 19, frontier_capacity=1 << 17)
        assert part.depth == 16 and all(os.path.exists("%s.rank%d" % (ck, r)) for r in range(world))
        rest = mc.check_multi(world, stop_on_violation=False, recover_path=ck, table_capacity=1 << 20, frontier_capacity=1 << 17)
        assert (rest.rc, rest.complete, rest.distinct, rest.generated, rest.depth) == (0, True, 697364, 1831657, 30)
        assert rest.level_sizes[:16] == part.level_sizes


def test_recover_refuses_what_it_cannot_continue(pkg, tmp_path):
    ck = str(tmp_path / "vsr.ckpt")
    a = pkg.ModelChecker.from_constants(2, 2, 2)
    assert a.check(max_depth=8, checkpoint_path=ck, checkpoint_seconds=1e9, table_capacity=1 << 14, frontier_capacity=1 << 12).depth == 8
    other = pkg.ModelChecker.from_constants(2, 2, 2, symmetry=False)  # another state graph
    assert other.check(recover_path=ck, table_capacity=1 << 14, frontier_capacity=1 << 12).rc == 150
    bad = tmp_path / "garbage"
    bad.write_bytes(b"not a checkpoint" * 100)
    assert a.check(recover_path=str(bad), table_capacity=1 << 14, frontier_capacity=1 << 12).rc == 150
    with pytest.raises(pkg.VsrError):  # 153: the file cannot be opened
        a.check(recover_path=str(tmp_path / "missing"), table_capacity=1 << 14, frontier_capacity=1 << 12)
    assert a.check(recover_path=ck, table_capacity=64, frontier_capacity=1 << 12).rc == 152  # the seen-set does not fit


def test_cli_checkpoint_and_recover(pkg, tmp_path):
    """vsrmc -checkpoint 0 -metadir D -depth N, then vsrmc -recover D: the summary lines of the continued run are those of
    an uninterrupted one"""
    exe = os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc")
    cfg = tmp_path / "m.cfg"
    cfg.write_text(pkg.cfg_text(3, ["v1"], 1))
    meta = str(tmp_path / "states")
    common = [exe, "-deadlock", "-config", str(cfg), "-table", "1048576", "-frontier", "262144"]
    whole = subprocess.run(common, capture_output=True, text=True)
    first = subprocess.run(common + ["-checkpoint", "0", "-metadir", meta, "-depth", "11"], capture_output=True, text=True)
    assert first.returncode == 0 and "states left on queue" in first.stdout and os.path.exists(os.path.join(meta, "vsr.ckpt"))
    rest = subprocess.run(common + ["-recover", meta], capture_output=True, text=True)
    assert rest.returncode == whole.returncode
    pick = lambda out: [ln for ln in out.splitlines() if "states generated" in ln or "The depth of the complete" in ln or ln.startswith("Error: Invariant")]
    assert pick(rest.stdout) == pick(whole.stdout) and pick(whole.stdout)
