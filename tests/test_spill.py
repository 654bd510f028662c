"""Frontier spill (BASELINE configs[3]): a frontier buffer continues in pinned host memory once its part in HBM is full.  The
engine addresses the two parts in several places besides the one-launch BFS the parity tests run: a launch that expands a
part of the level (vsr_engine_step) and starts before, at, across or past the end of the HBM part; the checkpoint writer and
same-world recovery, which copy the frontier through host memory; and the level audit, which reads the level just finished.
Each must see the level exactly as a run without spill does.  State space: R=3, V=2, L=1 without SYMMETRY (697,364 states,
depth 30), with an HBM part far smaller than its widest level."""
import os

import pytest

pytestmark = pytest.mark.gpu

HBM = 5000          # frontier states per buffer in HBM
HOST = 1 << 19      # ... and in pinned host memory
CAPS = dict(table_capacity=1 << 21)
PART = 9973         # states per part past the boundary


def parts(n, depth):
    """[first, count) parts covering a level of n states.  Odd depths: two parts before the boundary, one across it
    ([HBM - 5, HBM + 3)), then parts wholly past it.  Even depths: one part ending at the boundary, then parts starting at it
    and past it."""
    cuts = [0, HBM // 3, HBM - 5, HBM + 3] if depth % 2 else [0, HBM]
    while cuts[-1] + PART < n:
        cuts.append(cuts[-1] + PART)
    cuts = sorted({c for c in cuts if c < n}) + [n]
    return [(a, b - a) for a, b in zip(cuts, cuts[1:])]


def bfs_levels(mc, spill):
    """The BFS pumped level by level through a one-rank GpuEngine, every level audited.  spill: frontiers of HBM + HOST states,
    every level expanded in parts(); else one launch per level in a frontier that holds every level in HBM.  Per level:
    (its states as a set, its size, the successors generated expanding it, its audit)."""
    from vsr_tlaplus_b200 import dist as vdist
    caps = dict(frontier_capacity=HBM, frontier_host_capacity=HOST) if spill else dict(frontier_capacity=1 << 18)
    eng = vdist.GpuEngine(mc, 0, 1, keep_trace=False, collect_levels=True, **CAPS, **caps)
    sb = mc.state_bytes
    out = []
    try:
        eng.reset()
        eng.seed()
        li = eng.finish()
        while li.new_states:
            assert li.error_code == 0 and li.overflow == 0
            depth, n = len(out) + 1, eng.frontier_size()
            a = eng.audit()
            raw = eng.collected(depth)
            assert len(raw) == n * sb
            if spill:
                for first, count in parts(n, depth):
                    eng.step(first, count, 0, None)
            else:
                eng.expand()
            li = eng.finish()
            out.append((frozenset(raw[i * sb:(i + 1) * sb] for i in range(n)), n, int(li.generated), a))
    finally:
        eng.close()
    return out


@pytest.fixture(scope="module")
def runs(pkg):
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    return mc, bfs_levels(mc, spill=False), bfs_levels(mc, spill=True)


def test_parts_across_the_boundary_expand_every_level_as_one_launch(runs):
    mc, ref, got = runs
    assert sum(n for _, n, _, _ in ref) == 697364 and len(ref) == 30
    # both part patterns reach past the boundary on several levels
    wide = [d for d, (_, n, _, _) in enumerate(got, start=1) if n > HBM + PART]
    assert len([d for d in wide if d % 2]) >= 2 and len([d for d in wide if d % 2 == 0]) >= 2
    assert max(n for _, n, _, _ in got) <= HBM + HOST
    for d, ((s0, n0, g0, _), (s1, n1, g1, _)) in enumerate(zip(ref, got), start=1):
        assert (n1, g1) == (n0, g0), "depth %d" % d
        assert s1 == s0, "depth %d: the spilled run's states differ" % d
    assert len(got) == len(ref)


def audit_sums(a):
    return (a.tagged, a.found, a.fp_sum, a.fp_xor, a.words_sum, a.words_xor, a.tagged_fp_sum, a.tagged_fp_xor)


def test_audit_reads_a_spilled_level(runs):
    _, ref, got = runs
    assert len(got) == len(ref)
    for d, ((_, n, _, a0), (_, _, _, a1)) in enumerate(zip(ref, got), start=1):
        assert a1.level == d and a1.size == n
        assert a1.found == a1.tagged == n, "depth %d: %d of %d states found in the seen-set" % (d, a1.found, n)
        assert audit_sums(a1) == audit_sums(a0), "depth %d" % d


def same_exploration(a, b):
    assert (a.rc, a.complete, a.generated, a.distinct, a.queue, a.depth) == (b.rc, b.complete, b.generated, b.distinct, b.queue, b.depth)
    assert a.level_sizes == b.level_sizes
    assert a.level_generated[:a.depth - 1] == b.level_generated[:b.depth - 1]
    assert a.violation_level == b.violation_level


def test_checkpoint_of_a_frontier_across_the_boundary(pkg, tmp_path):
    """a checkpoint written while the frontier straddles the end of its HBM part, recovered with the same split, another split
    and no host part at all"""
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    whole = mc.check(stop_on_violation=False, frontier_capacity=1 << 18, **CAPS)
    assert whole.complete and whole.distinct == 697364
    depth = next(d for d, n in enumerate(whole.level_sizes, start=1) if n > 3 * HBM)
    assert depth < whole.depth - 3
    ck = str(tmp_path / "spill.ckpt")
    part = mc.check(stop_on_violation=False, max_depth=depth, checkpoint_path=ck, checkpoint_seconds=1e9, frontier_capacity=HBM,
                    frontier_host_capacity=HOST, **CAPS)
    assert part.depth == depth and part.level_sizes == whole.level_sizes[:depth] and os.path.exists(ck)
    for caps in (dict(frontier_capacity=HBM, frontier_host_capacity=HOST),
                 dict(frontier_capacity=2 * HBM + 17, frontier_host_capacity=HOST // 2),
                 dict(frontier_capacity=1 << 18)):
        same_exploration(mc.check(stop_on_violation=False, recover_path=ck, **caps, **CAPS), whole)
