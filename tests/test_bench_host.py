"""Host-side checks of bench.py that need no GPU: bench.py runs only on a GPU machine, so a misspelt
name there would cost a whole measurement run."""
import builtins
import os
import symtable
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _unresolved_globals(path):
    src = open(path).read()
    top = symtable.symtable(src, path, "exec")
    module_names = set(top.get_identifiers())
    bad = []

    def walk(t):
        for c in t.get_children():
            for s in c.get_symbols():
                if s.is_global() and s.is_referenced() and not s.is_assigned():
                    n = s.get_name()
                    if n not in module_names and not hasattr(builtins, n):
                        bad.append((c.get_name(), n))
            walk(c)

    walk(top)
    return bad


@pytest.mark.parametrize("rel", ["bench.py", "__graft_entry__.py", "vsr-tlaplus_b200/dist.py", "vsr-tlaplus_b200/checker.py"])
def test_every_global_name_resolves(rel):
    assert _unresolved_globals(os.path.join(ROOT, rel)) == []


def test_usable_cores_is_within_the_machine():
    import bench
    n = bench.usable_cores()
    assert 1 <= n <= (os.cpu_count() or 1)


def test_sharded_result_carries_the_fields_the_bench_line_prints():
    import _pkg
    _pkg.load()
    from vsr_tlaplus_b200 import dist as vdist
    r = vdist.ShardedResult()
    assert set(r.phase_seconds) == {"expand", "exchange", "finish"}
    assert r.insert_ms_max == 0.0 and r.exchanged_records == 0 and r.level_sizes == [] and r.level_ms == [] and r.launches == 0


def test_level_reduce_on_one_rank_is_the_identity():
    import _pkg
    _pkg.load()
    from vsr_tlaplus_b200 import dist as vdist

    class _E:  # no engine call is made by _reduce_level
        pass

    b = vdist.ShardedBfs(_E(), 0, 1)
    assert b._reduce_level([1, 2], [3], [4, 5]) == ([1, 2], [3], [4, 5])


def test_readme_block_is_guarded_by_the_hosts_memory():
    """bench.py pins host memory for the README constants' frontier spill only when the job may have it (a box that is a slice
    of a machine kills a job that pins past its cgroup limit instead of returning an error): the guard reads MemAvailable and
    the cgroup limit and weighs the pinning of ALL ranks on the machine; the sizes of every GPU count are there and fit an
    80 GB H100"""
    import bench
    avail = bench.host_memory_available()
    assert avail is None or 0 < avail < 1 << 50
    state_bytes = 64  # Layout<3,3,4>
    for world in (2, 4, 8):
        assert bench.CFG3["table_total"][world] // world * 7 // 8 >= bench.CFG3["distinct"] // world  # the seen-set's 7/8 load limit
        per_gpu = bench.CFG3["frontier_total"][world] // world + bench.CFG3["frontier_host"][world]
        assert per_gpu * world >= 1_344_894_424  # depth 24 of the README constants (profiles/cfg3_counterexample)
        hbm = bench.CFG3["table_total"][world] // world * 23 + 2 * bench.CFG3["frontier_total"][world] // world * state_bytes
        assert hbm < 72e9  # seen-set (16 B) + trace (7 B) per slot and two frontiers of 64 B states, with room for the inboxes
        pinned = 2 * bench.CFG3["frontier_host"][world] * state_bytes  # per rank
        if pinned:
            # a share that one rank alone could pin is refused when all ranks of the machine together exceed the limit
            assert bench.pinning_fits(pinned, 1, pinned / 0.6)
            assert not bench.pinning_fits(pinned, world, pinned * world / 0.6 - 1)
            assert bench.pinning_fits(pinned, world, pinned * world / 0.6 + 1)
    # N = 2: 2 x 71.7 GB pinned on one machine; a job with 200 GB available must skip the block, not pin 143 GB
    pinned2 = 2 * bench.CFG3["frontier_host"][2] * state_bytes
    assert not bench.pinning_fits(pinned2, 2, 200e9) and bench.pinning_fits(pinned2, 2, 240e9)
    assert not bench.pinning_fits(1, 1, None)
