"""The seen-set near full: complete BFS of (R=3, V=2, L=1) without SYMMETRY in tables at loads 0.67 and 0.86.

At these loads many inserts walk past their home bucket, and probe chains of many buckets are common.  (The engine
refuses a level that would take the table past 7/8 full, so 0.86 is about as high as a complete run goes.)  Every level's
size and successor count must equal a run in a nearly empty table, and the totals must equal the answers the TLA+
evaluator gave on the spec's text (tests/golden/spec_text_results.json)."""
import pytest

pytestmark = pytest.mark.gpu

DISTINCT, GENERATED, DEPTH = 697364, 1831657, 30
LOADED = (1 << 20, 806_912)  # slots for the whole space: loads 0.67 and 0.86 at the end of the BFS (multiples of 4 x 64)


def _mc(pkg):
    return pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)


def _assert_same(res, ref):
    assert (res.rc, res.complete, res.error_code, res.queue) == (0, True, 0, 0)
    assert (res.distinct, res.generated, res.depth) == (DISTINCT, GENERATED, DEPTH)
    assert res.level_sizes == ref.level_sizes
    assert res.level_generated == ref.level_generated
    assert res.h2_ties == 0 and res.fp_collisions == 0


@pytest.fixture(scope="module")
def roomy(pkg):
    ref = _mc(pkg).check(stop_on_violation=False, table_capacity=1 << 23, frontier_capacity=1 << 18)
    assert (ref.rc, ref.complete, ref.distinct, ref.generated, ref.depth) == (0, True, DISTINCT, GENERATED, DEPTH)
    return ref


@pytest.mark.parametrize("slots", LOADED)
def test_one_rank_high_load_matches_roomy_table(pkg, roomy, slots):
    res = _mc(pkg).check(stop_on_violation=False, table_capacity=slots, frontier_capacity=1 << 18)
    _assert_same(res, roomy)
    assert res.table_capacity == slots
    # seen-set buckets probed per generated successor: well above 1, so many inserts went past their first bucket
    assert res.probe_total / res.generated > (1.5 if slots < (1 << 20) else 1.2)


@pytest.mark.parametrize("world", (2, 4))
@pytest.mark.parametrize("slots", LOADED)
def test_ranks_of_one_process_high_load_match_roomy_table(pkg, roomy, monkeypatch, world, slots):
    """vsr_bfs_multi with every rank on device 0: records from peers go through the same seen-set insert.
    Each rank owns about 1/world of the states, so its table is sized for the same load."""
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    res = _mc(pkg).check_multi(world, table_capacity=slots // world, frontier_capacity=1 << 18, stop_on_violation=False)
    _assert_same(res, roomy)
    # probe_total is rank 0's, which generated about 1/world of the successors
    assert res.probe_total * world / res.generated > (1.5 if slots < (1 << 20) else 1.2)
