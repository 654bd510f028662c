"""GPU parity proper: the CUDA BFS (through the C ABI) against the CPU oracle.

Bar (bit-exact, integer work): for every BFS depth the SET of canonical VIEW-projected states the GPU
found equals the oracle's set (compared through the oracle's own canonical digest of each unpacked GPU
state), and the four TLC scalars — states generated, distinct states, states left on queue, depth —
are equal.  Sizes are chosen so the oracle finishes in seconds.
"""
import ctypes as C

import pytest

import orc

pytestmark = pytest.mark.gpu


def level_digest_sets(pkg, mc, res, q):
    sb = mc.state_bytes
    out = []
    CH = 8192  # a VsrFlatState is 19 kB: unpack and digest wide levels in chunks
    flats = (pkg.checker.VsrFlatState * CH)()
    for raw in res.levels:
        n = len(raw) // sb
        digs = set()
        for c0 in range(0, n, CH):
            m = min(CH, n - c0)
            buf = (C.c_uint8 * (m * sb)).from_buffer_copy(raw[c0 * sb:(c0 + m) * sb])
            base = C.addressof(buf)
            for i in range(m):
                assert mc._lib.vsr_unpack(mc._h, base + i * sb, C.byref(flats[i])) == 0
            d, _ = orc.digests_of(q, flats, m)
            digs.update(d)
        assert len(digs) == n, "GPU level holds two states with the same canonical VIEW"
        out.append(digs)
    return out


def run_pair(pkg, R, V, L, symmetry=True, max_depth=0, inv=("AcknowledgedWriteNotLost",), table=1 << 23, frontier=1 << 21, **check_kw):
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=symmetry, invariants=inv)
    res = mc.check(collect_levels=True, max_depth=max_depth, table_capacity=table, frontier_capacity=frontier,
                   stop_on_violation=False, **check_kw)
    inv_id = 1 if "AcknowledgedWriteNotLost" in inv else (2 if "AcknowledgedWritesExistOnMajority" in inv else 4)
    q = orc.params(R, V, L, symmetry=symmetry and V > 1, invariant=inv_id)
    o = orc.bfs(q, workers=8, max_depth=max_depth, keep_trace=False, digests=True)
    return mc, res, q, o


def assert_same_exploration(pkg, mc, res, q, o, complete):
    assert res.error_code == 0
    assert sum(o.assumptions[:5]) + sum(o.assumptions[6:]) == 0, "oracle audit of the slot-encoding assumptions failed"
    assert res.level_sizes == o.level_sizes
    # successors generated while expanding each depth (the last depth reached is not expanded under -depth)
    ng = len(o.level_generated)
    assert res.level_generated[:ng] == o.level_generated
    gpu_sets = level_digest_sets(pkg, mc, res, q)
    assert len(gpu_sets) == len(o.level_digests)
    for d, (g, w) in enumerate(zip(gpu_sets, o.level_digests)):
        assert g == set(w), f"depth {d + 1}: GPU and oracle state sets differ"
    assert res.distinct == o.distinct
    assert res.generated == o.generated
    assert res.depth == o.depth
    assert res.h2_ties == o.h2_ties
    if complete:
        assert res.complete and o.complete and res.queue == 0 == o.queue


@pytest.mark.parametrize("R,V,L,sym", [(2, 1, 1, True), (2, 2, 2, True), (2, 2, 2, False), (3, 1, 1, True)])
def test_full_state_space_matches_oracle(pkg, R, V, L, sym):
    mc, res, q, o = run_pair(pkg, R, V, L, symmetry=sym)
    assert res.rc == 0
    assert_same_exploration(pkg, mc, res, q, o, complete=True)


def test_cfg1_scalars(pkg):
    """BASELINE configs[0]: ReplicaCount=2 Values={v1} StartViewOnTimerLimit=1, full BFS (deadlock checking off)."""
    mc = pkg.ModelChecker.from_constants(2, 1, 1)
    res = mc.check()
    assert (res.generated, res.distinct, res.queue, res.depth, res.rc, res.complete) == (100, 76, 0, 14, 0, True)


@pytest.mark.parametrize("R,V,L,depth", [(3, 2, 2, 15), (3, 3, 3, 13), (5, 2, 2, 9), (3, 2, 1, 14), (4, 2, 2, 8), (3, 3, 2, 10)])
def test_bounded_depth_matches_oracle(pkg, R, V, L, depth):
    """cfg2 (shipped VSR.cfg), cfg3 (README), cfg4 (R=5) and friends, as deep as the oracle goes in about a minute on eight
    threads (1.1 - 1.7 million states each for the three BASELINE configs): every depth's SET of states equal."""
    mc, res, q, o = run_pair(pkg, R, V, L, max_depth=depth)
    assert_same_exploration(pkg, mc, res, q, o, complete=False)
    assert res.queue == res.level_sizes[-1]


def test_no_symmetry_no_view_matches_oracle(pkg):
    mc = pkg.ModelChecker.from_cfg_text(pkg.cfg_text(3, ["a", "b"], 2, view=False, symmetry=False))
    res = mc.check(collect_levels=True, max_depth=9, table_capacity=1 << 22, frontier_capacity=1 << 20)
    q = orc.params(3, 2, 2, symmetry=False, view=False)
    o = orc.bfs(q, workers=8, max_depth=9, keep_trace=False, digests=True)
    assert_same_exploration(pkg, mc, res, q, o, complete=False)


def test_deterministic_across_runs(pkg):
    mc = pkg.ModelChecker.from_constants(3, 2, 2)
    a = mc.check(collect_levels=True, max_depth=10, table_capacity=1 << 21, frontier_capacity=1 << 19)
    b = mc.check(collect_levels=True, max_depth=10, table_capacity=1 << 23, frontier_capacity=1 << 19)
    sb = mc.state_bytes
    for la, lb in zip(a.levels, b.levels):
        sa = {la[i:i + sb] for i in range(0, len(la), sb)}
        sbb = {lb[i:i + sb] for i in range(0, len(lb), sb)}
        assert sa == sbb
    assert (a.generated, a.distinct, a.depth) == (b.generated, b.distinct, b.depth)


def test_counterexample_is_a_behaviour(pkg):
    """AcknowledgedWritesExistOnMajority is violated early; the GPU's counterexample must be a literal behaviour
    of the spec (every step in the oracle's Next, last state violating), of minimal length (BFS)."""
    inv = ("AcknowledgedWritesExistOnMajority",)
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=inv)
    res = mc.check(table_capacity=1 << 22, frontier_capacity=1 << 20)
    q = orc.params(3, 2, 1, invariant=2)
    o = orc.bfs(q, workers=8, keep_trace=False)
    if o.rc != 12:
        pytest.skip("invariant not violated in this configuration")
    assert res.rc == 12
    assert res.violation_level == o.depth
    assert len(res.trace) == o.depth
    assert res.trace[0][0] == "Initial predicate"
    L = orc.lib()
    flats = [mc.unpack(st) for _, st in res.trace]
    for i in range(len(flats) - 1):
        cap = 256
        succ = (pkg.checker.VsrFlatState * cap)()
        acts = (C.c_int * cap)()
        n = L.orc_successors_flat(q, C.byref(flats[i]), succ, acts, cap)
        want = orc.digests_full_of(orc.params(3, 2, 1, symmetry=False, invariant=2), (pkg.checker.VsrFlatState * 1)(flats[i + 1]))[0]
        got = orc.digests_full_of(orc.params(3, 2, 1, symmetry=False, invariant=2), succ)[:n]
        names = [pkg.ACTION_NAMES[acts[k]] for k in range(n)]
        assert any(g == want and nm == res.trace[i + 1][0] for g, nm in zip(got, names)), f"step {i + 1} is not a step of Next"
    assert L.orc_invariant_flat(q, C.byref(flats[-1])) == 0
    for f in flats[:-1]:
        assert L.orc_invariant_flat(q, C.byref(f)) == 1


@pytest.mark.parametrize("stop", [True, False])
def test_one_gpu_paths_agree(pkg, stop):
    """check() (vsr_bfs), check(collect_levels=True) and GpuEngine(mc, 0, 1).run() run the one level loop: the same verdict,
    totals, per-level tables and launches, whether the run stops at the violation or continues past it.  Which violating
    state a run reports, and which parent each state keeps, follow the order in which warps insert states, so the three
    counterexamples are compared as behaviours: as long as the BFS depth, every step a step of Next, only the last state
    violating."""
    from vsr_tlaplus_b200 import dist as vdist
    inv = ("AcknowledgedWritesExistOnMajority",)
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=inv)
    caps = dict(table_capacity=1 << 21, frontier_capacity=1 << 18)
    one = mc.check(stop_on_violation=stop, **caps)
    col = mc.check(stop_on_violation=stop, collect_levels=True, **caps)
    eng = vdist.GpuEngine(mc, 0, 1, **caps)
    try:
        run = eng.run(stop_on_violation=stop)
    finally:
        eng.close()
    k = len(run.level_generated)  # levels expanded
    assert run.rc == 12 and run.violation_level > 8 and run.complete == (not stop) and len(run.level_ms) == k
    lit = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False, invariants=inv)
    for r in (one, col):
        assert (r.rc, r.generated, r.distinct, r.queue, r.depth, r.complete) == (run.rc, run.generated, run.distinct, run.queue, run.depth, run.complete)
        assert r.level_sizes == run.level_sizes
        assert r.level_generated[:k] == run.level_generated and not any(r.level_generated[k:]) and not any(r.level_ms[k:])
        assert (r.violation_level, r.h2_ties, r.kernel_launches) == (run.violation_level, run.h2_ties, run.launches)
        assert r.violated_invariants == list(inv)
    for trace in (one.trace, col.trace, vdist.replay_trace(mc, run.trace_cands)):
        assert len(trace) == run.violation_level and trace[0] == ("Initial predicate", lit.init_state())
        for (_, a), (act, b) in zip(trace, trace[1:]):
            assert (b, act) in [(t, pkg.ACTION_NAMES[x]) for t, x, _ in lit.successors(a)]
        assert [lit.invariant(s) != 0 for _, s in trace] == [False] * (len(trace) - 1) + [True]


def test_frontier_overflow_is_loud(pkg):
    mc = pkg.ModelChecker.from_constants(3, 2, 2)
    res = mc.check(max_depth=12, table_capacity=1 << 20, frontier_capacity=256)
    assert res.rc == 152


def test_published_behaviour_is_inside_the_explored_set(pkg):
    """golden cross-check on the README constants (R=3, V=3, L=3): after a BFS to depth 12, the k-th state of the
    reference's published 24-state counterexample (k <= 12) is in the seen-set, first seen at a depth <= k"""
    import base64, json, os, zlib
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 3, 3)
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=1 << 22, frontier_capacity=1 << 20)
    try:
        res = vdist.ShardedBfs(eng, 0, 1).run(max_depth=12)
        assert res.rc == 0 and res.depth == 12
        fx = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "state_transfer_trace.json")))
        Flat = pkg.checker.VsrFlatState
        for k, s in enumerate(fx["states"][:12], start=1):
            packed = mc.pack(Flat.from_buffer_copy(zlib.decompress(base64.b64decode(s["flat_zlib_b64"]))))
            lvl, owner = eng.lookup(packed)
            assert owner == 0 and 0 < lvl <= k, (k, lvl)
        # and a state that cannot have been reached yet is absent
        last = mc.pack(Flat.from_buffer_copy(zlib.decompress(base64.b64decode(fx["states"][23]["flat_zlib_b64"]))))
        assert eng.lookup(last)[0] == 0
    finally:
        eng.close()


def test_view_ties_resolve_to_smallest_aux_key(pkg):
    """SURVEY H2: states with equal VIEW but different aux variables arriving in the SAME level.  No configuration explored so
    far produces one, so inject them through the engine's record interface: three candidates, aux_svc = 2, 0, 1, same VIEW.
    The level must keep exactly one state — the one with the smallest aux key, whatever the arrival order — with its own
    trace record, and report the ties."""
    import struct
    import torch
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 2)
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=1 << 12, frontier_capacity=1 << 10)
    try:
        eng.reset()
        eng.seed()
        assert eng.finish().new_states == 1
        base = [t for t, a, _ in mc.successors(mc.init_state()) if pkg.ACTION_NAMES[a] == "TimerSendSVC"][0]
        variants = []
        for aux in (2, 0, 1):
            f = mc.unpack(base)
            f.aux_svc = aux
            variants.append(mc.pack(f))
        assert len({mc.fingerprint(v) for v in variants}) == 1 and len({mc.aux_key(v) for v in variants}) == 3
        recs = b"".join(v + struct.pack("<QQ", mc.fingerprint(v), (0 << 12) | (100 + i) | (1 << 56)) for i, v in enumerate(variants))  # vsr_gpu.cuh RecHdr
        t = torch.frombuffer(bytearray(recs), dtype=torch.uint8).cuda()
        eng.insert(t, 3)
        li = eng.finish()
        assert (li.new_states, li.ties, li.generated) == (1, 2, 3)
        out = (C.c_uint8 * mc.state_bytes)()
        assert mc._lib.vsr_engine_read_frontier(eng._e, 0, 1, out) == 0
        assert bytes(out) == variants[1]                       # aux_svc = 0 wins
        assert eng.trace_record(1) == (0, 101)                 # ... with the trace record of the winner
    finally:
        eng.close()


def test_frontier_spill_and_odd_capacities_give_the_same_exploration(pkg):
    """BASELINE configs[3]'s capacity path at test size: 700 frontier states in HBM, the rest of every level in pinned host
    memory (levels of up to thousands of states: most of them straddle the boundary), and a seen-set whose capacity is not a
    power of two.  Same per-depth state SETS as the oracle."""
    mc, res, q, o = run_pair(pkg, 3, 1, 1, table=100_000, frontier=700, frontier_host_capacity=1 << 16)
    assert res.rc == 0 and res.table_capacity == 100_032 and res.frontier_capacity == 700 + (1 << 16)
    assert max(res.level_sizes) > 2000
    assert_same_exploration(pkg, mc, res, q, o, complete=True)
    # without the host part the same run must stop with TLC's "state space too large", not lose states
    small = mc.check(table_capacity=100_000, frontier_capacity=700, stop_on_violation=False)
    assert small.rc == 152 and not small.complete


def test_threads_of_one_process_shard_the_search(pkg, monkeypatch):
    """vsr_bfs_multi (what `vsrmc -gpus N` runs): one thread per rank, inboxes reached through plain peer pointers.  On a
    one-GPU box the test hook VSR_B200_MULTI_ONE_DEVICE puts every rank on device 0."""
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    for world in (2, 4):
        mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=("AcknowledgedWritesExistOnMajority",))
        res = mc.check_multi(world, table_capacity=1 << 20, frontier_capacity=1 << 18)
        o = orc.bfs(orc.params(3, 2, 1, invariant=2), workers=8, keep_trace=False, check_assumptions=False)
        assert res.rc == 12 == o.rc and res.violation_level == o.depth and len(res.trace) == o.depth
        assert res.violated_invariants == ["AcknowledgedWritesExistOnMajority"]
        assert res.level_sizes == o.level_sizes
        full = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False).check_multi(world, table_capacity=1 << 21, frontier_capacity=1 << 18, stop_on_violation=False)
        assert (full.rc, full.complete, full.distinct, full.generated, full.depth) == (0, True, 697364, 1831657, 30)


def test_shipped_cfg_full_size_properties(pkg):
    """BASELINE configs[1] at FULL size (the shipped VSR.cfg constants, 1.17e9 states: far beyond what the oracle can enumerate),
    through size-independent properties:
      * two complete explorations with different seen-set capacities (different probe sequences, different arrival orders)
        give identical per-depth counts, totals and depth: the result does not depend on scheduling;
      * distinct = sum of level sizes; generated = 1 + sum of per-level generated; the last level generates successors but no
        new state; no VIEW ties and no fingerprint collisions were detected;
      * the first violating depth is the same in both, and the counterexample of one run replays through the ORACLE's Next
        step by step with only its last state violating AcknowledgedWriteNotLost (checked up to value relabelling);
      * the bounded-depth prefix agrees with the oracle-verified level sizes of test_bounded_depth_matches_oracle."""
    mc = pkg.ModelChecker.from_cfg_text(pkg.cfg_text(3, ["v1", "v2"], 2))
    a = mc.check(stop_on_violation=False, table_capacity=1 << 31, frontier_capacity=130_000_000)
    b = mc.check(stop_on_violation=False, table_capacity=3_000_000_000, frontier_capacity=125_000_000, keep_trace=False)
    for r in (a, b):
        assert r.complete and r.error_code == 0 and r.queue == 0
        assert r.distinct == sum(r.level_sizes) == 1173992337
        assert r.generated == 1 + sum(r.level_generated) == 3129587684
        assert r.depth == len(r.level_sizes) == 47 and r.level_generated[-1] == 0
        assert r.h2_ties == 0 and r.fp_collisions == 0
        assert r.violation_level == 28
    assert a.level_sizes == b.level_sizes and a.level_generated == b.level_generated
    assert a.level_sizes[:11] == [1, 3, 10, 35, 124, 403, 1200, 3319, 8500, 20030, 43306]
    # the counterexample (run a kept parent records): literal behaviour, oracle-validated
    assert a.rc == 12 and len(a.trace) == 28
    q = orc.params(3, 2, 2, symmetry=False)
    L = orc.lib()
    flats = [mc.unpack(s) for _, s in a.trace]
    for i in range(27):
        cap = 256
        succ = (pkg.checker.VsrFlatState * cap)()
        acts = (C.c_int * cap)()
        n = L.orc_successors_flat(q, C.byref(flats[i]), succ, acts, cap)
        want = orc.digests_full_of(q, (pkg.checker.VsrFlatState * 1)(flats[i + 1]))[0]
        got = orc.digests_full_of(q, succ)[:n]
        assert any(g == want and pkg.ACTION_NAMES[acts[k]] == a.trace[i + 1][0] for k, g in enumerate(got)), f"step {i + 1}"
    assert [L.orc_invariant_flat(q, C.byref(f)) for f in flats] == [1] * 27 + [0]
