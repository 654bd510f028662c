"""Every BFS level's verdicts against the oracle, state by state: the invariant mask of a state, the name TLC gives a
violation, and the violation and deadlock fields of VsrLevelInfo (vsr_engine_finish_level).

Reference.  Each packed state is unpacked with vsr_unpack and judged by the oracle alone: AcknowledgedWriteNotLost (bit 1)
and AcknowledgedWritesExistOnMajority (bit 2) each by orc_invariant_flat with that one invariant; the test hook 256 ("no
replica has committed every value", vsr_model_create only) in Python from the replicas' commit numbers; a state is terminal
when orc_successors_flat finds no successor.  The product's vsr_invariant / vsr_successors are what is checked, never the
reference.

Ids on one GPU.  The engine numbers states in BFS order: Init has local id 0 and the states first seen at depth d follow
those of depths 1 .. d-1.  In vsr_gpu.cu a launch writes new state k of the level to row k of the next frontier with id
out_base + k (out_base = next_base: flush's atomicMin(viol_id, out_base + base + lane)); finish_level makes that frontier
the current one, cur_base = the old next_base, and advances next_base by the level's size.  A launch over frontier rows
[first, first + count) has in_base = cur_base + first, and the row a scanning thread holds is in_base + round_first +
pass * NS + tid, so its id is cur_base + its row.  Hence, with base = the number of states of the earlier levels:
    after finish(), row i of read_frontier() has id base + i;
    violation_id = base + the first row of the new level that violates an invariant;
    deadlock_id  = prev_base + the first row of the level just expanded that has no successor.
A checkpoint recovered by a world-1 engine keeps cur_base (vsr_ckpt.cu: the old files' cur_base summed over the one file),
so the same numbering continues after recovery.  A round of the expand kernel is NR = passes x NS rows of its launch (NS =
32 x warps): the deadlock id of a row in pass 1 needs the pass term, and only a two-pass layout has one, so one case puts the
level's only terminal row at offset NS + 100 of a two-pass round on purpose, and the two-pass parts case uses parts larger
than NR.

A state with an acknowledged value that no replica holds violates both invariants (mask 3).  None of the explorations here
reaches one (the shipped config first violates AcknowledgedWriteNotLost at depth 28: bench.py's EXPECT), so the crafted
states (CPU) and the tie injection (GPU) carry the mask-3 checks.

On one H100 the GPU cases of this module take about a minute, oracle work included.
"""
import ctypes as C
import itertools
import os
import struct

import pytest

import orc
from test_kernel_shapes import NEW_PARITY, shapes  # noqa: F401  (shapes: the module fixture of every layout's kernel shape)

NOT_LOST, MAJORITY, HOOK = 1, 2, 256
NAMES = {NOT_LOST: "AcknowledgedWriteNotLost", MAJORITY: "AcknowledgedWritesExistOnMajority"}
ACK_ABSENT, ACK_FALSE, ACK_TRUE = 0, 1, 2  # vsr_layout.h
ORDERS = [(NOT_LOST, MAJORITY), (MAJORITY, NOT_LOST)]


def model(pkg, R, V, L, mask, symmetry=True):
    """ModelChecker through vsr_model_create, which alone takes the test hook 256"""
    lib = pkg.checker.load_library()
    h, err = C.c_void_p(), C.create_string_buffer(512)
    assert lib.vsr_model_create(R, 1, V, L, 0, int(symmetry), 1, mask, C.byref(h), err, len(err)) == 0, err.value
    return pkg.ModelChecker(h, lib)


class Reference:
    """the oracle's verdicts on packed states of `mc` (whose INVARIANT mask is `mask`)"""

    def __init__(self, pkg, mc, mask):
        i = mc.info
        R, V, L = int(i.replica_count), int(i.value_count), int(i.start_view_on_timer_limit)
        self.mc, self.mask, self.R, self.V = mc, mask, R, V
        self.q = {b: orc.params(R, V, L, symmetry=bool(i.symmetry), invariant=b) for b in (NOT_LOST, MAJORITY)}
        self.flat = pkg.checker.VsrFlatState()
        self.lib = orc.lib()

    def _unpack(self, state):
        assert self.mc._lib.vsr_unpack(self.mc._h, state, C.byref(self.flat)) == 0

    def verdict(self, state, terminal=False):
        """(mask of the configured invariants the state violates, whether it has no successor or None)"""
        self._unpack(state)
        f, m = self.flat, 0
        for b in (NOT_LOST, MAJORITY):
            if self.mask & b and self.lib.orc_invariant_flat(self.q[b], C.byref(f)) == 0:
                m |= b
        if self.mask & HOOK and any(f.rep[r].commit == self.V for r in range(self.R)):
            m |= HOOK
        t = self.lib.orc_successors_flat(self.q[NOT_LOST], C.byref(f), None, None, 0) == 0 if terminal else None
        return m, t

    def masks(self, rows):
        sb = self.mc.state_bytes
        return [self.verdict(rows[k:k + sb])[0] for k in range(0, len(rows), sb)]

    def terminals(self, rows):
        sb = self.mc.state_bytes
        return [self.verdict(rows[k:k + sb], True)[1] for k in range(0, len(rows), sb)]


def reported(order, mask):
    """TLC's rule: the first invariant of the INVARIANT list that the state violates"""
    return next((NAMES[b] for b in order if mask & b), None)


# ------------------------------------------------------------------------------------------------------------ CPU part
def host_space(mc, limit):
    """the states reachable in `mc` (canonical, distinct by VIEW fingerprint), breadth first, at most `limit`; and whether
    that is all of them"""
    init = mc.canon(mc.init_state())
    seen, order, k = {mc.fingerprint(init)}, [init], 0
    while k < len(order):
        for s, _, _ in mc.successors(order[k]):
            s = mc.canon(s)
            fp = mc.fingerprint(s)
            if fp not in seen:
                if len(order) >= limit:
                    return order, False
                seen.add(fp)
                order.append(s)
        k += 1
    return order, True


def holders(mc, state):
    """replicas whose log holds each value"""
    f = mc.unpack(state)
    return tuple(sum(any(f.rep[r].log[i].operation == x + 1 for i in range(f.rep[r].log_n)) for r in range(f.R)) for x in range(f.V))


def with_dropped_entries(pkg, mc, states):
    """the states, and each with the last log entry of one or two replicas dropped, that the packed encoding holds"""
    def dropped(f):
        for r in range(f.R):
            if f.rep[r].log_n:
                g = pkg.checker.VsrFlatState.from_buffer_copy(f)
                g.rep[r].log_n -= 1
                g.rep[r].op = g.rep[r].log_n
                g.rep[r].commit = min(g.rep[r].commit, g.rep[r].op)
                yield g

    for s in states:
        f = mc.unpack(s)
        for g in [f] + list(dropped(f)) + [h for d in dropped(f) for h in dropped(d)]:
            try:
                yield mc.pack(g)
            except pkg.VsrError:  # not representable (the slot encoding ties log entries to the messages)
                pass


def crafted_states(pkg, R):
    """states of (R, 2, 1) without symmetry: reachable ones with both values requested, and the same with the last log entry
    of one or two replicas dropped (so that with R = 2 too a requested value can have no holder), one per vector of holder
    counts, each with every assignment of `acked` (FALSE, TRUE) to the two values; the packed encoding must hold them"""
    mc = model(pkg, R, 2, 1, 0, symmetry=False)
    by_holders = {}
    for t in with_dropped_entries(pkg, mc, [s for s in host_space(mc, 10_000)[0] if all(mc.unpack(s).acked[:2])]):
        by_holders.setdefault(holders(mc, t), t)
    out = []
    for h, s in sorted(by_holders.items()):
        for a in itertools.product((ACK_FALSE, ACK_TRUE), repeat=2):
            f = mc.unpack(s)
            f.acked[0], f.acked[1] = a
            out.append((h, a, mc.pack(f)))
    return out


COMPLETE_SPACES = [(2, 1, 1, False), (2, 2, 2, True), (2, 2, 2, False), (3, 1, 1, False)]  # test_host_parity's complete spaces
SUBSETS = [NOT_LOST, MAJORITY, NOT_LOST | MAJORITY, HOOK, NOT_LOST | MAJORITY | HOOK]


@pytest.mark.parametrize("R,V,L,sym", COMPLETE_SPACES)
def test_invariant_mask_matches_oracle_on_complete_spaces(pkg, R, V, L, sym):
    """vsr_invariant returns every configured invariant a state violates, on every reachable state"""
    space, complete = host_space(model(pkg, R, V, L, 0, symmetry=sym), 100_000)
    assert complete
    ref = Reference(pkg, model(pkg, R, V, L, NOT_LOST | MAJORITY | HOOK, symmetry=sym), NOT_LOST | MAJORITY | HOOK)
    want = [ref.verdict(s)[0] for s in space]
    assert any(w & HOOK for w in want)
    for sub in SUBSETS:
        mc = model(pkg, R, V, L, sub, symmetry=sym)
        bad = [(i, mc.invariant(s), w & sub) for i, (s, w) in enumerate(zip(space, want)) if mc.invariant(s) != w & sub]
        assert not bad, "INVARIANT mask %d: (state, vsr_invariant, oracle) %s" % (sub, bad[:5])


@pytest.mark.parametrize("R", [2, 3])
def test_invariant_mask_matches_oracle_on_crafted_states(pkg, R):
    """acknowledged values with no holder, a minority and a majority, alone and together in both value orders: the full mask"""
    states = crafted_states(pkg, R)
    ref = Reference(pkg, model(pkg, R, 2, 1, NOT_LOST | MAJORITY | HOOK, symmetry=False), NOT_LOST | MAJORITY | HOOK)
    seen = set()
    for sub in SUBSETS:
        mc = model(pkg, R, 2, 1, sub, symmetry=False)
        for h, a, s in states:
            want = ref.verdict(s)[0] & sub
            assert mc.invariant(s) == want, (sub, h, a)
            seen.add((h, a, want))
    # the cases that tell a full mask from a first hit: both values acknowledged, one with no holder beside one with a
    # minority, in both orders (with R = 2 a minority is one replica of two)
    for h in ((1, 0), (0, 1)):
        assert (h, (ACK_TRUE, ACK_TRUE), NOT_LOST | MAJORITY) in seen
        assert (h, (ACK_TRUE, ACK_TRUE), MAJORITY) in seen
    assert ((1, 0), (ACK_TRUE, ACK_FALSE), MAJORITY) in seen and ((1, 0), (ACK_FALSE, ACK_TRUE), NOT_LOST | MAJORITY) in seen


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("order", ORDERS)
def test_reported_invariant_is_the_first_violated_in_cfg_order(pkg, R, order):
    """TLC names the first invariant of the INVARIANT list that the state violates: the same rule from cfg text and from
    from_constants(invariants=...), whichever order the list has"""
    names = [NAMES[b] for b in order]
    by_cfg = pkg.ModelChecker.from_cfg_text(pkg.cfg_text(R, ["v1", "v2"], 1, symmetry=False, invariants=names))
    by_constants = pkg.ModelChecker.from_constants(R, 2, 1, symmetry=False, invariants=tuple(names))
    ref = Reference(pkg, model(pkg, R, 2, 1, NOT_LOST | MAJORITY, symmetry=False), NOT_LOST | MAJORITY)
    both = 0
    for h, a, s in crafted_states(pkg, R):
        mask = ref.verdict(s)[0]
        both += mask == NOT_LOST | MAJORITY
        for mc in (by_cfg, by_constants):
            assert mc.invariant(s) == mask, (h, a)
            assert mc.reported_invariant(s) == reported(order, mask), (h, a, mask)
    assert both >= 4
    # the order is kept when only one of the two is listed, too
    one = pkg.ModelChecker.from_constants(R, 2, 1, symmetry=False, invariants=(NAMES[order[1]],))
    for h, a, s in crafted_states(pkg, R):
        assert one.reported_invariant(s) == reported((order[1],), ref.verdict(s)[0])


# the layouts whose verdicts are checked level by level on the GPU, one per kernel shape: (R, V, L, depth), each from
# test_kernel_shapes.NEW_PARITY and no deeper than there.  The 32-warp two-pass shape runs a complete space with deadlocks
# and up to 69 hook violators per level; the 28-warp one-pass shape reaches hook violators at depths 9 - 11 (235,044
# states); the 22-warp and the two-block shapes reach none within about 10,000 states, so there the case checks that no
# verdict is reported where the oracle finds none
SHAPE_CASES = [(2, 3, 2, 0), (3, 2, 3, 11), (4, 3, 2, 7), (5, 3, 2, 6)]
# (R, V, L, depth, part): a two-pass and a one-pass layout, parts longer than a round (NR rows) that NR does not divide, so
# that a part's later rounds start at round_first > 0 and, on the two-pass layout, reach pass 1
PART_CASES = [(3, 2, 1, 17, 3001), (3, 2, 3, 11, 997)]


def test_every_shape_has_a_verdict_case(shapes):  # noqa: F811
    """a layout or tuning change that creates a new kernel shape fails here until a verdict case covers it"""
    parity = {p[:3]: p[3] for p in NEW_PARITY}
    covered = {shapes[c[:3]] for c in SHAPE_CASES}
    assert set(shapes.values()) <= covered, "kernel shapes without a verdict case: %s" % sorted(set(shapes.values()) - covered)
    for R, V, L, depth in SHAPE_CASES:
        assert (R, V, L) in parity and (parity[(R, V, L)] == 0 or depth <= parity[(R, V, L)])
    assert {shapes[c[:3]][2] for c in PART_CASES} == {1, 2}
    for R, V, L, _, part in PART_CASES:
        warps, _, passes, _ = shapes[(R, V, L)]
        assert part > passes * 32 * warps and part % (passes * 32 * warps)


# ------------------------------------------------------------------------------------------------------------ GPU part
class Tally:
    def __init__(self):
        self.viol_levels = self.dead_levels = self.max_violators = self.levels = 0
        self.masks = set()
        self.recovered = False
        self.sides = set()  # ("viol" | "dead", row < frontier_capacity)


def check_level(li, depth, rows, masks, base, prev_terms, prev_base, tally, split):
    assert li.error_code == 0 and li.overflow == 0, (depth, li.error_code, li.overflow)
    assert len(masks) == li.new_states, depth
    bad = [i for i, m in enumerate(masks) if m]
    mask = 0
    for m in masks:
        mask |= m
    assert bool(li.violation) == bool(bad), "depth %d: violation %d, the oracle finds %d violating states" % (depth, li.violation, len(bad))
    assert li.violation_mask == mask, "depth %d: violation_mask %d, the oracle's OR of the masks %d" % (depth, li.violation_mask, mask)
    if bad:
        assert li.violation_id == base + bad[0], "depth %d: violation_id %d, first violating row %d + base %d" % (depth, li.violation_id, bad[0], base)
        tally.viol_levels += 1
        tally.max_violators = max(tally.max_violators, len(bad))
        tally.masks.add(mask)
        if split:
            tally.sides |= {("viol", i < split) for i in bad}
    terms = [i for i, t in enumerate(prev_terms or []) if t]
    assert bool(li.deadlock) == bool(terms), "depth %d: deadlock %d, the oracle finds %d terminal states in the expanded level" % (depth, li.deadlock, len(terms))
    if terms:
        assert li.deadlock_id == prev_base + terms[0], "depth %d: deadlock_id %d, first terminal row %d + base %d" % (depth, li.deadlock_id, terms[0], prev_base)
        tally.dead_levels += 1
        if split:
            tally.sides |= {("dead", i < split) for i in terms}
    tally.levels += 1


def explore(pkg, mc, ref, depth, part=0, frontier=1 << 18, host=0, checkpoint_at=0, tmp_path=None):
    """the BFS level by level on a world-1 engine (deadlock checking on, past every violation and deadlock) to `depth` or
    the end of the space, every level's verdicts checked against the reference.  part: expand in steps of that many
    frontier states; checkpoint_at: write a checkpoint after that depth and continue in a fresh engine recovered from it"""
    from vsr_tlaplus_b200 import dist as vdist
    kw = dict(table_capacity=1 << 22, frontier_capacity=frontier, frontier_host_capacity=host, check_deadlock=True, keep_trace=True)
    eng = vdist.GpuEngine(mc, 0, 1, **kw)
    tally = Tally()
    try:
        eng.reset()
        eng.seed()
        li, d, base, prev_base, prev_terms = eng.finish(), 1, 0, 0, None
        while True:
            rows = eng.read_frontier()
            check_level(li, d, rows, ref.masks(rows), base, prev_terms, prev_base, tally, frontier if host else 0)
            n = int(li.new_states)
            if n == 0 or d == depth:
                return tally, d
            if d == checkpoint_at:
                path = str(tmp_path / "verdicts.ckpt")
                assert eng.lib.vsr_engine_checkpoint(eng._e, path.encode(), None) == 0
                eng.close()
                eng = vdist.GpuEngine(mc, 0, 1, **kw)
                assert eng.lib.vsr_engine_recover(eng._e, path.encode(), None) == 0, eng.lib.vsr_engine_last_error(eng._e)
                assert eng.read_frontier() == rows and eng.stats().distinct == base + n
                tally.recovered = True
            prev_terms, prev_base = ref.terminals(rows), base
            if part:
                for first in range(0, n, part):
                    eng.step(first, part, 0, None)
            else:
                eng.expand()
            li, d, base = eng.finish(), d + 1, base + n
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth", SHAPE_CASES)
@pytest.mark.parametrize("mask", [NOT_LOST | MAJORITY, HOOK])
def test_level_verdicts_on_every_kernel_shape(pkg, R, V, L, depth, mask):
    mc = model(pkg, R, V, L, mask, symmetry=V > 1)
    tally, reached = explore(pkg, mc, Reference(pkg, mc, mask), depth)
    print((R, V, L), mask, "depth", reached, "levels with violators", tally.viol_levels, "max", tally.max_violators,
          "with deadlocks", tally.dead_levels, "masks", sorted(tally.masks))
    assert reached == depth or depth == 0
    assert tally.masks <= {mask if mask == HOOK else MAJORITY}
    if (R, V, L) == (2, 3, 2):
        assert tally.dead_levels >= 5 and (mask != HOOK or (tally.viol_levels >= 10 and tally.max_violators > 32))
    if (R, V, L) == (3, 2, 3) and mask == HOOK:
        assert tally.viol_levels == 3


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth,part", PART_CASES)
def test_level_verdicts_when_levels_are_expanded_in_parts(pkg, R, V, L, depth, part):
    mask = NOT_LOST | MAJORITY | HOOK
    mc = model(pkg, R, V, L, mask, symmetry=V > 1)
    tally, reached = explore(pkg, mc, Reference(pkg, mc, mask), depth, part=part)
    print((R, V, L), "part", part, "levels with violators", tally.viol_levels, "max", tally.max_violators, "with deadlocks", tally.dead_levels)
    assert reached == depth and tally.viol_levels >= 3
    if (R, V, L) == (3, 2, 1):
        assert tally.dead_levels >= 2 and tally.max_violators > 32


@pytest.mark.gpu
def test_level_verdicts_across_the_frontier_spill_boundary(pkg):
    """8000 frontier states in HBM, the rest of each level (up to 24,159 states) in pinned host memory: violating and
    terminal rows on both sides (depth 16 has 24 terminal states among 17,992)"""
    mask = NOT_LOST | MAJORITY | HOOK
    mc = model(pkg, 3, 2, 1, mask)
    tally, reached = explore(pkg, mc, Reference(pkg, mc, mask), 17, frontier=8000, host=1 << 16)
    assert reached == 17 and tally.dead_levels >= 1
    assert tally.sides == {("viol", True), ("viol", False), ("dead", True), ("dead", False)}, tally.sides


@pytest.mark.gpu
def test_level_verdicts_after_recovering_a_checkpoint(pkg, tmp_path):
    mask = NOT_LOST | MAJORITY | HOOK
    mc = model(pkg, 3, 2, 1, mask)
    tally, reached = explore(pkg, mc, Reference(pkg, mc, mask), 17, checkpoint_at=12, tmp_path=tmp_path)
    assert reached == 17 and tally.recovered and tally.viol_levels >= 2 and tally.dead_levels >= 1


def inject(eng, mc, states):
    """one launch that inserts `states` as records of the level being generated (parent Init): they take the next rows of
    the level, after every row of earlier launches, in an order the launch chooses"""
    import torch
    recs = b"".join(s + struct.pack("<QQ", mc.fingerprint(s), (0 << 12) | (1 << 56)) for s in states)  # vsr_gpu.cuh RecHdr
    eng.insert(torch.frombuffer(bytearray(recs), dtype=torch.uint8).cuda(), len(states))


def rows_of(mc, raw):
    sb = mc.state_bytes
    return [raw[k:k + sb] for k in range(0, len(raw), sb)]


@pytest.mark.gpu
def test_deadlock_id_of_a_terminal_row_in_pass_one(pkg):
    """On a two-pass layout, a level of NS + 101 states whose only terminal state is the last row: the level is one round
    and that row is in its pass 1 (thread 100), so deadlock_id = 1 + NS + 100 holds only with the pass term of the id."""
    from vsr_tlaplus_b200 import dist as vdist
    mask = NOT_LOST | MAJORITY | HOOK
    mc = model(pkg, 3, 2, 1, mask)
    warps, _, passes, _ = mc.expand_shape()
    NS = 32 * warps
    assert passes == 2
    ref = Reference(pkg, mc, mask)
    deep = rows_of(mc, mc.check(collect_levels=True, max_depth=15, table_capacity=1 << 20, frontier_capacity=1 << 16,
                                stop_on_violation=False).levels[14])
    terms = ref.terminals(b"".join(deep))
    live = [s for s, t in zip(deep, terms) if not t]
    dead = [s for s, t in zip(deep, terms) if t]
    assert dead and len(live) >= NS + 100
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=1 << 20, frontier_capacity=1 << 16, check_deadlock=True)
    try:
        eng.reset()
        eng.seed()
        assert eng.finish().new_states == 1
        inject(eng, mc, live[:NS + 100])
        inject(eng, mc, dead[:1])
        li = eng.finish()
        rows = eng.read_frontier()
        check_level(li, 2, rows, ref.masks(rows), 1, None, 0, Tally(), 0)
        assert rows_of(mc, rows)[NS + 100] == dead[0]
        prev = ref.terminals(rows)
        assert prev.count(True) == 1 and prev[NS + 100]
        eng.expand()
        li = eng.finish()
        rows = eng.read_frontier()
        check_level(li, 3, rows, ref.masks(rows), 1 + NS + 101, prev, 1, Tally(), 0)
        assert li.deadlock and li.deadlock_id == 1 + NS + 100
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L", [c[:3] for c in SHAPE_CASES])
def test_injected_violators_on_every_kernel_shape(pkg, R, V, L):
    """Every shape, whether or not its exploration above reaches a violation: a level of 40 states that hold the
    invariants, then 40 that break one (reachable states with every requested value's `acked` set TRUE while a minority
    holds it), injected in two launches.  The violation id is the first of the second launch's rows; the level after it is
    checked as any other."""
    from vsr_tlaplus_b200 import dist as vdist
    mask = NOT_LOST | MAJORITY
    mc = model(pkg, R, V, L, mask, symmetry=False)
    ref = Reference(pkg, mc, mask)
    space, _ = host_space(mc, 3000)
    clean = [s for s in space[2::2] if ref.verdict(s)[0] == 0][:40]  # space[0] is Init, already seen at depth 1
    bad = []
    for s in space[1::2]:
        f = mc.unpack(s)
        for x in range(V):
            if f.acked[x]:
                f.acked[x] = ACK_TRUE
        t = mc.pack(f)
        if ref.verdict(t)[0]:
            bad.append(t)
    bad = bad[:40]
    assert len(clean) == len(bad) == 40
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=1 << 20, frontier_capacity=1 << 16, check_deadlock=True)
    tally = Tally()
    try:
        eng.reset()
        eng.seed()
        assert eng.finish().new_states == 1
        inject(eng, mc, clean)
        inject(eng, mc, bad)
        li = eng.finish()
        rows = eng.read_frontier()
        check_level(li, 2, rows, ref.masks(rows), 1, None, 0, tally, 0)
        assert li.new_states == 80 and li.violation_id == 1 + 40
        prev = ref.terminals(rows)
        eng.expand()
        li = eng.finish()
        rows = eng.read_frontier()
        check_level(li, 3, rows, ref.masks(rows), 81, prev, 1, tally, 0)
        assert tally.max_violators > 32
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("reverse", [False, True])
def test_level_verdicts_follow_the_winner_of_a_view_tie(pkg, reverse):
    """Same-VIEW variants that differ only in aux variables (aux_svc, acked) tie; the smallest aux key wins (vsr_gpu.cu's
    patch pass).  acked TRUE on a value nobody holds violates both invariants; FALSE violates none.  Each level injects
    its records one launch at a time, in both arrival orders: the level's flag, mask and id must follow the winners."""
    import torch
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 1, 1, invariants=(NAMES[NOT_LOST], NAMES[MAJORITY]))
    ref = Reference(pkg, mc, NOT_LOST | MAJORITY)
    # two states (distinct VIEWs) whose one value is requested and held by no replica
    bases = []
    for s in with_dropped_entries(pkg, mc, [s for s in host_space(mc, 2000)[0] if mc.unpack(s).acked[0]]):
        if holders(mc, s) == (0,) and all(mc.fingerprint(s) != mc.fingerprint(b) for b in bases):
            bases.append(s)
            if len(bases) == 2:
                break
    assert len(bases) == 2

    def variant(base, aux_svc, acked):
        f = mc.unpack(base)
        f.aux_svc, f.acked[0] = aux_svc, acked
        return mc.pack(f)

    bad_wins = lambda b: [variant(b, 0, ACK_TRUE), variant(b, 1, ACK_FALSE)]    # winner (aux_svc 0) violates
    clean_wins = lambda b: [variant(b, 0, ACK_FALSE), variant(b, 1, ACK_TRUE)]  # winner clean, loser violates
    scenarios = [[clean_wins(bases[0])], [bad_wins(bases[0])], [clean_wins(bases[0]), bad_wins(bases[1])],
                 [bad_wins(bases[0]), clean_wins(bases[1])]]
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=1 << 12, frontier_capacity=1 << 10, check_deadlock=True)
    try:
        for groups in scenarios:
            for g in groups:
                assert ref.verdict(g[0])[0] != ref.verdict(g[1])[0] and NOT_LOST | MAJORITY in (ref.verdict(g[0])[0], ref.verdict(g[1])[0])
                assert mc.fingerprint(g[0]) == mc.fingerprint(g[1]) and mc.aux_key(g[0]) < mc.aux_key(g[1])
            eng.reset()
            eng.seed()
            assert eng.finish().new_states == 1
            arrivals = [v for g in groups for v in (g[::-1] if reverse else g)]
            for i, v in enumerate(arrivals):  # one launch each: the arrival order is the order of the calls
                rec = v + struct.pack("<QQ", mc.fingerprint(v), (0 << 12) | (100 + i) | (1 << 56))  # vsr_gpu.cuh RecHdr
                eng.insert(torch.frombuffer(bytearray(rec), dtype=torch.uint8).cuda(), 1)
            li = eng.finish()
            rows = eng.read_frontier()
            sb = mc.state_bytes
            assert li.new_states == len(groups) and li.ties == len(groups)
            assert sorted(rows[k:k + sb] for k in range(0, len(rows), sb)) == sorted(g[0] for g in groups)
            masks = ref.masks(rows)
            check_level(li, 2, rows, masks, 1, None, 0, Tally(), 0)
            want = [ref.verdict(g[0])[0] for g in groups]
            assert li.violation_mask == (NOT_LOST | MAJORITY if any(want) else 0)
    finally:
        eng.close()


def assert_behaviour(pkg, mc, ref, trace, last):
    """the trace is a behaviour of the oracle's Next from Init whose last state alone is `last` ("violating" | "terminal")"""
    L = orc.lib()
    q = ref.q[NOT_LOST]
    Flat = pkg.checker.VsrFlatState
    flats = [mc.unpack(s) for _, s in trace]
    init = Flat()
    L.orc_init_flat(q, C.byref(init))
    assert orc.digests_full_of(q, (Flat * 1)(flats[0]))[0] == orc.digests_full_of(q, (Flat * 1)(init))[0]
    for i in range(len(flats) - 1):
        cap = 256
        succ, acts = (Flat * cap)(), (C.c_int * cap)()
        n = L.orc_successors_flat(q, C.byref(flats[i]), succ, acts, cap)
        want = orc.digests_full_of(q, (Flat * 1)(flats[i + 1]))[0]
        got = orc.digests_full_of(q, succ)[:n]
        assert any(g == want and pkg.ACTION_NAMES[acts[k]] == trace[i + 1][0] for k, g in enumerate(got)), "step %d is not a step of Next" % (i + 1)
    verdicts = [ref.verdict(s, True) for _, s in trace]
    if last == "violating":
        assert [m != 0 for m, _ in verdicts] == [False] * (len(trace) - 1) + [True]
    else:
        assert [t for _, t in verdicts] == [False] * (len(trace) - 1) + [True]
    return verdicts[-1][0]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 4])
def test_deadlock_trace_ends_in_a_terminal_state(pkg, monkeypatch, world):
    """the BFS stops at the oracle's deadlock depth and its trace is a behaviour whose last state alone has no successor"""
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(3, 1, 1)
    o = orc.bfs(orc.params(3, 1, 1, symmetry=False, invariant=4), workers=8, check_deadlock=True, keep_trace=False, check_assumptions=False)
    caps = dict(deadlock=True, table_capacity=1 << 20, frontier_capacity=1 << 16)
    res = mc.check(**caps) if world == 1 else mc.check_multi(world, **caps)
    # TLC's depth counts the level whose generation found the deadlock: the terminal state is one level shallower
    assert o.rc == 11 == res.rc and res.depth == o.depth and res.violated_invariants == []
    assert len(res.trace) == o.depth - 1
    lit = pkg.ModelChecker.from_constants(3, 1, 1, symmetry=False)
    assert_behaviour(pkg, lit, Reference(pkg, lit, 0), res.trace, "terminal")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("order", ORDERS)
def test_ranks_report_the_first_violation_and_name_it_as_tlc(pkg, monkeypatch, world, order):
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    names = tuple(NAMES[b] for b in order)
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=names)
    res = mc.check_multi(world, table_capacity=1 << 20, frontier_capacity=1 << 18)
    # both invariants: a violation of AcknowledgedWriteNotLost is one of AcknowledgedWritesExistOnMajority too
    o = orc.bfs(orc.params(3, 2, 1, invariant=MAJORITY), workers=8, keep_trace=False, check_assumptions=False)
    assert res.rc == 12 == o.rc and res.violation_level == o.depth == len(res.trace)
    lit = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False, invariants=names)
    mask = assert_behaviour(pkg, lit, Reference(pkg, lit, NOT_LOST | MAJORITY), res.trace, "violating")
    assert res.violated_invariants == [reported(order, mask)]


@pytest.mark.gpu
@pytest.mark.parametrize("order", ORDERS)
def test_vsrmc_names_one_invariant(pkg, tmp_path, order):
    """vsrmc prints TLC's single "Error: Invariant X is violated." line, X by the naming rule on the reported state.  On
    (3, 2, 1) no reachable state loses an acknowledged value, so the first violating state breaks the majority only"""
    import subprocess
    from conftest import ROOT
    cfg = tmp_path / "m.cfg"
    cfg.write_text(pkg.cfg_text(3, ["v1", "v2"], 1, invariants=[NAMES[b] for b in order]))
    r = subprocess.run([os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc"), "-deadlock", "-config", str(cfg), "-table", "1048576",
                        "-frontier", "200000"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 12
    assert [ln for ln in r.stdout.splitlines() if ln.startswith("Error: Invariant")] == ["Error: Invariant %s is violated." % NAMES[MAJORITY]]
