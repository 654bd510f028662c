"""The seen-set host tier where it removes states (csrc/vsr_seen_host.cu), against a plain model of the tier.

VSR's own successors never lie two levels back, so its runs find no state of the tier again: the tier pass, the compaction,
the verdict and coverage repairs and the eviction's level window run only on states injected through the engine's record
interface.  The driver here pumps a world-1 engine level by level and, before each expansion, injects records drawn only
from states already seen (Init, the frontier's depth, states injected at the level before, one state twice, violators).
Every injected record is therefore a duplicate or a false new state, and none changes what is explored: the HBM-only
engine fed the same records is the reference, level by level, and TierModel predicts the tier's figures exactly.

TierModel follows DESIGN §2 and vsr_seen_host.cu, per rank:
  * injected state s at the level generating depth g: a duplicate when resident (its depth is at least evict_floor, or it
    carries a mark); otherwise the tier holds it, it is a false new state and stays resident with the mark depth(s);
  * end of a level: table_resident grows by new + false new states (the pre-filter out_count); above cap - cap/8: 152;
  * boundary at frontier depth d: when table_resident > load * cap, entries tagged [evict_floor, d) move to the tier, marks
    tagged below evict_floor are dropped, only depth-d entries stay, evict_floor = d.
The tier holds every state of depth < evict_floor, so the model keeps the real states as counts per depth and the injected
ones by value.
"""
import ctypes as C
import os
import random
import struct
import types
from collections import Counter

import pytest

import test_kernel_shapes as tks
from conftest import ROOT
from test_coverage import host_walk
from test_reshard import INV, assert_behaviour
from test_seen_host import HOOK, TIER

TRACE_HOOK = "VSR_B200_TRACE_HBM_RECORDS"


# -------------------------------------------------------------------------------------------------- 1. the model
class TierModel:
    """One rank's tier.  level(g, injected, new) plays the level generating depth g: `injected` are (state, depth) in
    arrival order, `new` its real new states; the result has the level's false_new, overflow (4 or 0) with the 7/8
    check's numbers, evicted and host_entries, as VsrLevelInfo reports them."""

    def __init__(self, cap, load):
        self.cap, self.load = cap, load
        self.tier = Counter()      # depth -> states in the tier
        self.real = Counter()      # depth -> real states resident in the table
        self.marks = {}            # state -> (tag, level that marked it): false new states resident with their mark
        self.evict_floor = 0
        self.table_resident = 0
        self.mark_hits = 0         # injected states found as duplicates of a mark made at an earlier level
        self.batch_dups = 0        # ... of a mark made in the same batch
        self.marks_dropped = 0     # marks dropped by an eviction (in the tier already)
        self.evictions = 0

    def host_entries(self):
        return sum(self.tier.values())

    def inject(self, g, states):
        false_new = 0
        for item in states:  # (state, depth) or (state, depth, the state whose seen-set key it shares)
            s, depth = item[-1] if len(item) > 2 else item[0], item[1]
            if s in self.marks:
                if self.marks[s][1] < g:
                    self.mark_hits += 1
                else:
                    self.batch_dups += 1
            elif depth < self.evict_floor:
                self.marks[s] = (depth, g)
                false_new += 1
        return false_new

    def level(self, g, injected, new):
        false_new = self.inject(g, injected)
        out = types.SimpleNamespace(false_new=false_new, overflow=0, evicted=0, host_entries=0, numbers=None)
        pre = new + false_new
        if self.table_resident + pre > self.cap - self.cap // 8:
            out.overflow = 4
            out.numbers = (self.table_resident + pre, pre, self.cap, self.host_entries())
        self.table_resident += pre
        self.real[g] += new
        if out.overflow:
            return out
        d = g
        if self.table_resident > self.load * self.cap:
            moved = 0
            for t in [t for t in self.real if self.evict_floor <= t < d]:
                moved += self.real[t]
                self.tier[t] += self.real.pop(t)
            for s, (t, _) in list(self.marks.items()):
                if t < self.evict_floor:
                    self.marks_dropped += 1
                elif t < d:
                    moved += 1
                    self.tier[t] += 1
                del self.marks[s]
            self.evict_floor = d
            self.table_resident = self.real[d]
            self.evictions += 1
            out.evicted = moved
        out.host_entries = self.host_entries()
        return out


def test_model_reinjection_across_boundaries():
    """64 slots (7/8: 56), eviction above 16 entries; depths: i = 1, a = 2, b = 3, c... = 1 - 4"""
    m = TierModel(64, 0.25)
    lv = m.level(1, [], 1)
    assert (lv.false_new, lv.evicted, lv.host_entries, m.table_resident) == (0, 0, 0, 1)
    lv = m.level(2, [("i", 1)], 4)                       # Init is resident: a duplicate
    assert (lv.false_new, lv.evicted, m.table_resident) == (0, 0, 5)
    lv = m.level(3, [("i", 1), ("a", 2)], 12)            # 17 > 16: depths 1 and 2 move
    assert (lv.false_new, lv.evicted, lv.host_entries, m.evict_floor, m.table_resident) == (0, 5, 5, 3, 12)
    # with eviction behind it: Init and a are false new states; a twice in one batch counts once
    lv = m.level(4, [("i", 1), ("a", 2), ("a", 2), ("b", 3)], 1)
    assert (lv.false_new, lv.evicted, lv.host_entries, m.table_resident) == (2, 0, 5, 15)
    assert m.marks == {"i": (1, 4), "a": (2, 4)} and (m.mark_hits, m.batch_dups) == (0, 1)
    # no eviction at that boundary: the marks linger and the same states are duplicates of them
    lv = m.level(5, [("i", 1), ("a", 2), ("b", 3)], 2)
    assert (lv.false_new, m.mark_hits) == (0, 2)
    # 12 + 1 + 2 + 2 = 17 entries: this boundary evicts, drops the marks (their states are in the tier) and moves only
    # depths 3 and 4
    assert (lv.evicted, lv.host_entries, m.marks_dropped, m.marks, m.evict_floor, m.table_resident) == (13, 18, 2, {}, 5, 2)
    lv = m.level(6, [("i", 1)], 1)                       # a false new state again
    assert (lv.false_new, lv.evicted, m.table_resident) == (1, 0, 4)


def test_model_false_new_states_take_table_room():
    m = TierModel(64, 0.0)
    for g, n in ((1, 1), (2, 2), (3, 2)):
        m.level(g, [], n)
    assert (m.evict_floor, m.table_resident, m.host_entries()) == (3, 2, 3)
    lv = m.level(4, [("c%d" % k, 1 + k % 2) for k in range(5)], 50)  # 2 + 50 fits in 56 slots, 2 + 55 does not
    assert (lv.false_new, lv.overflow, lv.numbers, lv.host_entries) == (5, 4, (57, 55, 64, 3), 0)
    m = TierModel(64, 0.0)
    for g, n in ((1, 1), (2, 2), (3, 2)):
        m.level(g, [], n)
    assert m.level(4, [("c%d" % k, 1 + k % 2) for k in range(4)], 50).overflow == 0


def test_model_without_a_tier_entry_finds_no_false_new_state():
    """nothing was evicted (evict_floor 0): every injected state is resident"""
    m = TierModel(1 << 20, 0.5)
    for g in range(1, 6):
        assert m.level(g, [("i", 1), ("x%d" % g, g - 1 or 1)], 100).false_new == 0
    assert m.host_entries() == 0 and m.evictions == 0


# -------------------------------------------------------------------------------------------------- 2. the driver
def split(mc, rows):
    sb = mc.state_bytes
    return [rows[i:i + sb] for i in range(0, len(rows), sb)]


def records(mc, states, cands):
    """RecHdr records (vsr_gpu.cuh): the state's words, fp, parent << 12 | candidate | 1 << 56; parent = Init's id 0.  The
    seen-set stores fingerprint 0 as 1 (0 marks an empty slot), and a weak0 build gives every state fingerprint 0"""
    return b"".join(s[0] + struct.pack("<QQ", mc.fingerprint(s[0]) or 1, cands[k % len(cands)] | (1 << 56)) for k, s in enumerate(states))


def insert(eng, mc, states, cands):
    import torch
    if states:
        t = torch.frombuffer(bytearray(records(mc, states, cands)), dtype=torch.uint8).cuda()
        eng.insert(t, len(states))


def spread_cands(mc):
    """one candidate index of each action met near Init, so the coverage give-back touches several counters"""
    _, cand_action, _ = host_walk(mc, max_states=4000)
    by_action = {}
    for c, a in sorted(cand_action.items()):
        by_action.setdefault(a, c)
    assert len(by_action) >= 3
    return sorted(by_action.values())


class Draw:
    """the injected records of each level: seeded, only states already seen, at depths up to the frontier's"""

    def __init__(self, mc, seed=1, per_level=24, viol=True):
        self.mc, self.rng, self.per_level, self.viol = mc, random.Random(seed), per_level, viol
        self.levels = []       # per depth: the reference run's rows
        self.violators = []    # (state, depth)
        self.prev = []

    def add_level(self, rows):
        states = split(self.mc, rows)
        self.levels.append(states)
        if self.viol:
            for s in self.rng.sample(states, min(len(states), 300)):
                if self.mc.invariant(s):
                    self.violators.append((s, len(self.levels)))

    def any(self, lo, hi):
        d = self.rng.randint(lo, hi)
        return self.rng.choice(self.levels[d - 1]), d

    def __call__(self, d):
        """records injected before the frontier of depth d is expanded"""
        out = [(self.levels[0][0], 1)]
        out += [self.any(d, d) for _ in range(2)]                      # the frontier's own depth: duplicates in the table
        out += [self.any(1, d) for _ in range(self.per_level)]
        out += self.rng.sample(self.prev, len(self.prev) // 2)         # again at the next level: lingering marks
        old = [v for v in self.violators if v[1] < d]
        out += self.rng.sample(old, min(4, len(old)))
        self.rng.shuffle(out)
        out.append(out[len(out) // 2])                                 # the same state twice in one batch
        self.prev = out
        return out


class Revisits:
    """The tier engine and the HBM-only engine pumped side by side with the same injected records, compared level by
    level with each other and with TierModel.  levels: per finished level (depth, VsrLevelInfo of the tier run, the
    model's prediction)."""

    def __init__(self, pkg, mc, load, table=1 << 20, frontier=1 << 17, hbm_table=None, keep_trace=True, coverage=False,
                 frontier_host_capacity=0, cands=None, trace_rows=20_000):
        from vsr_tlaplus_b200 import dist as vdist
        self.pkg, self.mc, self.load = pkg, mc, load
        kw = dict(frontier_capacity=frontier, keep_trace=keep_trace, collect_levels=True, coverage=coverage,
                  frontier_host_capacity=frontier_host_capacity)
        self.hbm = vdist.GpuEngine(mc, 0, 1, table_capacity=hbm_table or table, **kw)
        try:
            self.eng = vdist.GpuEngine(mc, 0, 1, table_capacity=table, table_host_capacity=TIER, **kw)
        except BaseException:
            self.hbm.close()
            raise
        self.model = TierModel(int(self.eng.stats().table_capacity), load)
        self.keep_trace, self.trace_rows = keep_trace, trace_rows
        self.cands = cands or [0]
        self.levels, self.hbm_levels, self.base = [], [], [0]
        self.dropped_levels = 0
        self.complete = False
        self.overflow = None

    def close(self):
        self.eng.close()
        self.hbm.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def run(self, max_depth, draw):
        """to max_depth (0: the end of the space) or a 152; draw(d) -> [(state, depth)] before expanding depth d"""
        for e in (self.eng, self.hbm):
            e.reset()
            e.seed()
        self._finish(1, [])
        d = 1
        while not self.complete and self.overflow is None and d != max_depth:
            inj = draw(d)
            for e in (self.eng, self.hbm):
                insert(e, self.mc, inj, self.cands)
                e.expand()
            d += 1
            self._finish(d, inj)
        st = self.eng.stats()
        assert int(st.host_false_new) == sum(lv.false_new for _, lv, _ in self.levels)
        return self

    def _finish(self, g, inj):
        mc = self.mc
        li, ref = self.eng.finish(), self.hbm.finish()
        want = self.model.level(g, inj, int(ref.new_states))
        self.levels.append((g, li, want))
        self.hbm_levels.append(ref)
        assert ref.overflow == 0 and ref.error_code == 0 and li.error_code == 0, g
        assert (li.false_new, li.overflow) == (want.false_new, want.overflow), (g, li.false_new, li.overflow, want)
        assert (li.new_states, li.generated) == (ref.new_states, ref.generated), g
        if li.overflow:
            msg = self.eng.lib.vsr_engine_last_error(self.eng._e).decode()
            self.overflow = msg
            assert "capacity exceeded (seen-set)" in msg and "(false ones included)" in msg, msg
            n = want.numbers
            assert ("%d entries in HBM with this level's %d new states" % n[:2]) in msg and ("in %d slots" % n[2]) in msg, (msg, n)
            assert ("the host tier holds %d of %d entries" % (n[3], TIER)) in msg, (msg, n)
            return
        assert (li.evicted, li.host_entries) == (want.evicted, want.host_entries), (g, li.evicted, li.host_entries, want)
        n = int(li.new_states)
        if n == 0:
            self.complete = True
            return
        rows, ref_rows = self.eng.read_frontier(), self.hbm.read_frontier()
        assert sorted(split(mc, rows)) == sorted(split(mc, ref_rows)), "depth %d: the tier run's states are not the HBM run's" % g
        assert self.eng.collected(g) == rows, g
        tks.check_audit(self.eng.audit(), g, n)
        assert (li.violation, li.violation_mask) == (ref.violation, ref.violation_mask), g
        base = self.base[-1]
        if li.false_new:
            self.dropped_levels += 1
            self._check_verdict(g, li, rows, base)
            if self.keep_trace:
                self._check_trace(g, rows, base, n, int(li.false_new))
        self.base.append(base + n)
        self.last_rows = rows

    def _check_verdict(self, g, li, rows, base):
        """over the kept rows: the OR of the invariant masks, and the first row that violates"""
        masks = [self.mc.invariant(s) for s in split(self.mc, rows)]
        mask = 0
        for m in masks:
            mask |= m
        bad = [i for i, m in enumerate(masks) if m]
        assert bool(li.violation) == bool(bad) and li.violation_mask == mask, (g, li.violation, li.violation_mask, mask)
        if bad:
            assert li.violation_id == base + bad[0], (g, li.violation_id, base, bad[0])

    def _check_trace(self, g, rows, base, n, dropped):
        """every row's trace record has its parent in the previous level (all rows of small levels; otherwise the rows that
        can have moved, [0, dropped), and a sample), and the trace built from some of them ends in the row"""
        prev = self.base[-2] if len(self.base) > 1 else 0
        rng = random.Random(g)
        idx = range(n) if n <= self.trace_rows else sorted(set(range(min(n, dropped + 64))) | set(rng.sample(range(n), 2000)) | {n - 1})
        for i in idx:
            parent, _ = self.eng.trace_record(base + i)
            assert prev <= parent < base, "depth %d row %d: parent %d outside the previous level [%d, %d)" % (g, i, parent, prev, base)
        sb, cap = self.mc.state_bytes, g + 2
        tr, acts = self.mc._buf(cap), (C.c_uint8 * cap)()
        for i in sorted(set(range(min(n, 24))) | set(rng.sample(range(n), min(n, 24)))):
            m = self.mc._lib.vsr_engine_build_trace(self.eng._e, base + i, tr, acts, cap)
            assert m == g and bytes(tr)[(m - 1) * sb:m * sb] == rows[i * sb:(i + 1) * sb], (g, i, m)

    def check_lookup(self, draw, per_depth=12):
        rng = random.Random(5)
        for d, states in enumerate(draw.levels, 1):
            for s in rng.sample(states, min(per_depth, len(states))):
                assert self.eng.lookup(s) == (d, 0), d

    def false_new(self):
        return sum(lv.false_new for _, lv, _ in self.levels)


# -------------------------------------------------------------------------------------------------- 3. cases
SHAPES = [(2, 1, 1, True, 0), (3, 2, 1, False, 0), (3, 2, 2, True, 12), (3, 3, 3, True, 10), (5, 2, 2, True, 7),
          (2, 4, 2, True, 12),   # a layout compiled as a plug-in
          (3, 4, 10, True, 9)]   # test_layout_edges.WIDE: a 64-word plug-in


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,sym,depth", SHAPES)
def test_revisits_on_every_row_shape(pkg, monkeypatch, R, V, L, sym, depth):
    """the compaction kernel at every NW and kernel shape: the evicted states injected at every level are removed, rows,
    trace records and verdicts as in the HBM run, the tier's figures as the model's"""
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=sym)
    draw = Draw(mc, seed=R * 100 + V * 10 + L)
    with Revisits(pkg, mc, 0.0, table=1 << 21, frontier=1 << 18, cands=spread_cands(mc)) as r:
        _run_drawing(r, draw, depth)
        assert r.false_new() > 0 and r.dropped_levels >= 2, (r.false_new(), r.dropped_levels)
        assert r.complete == (depth == 0)
        r.check_lookup(draw)


def _run_drawing(r, draw, depth):
    """Revisits.run with the draw fed the reference run's rows of every level before it draws"""
    def pick(d):
        while len(draw.levels) < d:
            draw.add_level(r.hbm.collected(len(draw.levels) + 1))
        return draw(d)
    return r.run(depth, pick)


@pytest.fixture(scope="module")
def sizes_321():
    """(3, 2, 1) without SYMMETRY: the oracle's level sizes, for the thresholds the cases below choose"""
    import orc
    o = orc.bfs(orc.params(3, 2, 1, symmetry=False), workers=8, keep_trace=False)
    assert o.distinct == 697_364
    return o.level_sizes


def eviction_plan(sizes, cap, load):
    """the boundaries TierModel evicts at without injection: (depth, entries moved)"""
    m = TierModel(cap, load)
    out = []
    for g, n in enumerate(sizes, 1):
        lv = m.level(g, [], n)
        if lv.evicted or m.evict_floor == g:
            out.append((g, lv.evicted))
    return out


LINGER_LOAD = 0.2


@pytest.mark.gpu
def test_lingering_marks_under_a_threshold(pkg, monkeypatch, sizes_321):
    """marks that stay in the table across boundaries: a later injection finds them as duplicates (the tier pass's level
    test must not count them again), and the next eviction drops them instead of moving them to the tier a second time
    (the [evict_floor, d) window)"""
    plan = eviction_plan(sizes_321, 1 << 20, LINGER_LOAD)
    assert len(plan) >= 3 and len(plan) < len(sizes_321) - 3, plan
    monkeypatch.setenv(HOOK, str(LINGER_LOAD))
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    draw = Draw(mc, seed=11, per_level=30)
    with Revisits(pkg, mc, LINGER_LOAD, table=1 << 20, frontier=1 << 17, cands=spread_cands(mc)) as r:
        _run_drawing(r, draw, 0)
        m = r.model
        print("evictions", m.evictions, "mark hits", m.mark_hits, "marks dropped", m.marks_dropped, "false new", r.false_new())
        assert r.complete and m.evictions >= 3 and m.mark_hits >= 1 and m.marks_dropped >= 1 and r.false_new() > 0
        assert r.eng.stats().host_entries == m.host_entries() < FULL_321
        r.check_lookup(draw)


FULL_321 = 697_364


@pytest.mark.gpu
def test_false_new_takes_table_room(pkg, monkeypatch, sizes_321):
    """a table in which a level's real states pass 7/8 only together with the injected false ones: the 152 with the
    model's numbers; the HBM run with the same injection goes on"""
    monkeypatch.setenv(HOOK, "0")
    # the level g whose real states with the previous level's fill the table to just below 7/8
    g = max(range(3, len(sizes_321)), key=lambda k: sizes_321[k - 1] + sizes_321[k - 2])
    resident = sizes_321[g - 2] + sizes_321[g - 1]
    extra = 3000
    cap = ((resident + extra // 2) * 8 // 7 + 64) & ~63   # resident fits under 7/8, resident + extra does not
    assert resident <= cap - cap // 8 < resident + extra, (g, resident, cap)
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    draw = Draw(mc, seed=3, per_level=0, viol=False)

    def pick(d):
        while len(draw.levels) < d:
            draw.add_level(r.hbm.collected(len(draw.levels) + 1))
        if d != g - 1:
            return []
        older = [(s, k) for k in range(1, d - 1) for s in draw.levels[k - 1]]
        return draw.rng.sample(older, extra)
    with Revisits(pkg, mc, 0.0, table=cap, hbm_table=1 << 21, frontier=1 << 17, cands=spread_cands(mc)) as r:
        r.run(g + 1, pick)
        assert r.overflow is not None and r.levels[-1][0] == g, (r.overflow, r.levels[-1][0], g)
        assert r.levels[-1][1].false_new == extra and r.levels[-1][1].overflow == 4
        ref = r.hbm_levels[-1]
        assert ref.overflow == 0 and ref.new_states == sizes_321[g - 1]
        r.hbm.expand()
        assert r.hbm.finish().new_states == sizes_321[g]  # the HBM run does not stop


def _only_false_new_violators(pkg, mc, max_depth):
    """(first violating depth V, a depth g > V + 1 whose own states all hold the invariant), from a plain run"""
    res, _ = tks.engine_bfs(pkg, mc, max_depth=max_depth, table=1 << 22, frontier=1 << 20)
    bad = [any(mc.invariant(s) for s in split(mc, lv)) for lv in res.levels]
    res.engine = None
    v = bad.index(True) + 1
    clean = [d for d in range(v + 2, len(bad) + 1) if not bad[d - 1]]
    return v, clean, res


VERDICT_CASE = (3, 2, 1, True, INV)  # violators at depths 19 - 23 only: depth 24 on holds the invariant


@pytest.mark.gpu
def test_verdict_of_a_level_whose_only_violators_are_false_new(pkg, monkeypatch):
    """violators of an earlier depth injected into a level whose own states all hold the invariant: inserted as new they
    set the level's verdict, and the repair after their removal must turn it off"""
    R, V, L, sym, inv = VERDICT_CASE
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=sym, invariants=inv)
    v, clean, plain = _only_false_new_violators(pkg, mc, 0)
    assert clean, "no level after the first violating depth %d holds the invariant in all its states" % v
    g = clean[0]
    monkeypatch.setenv(HOOK, "0")
    draw = Draw(mc, seed=9, per_level=8)

    def pick(d):
        while len(draw.levels) < d:
            draw.add_level(r.hbm.collected(len(draw.levels) + 1))
        if d == g - 1:
            bad = [(s, k) for k in range(v, d - 1) for s in draw.levels[k - 1] if mc.invariant(s)]
            return draw.rng.sample(bad, min(50, len(bad)))
        return draw(d)
    with Revisits(pkg, mc, 0.0, table=1 << 21, frontier=1 << 18, cands=spread_cands(mc)) as r:
        r.run(g + 1, pick)
        _, li, _ = r.levels[g - 1]
        assert li.false_new > 0 and not li.violation and li.violation_mask == 0, (g, li.false_new, li.violation, li.violation_mask)
        print("first violating depth", v, "clean depths after it", clean, "flipped level", g, "false new", li.false_new)


def _liveness(eng):
    from vsr_tlaplus_b200 import checker as ck
    ls = ck.VsrLiveStats()
    cap = 4096
    cands = (C.c_uint32 * cap)()
    rc = eng.lib.vsr_engine_liveness(eng._e, C.byref(ls), cands, cap)
    assert rc in (0, 13), (rc, eng.lib.vsr_engine_last_error(eng._e))
    return rc, ls, cands


def _liveness_pair(pkg, r, mc, hooks):
    import test_liveness as tl
    rc, ls, cands = _liveness(r.eng)
    rc_h, ls_h, _ = _liveness(r.hbm)
    assert (rc, int(ls.stored), int(ls.sinks)) == (rc_h, int(ls_h.stored), int(ls_h.sinks)), (rc, ls.stored, ls.sinks, rc_h, ls_h.stored, ls_h.sinks)
    if rc == 13:
        res = types.SimpleNamespace(trace=mc._trace_from_cands(cands, int(ls.trace_len)), trace_loop=int(ls.trace_loop))
        assert tl.lasso_errors(pkg, mc, res, __import__("orc").params(3, 1, 1), hooks) == []
    return rc, ls


@pytest.mark.gpu
def test_a_level_of_only_false_new_states(pkg, monkeypatch):
    """tier states injected into the expansion of the last level: every row of that level is dropped, the run ends
    complete at the reference's depth, no extra level is reported, and the liveness pass still runs"""
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(3, 1, 1, property=True, live_test_hooks=0)
    last = mc.check(deadlock=False, table_capacity=1 << 20, frontier_capacity=1 << 17).depth
    draw = Draw(mc, seed=4, per_level=6, viol=False)

    def pick(d):
        while len(draw.levels) < d:
            draw.add_level(r.hbm.collected(len(draw.levels) + 1))
        if d == last:
            return [(s, k) for k in range(1, d) for s in draw.levels[k - 1][:40]]
        return draw(d)
    with Revisits(pkg, mc, 0.0, cands=spread_cands(mc)) as r:
        r.run(0, pick)
        g, li, _ = r.levels[-1]
        assert r.complete and g == last + 1 and li.new_states == 0 and li.false_new > 40, (g, last, li.new_states, li.false_new)
        st, sh = r.eng.stats(), r.hbm.stats()
        assert (st.num_levels, st.distinct, st.generated) == (sh.num_levels, sh.distinct, sh.generated) and st.num_levels == last
        rc, ls = _liveness_pair(pkg, r, mc, 0)
        assert rc == 0 and int(ls.stored) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("hooks", [0, 1])
def test_revisits_before_the_liveness_pass(pkg, monkeypatch, hooks):
    """the liveness store collected after compactions: stored, sinks and the verdict equal the HBM run's"""
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(3, 1, 1, property=True, live_test_hooks=hooks)
    draw = Draw(mc, seed=20 + hooks, per_level=30)
    with Revisits(pkg, mc, 0.0, cands=spread_cands(mc)) as r:
        _run_drawing(r, draw, 0)
        assert r.complete and r.dropped_levels >= 5
        rc, ls = _liveness_pair(pkg, r, mc, hooks)
        if hooks == 1:
            assert rc == 13 and int(ls.sinks) == 55
        else:
            assert rc == 0


SPILL_HBM = 700


@pytest.mark.gpu
def test_revisits_across_the_spill_boundaries(pkg, monkeypatch, sizes_321):
    """a frontier of 700 rows in HBM, the rest in host memory, and the trace's boundary inside the level with the most
    false new states: more of them than the HBM part of the parent buffer holds as 8-byte hole rows (2,800 of them for
    32-byte rows), so holes, moved rows and moved trace records lie in host memory"""
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    holes_hbm = SPILL_HBM * mc.state_bytes // 8
    big = holes_hbm + 1500
    g = next(k for k in range(4, len(sizes_321)) if sizes_321[k - 1] > big + 2000 and sum(sizes_321[:k - 2]) > big)
    start = sum(sizes_321[:g - 1])
    monkeypatch.setenv(HOOK, "0")
    monkeypatch.setenv(TRACE_HOOK, str(start + sizes_321[g - 1] // 2))
    draw = Draw(mc, seed=6, per_level=20)

    def pick(d):
        while len(draw.levels) < d:
            draw.add_level(r.hbm.collected(len(draw.levels) + 1))
        if d == g - 1:  # the tier holds every depth below the frontier's
            older = [(s, k) for k in range(1, d) for s in draw.levels[k - 1]]
            return draw.rng.sample(older, big)
        return draw(d)
    with Revisits(pkg, mc, 0.0, table=1 << 21, frontier=SPILL_HBM, frontier_host_capacity=1 << 17, cands=spread_cands(mc),
                  trace_rows=1 << 17) as r:
        r.run(g + 2, pick)
        _, li, _ = r.levels[g - 1]
        assert li.false_new == big > holes_hbm, (li.false_new, holes_hbm)
        assert r.complete is False and len(r.levels) == g + 2


@pytest.mark.gpu
def test_revisits_with_weak_fingerprints(monkeypatch, tmp_path):
    """the tier pass's own probe walk and check-hash comparison against the insert's: 16-bit fingerprints, one
    fingerprint for every state (one probe chain wrapping the table), 4-entry buckets; in child processes"""
    variants = {"weak16": ("-DVSR_WEAK_FP_BITS=16", [(3, 2, 1)]), "weak0": ("-DVSR_WEAK_FP_BITS=0", [(2, 2, 2)]),
                "bucket4": ("-DVSR_BUCKET=4", [(3, 2, 1)])}
    libs = tks.build_variants(str(tmp_path), variants)
    monkeypatch.setenv(HOOK, "0")
    for (name, R, V, L), so in sorted(libs.items()):
        table = 4672 if name == "weak0" else 1 << 20
        out = tks._child("import os; os.environ['VSR_B200_LIB'] = %r\nimport _pkg; pkg = _pkg.load()\n"
                         "import test_seen_host_revisits as t\nt.weak_case(pkg, %d, %d, %d, %d, %r)\nprint('CHILD-OK')\n"
                         % (so, R, V, L, table, name))
        print(name, out.strip().splitlines()[-2])


def weak_case(pkg, R, V, L, table, name):
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=False)
    draw = Draw(mc, seed=R + V + L, per_level=30)
    with Revisits(pkg, mc, 0.0, table=table, hbm_table=table, frontier=1 << 17, cands=spread_cands(mc)) as r:
        _run_drawing(r, draw, 0)
        colls = sum(int(lv.collisions) for _, lv, _ in r.levels)
        st = r.eng.stats()
        assert r.complete and r.false_new() > 0 and r.dropped_levels >= 3
        assert int(st.distinct) == int(r.hbm.stats().distinct)
        if name != "bucket4":
            assert colls > 0
        r.check_lookup(draw)
        print("RESULT", name, "false new", r.false_new(), "collisions", colls, "distinct", int(st.distinct))


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth", [(3, 1, 1, 0), (3, 2, 1, 12)])
def test_revisits_with_coverage(pkg, monkeypatch, R, V, L, depth):
    """distinct per level and action equals the HBM run's (the give-back of the dropped rows), generated equals the HBM
    run's with the same injection, and distinct is the histogram of the kept trace records' actions"""
    import numpy as np
    from vsr_tlaplus_b200 import dist as vdist
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=False)
    _, cand_action, _ = host_walk(mc, max_states=30_000)  # expands every level up to 12 of (3, 2, 1): their candidates
    draw = Draw(mc, seed=8, per_level=30)
    with Revisits(pkg, mc, 0.0, coverage=True, cands=spread_cands(mc)) as r:
        _run_drawing(r, draw, depth)
        assert r.false_new() > 0
        dis, gen = r.eng.coverage().levels
        hdis, hgen = r.hbm.coverage().levels
        # distinct per level (per action it depends on which of a state's arrivals is first), generated per level and action
        assert dis.sum(1).tolist() == hdis.sum(1).tolist() and gen.tolist() == hgen.tolist()
        dropped_actions = {cand_action[c] for c in r.cands}
        assert len(dropped_actions) >= 3
        hist = np.zeros_like(dis)
        gid = 0
        for d, (_, li, _) in enumerate(r.levels):
            for _ in range(int(li.new_states)):
                parent, cand = r.eng.trace_record(gid)
                hist[d][0 if parent == vdist.ROOT_PARENT else cand_action[cand]] += 1
                gid += 1
        assert hist.tolist() == dis.tolist()


@pytest.mark.gpu
def test_false_new_with_a_view_tie(pkg, monkeypatch):
    """a tier state and a copy that differs only in its aux bits, in one level: the tie patch runs on a false new state
    before the tier pass drops it.  Rows, trace and coverage equal the HBM run's.  The tier run counts the tie (li.ties,
    h2_ties), which the HBM run, where both arrivals are duplicates of an older level, does not"""
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(3, 2, 2)
    draw = Draw(mc, seed=12, per_level=4, viol=False)
    tie_at = 6
    tied = {}

    def pick(d):
        while len(draw.levels) < d:
            draw.add_level(r.hbm.collected(len(draw.levels) + 1))
        if d != tie_at:
            return draw(d)
        for k in range(2, d - 1):
            for s in draw.levels[k - 1]:
                f = mc.unpack(s)
                for aux in (0, 1, 2):
                    if aux == f.aux_svc:
                        continue
                    f2 = mc.unpack(s)
                    f2.aux_svc = aux
                    t = mc.pack(f2)
                    if mc.fingerprint(t) == mc.fingerprint(s) and mc.aux_key(t) != mc.aux_key(s):
                        tied.update(state=s, copy=t, depth=k)
                        return [(s, k), (t, k, s)]
        raise AssertionError("no state of depths 2 .. %d has an aux-only copy" % (d - 2))
    with Revisits(pkg, mc, 0.0, table=1 << 21, frontier=1 << 18, coverage=True, cands=spread_cands(mc)) as r:
        r.run(tie_at + 2, pick)
        _, li, _ = r.levels[tie_at]
        ref = r.hbm_levels[tie_at]
        assert tied and li.false_new == 1 and (int(li.ties), int(ref.ties)) == (1, 0), (li.false_new, li.ties, ref.ties)
        assert (int(r.eng.stats().h2_ties), int(r.hbm.stats().h2_ties)) == (1, 0)
        assert r.eng.coverage().levels[0].sum(1).tolist() == r.hbm.coverage().levels[0].sum(1).tolist()
        assert r.eng.coverage().levels[1].tolist() == r.hbm.coverage().levels[1].tolist()
        assert r.eng.lookup(tied["state"]) == (tied["depth"], 0)


# -------------------------------------------------------------------------------------------------- several ranks
class _Injecting:
    """a staged engine that inserts this rank's own injected states before each level's first step"""

    def __init__(self, eng, mc, plan, cands, rank, world):
        self.e, self.mc, self.plan, self.cands, self.rank, self.world = eng, mc, plan, cands, rank, world
        self.level, self.pending, self.false_new = 0, False, 0

    def __getattr__(self, k):
        return getattr(self.e, k)

    def reset(self):
        self.level, self.pending, self.false_new = 0, False, 0
        self.e.reset()

    def finish(self):
        li = self.e.finish()
        self.level += 1
        self.pending = True
        self.false_new += int(li.false_new)
        return li

    def step(self, first, count, parity, drain):
        if self.pending:
            self.pending = False
            mine = [(s, d) for s, d in self.plan.get(self.level, []) if self.mc._lib.vsr_owner_rank(self.mc.fingerprint(s), self.world) == self.rank]
            insert(self.e, self.mc, mine, self.cands)
        return self.e.step(first, count, parity, drain)


def _ranks_worker(rank, world, port, plan, cands, depth, q):
    import torch.distributed as tdist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), **{HOOK: "0"})
    tdist.init_process_group("gloo", rank=rank, world_size=world)
    import _pkg
    pkg = _pkg.load()
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    eng = vdist.GpuEngine(mc, rank, world, device=0, table_capacity=1 << 20, frontier_capacity=1 << 17, collect_levels=True,
                          exchange="staged", table_host_capacity=TIER)
    try:
        w = _Injecting(eng, mc, plan, cands, rank, world)
        res = vdist.ShardedBfs(w, rank, world, part_states=3000).run(max_depth=depth, stop_on_violation=False)
        levels = [sorted(split(mc, eng.collected(d))) for d in range(1, res.depth + 1)]
        go_on = dict(rc=res.rc, generated=res.generated, distinct=res.distinct, level_sizes=res.level_sizes, false_new=w.false_new,
                     stats_false_new=int(eng.stats().host_false_new))
        res = vdist.ShardedBfs(w, rank, world, part_states=3000).run(stop_on_violation=True)
        trace = vdist.replay_trace(mc, res.trace_cands) if rank == 0 and res.trace_cands else []
        stop = dict(rc=res.rc, violation_level=res.violation_level, false_new=w.false_new)
        q.put((rank, go_on, levels, stop, trace))
    finally:
        eng.close()
        tdist.destroy_process_group()


@pytest.mark.gpu
def test_ranks_remove_their_own_false_new_states(pkg, monkeypatch, viol_depth_321):
    """world 2 and 4 over gloo, every rank on cuda:0: each rank filters the false new states it owns.  Per-depth sets,
    level sizes, generated and the summed host_false_new equal the world-1 run and the model; stopping at the violation,
    the counterexample is a behaviour"""
    import torch.multiprocessing as mp
    monkeypatch.setenv(HOOK, "0")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    depth = viol_depth_321 + 3
    cands = spread_cands(mc)
    draw = Draw(mc, seed=31, per_level=30)
    plan = {}

    def pick(d):
        while len(draw.levels) < d:
            draw.add_level(r.hbm.collected(len(draw.levels) + 1))
        plan[d] = draw(d)
        return plan[d]
    with Revisits(pkg, mc, 0.0, cands=cands) as r:
        r.run(depth, pick)
        one_levels = [sorted(lv) for lv in draw.levels] + [sorted(split(mc, r.eng.collected(depth)))]
        one = dict(generated=sum(int(lv.generated) for _, lv, _ in r.levels), distinct=int(r.eng.stats().distinct),
                   level_sizes=[int(lv.new_states) for _, lv, _ in r.levels], false_new=r.false_new())
    assert one["false_new"] > 0
    ctx = mp.get_context("spawn")
    for world in (2, 4):
        q = ctx.Queue()
        procs = [ctx.Process(target=_ranks_worker, args=(k, world, 29650 + world, plan, cands, depth, q)) for k in range(world)]
        for p in procs:
            p.start()
        got = sorted((q.get(timeout=600) for _ in procs), key=lambda x: x[0])
        for p in procs:
            p.join(60)
            assert p.exitcode == 0
        for _, go_on, _, _, _ in got:
            assert go_on["rc"] in (0, 12) and (go_on["generated"], go_on["distinct"], go_on["level_sizes"]) == \
                (one["generated"], one["distinct"], one["level_sizes"]), (world, go_on, one)
        assert sum(g["false_new"] for _, g, _, _, _ in got) == sum(g["stats_false_new"] for _, g, _, _, _ in got) == one["false_new"], world
        assert all(g["false_new"] > 0 for _, g, _, _, _ in got), world
        for d in range(depth):
            union = sorted(s for _, _, lv, _, _ in got for s in lv[d])
            assert union == one_levels[d], (world, d + 1)
        _, _, _, stop, trace = got[0]
        res = types.SimpleNamespace(rc=stop["rc"], violation_level=stop["violation_level"], trace=trace)
        assert_behaviour(pkg, res, viol_depth_321)
        assert sum(s["false_new"] for _, _, _, s, _ in got) > 0


@pytest.fixture(scope="module")
def viol_depth_321():
    import orc
    o = orc.bfs(orc.params(3, 2, 1, invariant=2), workers=8, keep_trace=False, check_assumptions=False)
    assert o.rc == 12 and o.depth > 8
    return o.depth
