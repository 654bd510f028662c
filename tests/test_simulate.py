"""Simulation mode (TLC's `-simulate`): simulate_kernel walk by walk against the host, the oracle and the command line.

The kernel runs one thread per random walk from Init in a grid-stride loop over T = SMs x 16 blocks x 128 threads
(vsr_simulate), and calls Ops<L>::step<true> and random_enabled on plain word arrays; the host's vsr_walk runs the same
templates built by g++.  Runs of 2T + 777 walks send threads through the loop a second and a third time.  Where walks
are compared no invariant is configured, so a walk ends at the depth bound or in a state without an enabled candidate;
a step that failed to apply would end a walk silently on both sides, and the check that every walk that stopped early
ends in a state without enabled candidates tells the two apart.
"""
import collections
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy import stats

import orc
from conftest import ROOT
from test_kernel_shapes import builtin_layouts

TESTS = os.path.join(ROOT, "tests")
VSRMC = os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc")
BOTH = ("AcknowledgedWriteNotLost", "AcknowledgedWritesExistOnMajority")
HOOK = 256  # vsr_model_create's test-hook invariant: "no replica has committed every value", violated often


def hook_model(pkg, R, V, L, symmetry=False):
    lib = pkg.load_library()
    h = C.c_void_p()
    err = C.create_string_buffer(256)
    assert lib.vsr_model_create(R, 1, V, L, 0, int(symmetry), 1, HOOK, C.byref(h), err, len(err)) == 0, err.value
    return pkg.ModelChecker(h, lib)


class Walker:
    """The host side of one model: re-walks (vsr_walk), literal replays (vsr_replay_candidates), the all-word FP64 of a
    state's canonical form (what simulate_kernel probes), and the number of enabled candidates of a state."""

    def __init__(self, pkg, R, V, L, symmetry=True, invariants=(), mc=None):
        self.mc = mc or pkg.ModelChecker.from_constants(R, V, L, symmetry=symmetry, invariants=invariants)
        self.nv = pkg.ModelChecker.from_constants(R, V, L, symmetry=symmetry, view=False, invariants=())
        self.lib, self.sb = self.mc._lib, self.mc.state_bytes
        self.cands = (C.c_uint32 * 4096)()
        self.va = C.c_int()
        self.en = (C.c_uint32 * 4096)()

    def walk(self, seed, k, depth):
        """(transitions, depth of the first violating state or 0) of walk k; its candidates are in self.cands"""
        n = self.lib.vsr_walk(self.mc._h, seed, k, depth, self.cands, C.byref(self.va))
        return n, self.va.value

    def replay(self, cands):
        """the literal behaviour of a candidate chain from Init: [(action name, packed state)]"""
        arr = (C.c_uint32 * max(len(cands), 1))(*cands)
        return self.mc._trace_from_cands(arr, len(cands))

    def canonical_last(self, cands):
        """the state the device holds after the chain: the literal last state, canonicalised under SYMMETRY"""
        buf = (C.c_uint8 * self.sb).from_buffer_copy(self.replay(cands)[-1][1])
        assert self.lib.vsr_canon(self.mc._h, buf) == 0
        return buf

    def fp(self, buf):
        return int(self.lib.vsr_fingerprint_bytewise(self.nv._h, buf))

    def enabled(self, buf):
        n = self.lib.vsr_enabled_candidates(self.mc._h, buf, self.en, len(self.en))
        assert 0 <= n <= len(self.en), n
        return [int(self.en[i]) for i in range(n)]

    def successor_fps(self, prefix):
        """for the state a candidate chain reaches: [(candidate, fingerprint of the state it steps to)] over its enabled candidates"""
        return [(c, self.fp(self.canonical_last(list(prefix) + [c]))) for c in self.enabled(self.canonical_last(prefix))]


def threads():
    """T: the simulate kernel's thread count on device 0 (vsr_simulate launches SMs x 16 blocks of 128 threads)"""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 128


def sample_walks(T, n):
    """walks 0-511, T-256 .. T+255, 2T-256 .. 2T+255 and the last 256 (the first and later rounds of the grid-stride loop)"""
    idx = set(range(min(512, n))) | set(range(max(0, n - 256), n))
    for c in (T, 2 * T):
        idx |= set(range(max(0, c - 256), min(n, c + 256)))
    return sorted(idx)


def probe_array(mc):
    return np.array(mc.last_probe, dtype=np.uint64).reshape(-1, 2)


def check_walks_like_the_host(pkg, R, V, L, symmetry, depth, seed, T, num_walks=None, every=False):
    """One device run of num_walks (default 2T + 777) walks, every walk probed.  Over all walks: the probes' transitions
    add up to the kernel's steps, and the walks shorter than depth - 1 transitions are its dead ends.  On the sampled
    walks (every walk with every=True): the host re-walk has the same length and the same last state, and a walk that
    stopped early stopped in a state without an enabled candidate.  Returns the stats."""
    w = Walker(pkg, R, V, L, symmetry)
    n = 2 * T + 777 if num_walks is None else num_walks
    st, trace = w.mc.simulate(num_walks=n, depth=depth, seed=seed, probe_walks=n, deadlock=False)
    assert (st.rc, trace, st.walks) == (0, [], n)
    probe = probe_array(w.mc)
    assert probe.shape == (n, 2)
    assert int(probe[:, 1].sum()) == st.steps, "the probes' transitions do not add up to the kernel's steps"
    assert int((probe[:, 1] < depth - 1).sum()) == st.dead_ends, "walks shorter than the bound are not the dead ends"
    assert int(probe[:, 1].max(initial=0)) <= depth - 1
    for k in (range(n) if every else sample_walks(T, n)):
        nh, viol = w.walk(seed, k, depth)
        assert viol == 0 and nh == int(probe[k, 1]), (k, nh, int(probe[k, 1]))
        last = w.canonical_last(list(w.cands[:nh]))
        assert w.fp(last) == int(probe[k, 0]), "walk %d: device and host end in different states" % k
        if nh < depth - 1:
            assert w.enabled(last) == [], "walk %d stopped after %d transitions in a state with enabled candidates" % (k, nh)
    return st


# -------------------------------------------------------------------------------------------------- 1. device = host
SYM_OFF = [(3, 2, 2), (3, 3, 3), (5, 2, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,symmetry", [c + (True,) for c in builtin_layouts()] + [c + (False,) for c in SYM_OFF])
def test_device_walks_are_host_walks(pkg, R, V, L, symmetry):
    st = check_walks_like_the_host(pkg, R, V, L, symmetry, 100, seed=1000 + 100 * R + 10 * V + L, T=threads())
    assert st.steps > st.walks


@pytest.mark.gpu
def test_plugin_layout_walks_are_host_walks(pkg):
    """(2, 4, 2) is not built in: its kernels come from the plug-in path.  In a child process, as the plug-in's BFS test."""
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "import _pkg; pkg = _pkg.load()\n"
            "import test_simulate as t\n"
            "t.check_walks_like_the_host(pkg, 2, 4, 2, True, 100, 77, t.threads())\n"
            "print('PLUGIN-SIM-OK')\n" % (ROOT, TESTS))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    assert "PLUGIN-SIM-OK" in r.stdout, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])


# -------------------------------------------------------------------------------------------------- 2. exact totals
@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L", [(2, 1, 1), (2, 2, 1)])
def test_small_spaces_every_walk_rewalked(pkg, R, V, L):
    st = check_walks_like_the_host(pkg, R, V, L, True, 40, seed=21, T=threads(), every=True)
    assert st.dead_ends > 0


# -------------------------------------------------------------------------------------------------- 3. oracle
@pytest.mark.parametrize("R,V,L", [(3, 2, 2), (3, 3, 3), (4, 3, 2), (5, 2, 2)])
def test_walks_are_behaviours_of_the_spec_per_the_oracle(pkg, R, V, L):
    """64 walks at depth 100 with both invariants, replayed literally: every step is a step of the oracle's Next with the
    same action name, every state's verdict is the oracle's, a walk stops at its first violating state, and a walk that
    ended early ends where the oracle has no successor.  Independent of vsr_actions.h, which host and device share."""
    depth = 100
    w = Walker(pkg, R, V, L, True, invariants=BOTH)
    q = orc.params(R, V, L, symmetry=False)
    qs = [orc.params(R, V, L, symmetry=False, invariant=i) for i in (1, 2)]
    O = orc.lib()
    Flat = pkg.checker.VsrFlatState
    cap = 1024
    succ, acts, dig = (Flat * cap)(), (C.c_int * cap)(), (C.c_uint64 * (2 * cap))()
    ended_early = 0
    for k in range(64):
        n, viol = w.walk(3, k, depth)
        trace = w.replay(list(w.cands[:n]))
        assert len(trace) == n + 1 and trace[0][0] == "Initial predicate"
        flats = [w.mc.unpack(s) for _, s in trace]
        for i, ((name, s), f) in enumerate(zip(trace, flats)):
            mask = w.mc.invariant(s)
            for b, qi in zip((1, 2), qs):
                assert bool(mask & b) == (O.orc_invariant_flat(qi, C.byref(f)) == 0), (k, i + 1, b)
            assert (mask != 0) == (viol == i + 1), (k, i + 1, mask, viol)
            m = O.orc_successors_flat(q, C.byref(f), succ, acts, cap)
            assert 0 <= m <= cap
            if i + 1 < len(trace):
                want = orc.digests_full_of(q, (Flat * 1)(flats[i + 1]))[0]
                O.orc_digest_full_flat(q, succ, m, dig)
                got = bytes(dig)[:16 * m]
                assert any(got[16 * j:16 * j + 16] == want and pkg.ACTION_NAMES[acts[j]] == trace[i + 1][0] for j in range(m)), \
                    "walk %d: step %d is not a step of Next" % (k, i + 1)
            elif not viol and n < depth - 1:
                assert m == 0, "walk %d stopped after %d transitions where the oracle has %d successors" % (k, n, m)
                ended_early += 1
    print("(%d,%d,%d): %d of 64 walks ended early" % (R, V, L, ended_early))


# -------------------------------------------------------------------------------------------------- 4. uniform choice
@pytest.mark.gpu
@pytest.mark.parametrize("symmetry", [True, False])
def test_steps_are_drawn_uniformly_among_enabled_candidates(pkg, symmetry):
    """2^20 walks of depth 2 and of depth 3 with the same seed: walk k takes the same first step in both, so the two probes
    give its first and its second state.  The first step's state is counted against Init's enabled candidates, the second
    against the enabled candidates of the first step's state; a chi-square test of each against uniform (candidates that
    lead to the same state pooled) must give p >= 1e-6.  The seeds are fixed, so the result is too."""
    R, V, L, N, seed = 3, 2, 2, 1 << 20, 4242
    w = Walker(pkg, R, V, L, symmetry)
    first = []
    for depth in (2, 3):
        st, _ = w.mc.simulate(num_walks=N, depth=depth, seed=seed, probe_walks=N)
        assert st.rc == 0
        first.append(probe_array(w.mc))
    p2, p3 = first
    assert (p2[:, 1] == 1).all() and st.dead_ends == int((p3[:, 1] < 2).sum())

    def chi2(observed, expected_cands):
        """(statistic, degrees of freedom) of the observed fingerprints against a uniform choice among the candidates"""
        k = collections.Counter(fp for _, fp in expected_cands)
        assert set(observed) <= set(k), "a step to a state that is not a successor"
        tot = sum(observed.values())
        obs = np.array([observed.get(f, 0) for f in k], dtype=float)
        exp = np.array([tot * k[f] / len(expected_cands) for f in k])
        return float(((obs - exp) ** 2 / exp).sum()), len(k) - 1

    init = w.successor_fps([])
    assert len(init) >= 3
    s1, df1 = chi2(collections.Counter(p2[:, 0].tolist()), init)
    p_first = stats.chi2.sf(s1, df1)
    by_first = collections.defaultdict(collections.Counter)
    for f1, f2 in zip(p2[:, 0].tolist(), p3[:, 0].tolist()):
        by_first[f1][f2] += 1
    via = dict((fp, c) for c, fp in init)
    s2, df2 = 0.0, 0
    for f1, obs in by_first.items():
        nxt = w.successor_fps([via[f1]])
        assert nxt, "Init's successors all have successors"
        s, d = chi2(obs, nxt)
        s2, df2 = s2 + s, df2 + d
    p_second = stats.chi2.sf(s2, df2)
    print("symmetry %d: first step chi2 %.1f df %d p %.3g; second step chi2 %.1f df %d p %.3g" % (symmetry, s1, df1, p_first, s2, df2, p_second))
    assert p_first >= 1e-6 and p_second >= 1e-6


# -------------------------------------------------------------------------------------------------- 5. smallest walk
@pytest.mark.gpu
def test_reported_violation_is_the_smallest_walk_and_a_behaviour(pkg):
    """Uniform random walks essentially never violate the spec's invariants, so the violation path runs on the test-hook
    invariant.  The reported walk is the smallest violating index (every walk below it is re-walked on the host), its
    trace is a literal behaviour of the spec per the oracle with only its last state violating, and the same seed gives
    the same trace."""
    hook = hook_model(pkg, 3, 1, 1)
    st, trace = hook.simulate(num_walks=1 << 16, depth=40, seed=5)
    assert st.rc == 12 and len(trace) == st.violation_depth and trace[0][0] == "Initial predicate"
    w = Walker(pkg, 3, 1, 1, False, mc=hook)
    for k in range(int(st.violating_walk)):
        assert w.walk(5, k, 40)[1] == 0, "walk %d violates, below the reported walk %d" % (k, st.violating_walk)
    n, viol = w.walk(5, int(st.violating_walk), 40)
    assert viol == st.violation_depth and n == viol - 1
    assert [s for _, s in w.replay(list(w.cands[:n]))] == [s for _, s in trace]
    assert_oracle_behaviour(pkg, 3, 1, 1, trace)
    flats = [hook.unpack(s) for _, s in trace]
    assert max(f.rep[r].commit for f in flats[-1:] for r in range(3)) == 1
    assert all(max(f.rep[r].commit for r in range(3)) == 0 for f in flats[:-1])
    st2, trace2 = hook.simulate(num_walks=1 << 16, depth=40, seed=5)
    assert (st2.violating_walk, st2.violation_depth, st2.steps, st2.dead_ends) == (st.violating_walk, st.violation_depth, st.steps, st.dead_ends)
    assert trace2 == trace


def assert_oracle_behaviour(pkg, R, V, L, trace):
    """every step of a literal trace is a step of the oracle's Next with the same action name; returns the oracle's
    number of successors of the last state"""
    q = orc.params(R, V, L, symmetry=False)
    O = orc.lib()
    Flat = pkg.checker.VsrFlatState
    cap = 1024
    succ, acts = (Flat * cap)(), (C.c_int * cap)()
    flats = [pkg.ModelChecker.from_constants(R, V, L, symmetry=False).unpack(s) for _, s in trace]
    for i in range(len(flats) - 1):
        n = O.orc_successors_flat(q, C.byref(flats[i]), succ, acts, cap)
        assert 0 <= n <= cap
        want = orc.digests_full_of(q, (Flat * 1)(flats[i + 1]))[0]
        got = orc.digests_full_of(q, succ)[:n]
        assert any(g == want and pkg.ACTION_NAMES[acts[k]] == trace[i + 1][0] for k, g in enumerate(got)), f"step {i + 1}"
    return O.orc_successors_flat(q, C.byref(flats[-1]), succ, acts, cap)


# -------------------------------------------------------------------------------------------------- 6. edges
@pytest.mark.gpu
def test_depth_one_and_two(pkg):
    w = Walker(pkg, 3, 2, 2)
    init = w.fp(w.canonical_last([]))
    st, _ = w.mc.simulate(num_walks=10_000, depth=1, seed=9, probe_walks=10_000)
    assert (st.rc, st.steps, st.dead_ends) == (0, 0, 0)
    assert set(w.mc.last_probe) == {(init, 0)}
    st, _ = w.mc.simulate(num_walks=10_000, depth=2, seed=9, probe_walks=10_000)
    assert (st.rc, st.steps, st.dead_ends) == (0, 10_000, 0)
    succ = {fp for _, fp in w.successor_fps([])}
    assert {t for _, t in w.mc.last_probe} == {1} and {fp for fp, _ in w.mc.last_probe} == succ


@pytest.mark.gpu
@pytest.mark.parametrize("num_walks", [0, 1, 1_000_003])
def test_walk_counts_off_the_grid(pkg, num_walks):
    """no walk, one walk, and a count that is not a multiple of a warp or of a block"""
    st = check_walks_like_the_host(pkg, 3, 2, 2, True, 40, seed=13, T=threads(), num_walks=num_walks)
    assert st.walks == num_walks and (st.steps > 0) == (num_walks > 0)


@pytest.mark.gpu
def test_probes_beyond_the_walks_are_not_reported(pkg):
    mc = pkg.ModelChecker.from_constants(3, 2, 2, invariants=())
    st, _ = mc.simulate(num_walks=1000, depth=40, seed=2, probe_walks=5000)
    assert st.rc == 0 and len(mc.last_probe) == 1000
    assert sum(t for _, t in mc.last_probe) == st.steps


@pytest.mark.gpu
def test_same_seed_same_walks_other_seed_other_walks(pkg):
    mc = pkg.ModelChecker.from_constants(3, 2, 2, invariants=())
    runs = []
    for seed in (17, 17, 18):
        st, _ = mc.simulate(num_walks=100_000, depth=40, seed=seed, probe_walks=100_000)
        runs.append((probe_array(mc).tobytes(), st.steps, st.dead_ends))
    assert runs[0] == runs[1]
    assert runs[0][0] != runs[2][0]


# -------------------------------------------------------------------------------------------------- 7. deadlock
def first_reported(w, seed, depth, num_walks):
    """(rc, walk, depth) the host expects: the smallest walk that violates (12) or stops before the bound (11)"""
    for k in range(num_walks):
        n, viol = w.walk(seed, k, depth)
        if viol:
            return 12, k, viol
        if n < depth - 1:
            return 11, k, n + 1
    return 0, 0, 0


@pytest.mark.gpu
def test_deadlock_is_reported_like_tlc(pkg):
    """TLC's simulator stops with "Deadlock reached" (11) at a state without successors unless -deadlock is given.
    Reported: the smallest walk that stops before the bound, its last state without a successor per the oracle."""
    mc = pkg.ModelChecker.from_constants(2, 1, 1, invariants=())
    w = Walker(pkg, 2, 1, 1, True, mc=mc)
    N, depth, seed = 1 << 16, 40, 3
    st, trace = mc.simulate(num_walks=N, depth=depth, seed=seed, deadlock=True)
    assert (st.rc, st.violating_walk, st.violation_depth) == first_reported(w, seed, depth, N) and st.rc == 11
    assert len(trace) == st.violation_depth and trace[0][0] == "Initial predicate"
    assert assert_oracle_behaviour(pkg, 2, 1, 1, trace) == 0
    off, tr = mc.simulate(num_walks=N, depth=depth, seed=seed, deadlock=False)
    assert off.rc == 0 and tr == [] and off.dead_ends > 0
    assert (off.steps, off.dead_ends) == (st.steps, st.dead_ends)
    # deadlock=None: the cfg's CHECK_DEADLOCK, off when it has none
    assert mc.simulate(num_walks=N, depth=depth, seed=seed)[0].rc == 0
    on = pkg.ModelChecker.from_cfg_text(pkg.cfg_text(2, ["v1"], 1, invariants=()) + "CHECK_DEADLOCK TRUE\n")
    assert on.simulate(num_walks=N, depth=depth, seed=seed)[0].rc == 11


@pytest.mark.gpu
def test_violation_and_deadlock_the_smaller_walk_wins(pkg):
    """test-hook invariant and deadlock checking together: the status and the trace are those of whichever walk comes
    first, a violation or a state without successors; over these seeds each kind comes first at least once"""
    hook = hook_model(pkg, 3, 1, 1)
    w = Walker(pkg, 3, 1, 1, False, mc=hook)
    seen = set()
    for seed in range(5, 13):
        st, trace = hook.simulate(num_walks=1 << 16, depth=40, seed=seed, deadlock=True)
        assert (st.rc, st.violating_walk, st.violation_depth) == first_reported(w, seed, 40, 1 << 16), seed
        assert len(trace) == st.violation_depth
        n = assert_oracle_behaviour(pkg, 3, 1, 1, trace)
        assert st.rc == 12 or n == 0, "seed %d: a deadlock reported where the oracle has %d successors" % (seed, n)
        assert (hook.invariant(trace[-1][1]) != 0) == (st.rc == 12)
        seen.add(st.rc)
    assert seen == {11, 12}


# -------------------------------------------------------------------------------------------------- 8. vsrmc
def run_cli(args, tmp_path, cfg):
    p = tmp_path / "m.cfg"
    p.write_text(cfg)
    r = subprocess.run([VSRMC, "-config", str(p)] + args, capture_output=True, text=True, timeout=300)
    return r.returncode, r.stdout + r.stderr


@pytest.mark.gpu
def test_cli_simulate_checks_deadlock_like_tlc(pkg, tmp_path):
    cfg = pkg.cfg_text(2, ["v1"], 1)
    sim = ["-simulate", "-num", "300000", "-depth", "40", "-seed", "7"]
    dump = tmp_path / "trace.txt"
    rc, out = run_cli(sim + ["-dumpTrace", "tlc", str(dump)], tmp_path, cfg)
    mc = pkg.ModelChecker.from_cfg_text(cfg)
    st, trace = mc.simulate(num_walks=300000, depth=40, seed=7, deadlock=True)
    assert rc == 11 == st.rc, out[-3000:]
    assert "Error: Deadlock reached." in out and "Error: The behavior up to this point is:" in out
    assert "State 1: <Initial predicate>" in out and "State %d: <%s " % (len(trace), trace[-1][0]) in out
    r = subprocess.run([os.path.join(ROOT, "oracle", "_build", "vsr_oracle"), "replay", str(dump)], capture_output=True, text=True)
    assert "NOT A STEP" not in r.stdout and r.stdout.count(" ok (") == len(trace) - 1, r.stdout[-2000:]
    rc, out = run_cli(sim + ["-deadlock"], tmp_path, cfg)
    st, _ = mc.simulate(num_walks=300000, depth=40, seed=7, deadlock=False)
    assert rc == 0, out[-3000:]
    assert "%d behaviours, %d states checked (%d ended in a state without successors)" % (st.walks, st.steps + st.walks, st.dead_ends) in out
    rc, out = run_cli(sim, tmp_path, cfg + "CHECK_DEADLOCK FALSE\n")
    assert rc == 0 and "Deadlock" not in out, out[-3000:]
