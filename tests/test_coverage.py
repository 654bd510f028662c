"""TLC's action coverage (`-coverage`; include/vsr_b200.h VsrCoverage): per action of Next and per BFS level, states generated
and distinct states found.

Reference: a Python BFS over the CPU oracle's successor function (it enumerates bindings literally, so its successors per
action are TLC's "states generated"), with for every state the set of actions on its discovery edges (edges from the level
before).  Checked, on every run:
  1. sums: per level and in all, generated / distinct add up to the run's own statistics;
  2. generated[d][a] equals the oracle's, exactly, at every number of ranks;
  3. with parent records kept, distinct[d][.] is the histogram of the trace records' actions (also after a VIEW tie);
  4. lo[d][a] <= distinct[d][a] <= hi[d][a]: states all of whose discovery edges are by a / at least one of them.
"""
import ctypes as C
import functools
import os
import re
import struct
import subprocess

import numpy as np
import pytest

import orc
from conftest import ROOT

EXE = os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc")
NA = 20
SPACES = [(2, 1, 1), (2, 2, 2), (3, 1, 1)]
# generated / distinct of the complete spaces with SYMMETRY (tests/golden/spec_text_results.json has the same from the spec's text)
TOTALS = {(2, 1, 1): (100, 76), (2, 2, 2): (2_812, 2_073), (3, 1, 1): (118_746, 43_941)}
FULL_321 = 697_364  # (3, 2, 1) without SYMMETRY


@functools.lru_cache(maxsize=None)
def reference(R, V, L, symmetry=True, max_depth=0):
    """(generated rows, lo rows, hi rows, level sizes) from the oracle; row d - 1 = successors of depth d"""
    import _pkg
    Flat = _pkg.load().checker.VsrFlatState
    q = orc.params(R, V, L, symmetry=symmetry)
    lib = orc.lib()
    init = Flat()
    lib.orc_init_flat(q, C.byref(init))
    depth_of = {orc.digests_of(q, (Flat * 1)(init))[0][0]: 1}
    one = [1] + [0] * (NA - 1)
    gen, lo, hi, sizes = [one], [one], [one], [1]
    cap = 512
    out, acts = (Flat * cap)(), (C.c_int * cap)()
    level, d = [init], 1
    while level and not (max_depth and d >= max_depth):
        d += 1
        row, found, nxt = [0] * NA, {}, []
        for f in level:
            n = lib.orc_successors_flat(q, C.byref(f), out, acts, cap)
            assert 0 <= n <= cap
            digs = orc.digests_of(q, out, n)[0] if n else []
            for k, dig in enumerate(digs):
                a = int(acts[k])
                row[a] += 1
                if depth_of.get(dig, d) != d:
                    continue
                if dig not in found:
                    depth_of[dig] = d
                    found[dig] = set()
                    nxt.append(Flat.from_buffer_copy(out[k]))
                found[dig].add(a)
        if not any(row):
            break
        gen.append(row)
        lo.append([sum(1 for s in found.values() if s == {a}) for a in range(NA)])
        hi.append([sum(1 for s in found.values() if a in s) for a in range(NA)])
        if nxt:
            sizes.append(len(nxt))
        level = nxt
    return np.array(gen, dtype=np.uint64), np.array(lo, dtype=np.uint64), np.array(hi, dtype=np.uint64), sizes


def host_walk(mc, max_states=1 << 20):
    """BFS with the library's host successor function: per-action sum of mult, and the action of every candidate index met"""
    lib = mc._lib
    gen, cand_action = [0] * NA, {}
    seen, level = {mc.init_state()}, [mc.init_state()]
    gen[0] = 1
    while level and len(seen) < max_states:
        nxt = []
        for s in level:
            succ = mc.successors(s)
            en = (C.c_uint32 * 1024)()
            n = lib.vsr_enabled_candidates(mc._h, (C.c_uint8 * mc.state_bytes).from_buffer_copy(s), en, 1024)
            assert n == len(succ)
            for k, (t, a, mult) in enumerate(succ):
                gen[a] += mult
                assert cand_action.setdefault(int(en[k]), a) == a
                if t not in seen:
                    seen.add(t)
                    nxt.append(t)
        level = nxt
    return gen, cand_action, len(seen)


def identities(res, cov, ref=None):
    dis, gen = cov.levels
    assert dis.shape == gen.shape and gen.shape[1] == NA and dis.dtype == np.uint64
    assert int(gen.sum()) == res.generated and int(dis.sum()) == res.distinct
    assert [int(x) for x in gen.sum(0)] == [g for _, g in cov.by_action.values()]
    assert [int(x) for x in dis.sum(0)] == [d for d, _ in cov.by_action.values()]
    assert gen[0].tolist() == [1] + [0] * (NA - 1) and dis[0].tolist() == gen[0].tolist()
    for d, n in enumerate(res.level_sizes):
        assert int(dis[d].sum()) == n, d
    assert not dis[len(res.level_sizes):].any()
    for d in range(1, gen.shape[0]):
        assert int(gen[d].sum()) == res.level_generated[d - 1], d
    assert not gen[:, 16:].any() and not dis[:, 16:].any()  # the recovery actions need RestartEmptyLimit > 0
    if ref is not None:
        rgen, lo, hi, sizes = ref
        assert gen.tolist() == rgen.tolist()
        assert res.level_sizes == sizes
        assert (lo <= dis).all() and (dis <= hi).all()


# -------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("rvl", SPACES)
def test_reference_table_adds_up_to_the_pinned_totals(pkg, rvl):
    gen, lo, hi, sizes = reference(*rvl)
    assert (int(gen.sum()), sum(sizes)) == TOTALS[rvl]
    assert gen.shape[0] in (len(sizes), len(sizes) + 1) and not hi[len(sizes):].any()  # a last row: successors of the deepest level, none new
    assert (lo <= hi).all() and all(int(lo[d].sum()) <= n for d, n in enumerate(sizes))
    assert all(int(hi[d].sum()) >= sizes[d] for d in range(len(sizes)))


@pytest.mark.parametrize("rvl", SPACES)
def test_host_successors_generate_the_same_per_action(pkg, rvl):
    mc = pkg.ModelChecker.from_constants(*rvl)
    gen, cand_action, n = host_walk(mc)
    assert n == TOTALS[rvl][1]
    assert gen == [int(x) for x in reference(*rvl)[0].sum(0)]
    assert set(cand_action.values()) <= set(range(1, 16))


def test_struct_mirrors_have_the_c_sizes(pkg):
    lib, ck = pkg.load_library(), pkg.checker
    for name in ("VsrRunOpts", "VsrCoverage", "VsrStats", "VsrLevelInfo"):
        assert lib.vsr_sizeof(name.encode()) == C.sizeof(getattr(ck, name)), name
    assert lib.vsr_sizeof(b"nothing") == 0
    assert ck.VsrRunOpts.coverage.offset + C.sizeof(C.c_void_p) == C.sizeof(ck.VsrRunOpts)  # the trailing field
    assert not ck.VsrRunOpts().coverage                                                      # a zeroed struct: off


@pytest.mark.parametrize("args,frag", [
    (["-simulate"], "-simulate"),
    (["-checkpoint", "0"], "-checkpoint"),
    (["-recover", "nowhere"], "-recover"),
])
def test_cli_refuses_coverage_where_it_cannot_count(pkg, tmp_path, args, frag):
    cfg = tmp_path / "VSR.cfg"
    cfg.write_text(pkg.cfg_text(2, ["v1"], 1))
    r = subprocess.run([EXE, "-deadlock", "-coverage", "1", "-metadir", str(tmp_path / "states")] + args + ["-config", str(cfg)],
                       capture_output=True, text=True)
    assert r.returncode == 151 and "-coverage" in r.stderr and frag in r.stderr, r.stdout + r.stderr


def test_cli_coverage_without_an_argument_is_not_an_option(pkg, tmp_path):
    cfg = tmp_path / "VSR.cfg"
    cfg.write_text(pkg.cfg_text(2, ["v1"], 1))
    r = subprocess.run([EXE, "-deadlock", "-config", str(cfg), "-coverage"], capture_output=True, text=True)
    assert r.returncode == 255 and "unrecognized option -coverage" in r.stderr


def test_staged_exchange_refuses_coverage_by_name(pkg):
    from vsr_tlaplus_b200 import dist as vdist
    with pytest.raises(pkg.VsrError) as e:
        vdist.GpuEngine(pkg.ModelChecker.from_constants(2, 1, 1), 0, 2, exchange="staged", coverage=True)
    assert e.value.rc == 151 and "coverage" in str(e.value) and "staged" in str(e.value)


# -------------------------------------------------------------------------------------------------- GPU
SMALL = dict(table_capacity=1 << 18, frontier_capacity=1 << 16)


@pytest.mark.gpu
@pytest.mark.parametrize("rvl", SPACES)
def test_complete_spaces_on_one_gpu(pkg, rvl):
    mc = pkg.ModelChecker.from_constants(*rvl)
    off = mc.check(**SMALL)
    on = mc.check(coverage=True, **SMALL)
    assert off.coverage is None and off.rc == 0 and off.complete
    assert (on.rc, on.generated, on.distinct, on.queue, on.depth, on.level_sizes) == (0, off.generated, off.distinct, off.queue, off.depth, off.level_sizes)
    assert (on.generated, on.distinct) == TOTALS[rvl]
    assert on.kernel_launches == off.kernel_launches
    identities(on, on.coverage, reference(*rvl))
    assert list(on.coverage.by_action) == pkg.ACTION_NAMES


@pytest.mark.gpu
def test_a_run_without_coverage_launches_what_it_always_did(pkg):
    """(2, 1, 1): Init's launch and one launch per expanded level, nothing for the counters"""
    res = pkg.ModelChecker.from_constants(2, 1, 1).check(**SMALL)
    assert res.coverage is None and res.kernel_launches == 1 + res.depth == 15


@pytest.mark.gpu
@pytest.mark.parametrize("gpus", [2, 4])
@pytest.mark.parametrize("rvl", SPACES)
def test_ranks_count_the_same(pkg, monkeypatch, rvl, gpus):
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(*rvl)
    res = mc.check_multi(gpus, coverage=True, **SMALL)
    assert res.rc == 0 and res.complete and (res.generated, res.distinct) == TOTALS[rvl]
    identities(res, res.coverage, reference(*rvl))
    assert mc.check_multi(gpus, **SMALL).coverage is None


@pytest.mark.gpu
def test_the_space_without_symmetry_and_its_ranks(pkg, monkeypatch):
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    mc = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)
    one = mc.check(coverage=True, table_capacity=1 << 21, frontier_capacity=1 << 19)
    assert one.rc == 0 and one.complete and one.distinct == FULL_321
    identities(one, one.coverage)
    two = mc.check_multi(2, coverage=True, table_capacity=1 << 20, frontier_capacity=1 << 19)
    identities(two, two.coverage)
    assert two.coverage.levels[1].tolist() == one.coverage.levels[1].tolist()           # generated: the same at every world size
    assert two.coverage.levels[0].sum(1).tolist() == one.coverage.levels[0].sum(1).tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("rvl,depth", [((3, 2, 2), 9), ((3, 3, 3), 8), ((5, 2, 2), 6), ((2, 4, 1), 12)])
def test_bounded_prefixes_of_the_larger_configurations(pkg, rvl, depth):
    """cfg2, cfg3, cfg4 (a two-pass, a one-pass and a two-blocks-per-SM layout) and a layout compiled as a plug-in, as deep as
    the oracle follows in seconds; a run stopped by -depth reports what it counted so far"""
    mc = pkg.ModelChecker.from_constants(*rvl)
    res = mc.check(coverage=True, max_depth=depth, table_capacity=1 << 21, frontier_capacity=1 << 19)
    assert res.rc == 0 and not res.complete and res.depth == depth
    identities(res, res.coverage, reference(*rvl, max_depth=depth))
    assert res.coverage.levels[1].shape[0] == depth


@pytest.mark.gpu
@pytest.mark.parametrize("rvl", [(2, 1, 1), (2, 2, 2)])
def test_distinct_is_the_histogram_of_the_trace_records(pkg, rvl):
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(*rvl)
    _, cand_action, _ = host_walk(mc)
    eng = vdist.GpuEngine(mc, 0, 1, coverage=True, **SMALL)
    try:
        res = eng.run()
        assert res.rc == 0 and res.complete
        hist = np.zeros_like(res.coverage.levels[0])
        gid = 0
        for d, n in enumerate(res.level_sizes):
            for _ in range(n):
                parent, cand = eng.trace_record(gid)
                hist[d][0 if parent == vdist.ROOT_PARENT else cand_action[cand]] += 1
                gid += 1
        assert hist.tolist() == res.coverage.levels[0].tolist()
        assert eng.coverage().levels[1].tolist() == res.coverage.levels[1].tolist()  # one rank: the engine's own counts are the job's
    finally:
        eng.close()


@pytest.mark.gpu
def test_a_resolved_view_tie_moves_the_count_to_the_winner(pkg):
    """three arrivals with one VIEW in one level (injected, as in test_view_ties_resolve_to_smallest_aux_key): the first one,
    through one action, loses to a later one through another action; distinct follows the trace record"""
    import torch
    from vsr_tlaplus_b200 import dist as vdist
    mc = pkg.ModelChecker.from_constants(3, 2, 2)
    _, cand_action, _ = host_walk(mc, max_states=2000)
    by_action = {}
    for c, a in sorted(cand_action.items()):
        by_action.setdefault(a, c)
    (a_first, c_first), (a_win, c_win) = sorted(by_action.items())[:2]
    eng = vdist.GpuEngine(mc, 0, 1, coverage=True, table_capacity=1 << 12, frontier_capacity=1 << 10)
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
            return v + struct.pack("<QQ", mc.fingerprint(v), (0 << 12) | cand | (mult << 56))

        for blob, n in ((rec(2, c_first, 2), 1), (rec(0, c_win, 1) + rec(1, c_first, 3), 2)):
            eng.insert(torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda(), n)
        li = eng.finish()
        assert (li.new_states, li.ties, li.generated) == (1, 2, 6)
        assert eng.trace_record(1) == (0, c_win)
        dis, gen = eng.coverage().levels
        want_gen, want_dis = [0] * NA, [0] * NA
        want_gen[a_first], want_gen[a_win], want_dis[a_win] = 5, 1, 1
        assert gen[1].tolist() == want_gen and dis[1].tolist() == want_dis
    finally:
        eng.close()


def _sharded_worker(rank, world, name, q):
    import _pkg
    pkg = _pkg.load()
    from vsr_tlaplus_b200 import dist as vdist
    g = vdist.Group(name, rank, world, timeout_s=120)
    try:
        res = vdist.check_sharded(pkg.ModelChecker.from_constants(2, 2, 2), g, coverage=True, **SMALL)
        q.put((rank, res.rc, res.generated, res.distinct, res.level_sizes, res.level_generated, res.coverage.levels[0].tolist(),
               res.coverage.levels[1].tolist()))
    finally:
        g.close()


@pytest.mark.gpu
def test_sharded_processes_report_the_jobs_totals_on_every_rank(pkg):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    name = "/vsr-cov-%d" % os.getpid()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, name, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = sorted(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    rgen, lo, hi, sizes = reference(2, 2, 2)
    assert got[0][1:] == got[1][1:]
    _, rc, generated, distinct, level_sizes, _, dis, gen = got[0]
    assert (rc, generated, distinct, level_sizes) == (0,) + TOTALS[(2, 2, 2)] + (sizes,)
    assert gen == rgen.tolist()
    dis = np.array(dis, dtype=np.uint64)
    assert (lo <= dis).all() and (dis <= hi).all() and [int(x) for x in dis.sum(1)[:len(sizes)]] == sizes


def _coverage_block(out):
    lines = out.splitlines()
    a = next(i for i, l in enumerate(lines) if l.startswith("The coverage statistics at "))
    b = lines.index("End of statistics.")
    return lines[a + 1:b], lines[b + 1], lines[b + 2]


@pytest.mark.gpu
def test_cli_prints_tlcs_block(pkg, tmp_path):
    cfg = tmp_path / "VSR.cfg"
    cfg.write_text(pkg.cfg_text(2, ["v1"], 1))
    r = subprocess.run([EXE, "-deadlock", "-coverage", "1", "-config", str(cfg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    block, project_line, next_line = _coverage_block(r.stdout)
    assert len(block) == NA and next_line.startswith("100 states generated, 76 distinct states found")
    rows = [re.match(r"^<(\w+) .*>: (\d+):(\d+)$", l) for l in block]
    assert all(rows)
    assert [m.group(1) for m in rows] == ["Init"] + pkg.ACTION_NAMES[1:]
    api = pkg.ModelChecker.from_constants(2, 1, 1).check(coverage=True, **SMALL).coverage
    assert [int(m.group(3)) for m in rows] == [g for _, g in api.by_action.values()]
    assert sum(int(m.group(2)) for m in rows) == 76
    assert [(m.group(2), m.group(3)) for m in rows[16:]] == [("0", "0")] * 4
    never = [pkg.ACTION_NAMES[a] for a in range(1, 16) if not reference(2, 1, 1)[0][:, a].any()]
    assert never and never == api.never_enabled
    assert project_line == "Coverage: %d of 15 lowered actions never enabled: %s" % (len(never), ", ".join(never))


@pytest.mark.gpu
def test_cli_coverage_beside_the_temporal_property(pkg, tmp_path):
    cfg = tmp_path / "VSR.cfg"
    text = pkg.cfg_text(2, ["v1"], 1).replace("INIT Init\nNEXT Next\n", "SPECIFICATION Spec\n") + "PROPERTY\nViewChangeCompletes\n"
    cfg.write_text(text)
    r = subprocess.run([EXE, "-deadlock", "-coverage", "1", "-config", str(cfg)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "Finished checking temporal properties" in r.stdout
    assert len(_coverage_block(r.stdout)[0]) == NA
