"""The expand kernel's shapes against the oracle, and a per-level audit of the seen-set and the frontier.

Which code a layout runs depends on its shape (ExpandCfg in vsr_gpu.cuh): warps per block, blocks per SM, one or two scan
passes per round, and a 32- or 64-row staging area per warp.  The CPU tests list the shape of every built-in layout and
require an oracle-parity case for every shape in use and for every built-in layout.  The GPU tests run the layouts the
older parity tests leave out, kernel variants built with the experiment flags of tools/variants.sh (pool overflow on every
round, one pass on a two-pass layout, 16 warps, 1- and 4-entry buckets), multi-rank expansion on the one-pass shapes, and
the per-level audit (vsr_engine_audit_level) at sizes the oracle cannot enumerate.
"""
import concurrent.futures
import os
import pickle
import re
import subprocess
import sys
import tempfile
import types

import pytest

import orc
import test_gpu_parity as tgp
from conftest import ROOT, REF_CFG

CSRC = os.path.join(ROOT, "vsr-tlaplus_b200", "csrc")
TESTS = os.path.join(ROOT, "tests")


def builtin_layouts():
    """Layout<R, V, K> of VSR_FOR_EACH_CONFIG (vsr_model.h), as constants (R, V, L = K - 1)"""
    text = open(os.path.join(CSRC, "vsr_model.h")).read()
    return [(int(r), int(v), int(k) - 1) for r, v, k in re.findall(r"X\((\d+), (\d+), (\d+)\)", text)]


# -------------------------------------------------------------------------------------------------- parity cases
# (R, V, L, depth): the built-in layouts the parity tests of test_gpu_parity.py do not run.  depth 0 = the complete
# space; otherwise the oracle stays at 0.3 - 0.7 million states (a few seconds on eight threads).  (4, 3, 2) is
# Layout<4,3,3>, the only 22-warp two-pass layout (704 parents per pass); it goes as deep as the oracle affords
# (1.46 million states), and its levels exceed 2 x 704 states from depth 7 on.
NEW_PARITY = [(2, 2, 1, 0), (2, 3, 2, 0), (3, 1, 2, 14), (3, 2, 3, 12), (3, 3, 1, 22), (4, 1, 1, 15), (4, 2, 1, 15), (4, 3, 2, 11),
              (5, 1, 1, 9), (5, 2, 1, 9), (5, 3, 2, 8)]
# multi-rank expansion on one device: a 64-row one-pass layout and the two-block layout
MULTI_CASES = [(4, 2, 2, 7), (5, 2, 2, 7)]
# kernel variants (the flags of tools/variants.sh), each built for the single layouts listed with it
VARIANTS = {
    "qps1": ("-DVSR_QPS=1", [(3, 2, 2), (4, 3, 2)]),           # pool overflow (leftovers) on every round
    "passes1": ("-DVSR_ROUND_PASSES=1", [(3, 2, 2), (4, 3, 2)]),  # one scan pass and the 64-row staging on a two-pass layout
    "warps16": ("-DVSR_FORCE_WARPS=16", [(3, 2, 2)]),          # two blocks of 16 warps (fit on Layout<3,2,3> only)
    "bucket1": ("-DVSR_BUCKET=1", [(3, 2, 2), (4, 3, 2)]),
    "bucket4": ("-DVSR_BUCKET=4", [(3, 2, 2), (4, 3, 2)]),
}
VARIANT_DEPTH = {(3, 2, 2): 13, (4, 3, 2): 10}


def parametrized(fn):
    return [tuple(p) for m in getattr(fn, "pytestmark", []) if m.name == "parametrize" for p in m.args[1]]


def oracle_parity_layouts():
    """constants (R, V, L) of every per-depth state-set comparison with the oracle on the GPU"""
    cases = {p[:3] for p in parametrized(tgp.test_full_state_space_matches_oracle)}
    cases |= {p[:3] for p in parametrized(tgp.test_bounded_depth_matches_oracle)}
    cases |= {p[:3] for p in NEW_PARITY}
    return cases


@pytest.fixture(scope="module")
def shapes(pkg):
    return {c: pkg.ModelChecker.from_constants(*c).expand_shape() for c in builtin_layouts()}


def test_shape_of_every_builtin_layout(shapes):
    """(warps, blocks, passes, staging rows) per layout; the shapes obey ExpandCfg's rules"""
    assert len(shapes) == 20
    for c, (warps, blocks, passes, rows) in sorted(shapes.items()):
        print("R=%d V=%d L=%d  Layout<%d,%d,%d>  %2d warps x %d blocks, %d pass(es), %d-row staging" % (c + (c[0], c[1], c[2] + 1, warps, blocks, passes, rows)))
        assert blocks == (1 if warps > 16 else 2)
        assert rows == (32 if passes == 2 else 64)
        assert passes == 1 or blocks == 1
    # the shape the profile's unexplained (4,3,2) result ran on: 22 warps, two passes
    assert shapes[(4, 3, 2)] == (22, 1, 2, 32)


def test_every_shape_and_layout_has_oracle_parity(shapes):
    """a layout or tuning change that creates a new kernel shape fails here until a parity case covers it"""
    covered = oracle_parity_layouts()
    assert set(shapes) <= covered, "built-in layouts without oracle parity: %s" % sorted(set(shapes) - covered)
    for shape in set(shapes.values()):
        assert any(shapes[c] == shape for c in covered if c in shapes), "no oracle-parity case for shape %s" % (shape,)
    # the multi-rank and variant cases run the shapes they are meant for
    assert {shapes[c[:3]][3] for c in MULTI_CASES} == {64} and {shapes[c[:3]][1] for c in MULTI_CASES} == {1, 2}
    assert all(shapes[c][2] == 2 for _, cs in VARIANTS.values() for c in cs)


# -------------------------------------------------------------------------------------------------- variant libraries
def _variant_jobs(out, name, flags, R, V, L):
    only = ["-DVSR_ONLY_R=%d" % R, "-DVSR_ONLY_V=%d" % V, "-DVSR_ONLY_K=%d" % (L + 1)] + flags.split()
    tag = "%s_%d_%d_%d" % (name, R, V, L)
    nv = [os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
          "-Xcompiler", "-fPIC", "-diag-suppress", "128"] + only
    objs = {src: os.path.join(out, "%s_%s.o" % (src.split(".")[0], tag)) for src in ("vsr_gpu.cu", "vsr_shard.cu", "vsr_ckpt.cu", "vsr_host.cpp")}
    jobs = [nv + ["-c", src, "-o", o] for src, o in objs.items() if src.endswith(".cu")]
    jobs.append(["g++", "-O2", "-std=c++17", "-fPIC"] + only + ["-c", "vsr_host.cpp", "-o", objs["vsr_host.cpp"]])
    return tag, list(objs.values()), jobs


def _run(cmd):
    r = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert r.returncode == 0, (cmd, r.stderr[-3000:])


def build_variants(out, variants):
    """single-layout libvsr_b200 builds with extra -D flags (the command lines of tools/variants.sh), objects in parallel.
    Returns {(name, R, V, L): path of the library}."""
    group = os.path.join(out, "vsr_group.o")
    jobs, links = [["g++", "-O2", "-std=c++17", "-fPIC", "-c", "vsr_group.cpp", "-o", group]], {}
    for name, (flags, cases) in variants.items():
        for R, V, L in cases:
            tag, objs, j = _variant_jobs(out, name, flags, R, V, L)
            jobs += j
            links[(name, R, V, L)] = (os.path.join(out, "libvsr_b200_%s.so" % tag), objs)
    with concurrent.futures.ThreadPoolExecutor(max(2, os.cpu_count() or 2)) as ex:
        list(ex.map(_run, jobs))
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with concurrent.futures.ThreadPoolExecutor(max(2, os.cpu_count() or 2)) as ex:
        list(ex.map(_run, [[nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xlinker", "-Bsymbolic", "-o", so] + objs + [group, "-ldl", "-lpthread", "-lrt"]
                           for so, objs in links.values()]))
    return {k: so for k, (so, _) in links.items()}


@pytest.fixture(scope="module")
def variant_libs():
    with tempfile.TemporaryDirectory(prefix="vsr-variants-") as d:
        yield build_variants(d, VARIANTS)


def variant_shape(so, R, V, L):
    """in a child process: the template thunks' static tables are unique symbols, which the dynamic linker would share
    with an already loaded libvsr_b200.so"""
    out = _child("import os; os.environ['VSR_B200_LIB'] = %r\nimport _pkg; pkg = _pkg.load()\n"
                 "print('SHAPE', *pkg.ModelChecker.from_constants(%d, %d, %d).expand_shape())\nprint('CHILD-OK')\n" % (so, R, V, L))
    return tuple(int(x) for x in out.split("SHAPE", 1)[1].split()[:4])


def test_variant_libraries_build_with_their_shapes(variant_libs, shapes):
    """every variant builds for sm_90a, and the flags reach the kernel's shape"""
    for (name, R, V, L), so in variant_libs.items():
        w, b, p, rows = variant_shape(so, R, V, L)
        base = shapes[(R, V, L)]
        if name == "passes1":
            assert (w, b, p, rows) == (base[0], base[1], 1, 64)
        elif name == "warps16":
            assert (w, b) == (16, 2)
        elif name == "qps1":  # a tenth of the pool: more warps may fit
            assert w >= base[0] and (b, p, rows) == base[1:]
        else:
            assert (w, b, p, rows) == base


# -------------------------------------------------------------------------------------------------- the BFS, audited
def check_audit(a, level, size):
    assert a.level == level and a.size == size
    assert a.found == a.tagged == size, "depth %d: %d states, %d in the seen-set with this tag, %d seen-set entries with it" % (level, size, a.found, a.tagged)
    assert (a.fp_sum, a.fp_xor) == (a.tagged_fp_sum, a.tagged_fp_xor), "depth %d: the frontier's fingerprints are not the tagged entries'" % level


def engine_bfs(pkg, mc, max_depth=0, table=1 << 23, frontier=1 << 21, collect=True, audit=True, **kw):
    """The BFS pumped level by level through GpuEngine (reset / seed / expand / finish), every level audited.  Returns an
    object with the fields assert_same_exploration compares and the seen-set's fingerprint collisions per level, and per
    level (size, generated, fingerprint sum, fingerprint xor, words sum, words xor)."""
    from vsr_tlaplus_b200 import dist as vdist
    keep = kw.pop("keep", False)  # leave the engine open (res.engine) for the caller
    eng = vdist.GpuEngine(mc, 0, 1, table_capacity=table, frontier_capacity=frontier, keep_trace=kw.pop("keep_trace", False),
                          collect_levels=collect, **kw)
    try:
        eng.reset()
        eng.seed()
        li = eng.finish()
        sizes, gens, colls, rows, ties, generated, complete = [], [], [], [], 0, int(li.generated), False
        while True:
            assert li.error_code == 0 and li.overflow == 0, ("depth", len(sizes) + 1, "error", li.error_code, "overflow", li.overflow,
                                                             "new states", li.new_states)
            ties += int(li.ties)
            if li.new_states == 0:
                complete = True
                break
            sizes.append(int(li.new_states))
            colls.append(int(li.collisions))
            if audit:
                a = eng.audit()
                check_audit(a, len(sizes), sizes[-1])
                rows.append((sizes[-1], int(li.generated), a.fp_sum, a.fp_xor, a.words_sum, a.words_xor))
            if max_depth and len(sizes) >= max_depth:
                break
            eng.expand()
            li = eng.finish()
            gens.append(int(li.generated))
            generated += int(li.generated)
        res = types.SimpleNamespace(rc=0, error_code=0, level_sizes=sizes, level_generated=(gens + [0])[:len(sizes)] if not complete else gens,
                                    distinct=sum(sizes), generated=generated, depth=len(sizes), h2_ties=ties, complete=complete, level_collisions=colls,
                                    queue=0 if complete else sizes[-1], levels=[eng.collected(d) for d in range(1, len(sizes) + 1)] if collect else [],
                                    engine=eng)
        if not keep:
            eng.close()
        return res, rows
    except BaseException:
        eng.close()
        raise


_oracle = {}


def oracle(R, V, L, depth, symmetry=True):
    key = (R, V, L, depth, symmetry and V > 1)
    if key not in _oracle:
        q = orc.params(R, V, L, symmetry=key[-1])
        _oracle[key] = (q, orc.bfs(q, workers=8, max_depth=depth, keep_trace=False, digests=True))
    return _oracle[key]


def assert_parity(pkg, R, V, L, depth, res, mc):
    q, o = oracle(R, V, L, depth)
    tgp.assert_same_exploration(pkg, mc, res, q, o, complete=depth == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth", NEW_PARITY)
def test_layout_matches_oracle(pkg, R, V, L, depth):
    """every depth's SET of states equal to the oracle's, TLC's scalars equal, every level's audit holds"""
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=V > 1)
    res, _ = engine_bfs(pkg, mc, max_depth=depth)
    assert_parity(pkg, R, V, L, depth, res, mc)
    warps, _, passes, _ = mc.expand_shape()
    if passes == 2 and depth:
        # the second pass of a round runs, and batches map to pass-1 parents, at several expanded depths
        assert sum(s > 2 * 32 * warps for s in res.level_sizes[:-1]) >= 3


def release_device_memory(device=0):
    """Give the device memory this process keeps cached back to the driver, so that a child process can have it.  An
    engine keeps freed memory in the device's default pool (release threshold: everything, see vsr_engine_create), and
    earlier tests of this process allocated seen-sets of tens of GB there.  Returns the free device memory in bytes."""
    import ctypes as C
    import torch
    torch.cuda.synchronize(device)
    torch.cuda.empty_cache()
    cu = C.CDLL("libcuda.so.1")
    dev, pool = C.c_int(), C.c_void_p()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    cu.cuMemPoolTrimTo.argtypes = [C.c_void_p, C.c_size_t]
    assert cu.cuMemPoolTrimTo(pool, 0) == 0
    return torch.cuda.mem_get_info(device)[0]


def _child(code, timeout=900):
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path[:0] = [%r, %r]\n" % (ROOT, TESTS) + code], capture_output=True, text=True,
                       timeout=timeout)
    assert r.returncode == 0 and "CHILD-OK" in r.stdout, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def run_in_child(so, R, V, L, depth, out, collect=True, **kw):
    """the audited engine BFS with the library `so` in a child process (a variant's kernels may not have run on a GPU
    before: a fault there must not take the suite with it); per-depth canonical digest sets and audit rows to `out`"""
    env_code = "import os; os.environ['VSR_B200_LIB'] = %r\n" % so if so else ""
    _child(env_code + (
        "import pickle, _pkg; pkg = _pkg.load()\n"
        "import orc, test_kernel_shapes as t, test_gpu_parity as tgp\n"
        "mc = pkg.ModelChecker.from_constants(%d, %d, %d, symmetry=%d > 1)\n"
        "res, rows = t.engine_bfs(pkg, mc, max_depth=%d, collect=%r, **%r)\n"
        "sets = tgp.level_digest_sets(pkg, mc, res, orc.params(%d, %d, %d, symmetry=%d > 1)) if %r else []\n"
        "res.levels = []; del res.engine\n"
        "pickle.dump((vars(res), rows, sets), open(%r, 'wb'))\n"
        "print('CHILD-OK')\n") % (R, V, L, V, depth, collect, kw, R, V, L, V, collect, out))
    d, rows, sets = pickle.load(open(out, "rb"))
    return types.SimpleNamespace(**d), rows, sets


def assert_child_parity(R, V, L, depth, res, sets, symmetry=True):
    q, o = oracle(R, V, L, depth, symmetry)
    assert res.level_sizes == o.level_sizes
    assert res.level_generated[:len(o.level_generated)] == o.level_generated
    assert (res.distinct, res.generated, res.depth, res.h2_ties) == (o.distinct, o.generated, o.depth, o.h2_ties)
    assert len(sets) == len(o.level_digests)
    for d, (g, w) in enumerate(zip(sets, o.level_digests)):
        assert g == set(w), f"depth {d + 1}: GPU and oracle state sets differ"


@pytest.mark.gpu
@pytest.mark.parametrize("name,R,V,L", [(n, *c) for n, (_, cs) in VARIANTS.items() for c in cs])
def test_kernel_variant_matches_oracle(variant_libs, tmp_path, name, R, V, L):
    depth = VARIANT_DEPTH[(R, V, L)]
    res, rows, sets = run_in_child(variant_libs[(name, R, V, L)], R, V, L, depth, str(tmp_path / "out.pkl"))
    assert_child_parity(R, V, L, depth, res, sets)


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth", MULTI_CASES)
def test_multi_rank_on_one_pass_shapes_matches_oracle(pkg, monkeypatch, R, V, L, depth):
    """expand_kernel<L, true> (push_records + drain) on the 64-row staging area and on the two-block shape: outgoing
    records fill rows 32..63 while rows 0..sn-1 hold staged states"""
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")
    q, o = oracle(R, V, L, depth)
    mc = pkg.ModelChecker.from_constants(R, V, L)
    for world in (2, 4):
        res = mc.check_multi(world, max_depth=depth, table_capacity=1 << 22, frontier_capacity=1 << 20, stop_on_violation=False)
        assert res.error_code == 0 and res.rc in (0, 12), res.rc
        assert res.level_sizes == o.level_sizes, world
        assert res.level_generated[:len(o.level_generated)] == o.level_generated, world
        assert (res.distinct, res.generated, res.depth) == (o.distinct, o.generated, o.depth), world
        assert res.records_sent > 0


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth", [(3, 2, 2, 11), (4, 3, 2, 11)])
def test_trace_records_of_two_pass_layouts_rebuild_the_states(pkg, R, V, L, depth):
    """every sampled state's trace chain (parent id, candidate), replayed from Init, ends in that very state.  States
    expanded from the second scan pass of a round must point at their own parents (si = pass * NS + thread)."""
    import ctypes as C
    mc = pkg.ModelChecker.from_constants(R, V, L)
    res, _ = engine_bfs(pkg, mc, max_depth=depth, keep_trace=True, keep=True)
    eng = res.engine
    try:
        sb, cap = mc.state_bytes, depth + 2
        first = 0
        checked = 0
        for d, raw in enumerate(res.levels, start=1):
            n = len(raw) // sb
            for i in sorted({(k * 7919) % n for k in range(min(n, 200))}):
                tr, acts = mc._buf(cap), (C.c_uint8 * cap)()
                m = mc._lib.vsr_engine_build_trace(eng._e, first + i, tr, acts, cap)
                assert m == d, (d, i, m)
                assert bytes(tr)[(m - 1) * sb:m * sb] == raw[i * sb:(i + 1) * sb], f"depth {d} state {i}: its trace leads elsewhere"
                checked += 1
            first += n
        assert checked > 1000
    finally:
        eng.close()


# -------------------------------------------------------------------------------------------------- beyond the oracle
@pytest.mark.gpu
def test_r4_v3_l2_depth18_is_deterministic_under_audit(pkg, variant_libs, tmp_path):
    """(4,3,2) to depth 18, where depth-bounded runs once reported different distinct counts: a 1.25e9-slot seen-set, a
    2^31-slot one, and the one-pass build.  Each runs once; per-level sizes, successor counts and both frontier digests
    must be identical, and every level's audit must hold (found == tagged == size).  Depth 18 alone holds 349 million
    states of 80 bytes, more than a frontier sized from the free memory of an 80 GB card (about 211 million per buffer):
    such a run ends with 152 and a last level truncated to the frontier's capacity, which moves with the free memory.  So
    every level fits here: 200 million states per buffer in device memory and 200 million more in pinned host memory.
    Each run has a process to itself, and this process first hands back the device memory it keeps cached: the largest
    run needs 66 GB of device memory (2^31 slots of 16 bytes and two frontier buffers)."""
    free = release_device_memory()
    assert free >= 68e9, "%.1f GB of device memory free; the 2^31-slot run needs 66 GB" % (free / 1e9)
    caps = dict(collect=False, frontier=200_000_000, frontier_host_capacity=200_000_000)
    a, rows_a, _ = run_in_child(None, 4, 3, 2, 18, str(tmp_path / "a.pkl"), table=1_250_000_000, **caps)
    b, rows_b, _ = run_in_child(None, 4, 3, 2, 18, str(tmp_path / "b.pkl"), table=1 << 31, **caps)
    c, rows_c, _ = run_in_child(variant_libs[("passes1", 4, 3, 2)], 4, 3, 2, 18, str(tmp_path / "p1.pkl"), table=1_250_000_000, **caps)
    print("(4,3,2) depth 18: distinct", a.distinct, b.distinct, c.distinct, "generated", a.generated, b.generated, c.generated, "levels", a.level_sizes)
    assert len(rows_a) == 18 and max(a.level_sizes) > 200_000_000  # the last level continues in host memory
    assert rows_a == rows_b, [i + 1 for i, (x, y) in enumerate(zip(rows_a, rows_b)) if x != y]
    assert rows_a == rows_c, [i + 1 for i, (x, y) in enumerate(zip(rows_a, rows_c)) if x != y]
    assert (a.distinct, a.generated) == (b.distinct, b.generated) == (c.distinct, c.generated) == (705_737_513, 2_883_924_044)
    assert a.level_sizes[-1] == 349_206_481


@pytest.mark.gpu
def test_shipped_cfg_complete_under_audit(pkg):
    """the shipped VSR.cfg, complete (1.17e9 states): every level's audit holds, and TLC's totals"""
    mc = pkg.ModelChecker.from_cfg(REF_CFG)
    res, rows = engine_bfs(pkg, mc, table=1 << 31, frontier=130_000_000, collect=False)
    assert res.complete
    assert (res.distinct, res.generated, res.depth) == (1_173_992_337, 3_129_587_684, 47)
    assert len(rows) == 47
