"""Layout plug-ins at the edges of the packed encoding.

Every ReplicaCount / |Values| / StartViewOnTimerLimit outside the built-in layouts reaches the GPU through a plug-in
(csrc/vsr_layout_plugin.cu, compiled on first use).  Only some of the encoding's 630 layouts can be built: the packed state
must fit VSR_MAX_STATE_BYTES, the expand kernel's shared memory one SM, and the largest action group the kernel's 16-bit
pool item.  tests/harness/layout_table.cu lists, for every layout, its sizes, its expand-kernel shape and these limits,
from the very constexprs the kernel asserts.  On the CPU the tests hold that table against the layout restatement, the
built-in shapes, the loader's refusals and the documents, and run the host differential on the edge layouts.  On the GPU
the edge layouts -- the shapes no built-in layout has, the widest state, the largest action group, R = 7, V = 7, L = 14
and L = 0 -- must explore the oracle's per-depth state sets, walk as the host walks, find the oracle's violations, and
keep the oracle's levels across two ranks and across the end of the frontier's HBM part.
"""
import concurrent.futures
import ctypes as C
import json
import os
import re
import subprocess
import sys
import types

import pytest

import test_kernel_shapes as tks
from conftest import ROOT
from test_fp_collisions import layout_bits

CSRC = os.path.join(ROOT, "vsr-tlaplus_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

# (R, V, L, SYMMETRY, depth; 0 = the complete space).  Depths keep the oracle at a few hundred thousand states at most.
EDGE = [
    (2, 6, 14, True, 17),   # widest state (64 words), views up to 15; 8 warps whose shared memory leaves one block per SM
    (6, 5, 2, True, 6),     # largest action group (125 candidates), 449 candidates; R = 6
    (3, 4, 10, True, 10),   # 64 words, a group of 120, the most message slots (236)
    (4, 7, 4, False, 8),    # V = 7 at 64 words
    (5, 7, 2, False, 7),    # V = 7, R = 5, a group of 112
    (2, 7, 12, True, 12),   # the canonical labelling of 7 values
    (2, 7, 12, False, 18),  # the same layout, deeper
    (7, 1, 1, True, 7),     # R = 7: 4-bit replica indices, a majority of 4; 12 warps x 2 blocks
    (7, 3, 0, True, 23),    # R = 7 with L = 0, a group of 108
    (2, 2, 14, True, 22),   # 20 warps, one block, one pass; L = 14
    (2, 1, 0, True, 0),     # L = 0: the view-change and state-transfer groups are empty
    (3, 2, 0, False, 0),    # L = 0, the complete space of the host test, on the GPU
]
EDGE_LAYOUTS = sorted({c[:3] for c in EDGE})
WIDE = (3, 4, 10)           # the 64-word layout of the two-rank, spill and counterexample cases
WIDE_DEPTH = 9


# -------------------------------------------------------------------------------------------------- the table
@pytest.fixture(scope="session")
def table(tmp_path_factory):
    """{(R, V, L): row} of tests/harness/layout_table.cu for every layout of the encoding"""
    exe = str(tmp_path_factory.mktemp("layout-table") / "layout_table")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I", CSRC,
                    os.path.join(ROOT, "tests", "harness", "layout_table.cu"), "-o", exe], check=True, capture_output=True)
    lines = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split("\n")
    cols = lines[0].split()
    out = {}
    for ln in lines[1:]:
        if ln.strip():
            r = types.SimpleNamespace(**dict(zip(cols, map(int, ln.split()))))
            r.buildable = bool(r.state_ok and r.smem_ok and r.pool_ok)
            r.shape = (r.warps, r.blocks, r.passes, r.rows)
            out[(r.R, r.V, r.L)] = r
    return out


def buildable(table):
    return {c: r for c, r in table.items() if r.buildable}


def largest_l(table):
    """{R: [largest buildable L for |Values| = 1..7, None where none builds]}"""
    ok = buildable(table)
    return {R: [max([L for L in range(15) if (R, V, L) in ok], default=None) for V in range(1, 8)] for R in range(2, 8)}


def test_table_covers_the_encoding_and_matches_the_layout_restatement(table):
    assert set(table) == {(R, V, L) for R in range(2, 8) for V in range(1, 8) for L in range(15)}
    for (R, V, L), r in table.items():
        assert r.nw == layout_bits(R, V, L)[1], (R, V, L)
        assert r.state_ok == (4 * r.nw <= 256)
        assert r.maxgrp <= r.ncand
    ok = buildable(table)
    print("buildable layouts: %d of %d" % (len(ok), len(table)))
    print("shapes:", sorted({r.shape for r in ok.values()}))
    # the numbers the cases below are chosen by
    assert len(ok) == 259
    assert max(r.nw for r in ok.values()) == 64 and max(r.maxgrp for r in ok.values()) == 125
    assert max(r.ncand for r in ok.values()) == 449
    # the buildable L of each (R, V) are 0 .. largest: the documents can state the range by its end
    for (R, V), top in [((R, V), largest_l(table)[R][V - 1]) for R in range(2, 8) for V in range(1, 8)]:
        assert all(((R, V, L) in ok) == (top is not None and L <= top) for L in range(15)), (R, V)


def test_table_shapes_equal_the_builtin_layouts(pkg, table):
    builtin = tks.builtin_layouts()
    assert len(builtin) == 20
    for c in builtin:
        mc = pkg.ModelChecker.from_constants(*c)
        assert table[c].buildable
        assert table[c].shape == mc.expand_shape(), c
        assert table[c].nw * 4 == mc.state_bytes


def test_every_buildable_layout_fits_the_flat_message_bag(table):
    """the flat form holds VSR_MAX_MSGS messages; the oracle's to_flat stops there without a word, so no buildable layout may
    have more message slots"""
    cap = int(re.search(r"#define VSR_MAX_MSGS (\d+)", open(os.path.join(ROOT, "include", "vsr_flat.h")).read()).group(1))
    ok = buildable(table)
    most = max(ok, key=lambda c: ok[c].msgs)
    assert ok[most].msgs <= cap
    assert (most, ok[most].msgs) == ((3, 4, 10), 236)


def test_every_buildable_shape_has_oracle_parity(table):
    """a shape any buildable layout gets -- built in or a plug-in -- needs a per-depth parity case on the GPU: among the
    built-in layouts' cases (test_gpu_parity, test_kernel_shapes) or the edge cases here"""
    covered = {table[c].shape for c in tks.oracle_parity_layouts()} | {table[c[:3]].shape for c in EDGE}
    missing = {r.shape for r in buildable(table).values()} - covered
    assert not missing, "kernel shapes of buildable layouts without a GPU parity case: %s" % sorted(missing)
    assert all(table[c].buildable for c in EDGE_LAYOUTS)
    # and the edges the cases are there for
    edge = [table[c] for c in EDGE_LAYOUTS]
    assert max(r.nw for r in edge) == 64 and max(r.maxgrp for r in edge) == 125
    assert {7, 6} <= {r.R for r in edge} and 7 in {r.V for r in edge} and {0, 14} <= {r.L for r in edge}


# -------------------------------------------------------------------------------------------------- the loader
def _refusal(pkg, R, V, L):
    with pytest.raises(pkg.VsrError) as e:
        pkg.ModelChecker.from_constants(R, V, L)
    assert e.value.rc == 151
    msg = str(e.value)
    assert "\n" not in msg and "ReplicaCount=%d |Values|=%d StartViewOnTimerLimit=%d" % (R, V, L) in msg, msg
    assert "cannot be built" in msg and "log " not in msg, msg
    return msg


def _first(table, **want):
    return min(c for c, r in table.items() if all(getattr(r, k) == v for k, v in want.items()))


def test_loader_names_the_limit_a_layout_exceeds(pkg, table):
    """one refusal per limit, each a one-line 151 that names the numbers; the compiler stops at the limit in seconds"""
    # a state over 256 bytes takes more shared memory than an SM has, in every layout of the encoding
    assert all(r.smem_ok == r.state_ok for r in table.values())
    state = _first(table, state_ok=0, pool_ok=1)
    assert state == (2, 7, 13)
    msg = _refusal(pkg, *state)
    assert "the packed state would be %d bytes, more than 256" % (4 * table[state].nw) in msg, msg
    assert "the expand kernel's shared memory would be %d bytes, more than the 232448 of an SM" % table[state].smem in msg, msg
    assert "pool item" not in msg, msg
    pool = (7, 1, 7)
    assert not table[pool].pool_ok and table[pool].state_ok and table[pool].smem_ok
    msg = _refusal(pkg, *pool)
    assert "an action group of %d bindings does not fit the expand kernel's 16-bit pool items (at most 127)" % table[pool].maxgrp in msg, msg
    assert "packed state" not in msg, msg
    every = (7, 7, 14)
    assert not (table[every].state_ok or table[every].smem_ok or table[every].pool_ok)
    msg = _refusal(pkg, *every)
    assert "the packed state would be 1392 bytes" in msg and "an action group of 1176 bindings" in msg, msg
    assert "the expand kernel's shared memory would be %d bytes, more than the 232448 of an SM" % table[every].smem in msg, msg


def test_loader_builds_the_layouts_at_the_limits(plugins, table):
    """the accepted side of each limit: a 64-word state, the largest action group, the most shared memory"""
    ok = buildable(table)
    assert table[(2, 6, 14)].nw == 64 and table[(6, 5, 2)].maxgrp == 125
    assert table[(2, 2, 14)].smem == max(r.smem for r in ok.values())
    for c in ((2, 6, 14), (6, 5, 2), (2, 2, 14)):
        assert plugins[c] == "LOADED %d" % (4 * table[c].nw), (c, plugins[c])


def _load_in_child(c):
    code = ("import sys; sys.path.insert(0, %r); import _pkg; pkg = _pkg.load()\n"
            "print('LOADED', pkg.ModelChecker.from_constants(%d, %d, %d).state_bytes)\n" % ((ROOT,) + c))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    return r.stdout.strip() or r.stderr[-2000:]


@pytest.fixture(scope="session")
def plugins(pkg):
    """every edge layout's plug-in, built in parallel (one child process each; the loader locks per layout)"""
    with concurrent.futures.ThreadPoolExecutor(min(8, os.cpu_count() or 2)) as ex:
        return dict(zip(EDGE_LAYOUTS, ex.map(_load_in_child, EDGE_LAYOUTS)))


# -------------------------------------------------------------------------------------------------- the documents
DOCS = ["README.md", "INTEGRATION.md", "DESIGN.md", os.path.join("include", "vsr_b200.h")]


def doc_table(path):
    """the rows '| R | L | L | L | L | L | L | L |' of a document's table of the largest buildable L per (R, |Values|)"""
    text = open(os.path.join(ROOT, path)).read()
    rows = re.findall(r"^[ *]*\| ([2-7]) \|((?: (?:\d+|-) \|){7})[ \t]*$", text, re.M)
    return {int(R): [None if x == "-" else int(x) for x in re.findall(r"\d+|-", rest)] for R, rest in rows}


@pytest.mark.parametrize("path", DOCS)
def test_documents_state_the_buildable_range(table, path):
    assert doc_table(path) == largest_l(table), path
    text = open(os.path.join(ROOT, path)).read()
    assert "10 s" not in text, "%s: the plug-in compile time" % path


# -------------------------------------------------------------------------------------------------- host differential
@pytest.mark.parametrize("R,V,L", EDGE_LAYOUTS)
def test_edge_layout_matches_oracle_on_the_host(plugins, R, V, L):
    """pack, unpack, Next and the canonical form at the field widths' edges: random walks, successor by successor against
    the oracle, with SYMMETRY on and off"""
    assert plugins[(R, V, L)].startswith("LOADED"), plugins[(R, V, L)]
    exe = os.path.join(ROOT, "build", "diff_host")
    for sym in (1, 0):
        n = {6: 1000, 7: 150}.get(V, 4000) if sym else 4000  # with SYMMETRY, 720 or 5040 permutations per successor
        out = json.loads(subprocess.run([exe, str(R), str(V), str(L), str(sym), str(n), "1", "100000", str(7 + R + V + L)], check=True,
                                        capture_output=True, text=True).stdout)
        assert out["mismatches"] == 0 and out["assumption_violations"] == 0, out
        assert out["checked"] == n or (L == 0 and out["checked"] > 0), out


# -------------------------------------------------------------------------------------------------- on the GPU
def _gpu_child(code, timeout=1800):
    """in a child process: these layouts' kernels run on a GPU nowhere else, and a fault must be reported against the case"""
    return tks._child("import _pkg; pkg = _pkg.load()\n"
                      "import orc, test_gpu_parity as tgp, test_kernel_shapes as tks, test_simulate as ts, test_layout_edges as te\n" + code,
                      timeout=timeout)


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,sym,depth", EDGE)
def test_edge_layout_matches_oracle_on_the_gpu(plugins, R, V, L, sym, depth):
    """per-depth state sets, successors per level, ties and completeness equal to the oracle's, every level audited; then
    the simulation kernel's walks equal the host's"""
    out = _gpu_child(
        "mc = pkg.ModelChecker.from_constants(%d, %d, %d, symmetry=%r)\n"
        "res, _ = tks.engine_bfs(pkg, mc, max_depth=%d)\n"
        "q = orc.params(%d, %d, %d, symmetry=%r and %d > 1)\n"
        "o = orc.bfs(q, workers=8, max_depth=%d, keep_trace=False, digests=True)\n"
        "tgp.assert_same_exploration(pkg, mc, res, q, o, complete=%r)\n"
        "print('PARITY depth', res.depth, 'distinct', res.distinct, 'generated', res.generated, 'complete', res.complete)\n"
        "st = ts.check_walks_like_the_host(pkg, %d, %d, %d, %r, 100, %d, ts.threads())\n"
        "assert st.steps > st.walks\n"
        "print('CHILD-OK')\n" % (R, V, L, sym, depth, R, V, L, sym, V, depth, depth == 0, R, V, L, sym, 1000 + 100 * R + 10 * V + L))
    print(out)


def assert_counterexample_is_a_behaviour(pkg, mc, res, R, V, L):
    """every step of the GPU's trace a step of the oracle's Next with the action it names, only the last state violating"""
    import orc
    q = orc.params(R, V, L, symmetry=False, invariant=2)
    lib = orc.lib()
    flats = [mc.unpack(st) for _, st in res.trace]
    assert res.trace[0][0] == "Initial predicate"
    cap = 1024
    for i in range(len(flats) - 1):
        succ = (pkg.checker.VsrFlatState * cap)()
        acts = (C.c_int * cap)()
        n = lib.orc_successors_flat(q, C.byref(flats[i]), succ, acts, cap)
        assert 0 < n < cap
        want = orc.digests_full_of(q, (pkg.checker.VsrFlatState * 1)(flats[i + 1]))[0]
        got = orc.digests_full_of(q, succ)[:n]
        assert any(g == want and pkg.ACTION_NAMES[acts[k]] == res.trace[i + 1][0] for k, g in enumerate(got)), f"step {i + 1} is not a step of Next"
    assert [lib.orc_invariant_flat(q, C.byref(f)) for f in flats] == [1] * (len(flats) - 1) + [0]


def counterexample_case(pkg, R, V, L, depth):
    """AcknowledgedWritesExistOnMajority to `depth` on the GPU and in the oracle: the violation at the oracle's depth with a
    behaviour for its trace, or none within the bound in either"""
    import orc
    inv = ("AcknowledgedWritesExistOnMajority",)
    mc = pkg.ModelChecker.from_constants(R, V, L, invariants=inv)
    res = mc.check(max_depth=depth, table_capacity=1 << 23, frontier_capacity=1 << 21)
    o = orc.bfs(orc.params(R, V, L, symmetry=V > 1, invariant=2), workers=8, max_depth=depth, keep_trace=False)
    assert res.error_code == 0
    if o.rc != 12:
        print("(%d, %d, %d): AcknowledgedWritesExistOnMajority holds to depth %d (the bound stops short of any violation)" % (R, V, L, depth))
        assert res.rc == 0 and res.depth == o.depth == depth and res.distinct == o.distinct
        return
    assert res.rc == 12 and res.violated_invariants == list(inv)
    assert res.violation_level == o.depth and len(res.trace) == o.depth
    assert_counterexample_is_a_behaviour(pkg, mc, res, R, V, L)
    print("(%d, %d, %d): violated at depth %d, as in the oracle" % (R, V, L, o.depth))


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L,depth", [(7, 1, 1, 7), WIDE + (10,)])
def test_edge_counterexample_is_a_behaviour(plugins, R, V, L, depth):
    print(_gpu_child("te.counterexample_case(pkg, %d, %d, %d, %d)\nprint('CHILD-OK')\n" % (R, V, L, depth)))


def two_ranks_case(pkg, R, V, L, depth):
    """two ranks on one GPU: records of NW words + the 16-byte header pushed to the peer's inbox and drained there"""
    import orc
    os.environ["VSR_B200_MULTI_ONE_DEVICE"] = "1"
    o = orc.bfs(orc.params(R, V, L, symmetry=V > 1), workers=8, max_depth=depth, keep_trace=False)
    res = pkg.ModelChecker.from_constants(R, V, L).check_multi(2, max_depth=depth, table_capacity=1 << 22, frontier_capacity=1 << 20,
                                                               stop_on_violation=False)
    assert res.error_code == 0 and res.rc in (0, 12), res.rc
    assert res.level_sizes == o.level_sizes
    assert res.level_generated[:len(o.level_generated)] == o.level_generated
    assert (res.distinct, res.generated, res.depth) == (o.distinct, o.generated, o.depth)
    assert res.records_sent > 0
    print("two ranks: depth", res.depth, "distinct", res.distinct, "records sent", res.records_sent)


@pytest.mark.gpu
def test_wide_layout_on_two_ranks(plugins):
    print(_gpu_child("te.two_ranks_case(pkg, %d, %d, %d, %d)\nprint('CHILD-OK')\n" % (WIDE + (WIDE_DEPTH,))))


SPILL_HBM = 1000  # frontier states per buffer in HBM: the levels from depth 7 on continue in host memory


def spill_case(pkg, R, V, L, depth):
    """a frontier whose HBM part ends inside levels: the bulk stores of 256-byte rows split at the boundary"""
    import orc
    mc = pkg.ModelChecker.from_constants(R, V, L)
    res, _ = tks.engine_bfs(pkg, mc, max_depth=depth, frontier=SPILL_HBM, frontier_host_capacity=1 << 18)
    assert sum(n > SPILL_HBM for n in res.level_sizes) >= 3, res.level_sizes
    q = orc.params(R, V, L, symmetry=V > 1)
    o = orc.bfs(q, workers=8, max_depth=depth, keep_trace=False, digests=True)
    import test_gpu_parity as tgp
    tgp.assert_same_exploration(pkg, mc, res, q, o, complete=False)
    print("spill: levels", res.level_sizes)


@pytest.mark.gpu
def test_wide_layout_frontier_across_the_hbm_boundary(plugins):
    print(_gpu_child("te.spill_case(pkg, %d, %d, %d, %d)\nprint('CHILD-OK')\n" % (WIDE + (WIDE_DEPTH,))))
