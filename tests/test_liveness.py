"""PROPERTY ViewChangeCompletes == []<>AllReplicasMoveToSameView under SPECIFICATION Spec (VSR.tla:958-967).

CPU: the loader's matrix, the state predicate against a Python evaluation of it, and a reference verdict built from the
CPU oracle's complete quotient graph (canonical VIEW digests) with scipy's strongly connected components: the property is
violated iff a reachable not-P state has no successor but itself, or a cycle of not-P states exists.  GPU: the liveness
pass against that reference — the verdict, the number of stored not-P states, the BFS scalars unchanged — and, through the
test hooks of vsr_model_create (Q = "some replica has committed" instead of P; every state without successors steps to
Init), both kinds of counterexample, checked step by step against the oracle, also on a weak-fingerprint build.
"""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph

import orc
from conftest import ROOT

EXE = os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc")

# (R, V, L) with SYMMETRY: distinct states, states where P is false, states without a successor but themselves — the
# oracle's complete graph (reference_graph below); P holds eventually on every fair behaviour of all of them
TABLE = {
    (2, 1, 1): (76, 56, 5),
    (2, 2, 1): (163, 101, 11),
    (2, 1, 2): (811, 640, 51),
    (2, 2, 2): (2_073, 1_444, 128),
    (3, 1, 1): (43_941, 27_621, 2_067),
    (3, 2, 1): (349_365, 148_937, 13_244),
}
CPU_ROWS = [k for k in TABLE if k != (3, 2, 1)]  # (3, 2, 1) takes tens of seconds in Python: GPU tests only
Q_SINKS_311 = 55  # reachable not-Q states without successors in (3, 1, 1) (hook 1); none in the R = 2 spaces
FULL_321 = 697_364  # (3, 2, 1) without SYMMETRY: distinct states (tests/test_fp_collisions.py pins the same number)


def spec_cfg(pkg, R, values, L, props=("ViewChangeCompletes",), keyword="PROPERTY", symmetry=True):
    text = pkg.cfg_text(R, values, L, symmetry=symmetry).replace("INIT Init\nNEXT Next\n", "SPECIFICATION Spec\n")
    return text + keyword + "\n" + "\n".join(props) + "\n"


# -------------------------------------------------------------------------------------------------- Python definitions
def p_flat(f):
    """AllReplicasMoveToSameView on the flat form: every replica Normal (status 0), one view number"""
    reps = [f.rep[r] for r in range(f.R)]
    return all(x.status == 0 for x in reps) and len({x.view for x in reps}) == 1


def q_flat(f):
    return any(f.rep[r].commit >= 1 for r in range(f.R))


def reference_graph(pkg, R, V, L, symmetry=True):
    """the complete quotient graph from the oracle: per state (P, Q) and its successor ids (canonical VIEW digests)"""
    Flat = pkg.checker.VsrFlatState
    q = orc.params(R, V, L, symmetry=symmetry)
    lib = orc.lib()
    init = Flat()
    lib.orc_init_flat(q, C.byref(init))
    ids = {orc.digests_of(q, (Flat * 1)(init))[0][0]: 0}
    preds, succ = [(p_flat(init), q_flat(init))], []
    cap = 512
    out, acts = (Flat * cap)(), (C.c_int * cap)()
    level = [init]
    while level:
        nxt = []
        for f in level:
            n = lib.orc_successors_flat(q, C.byref(f), out, acts, cap)
            assert 0 <= n <= cap
            digs = orc.digests_of(q, out, n)[0] if n else []
            row = []
            for k, d in enumerate(digs):
                j = ids.get(d)
                if j is None:
                    j = ids[d] = len(preds)
                    g = Flat.from_buffer_copy(out[k])
                    preds.append((p_flat(g), q_flat(g)))
                    nxt.append(g)
                row.append(j)
            succ.append(row)
        level = nxt
    return preds, succ


def reference_verdict(preds, succ, use_q=False, init_edge=False):
    """holds?, #not-P, #states without a successor but themselves, #not-P such states, #non-trivial not-P SCCs"""
    n = len(preds)
    bad = np.array([not (pq[1] if use_q else pq[0]) for pq in preds])
    rows = [[j for j in set(s) if j != i] for i, s in enumerate(succ)]
    sinks = [i for i in range(n) if not rows[i]]
    if init_edge:
        for i in sinks:
            rows[i] = [0]
    bad_sinks = 0 if init_edge else sum(1 for i in sinks if bad[i])
    src = [i for i in range(n) for j in rows[i] if bad[i] and bad[j]]
    dst = [j for i in range(n) for j in rows[i] if bad[i] and bad[j]]
    g = scipy.sparse.csr_matrix((np.ones(len(src)), (src, dst)), shape=(n, n))
    k, lab = scipy.sparse.csgraph.connected_components(g, directed=True, connection="strong")
    sizes = np.bincount(lab[bad], minlength=k) if bad.any() else np.zeros(k, int)
    cycles = int((sizes >= 2).sum())
    return {"holds": bad_sinks == 0 and cycles == 0, "not_p": int(bad.sum()), "sinks": len(sinks), "bad_sinks": bad_sinks, "cycles": cycles}


# -------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("keyword", ["PROPERTY", "PROPERTIES"])
def test_spec_with_property_loads(pkg, keyword):
    mc = pkg.ModelChecker.from_cfg_text(spec_cfg(pkg, 3, ["v1", "v2"], 2, keyword=keyword))
    assert mc.info.property == 1
    spec_only = pkg.cfg_text(3, ["v1", "v2"], 2).replace("INIT Init\nNEXT Next\n", "SPECIFICATION Spec\n")
    assert pkg.ModelChecker.from_cfg_text(spec_only).info.property == 0


def test_property_without_spec_is_151(pkg):
    with pytest.raises(pkg.VsrError) as e:
        pkg.ModelChecker.from_cfg_text(pkg.cfg_text(3, ["v1", "v2"], 2) + "PROPERTY ViewChangeCompletes\n")
    assert e.value.rc == 151 and "PROPERTY" in str(e.value) and "SPECIFICATION Spec" in str(e.value)


@pytest.mark.parametrize("name", ["AllReplicasMoveToSameView", "Liveness", "ViewChangeCompletes2"])
def test_unknown_property_is_151_by_name(pkg, name):
    with pytest.raises(pkg.VsrError) as e:
        pkg.ModelChecker.from_cfg_text(spec_cfg(pkg, 3, ["v1", "v2"], 2, props=("ViewChangeCompletes", name)))
    assert e.value.rc == 151 and name in str(e.value)


def test_property_bits_of_model_create(pkg):
    mc = pkg.ModelChecker.from_constants(2, 1, 1, property=True, live_test_hooks=3)
    assert (mc.info.property, mc.info.invariant) == (1, 1)
    assert pkg.ModelChecker.from_constants(2, 1, 1).info.property == 0


@pytest.mark.parametrize("args,frag", [
    (["-simulate"], "-simulate"),
    (["-gpus", "2"], "-gpus"),
    (["-checkpoint", "0"], "-checkpoint"),
    (["-recover", "nowhere"], "-recover"),
])
def test_refused_combinations(pkg, tmp_path, args, frag):
    cfg = tmp_path / "VSR.cfg"
    cfg.write_text(spec_cfg(pkg, 2, ["v1"], 1))
    r = subprocess.run([EXE, "-deadlock", "-metadir", str(tmp_path / "states")] + args + ["-config", str(cfg)], capture_output=True, text=True)
    out = r.stdout + r.stderr
    assert r.returncode == 151 and frag in out and "ViewChangeCompletes" in out, out


def test_sharded_engine_refused(pkg):
    mc = pkg.ModelChecker.from_constants(2, 1, 1, property=True)
    e, err = C.c_void_p(), C.create_string_buffer(512)
    rc = mc._lib.vsr_engine_create(mc._h, C.byref(mc.run_opts()), 0, 2, C.byref(e), err, len(err))
    assert rc == 151 and b"one GPU" in err.value


@pytest.mark.parametrize("R,V,L", CPU_ROWS)
def test_vsr_property_matches_python(pkg, R, V, L):
    """vsr_property (one definition for host and device) against P and Q evaluated on the flat form, on every state"""
    Flat = pkg.checker.VsrFlatState
    mp = pkg.ModelChecker.from_constants(R, V, L, property=True)
    mq = pkg.ModelChecker.from_constants(R, V, L, property=True, live_test_hooks=1)
    q = orc.params(R, V, L)
    lib = orc.lib()
    init = Flat()
    lib.orc_init_flat(q, C.byref(init))
    seen = {orc.digests_of(q, (Flat * 1)(init))[0][0]}
    level, cap, checked = [init], 512, 0
    out, acts = (Flat * cap)(), (C.c_int * cap)()
    while level:
        nxt = []
        for f in level:
            s = mp.pack(f)
            assert mp.property_holds(s) == p_flat(f)
            assert mq.property_holds(s) == q_flat(f)
            checked += 1
            n = lib.orc_successors_flat(q, C.byref(f), out, acts, cap)
            for k, d in enumerate(orc.digests_of(q, out, n)[0] if n else []):
                if d not in seen:
                    seen.add(d)
                    nxt.append(Flat.from_buffer_copy(out[k]))
        level = nxt
    assert checked == TABLE[(R, V, L)][0]


@pytest.mark.parametrize("R,V,L", CPU_ROWS)
def test_reference_verdict_reproduces_table(pkg, R, V, L):
    preds, succ = reference_graph(pkg, R, V, L)
    v = reference_verdict(preds, succ)
    assert (len(preds), v["not_p"], v["sinks"]) == TABLE[(R, V, L)]
    assert v["holds"] and v["bad_sinks"] == 0 and v["cycles"] == 0
    vq = reference_verdict(preds, succ, use_q=True)
    assert vq["bad_sinks"] == (Q_SINKS_311 if (R, V, L) == (3, 1, 1) else 0)
    assert vq["cycles"] == 0


# -------------------------------------------------------------------------------------------------- GPU
def run_case(pkg, R, V, L, hooks=0, symmetry=True, **kw):
    """the liveness check of one space, with its lasso checked against the oracle; a dict a child process can print"""
    mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=symmetry, property=True, live_test_hooks=hooks)
    opts = dict(deadlock=False, table_capacity=1 << 22, frontier_capacity=1 << 20)
    opts.update(kw)
    res = mc.check(**opts)
    out = {"rc": res.rc, "distinct": res.distinct, "generated": res.generated, "depth": res.depth, "level_sizes": res.level_sizes,
           "trace_loop": res.trace_loop, "trace_len": len(res.trace), "live": {k: v for k, v in res.liveness.items()}}
    if res.rc == 13:
        out["lasso_errors"] = lasso_errors(pkg, mc, res, orc.params(R, V, L, symmetry=symmetry), hooks)
    return out


def lasso_errors(pkg, mc, res, q, hooks):
    """every way the lasso fails to be a counterexample: steps that are not Next steps (oracle), a stuttering end in a state
    with a successor, a loop state where the predicate holds, a back edge that is neither a Next step nor the hook's edge"""
    Flat = pkg.checker.VsrFlatState
    lib = orc.lib()
    states = [s for _, s in res.trace]
    flats = [mc.unpack(s) for s in states]
    digs = orc.digests_of(q, (Flat * len(flats))(*flats))[0]
    cap = 512
    out, acts = (Flat * cap)(), (C.c_int * cap)()

    def succ_digests(f):
        n = lib.orc_successors_flat(q, C.byref(f), out, acts, cap)
        return set(orc.digests_of(q, out, n)[0]) if n else set()
    errors = []
    if states[0] != mc.init_state():
        errors.append("the first state is not Init")
    for i in range(1, len(states)):
        if digs[i] not in succ_digests(flats[i - 1]):
            errors.append("step %d -> %d is not a Next step" % (i, i + 1))
    last = succ_digests(flats[-1])
    no_successor = last <= {digs[-1]}
    k = res.trace_loop
    if k == 0:
        if mc.property_holds(states[-1]) or not no_successor:
            errors.append("stuttering at a state where the predicate holds or that has a successor")
    else:
        if any(mc.property_holds(s) for s in states[k - 1:]):
            errors.append("the predicate holds on the loop")
        if digs[k - 1] not in last and not (hooks & 2 and k == 1 and no_successor):
            errors.append("the back edge to state %d is neither a Next step nor the edge to Init" % k)
    return errors


SPACES = list(TABLE) + [(3, 2, 1, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("space", SPACES, ids=lambda s: "_".join(map(str, s)))
def test_property_holds_on_gpu(pkg, space):
    R, V, L = space[:3]
    sym = space[3] if len(space) > 3 else True
    got = run_case(pkg, R, V, L, symmetry=sym)
    plain = pkg.ModelChecker.from_constants(R, V, L, symmetry=sym).check(deadlock=False, table_capacity=1 << 22, frontier_capacity=1 << 20)
    assert got["rc"] == 0, got
    assert (got["distinct"], got["generated"], got["depth"], got["level_sizes"]) == (plain.distinct, plain.generated, plain.depth, plain.level_sizes)
    live = got["live"]
    assert live["sinks"] == 0 and live["survivors"] == 0 and live["sweeps"] >= 1
    if sym:
        assert (got["distinct"], live["stored"]) == TABLE[(R, V, L)][:2]
    else:
        assert got["distinct"] == FULL_321
        mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=False, property=True)
        res = mc.check(deadlock=False, table_capacity=1 << 22, frontier_capacity=1 << 20, collect_levels=True)
        sb = mc.state_bytes
        not_p = sum(1 for lv in res.levels for i in range(0, len(lv), sb) if not mc.property_holds(lv[i:i + sb]))
        assert live["stored"] == not_p


@pytest.mark.gpu
def test_reference_verdict_321(pkg):
    preds, succ = reference_graph(pkg, 3, 2, 1)
    v = reference_verdict(preds, succ)
    assert (len(preds), v["not_p"], v["sinks"]) == TABLE[(3, 2, 1)] and v["holds"]


@pytest.mark.gpu
@pytest.mark.parametrize("R,V,L", CPU_ROWS)
def test_sink_counterexample(pkg, R, V, L):
    """hook 1: []<>Q, violated in (3, 1, 1) by not-Q states without successors, holds in the R = 2 spaces"""
    got = run_case(pkg, R, V, L, hooks=1)
    if (R, V, L) != (3, 1, 1):
        assert got["rc"] == 0 and got["live"]["sinks"] == 0, got
        return
    assert got["rc"] == 13 and got["trace_loop"] == 0, got
    assert got["live"]["sinks"] == Q_SINKS_311
    assert got["lasso_errors"] == [], got


@pytest.mark.gpu
def test_cycle_counterexample(pkg):
    """hooks 1 + 2: every state without successors steps to Init, so not-Q cycles through Init exist in (3, 1, 1)"""
    preds, succ = reference_graph(pkg, 3, 1, 1)
    want = reference_verdict(preds, succ, use_q=True, init_edge=True)
    got = run_case(pkg, 3, 1, 1, hooks=3)
    assert (got["rc"] == 0) == want["holds"], (got, want)
    assert got["rc"] == 13 and got["trace_loop"] >= 1 and got["live"]["survivors"] > 0, got
    assert got["lasso_errors"] == [], got
    for R, V, L in [(2, 1, 1), (2, 2, 2)]:
        preds, succ = reference_graph(pkg, R, V, L)
        want = reference_verdict(preds, succ, use_q=True, init_edge=True)
        got = run_case(pkg, R, V, L, hooks=3)
        assert (got["rc"] == 0) == want["holds"], (R, V, L, got, want)
        assert got["rc"] == 0 or got["lasso_errors"] == [], got


@pytest.mark.gpu
def test_store_continues_in_host_memory(pkg, monkeypatch):
    """the store's words past its HBM part go to pinned host memory when the run allows host memory"""
    monkeypatch.setenv("VSR_B200_LIVE_HBM_STATES", "1000")
    got = run_case(pkg, 3, 1, 1, frontier_host_capacity=1 << 10)
    assert got["rc"] == 0 and got["live"]["stored"] == TABLE[(3, 1, 1)][1] and got["live"]["bytes_host"] > 0, got
    got = run_case(pkg, 3, 1, 1, hooks=1, frontier_host_capacity=1 << 10)
    assert got["rc"] == 13 and got["lasso_errors"] == [], got


@pytest.mark.gpu
def test_store_overflow_is_152(pkg, monkeypatch):
    monkeypatch.setenv("VSR_B200_LIVE_HBM_STATES", "1000")
    mc = pkg.ModelChecker.from_constants(3, 1, 1, property=True)
    res = mc.check(deadlock=False, table_capacity=1 << 22, frontier_capacity=1 << 20)
    assert res.rc == 152 and res.liveness == {}


@pytest.mark.gpu
def test_bounded_run_checks_no_property(pkg):
    mc = pkg.ModelChecker.from_constants(3, 1, 1, property=True, live_test_hooks=1)
    res = mc.check(deadlock=False, max_depth=5, table_capacity=1 << 22, frontier_capacity=1 << 20)
    assert res.rc == 0 and not res.complete and res.liveness == {}


@pytest.mark.gpu
def test_one_call_bfs_reports_the_lasso(pkg):
    """vsr_bfs runs the liveness pass too: rc 13, the lasso as its trace, the back edge in trace_loop"""
    mc = pkg.ModelChecker.from_constants(3, 1, 1, property=True, live_test_hooks=3)
    o = mc.run_opts(deadlock=False, table_capacity=1 << 22, frontier_capacity=1 << 20)
    st = pkg.checker.VsrStats()
    cap = 4096
    tr, acts = mc._buf(cap), (C.c_uint8 * cap)()
    rc = mc._lib.vsr_bfs(mc._h, C.byref(o), C.byref(st), tr, acts, cap)
    ref = run_case(pkg, 3, 1, 1, hooks=3)
    assert rc == 13 and st.trace_len == ref["trace_len"] and st.trace_loop == ref["trace_loop"], (rc, st.trace_len, ref)


@pytest.mark.gpu
def test_vsrmc_temporal_lines(pkg, tmp_path):
    cfg = tmp_path / "VSR.cfg"
    cfg.write_text(spec_cfg(pkg, 2, ["v1", "v2"], 2))
    r = subprocess.run([EXE, "-deadlock", "-table", str(1 << 20), "-frontier", str(1 << 16), "-config", str(cfg)], capture_output=True, text=True)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out
    assert "Checking temporal properties for the complete state space with 2073 total distinct states" in out
    assert "Finished checking temporal properties in" in out
    assert "Model checking completed. No error has been found." in out


WEAK_CASES = [(2, 2, 2), (3, 1, 1)]


@pytest.mark.gpu
def test_weak_fingerprints(tmp_path):
    """a -DVSR_WEAK_FP_BITS=16 build: the live index keeps states with equal fingerprints apart by their check hash"""
    import test_kernel_shapes as tks
    libs = tks.build_variants(str(tmp_path), {"weak16": ("-DVSR_WEAK_FP_BITS=16", WEAK_CASES)})
    for R, V, L in WEAK_CASES:
        so = libs[("weak16", R, V, L)]
        outp = tks._child("import os, json; os.environ['VSR_B200_LIB'] = %r\nimport _pkg, test_liveness as tl; pkg = _pkg.load()\n"
                          "print('RES', json.dumps([tl.run_case(pkg, %d, %d, %d, hooks=h) for h in (0, 1, 3)]))\nprint('CHILD-OK')\n"
                          % (so, R, V, L))
        plain, sink, cycle = json.loads(outp.split("RES", 1)[1].splitlines()[0])
        assert plain["rc"] == 0 and (plain["distinct"], plain["live"]["stored"]) == TABLE[(R, V, L)][:2], plain
        if (R, V, L) == (3, 1, 1):
            assert sink["rc"] == 13 and sink["live"]["sinks"] == Q_SINKS_311 and sink["lasso_errors"] == [], sink
            assert cycle["rc"] == 13 and cycle["trace_loop"] >= 1 and cycle["lasso_errors"] == [], cycle
        else:
            assert sink["rc"] == 0, sink
