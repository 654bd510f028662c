"""Recovery on another number of GPUs (TLC's -recover works with any -workers): a checkpoint written by W_a ranks is
continued by W_b ranks, every new rank reading every old file and keeping the seen-set entries, frontier states and
trace records it owns.  The continued run must report exactly what the uninterrupted run reports; the shards it writes
back must be exactly the owners' shares; counterexamples found after the renumbering must still be behaviours.

Several ranks are threads of one process sharing device 0 (VSR_B200_MULTI_ONE_DEVICE), as in test_checkpoint.py."""
import json
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import orc
from test_checkpoint import same_exploration

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc")
CAPS = dict(table_capacity=1 << 20, frontier_capacity=1 << 17)
PINNED = (697_364, 1_831_657, 30)  # (3, 2, 1) without SYMMETRY, complete: distinct, generated, depth (the spec's text)
OWNER_MUL = 0xD6E8FEB86659FD93  # owner_of in csrc/vsr_layout.h


@pytest.fixture(autouse=True)
def one_device(monkeypatch):
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")


@pytest.fixture(scope="module")
def mc(pkg):
    return pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)


@pytest.fixture(scope="module")
def whole(mc):
    res = mc.check(stop_on_violation=False, **CAPS)
    assert (res.complete, res.distinct, res.generated, res.depth) == (True,) + PINNED
    return res


def run(mc, world, **kw):
    """the BFS on `world` ranks: one GPU through check(), several through check_multi()"""
    return mc.check(stop_on_violation=False, **kw) if world == 1 else mc.check_multi(world, stop_on_violation=False, **kw)


def checkpoint(mc, world, path, depth, **kw):
    kw = dict(CAPS, **kw)
    part = run(mc, world, max_depth=depth, checkpoint_path=path, checkpoint_seconds=1e9, **kw)
    assert part.depth == depth and not part.complete
    return part


def files_of(path, world):
    return [path] if world == 1 else ["%s.rank%d" % (path, r) for r in range(world)]


# -------------------------------------------------------------------------------------------------- checkpoint files
HDR = struct.Struct("<QIIII10i7Q")  # CkptHeader of csrc/vsr_ckpt.cu


def read_ckpt(path):
    """(header dict, frontier states as a list of bytes, seen-set entries as an (n, 2) uint64 array), at the offsets the
    header's own size fields give"""
    raw = open(path, "rb").read()
    f = HDR.unpack_from(raw, 0)
    h = dict(zip(["magic", "version", "header_bytes", "stats_bytes", "state_bytes", "R", "V", "K", "symmetry", "use_view", "invariant",
                  "rank", "world", "level", "keep_trace", "n_cur", "cur_base", "next_base", "n_entries", "n_trace", "sent", "received"], f))
    at = h["header_bytes"] + 2 * h["stats_bytes"]
    sb = h["state_bytes"]
    frontier = [raw[at + i * sb: at + (i + 1) * sb] for i in range(h["n_cur"])]
    at += h["n_cur"] * sb
    ents = np.frombuffer(raw, dtype="<u8", count=2 * h["n_entries"], offset=at).reshape(-1, 2)
    return h, frontier, ents


def owners(fps, world):
    if world == 1:
        return np.zeros(len(fps), dtype=np.int64)
    lg = world.bit_length() - 1
    with np.errstate(over="ignore"):
        return ((fps.astype(np.uint64) * np.uint64(OWNER_MUL)) >> np.uint64(64 - lg)).astype(np.int64)


def sorted_entries(ents):
    return ents[np.lexsort((ents[:, 1], ents[:, 0]))]


# -------------------------------------------------------------------------------------------------- 1. any world to any world
@pytest.mark.parametrize("w_a", [1, 2, 4])
def test_any_world_to_any_world(mc, whole, tmp_path, w_a):
    ck = str(tmp_path / "w.ckpt")
    checkpoint(mc, w_a, ck, 16)
    for w_b in (1, 2, 4, 8):
        if w_b != w_a:
            same_exploration(run(mc, w_b, recover_path=ck, **CAPS), whole)


# -------------------------------------------------------------------------------------------------- 2. the owners' shares
@pytest.mark.parametrize("w_a,w_b", [(1, 4), (4, 2), (2, 8)])
def test_shard_is_exactly_the_owners_share(pkg, mc, tmp_path, w_a, w_b):
    old, new = str(tmp_path / "old.ckpt"), str(tmp_path / "new.ckpt")
    checkpoint(mc, w_a, old, 16)
    # recovered and written straight back at the same boundary
    back = run(mc, w_b, recover_path=old, max_depth=16, checkpoint_path=new, checkpoint_seconds=0, **CAPS)
    assert back.depth == 16
    olds = [read_ckpt(p) for p in files_of(old, w_a)]
    news = [read_ckpt(p) for p in files_of(new, w_b)]
    for r, (h, frontier, ents) in enumerate(news):
        assert (h["rank"], h["world"], h["level"]) == (r, w_b, 16)
        assert (owners(ents[:, 0], w_b) == r).all()
        for s in frontier:
            fp = mc.fingerprint(s) or 1
            assert int(mc._lib.vsr_owner_rank(fp, w_b)) == r
    union = lambda parts: sorted_entries(np.concatenate([e for _, _, e in parts]))
    assert np.array_equal(union(olds), union(news))
    assert sorted(s for _, f, _ in olds for s in f) == sorted(s for _, f, _ in news for s in f)
    assert sum(h["n_entries"] for h, _, _ in news) == back.distinct


# -------------------------------------------------------------------------------------------------- 3. outgrowing one GPU
def test_space_that_outgrew_one_gpu_continues_on_two(mc, whole, tmp_path):
    ck = str(tmp_path / "one.ckpt")
    small = dict(table_capacity=1 << 19, frontier_capacity=1 << 17)  # load limit 458,752 < 697,364
    full = mc.check(stop_on_violation=False, checkpoint_path=ck, checkpoint_seconds=0, **small)
    assert full.rc == 152 and os.path.exists(ck)
    rest = mc.check_multi(2, stop_on_violation=False, recover_path=ck, **small)
    same_exploration(rest, whole)


# -------------------------------------------------------------------------------------------------- 4. counterexamples
INV = ("AcknowledgedWritesExistOnMajority",)


def assert_behaviour(pkg, res, depth):
    assert res.rc == 12 and res.violation_level == depth and len(res.trace) == depth
    lit = pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False, invariants=INV)
    assert res.trace[0][1] == lit.init_state()
    for (_, a), (_, b) in zip(res.trace, res.trace[1:]):
        assert b in [t for t, _, _ in lit.successors(a)]
    assert lit.invariant(res.trace[-1][1]) != 0 and all(lit.invariant(s) == 0 for _, s in res.trace[:-1])


def test_counterexample_survives_renumbering(pkg, tmp_path):
    sym = pkg.ModelChecker.from_constants(3, 2, 1, invariants=INV)
    o = orc.bfs(orc.params(3, 2, 1, invariant=2), workers=8, keep_trace=False, check_assumptions=False)
    assert o.rc == 12 and o.depth > 8
    ck = str(tmp_path / "before.ckpt")
    part = sym.check_multi(2, max_depth=o.depth - 6, checkpoint_path=ck, checkpoint_seconds=1e9, **CAPS)
    assert part.rc == 0
    for w_b in (1, 4):
        res = sym.check(recover_path=ck, **CAPS) if w_b == 1 else sym.check_multi(w_b, recover_path=ck, **CAPS)
        assert res.level_sizes == o.level_sizes
        assert_behaviour(pkg, res, o.depth)
    # a checkpoint written after the violation's level: the totals' violation id is renumbered
    whole = sym.check(stop_on_violation=False, **CAPS)
    ck2 = str(tmp_path / "after.ckpt")
    after = sym.check_multi(2, stop_on_violation=False, max_depth=o.depth + 2, checkpoint_path=ck2, checkpoint_seconds=1e9, **CAPS)
    assert after.violation_level == o.depth
    for w_b in (1, 4):
        kw = dict(stop_on_violation=False, recover_path=ck2, **CAPS)
        res = sym.check(**kw) if w_b == 1 else sym.check_multi(w_b, **kw)
        same_exploration(res, whole)
        assert_behaviour(pkg, res, o.depth)


# -------------------------------------------------------------------------------------------------- 5. two generations
def test_two_generations(mc, whole, tmp_path):
    ck1, ck2 = str(tmp_path / "g1.ckpt"), str(tmp_path / "g2.ckpt")
    checkpoint(mc, 1, ck1, 16)
    mid = mc.check_multi(4, stop_on_violation=False, recover_path=ck1, max_depth=23, checkpoint_path=ck2, checkpoint_seconds=0, **CAPS)
    assert mid.depth == 23 and mid.level_sizes == whole.level_sizes[:23]
    same_exploration(mc.check_multi(2, stop_on_violation=False, recover_path=ck2, **CAPS), whole)


# -------------------------------------------------------------------------------------------------- 6. frontier spill
def test_frontier_spill(mc, whole, tmp_path):
    ck = str(tmp_path / "s.ckpt")
    checkpoint(mc, 1, ck, 16)
    share = whole.level_sizes[15] // 2
    fcap = max(64, share // 4)  # far less than the frontier each of the two ranks owns at depth 16
    rest = mc.check_multi(2, stop_on_violation=False, recover_path=ck, table_capacity=1 << 20, frontier_capacity=fcap,
                          frontier_host_capacity=1 << 17)
    same_exploration(rest, whole)


# -------------------------------------------------------------------------------------------------- 7. without a trace
def test_without_trace(mc, whole, tmp_path):
    ck = str(tmp_path / "nt.ckpt")
    checkpoint(mc, 2, ck, 16, keep_trace=False)
    same_exploration(mc.check(stop_on_violation=False, recover_path=ck, keep_trace=False, **CAPS), whole)
    same_exploration(mc.check_multi(4, stop_on_violation=False, recover_path=ck, keep_trace=False, **CAPS), whole)


# -------------------------------------------------------------------------------------------------- 8. weak fingerprints
WEAK_CHILD = r"""
import os, json
os.environ['VSR_B200_LIB'] = %r
os.environ['VSR_B200_MULTI_ONE_DEVICE'] = '1'
import _pkg
pkg = _pkg.load()
mc = pkg.ModelChecker.from_constants(3, 1, 1)
caps = dict(table_capacity=1 << 18, frontier_capacity=1 << 16)
def run(world, **kw):
    r = mc.check(stop_on_violation=False, **kw) if world == 1 else mc.check_multi(world, stop_on_violation=False, **kw)
    return dict(rc=r.rc, complete=r.complete, generated=r.generated, distinct=r.distinct, queue=r.queue, depth=r.depth,
                level_sizes=r.level_sizes, level_generated=r.level_generated[:max(r.depth - 1, 0)], fp_collisions=r.fp_collisions)
whole = run(1, **caps)
out = dict(whole=whole, runs=[])
for w_a, w_b in ((1, 2), (2, 1)):
    ck = %r + '/w%%d.ckpt' %% w_a
    run(w_a, max_depth=whole['depth'] // 2, checkpoint_path=ck, checkpoint_seconds=1e9, **caps)
    out['runs'].append(run(w_b, recover_path=ck, **caps))
print('RES', json.dumps(out))
print('CHILD-OK')
"""


def test_weak_fingerprints(tmp_path):
    """a -DVSR_WEAK_FP_BITS=16 build, where equal fingerprints are common: they have one owner in every world, and the
    check hash keeps them apart there after the re-sharding as before it"""
    import test_kernel_shapes as tks
    so = tks.build_variants(str(tmp_path), {"weak16": ("-DVSR_WEAK_FP_BITS=16", [(3, 1, 1)])})[("weak16", 3, 1, 1)]
    out = tks._child(WEAK_CHILD % (so, str(tmp_path)))
    res = json.loads(out.split("RES", 1)[1].splitlines()[0])
    whole = res["whole"]
    assert whole["rc"] == 0 and whole["complete"] and whole["fp_collisions"] > 0, whole
    for r in res["runs"]:
        assert {k: r[k] for k in whole if k != "fp_collisions"} == {k: whole[k] for k in whole if k != "fp_collisions"}


# -------------------------------------------------------------------------------------------------- 9 / 10. the CLI
def vsrmc(pkg, tmp_path, *args):
    cfg = tmp_path / "m.cfg"
    if not cfg.exists():
        cfg.write_text(pkg.cfg_text(3, ["v1"], 1))
    cmd = [EXE, "-deadlock", "-config", str(cfg), "-table", "1048576", "-frontier", "262144"] + [str(a) for a in args]
    return subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, VSR_B200_MULTI_ONE_DEVICE="1"))


def summary(out):
    return [ln for ln in out.splitlines() if "states generated" in ln or "The depth of the complete" in ln or ln.startswith("Error: Invariant")]


def test_cli_recovers_on_another_number_of_gpus(pkg, tmp_path):
    whole = vsrmc(pkg, tmp_path)
    assert summary(whole.stdout)
    for w_a, w_bs in ((1, (2, 4)), (2, (1,))):
        meta = tmp_path / ("states%d" % w_a)
        first = vsrmc(pkg, tmp_path, "-gpus", w_a, "-checkpoint", 0, "-metadir", meta, "-depth", 11)
        assert first.returncode == 0 and "states left on queue" in first.stdout, first.stderr
        for w_b in w_bs:
            rest = vsrmc(pkg, tmp_path, "-gpus", w_b, "-recover", meta)
            assert rest.returncode == whole.returncode, rest.stderr
            assert summary(rest.stdout) == summary(whole.stdout), (w_a, w_b)


def test_refusals(pkg, tmp_path):
    def ckpt(name, gpus, depth):
        meta = tmp_path / name
        r = vsrmc(pkg, tmp_path, "-gpus", gpus, "-checkpoint", 0, "-metadir", meta, "-depth", depth)
        assert r.returncode == 0, r.stderr
        return meta
    a, b = ckpt("a", 2, 9), ckpt("b", 2, 8)
    # a rank file of another run
    swapped = tmp_path / "swapped"
    shutil.copytree(a, swapped)
    shutil.copy(b / "vsr.ckpt.rank1", swapped / "vsr.ckpt.rank1")
    r = vsrmc(pkg, tmp_path, "-gpus", 4, "-recover", swapped)
    assert r.returncode == 150 and str(swapped / "vsr.ckpt.rank1") in r.stderr, r.stderr
    # a missing rank file: the status of a missing file, with its name
    gone = tmp_path / "gone"
    shutil.copytree(a, gone)
    os.remove(gone / "vsr.ckpt.rank1")
    r = vsrmc(pkg, tmp_path, "-gpus", 1, "-recover", gone)
    assert r.returncode == 153 and str(gone / "vsr.ckpt.rank1") in r.stderr, r.stderr
    # a one-GPU checkpoint and a two-GPU one in the same place, recovered on four: which one is meant?
    both = tmp_path / "both"
    shutil.copytree(a, both)
    one = ckpt("one", 1, 9)
    shutil.copy(one / "vsr.ckpt", both / "vsr.ckpt")
    r = vsrmc(pkg, tmp_path, "-gpus", 4, "-recover", both)
    assert r.returncode == 151 and str(both / "vsr.ckpt") in r.stderr and str(both / "vsr.ckpt.rank0") in r.stderr, r.stderr
    # new ranks too small for their share
    r = vsrmc(pkg, tmp_path, "-gpus", 2, "-recover", one, "-table", 64)
    assert r.returncode == 152 and "capacity exceeded (recover)" in r.stderr, r.stderr
