"""Fingerprint collisions in the seen-set, made common by builds with weak fingerprints.

The seen-set keeps states with equal 64-bit fingerprints apart by a second, 32-bit check hash in each entry's meta (DESIGN
§2).  With 64-bit fingerprints no test space produces a collision, so the libraries here are built with VSR_WEAK_FP_BITS
(vsr_actions.h): weak16 keeps 16 bits of every fingerprint, weak0 none (every state has fingerprint 1 and lands in one
probe chain, which the capacities below make wrap past the table's end).  The oracle still gives the exact answer, so
under collisions on every path (expand and drain inserts, the VIEW-tie reduction and patch pass, lookups, the per-level
audit, checkpoint re-insertion) the GPU must find exactly the oracle's states.

The CPU tests pin FP64 to a plain bit-serial reference and the weak builds to its low bits.  Each GPU case runs in a child
process, as the kernel variants of test_kernel_shapes.py do.  What stays untested by design: states with equal fingerprint
AND equal check hash are merged without a word, as a fingerprint set would merge them.
"""
import collections
import ctypes as C
import os
import pickle
import struct
import tempfile
import types

import numpy as np
import pytest

import test_gpu_parity as tgp
import test_kernel_shapes as tks

# (name, flags, single layouts (R, V, L)), built by test_kernel_shapes.build_variants
WEAK = {
    "weak16": ("-DVSR_WEAK_FP_BITS=16", [(3, 2, 1), (3, 2, 2), (5, 2, 2)]),
    "weak0": ("-DVSR_WEAK_FP_BITS=0", [(2, 1, 1), (2, 2, 2)]),
}
BITS = {"weak16": 16, "weak0": 0}
POLY = 0x911498AE0E66BAD6
FULL_321 = (697_364, 1_831_657, 30)  # (3,2,1) without SYMMETRY, complete: distinct, generated, depth


# -------------------------------------------------------------------------------------------------- host definitions
def _pow2_width(m):
    return 1 if m < 2 else (2 if m < 4 else (4 if m < 16 else 8))


def layout_bits(R, V, L):
    """(VIEW_BITS, NW) of Layout<R, V, L + 1>, restated from the field list of vsr_layout.h: every field aligned to its own
    width, the aux variables last, so that the VIEW is the prefix before them"""
    K = L + 1
    VB, OB, RB, O, NV2 = _pow2_width(K), _pow2_width(V), _pow2_width(R - 1), R - 1, K - 1
    NSVC, NDVC, NSV, NPOK, NGS = NV2 * R * O, NV2 * O, NV2 * O, K * V * O, NV2 * O
    fields = [(2, R), (VB, R), (OB, R), (VB, R), (1, R), (1, R), (1, R * R), (1, R * R), (OB, R * R), (OB, R), (OB, R), (1, R), (VB, R),
              (OB, R), (OB, R * V), (OB, R * V), (OB, NDVC * V), (OB, NV2 * V), (OB, NGS * V), (2, NSVC), (2, NDVC), (VB, NDVC),
              (OB, NDVC), (2, NSV), (OB, NV2), (VB, V), (OB, V), (OB, V), (OB, V), (1, V * O), (2, NPOK), (2, NGS), (OB, NGS),
              (RB, NGS), (2, NGS), (OB, NGS)]
    end = 0
    for w, n in fields:
        end = (end + w - 1) // w * w + w * n
    view = end
    for w, n in [(_pow2_width(max(K - 1, 1)), 1), (2, V)]:
        end = (end + w - 1) // w * w + w * n
    return view, ((end + 31) // 32 + 3) // 4 * 4


def as_words(raw, nw):
    return np.frombuffer(raw, dtype="<u4").reshape(-1, nw)


def hashed_words(words, R, V, L, view=True):
    """the words FP64 and the check hash read: the VIEW prefix, its last word masked, or every word"""
    vb, _ = layout_bits(R, V, L)
    if not view:
        return words
    full, rem = divmod(vb, 32)
    w = words[:, :full + (1 if rem else 0)].copy()
    if rem:
        w[:, full] &= np.uint32((1 << rem) - 1)
    return w


def fp64_reference(words):
    """FP64, bit by bit: fp = POLY; for each byte of the little-endian words, fp ^= byte, then eight times
    fp = (fp >> 1) ^ (POLY if fp & 1 else 0).  The byte tables of fp64_build_table hold tab[j] = eight such steps from j."""
    fp = np.full(len(words), POLY, dtype=np.uint64)
    by = np.ascontiguousarray(words, dtype="<u4").view(np.uint8).reshape(len(words), -1)
    one, poly, zero = np.uint64(1), np.uint64(POLY), np.uint64(0)
    for j in range(by.shape[1]):
        fp ^= by[:, j].astype(np.uint64)
        for _ in range(8):
            fp = (fp >> one) ^ np.where((fp & one).astype(bool), poly, zero)
    return fp


def check_hash(words):
    """check_hash_t of vsr_gpu.cuh: per word h ^= w, h = rotl(h, 13) * 5 + 0xe6546b64, then the murmur3 finaliser"""
    h = np.full(len(words), 0x9747B28C, dtype=np.uint32)
    for i in range(words.shape[1]):
        h ^= words[:, i]
        h = ((h << np.uint32(13)) | (h >> np.uint32(19))) * np.uint32(5) + np.uint32(0xE6546B64)
    h ^= h >> np.uint32(16)
    h *= np.uint32(0x85EBCA6B)
    h ^= h >> np.uint32(13)
    h *= np.uint32(0xC2B2AE35)
    h ^= h >> np.uint32(16)
    return h


def seen_set_fp(fp, bits=64):
    """the fingerprint a seen-set entry holds: `bits` low bits of FP64, 0 remapped to 1"""
    fp = fp & np.uint64((1 << bits) - 1) if bits < 64 else fp
    return np.where(fp == 0, np.uint64(1), fp)


def table_home(cap, fp, bucket=2):
    """table_home of vsr_gpu.cuh: bucket floor(fp * 0x9E3779B97F4A7C15 mod 2^64 * (cap / bucket) / 2^64)"""
    return ((fp * 0x9E3779B97F4A7C15) % (1 << 64) * (cap // bucket) >> 64) * bucket


def host_call(mc, fn, raw):
    """fn(model, state) of the library for every packed state of raw"""
    sb = mc.state_bytes
    buf = (C.c_uint8 * max(len(raw), 1)).from_buffer_copy(raw)
    base, f = C.addressof(buf), getattr(mc._lib, fn)
    return np.array([f(mc._h, base + i * sb) for i in range(len(raw) // sb)], dtype=np.uint64)


def host_bfs(mc, n):
    """the first n states of a breadth-first search on the host (vsr_successors), packed back to back"""
    s0 = mc.init_state()
    seen, queue, i = {s0}, [s0], 0
    while i < len(queue) and len(queue) < n:
        for t, _, _ in mc.successors(queue[i]):
            if t not in seen:
                seen.add(t)
                queue.append(t)
        i += 1
    return b"".join(queue[:n])


def collision_bounds(level_fps):
    """per level: (the collisions the new states' inserts must count, the largest fingerprint class so far).  A new state
    walks past every entry of its class whose slot comes before its own, and slots are never freed: so past every entry of
    its class from earlier levels, and of each pair of new states of one class the later slot walks past the earlier."""
    seen, out = collections.Counter(), []
    for fps in level_fps:
        new = collections.Counter(fps.tolist())
        out.append(sum(seen[c] * k + k * (k - 1) // 2 for c, k in new.items()))
        seen.update(new)
        out[-1] = (out[-1], max(seen.values()))
    return out


# -------------------------------------------------------------------------------------------------- CPU tests
def test_layout_restatement_matches_the_library(pkg):
    """layout_bits gives every built-in layout's state size, and the VIEW prefixes end on odd and on even word counts"""
    odd_even = set()
    for R, V, L in tks.builtin_layouts():
        vb, nw = layout_bits(R, V, L)
        assert nw * 4 == pkg.ModelChecker.from_constants(R, V, L).state_bytes, (R, V, L)
        odd_even.add(((vb + 31) // 32) % 2)
    assert odd_even == {0, 1}


def test_fp64_reference_equals_both_host_forms(pkg):
    """the bit-serial FP64 of the VIEW-masked words equals vsr_fingerprint (slicing-by-8, what the GPU runs) and
    vsr_fingerprint_bytewise on reachable states of every built-in layout, with VIEW and without"""
    for R, V, L in tks.builtin_layouts():
        for view in (True, False):
            mc = pkg.ModelChecker.from_constants(R, V, L, view=view)
            raw = host_bfs(mc, 300)
            ref = fp64_reference(hashed_words(as_words(raw, mc.state_bytes // 4), R, V, L, view))
            assert (host_call(mc, "vsr_fingerprint", raw) == ref).all(), (R, V, L, view)
            assert (host_call(mc, "vsr_fingerprint_bytewise", raw) == ref).all(), (R, V, L, view)


@pytest.fixture(scope="module")
def weak_libs():
    with tempfile.TemporaryDirectory(prefix="vsr-weakfp-") as d:
        yield tks.build_variants(d, WEAK)


def in_child(so, fn, *args, multi_one_device=False, timeout=1500):
    """test_fp_collisions.fn(*args) in a child process with the library `so` (None: the product build); its pickled result.
    The template thunks' static tables are unique symbols, which the dynamic linker would share with a library this process
    has loaded already."""
    with tempfile.TemporaryDirectory(prefix="vsr-weakfp-out-") as d:
        out = os.path.join(d, "out.pkl")
        env = "import os\n" + ("os.environ['VSR_B200_LIB'] = %r\n" % so if so else "") + \
              ("os.environ['VSR_B200_MULTI_ONE_DEVICE'] = '1'\n" if multi_one_device else "")
        tks._child(env + "import pickle, test_fp_collisions as t\npickle.dump(t.%s(*%r), open(%r, 'wb'))\nprint('CHILD-OK')\n"
                   % (fn, args, out), timeout=timeout)
        return pickle.load(open(out, "rb"))


def _host_fps(R, V, L, bits):
    """(in a child) vsr_fingerprint, vsr_fingerprint_bytewise and the reference's low bits on reachable states"""
    import _pkg
    pkg = _pkg.load()
    out = []
    for view in (True, False):
        mc = pkg.ModelChecker.from_constants(R, V, L, view=view)
        raw = host_bfs(mc, 300)
        ref = fp64_reference(hashed_words(as_words(raw, mc.state_bytes // 4), R, V, L, view)) & np.uint64((1 << bits) - 1)
        out.append((host_call(mc, "vsr_fingerprint", raw), host_call(mc, "vsr_fingerprint_bytewise", raw), ref))
    return out


@pytest.mark.parametrize("name,R,V,L", [(n, *c) for n, (_, cs) in WEAK.items() for c in cs])
def test_weak_build_keeps_the_low_bits_of_fp64(weak_libs, name, R, V, L):
    """in a weak build both host forms equal the reference's low bits (host and device share fp64_view8 and fp64_view)"""
    for sliced, bytewise, ref in in_child(weak_libs[(name, R, V, L)], "_host_fps", R, V, L, BITS[name]):
        assert (sliced == ref).all() and (bytewise == ref).all()
        assert (len(set(ref.tolist())) > 100) if BITS[name] else not ref.any()


# -------------------------------------------------------------------------------------------------- GPU: child sides
def _load(R, V, L, symmetry, invariants=("AcknowledgedWriteNotLost",)):
    import _pkg
    pkg = _pkg.load()
    return pkg, pkg.ModelChecker.from_constants(R, V, L, symmetry=symmetry, invariants=invariants)


def _keys(mc, raw, R, V, L, bits, fps=None):
    """(seen-set fingerprint, check hash) of every packed state of raw; fps: the library's host fingerprints"""
    w = hashed_words(as_words(raw, mc.state_bytes // 4), R, V, L)
    fp = fps if fps is not None else fp64_reference(w)
    return seen_set_fp(fp, bits), check_hash(w)


def _parity(R, V, L, symmetry, depth, bits, table, frontier):
    """the audited engine BFS; per-depth digest sets, per-level collisions and their bounds from the variant's host
    fingerprint, and how many distinct (fingerprint, check) keys the states have"""
    import orc
    pkg, mc = _load(R, V, L, symmetry)
    res, rows = tks.engine_bfs(pkg, mc, max_depth=depth, table=table, frontier=frontier)
    sets = tgp.level_digest_sets(pkg, mc, res, orc.params(R, V, L, symmetry=symmetry and V > 1))
    fps = [seen_set_fp(host_call(mc, "vsr_fingerprint", raw)) for raw in res.levels]
    keys = set()
    for raw, fp in zip(res.levels, fps):
        _, chk = _keys(mc, raw, R, V, L, bits, fp)
        keys.update(zip(fp.tolist(), chk.tolist()))
    res.level_generated_in = [r[1] for r in rows]  # successors inserted while each level was built
    res.bounds = collision_bounds(fps)
    res.keys = len(keys)
    res.classes = len({f for fp in fps for f in fp.tolist()})
    res.levels = []
    del res.engine
    return vars(res), sets


def _entries(R, V, L, symmetry, bits, table, path):
    """a complete audited BFS, then a checkpoint: the multiset of its seen-set entries {(fp, check, level tag, aux key)}
    against the one computed on the host from the reference FP64, the check-hash restatement and vsr_aux_key"""
    pkg, mc = _load(R, V, L, symmetry)
    res, _ = tks.engine_bfs(pkg, mc, table=table, frontier=1 << 20, keep=True)
    try:
        assert res.complete and res.h2_ties == 0  # with ties, an entry keeps the first arrival's aux key
        assert mc._lib.vsr_engine_checkpoint(res.engine._e, path.encode(), None) == 0
    finally:
        res.engine.close()
    blob = open(path, "rb").read()
    header_bytes, stats_bytes, state_bytes = struct.unpack_from("<III", blob, 12)
    n_cur, n_entries = struct.unpack_from("<Q", blob, 64)[0], struct.unpack_from("<Q", blob, 88)[0]
    assert state_bytes == mc.state_bytes and n_cur == 0 and n_entries == res.distinct
    at = header_bytes + 2 * stats_bytes
    ent = np.frombuffer(blob, dtype="<u8", count=2 * n_entries, offset=at).reshape(-1, 2)
    gpu = np.stack([ent[:, 0], ent[:, 1] & np.uint64(0xFFFFFFFF), ent[:, 1] >> np.uint64(56), (ent[:, 1] >> np.uint64(32)) & np.uint64(0xFFFFFF)], 1)
    host = []
    for d, raw in enumerate(res.levels, start=1):
        fp, chk = _keys(mc, raw, R, V, L, bits)
        aux = host_call(mc, "vsr_aux_key", raw) & np.uint64(0xFFFFFF)
        host.append(np.stack([fp, chk.astype(np.uint64), np.full(len(fp), d, dtype=np.uint64), aux], 1))
    host = np.concatenate(host)
    srt = lambda a: a[np.lexsort(a.T[::-1])]
    gpu, host = srt(gpu), srt(host)
    assert gpu.shape == host.shape
    bad = np.nonzero((gpu != host).any(1))[0]
    assert len(bad) == 0, "%d of %d seen-set entries differ from the host's; first: gpu %s host %s" % (len(bad), len(host), gpu[bad[0]], host[bad[0]])
    return res.distinct, res.depth


def _multi(R, V, L, symmetry, depth, world, table, frontier):
    _, mc = _load(R, V, L, symmetry)
    r = mc.check_multi(world, max_depth=depth, table_capacity=table, frontier_capacity=frontier, stop_on_violation=False)
    return {k: v for k, v in vars(r).items() if k not in ("trace", "levels")}


def _recover(R, V, L, symmetry, stop, table, table2, frontier, bits, d):
    """uninterrupted (levels collected), stopped at depth `stop` with a checkpoint, continued from it in a table of
    capacity table2; with the collision lower bound of the whole run"""
    _, mc = _load(R, V, L, symmetry)
    ck = os.path.join(d, "weak.ckpt")
    whole = mc.check(collect_levels=True, stop_on_violation=False, table_capacity=table, frontier_capacity=frontier)
    part = mc.check(stop_on_violation=False, max_depth=stop, checkpoint_path=ck, checkpoint_seconds=1e9, table_capacity=table, frontier_capacity=frontier)
    rest = mc.check(stop_on_violation=False, recover_path=ck, table_capacity=table2, frontier_capacity=frontier)
    lb = sum(b for b, _ in collision_bounds([_keys(mc, raw, R, V, L, bits)[0] for raw in whole.levels]))
    strip = lambda r: types.SimpleNamespace(**{k: v for k, v in vars(r).items() if k not in ("trace", "levels")})
    return strip(whole), strip(part), strip(rest), lb


def _ties(R, V, L, bits):
    """VIEW ties and fingerprint collisions in one level, through the record interface.  A and B are reachable states with
    the same weak fingerprint and different VIEWs (different check hashes).  Returns what the two scenarios left."""
    import torch
    pkg, mc = _load(R, V, L, True)
    from vsr_tlaplus_b200 import dist as vdist  # importable once the package is loaded
    res, _ = tks.engine_bfs(pkg, mc, max_depth=10, table=1 << 20, frontier=1 << 18)
    raw = b"".join(res.levels[1:])  # not Init: the records go into depth 2, and Init's entry is in the seen-set
    res.engine.close()
    sb = mc.state_bytes
    states = [raw[i:i + sb] for i in range(0, len(raw), sb)]
    fp, chk = _keys(mc, raw, R, V, L, bits)
    aux = host_call(mc, "vsr_aux_key", raw)

    def variants(s, svcs):
        out = []
        for v in svcs:
            f = mc.unpack(s)
            f.aux_svc = v
            out.append(mc.pack(f))
        return out

    # A: aux_svc 2, 0, 1.  B: an aux key above A's with aux_svc 1, so that any of A's tie records beats B's own
    by_fp = collections.defaultdict(list)
    for i, f in enumerate(fp.tolist()):
        by_fp[f].append(i)
    pick = None
    for f, idx in by_fp.items():
        for a in idx:
            va = variants(states[a], (2, 0, 1))
            ka = [mc.aux_key(v) for v in va]
            if len(set(ka)) < 3 or len({mc.fingerprint(v) for v in va}) != 1:
                continue
            for b in idx:
                if chk[b] != chk[a] and aux[b] > ka[2]:
                    pick = (a, b, va)
                    break
            if pick:
                break
        if pick:
            break
    assert pick, "no two reachable states with one weak fingerprint, other VIEWs and the aux keys this test needs"
    a, b, va = pick
    B = states[b]
    vb = variants(B, (2, 0))
    assert mc.aux_key(vb[1]) < mc.aux_key(vb[0]) and len({mc.fingerprint(v) for v in va + [B] + vb}) == 1
    assert int(seen_set_fp(np.array([mc.fingerprint(B)], dtype=np.uint64))[0]) == int(fp[b])

    def rec(v, cand):
        f = mc.fingerprint(v) or 1
        return v + struct.pack("<QQ", f, (0 << 12) | cand | (1 << 56))  # vsr_gpu.cuh RecHdr: fp, trace record | mult << 56

    def run(batches):
        eng = vdist.GpuEngine(mc, 0, 1, table_capacity=1 << 12, frontier_capacity=1 << 10)
        try:
            eng.reset()
            eng.seed()
            assert eng.finish().new_states == 1
            for batch in batches:  # one insert launch each: later batches arrive later
                t = torch.frombuffer(bytearray(b"".join(batch)), dtype=torch.uint8).cuda()
                eng.insert(t, len(batch))
            li = eng.finish()
            n = int(li.new_states)
            out = (C.c_uint8 * (sb * max(n, 1)))()
            assert mc._lib.vsr_engine_read_frontier(eng._e, 0, n, out) == 0
            got = [bytes(out)[i * sb:(i + 1) * sb] for i in range(n)]
            return (n, int(li.ties), int(li.generated), int(li.collisions)), {s: eng.trace_record(1 + i) for i, s in enumerate(got)}
        finally:
            eng.close()

    # 1. the three variants of A interleaved with B (one launch): B is new, A's late arrivals tie
    one = run([[rec(va[0], 100), rec(B, 200), rec(va[1], 101), rec(va[2], 102)]])
    # 2. both with ties, the larger aux keys first: A's and B's tie records share the fingerprint, and each state must get
    #    its own smallest variant
    two = run([[rec(va[0], 100), rec(vb[0], 200)], [rec(va[2], 102), rec(vb[1], 201), rec(va[1], 101)]])
    return one, two, va, B, vb


def _counterexample(R, V, L):
    import _pkg
    tgp.test_counterexample_is_a_behaviour(_pkg.load())
    return True


# -------------------------------------------------------------------------------------------------- GPU tests
# (name, R, V, L, symmetry, depth (0: complete), table capacity): weak0's capacities make its one chain wrap
PARITY = [("weak16", 3, 2, 1, False, 0, 1 << 21), ("weak16", 3, 2, 2, True, 13, 1 << 22), ("weak0", 2, 1, 1, True, 0, 128),
          ("weak0", 2, 2, 2, False, 0, 4672)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,R,V,L,sym,depth,table", PARITY)
def test_parity_under_fingerprint_collisions(weak_libs, name, R, V, L, sym, depth, table):
    """every depth's state set, TLC's scalars and the ties equal to the oracle's, every level's audit holds, and each level
    counts at least the collisions its new states must walk past and at most generated x (largest class - 1)"""
    d, sets = in_child(weak_libs[(name, R, V, L)], "_parity", R, V, L, sym, depth, BITS[name], table, 1 << 20)
    res = types.SimpleNamespace(**d)
    assert res.keys == res.distinct, "two states share (weak fingerprint, check hash): exact parity is not the bar"
    assert res.classes <= 1 << BITS[name]
    tks.assert_child_parity(R, V, L, depth, res, sets, symmetry=sym)
    if depth == 0:
        assert res.complete
    if name == "weak0":
        home = table_home(table, 1)
        assert home + res.distinct > table and res.distinct <= table - table // 8, "the chain of fingerprint 1 must wrap"
    for lvl, (coll, gen, (low, big)) in enumerate(zip(res.level_collisions, res.level_generated_in, res.bounds), start=1):
        assert low <= coll <= gen * (big - 1), (lvl, low, coll, gen, big)
    assert sum(res.level_collisions) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", [None, "weak16"])
def test_seen_set_entries_equal_the_host_definitions(weak_libs, tmp_path, name):
    """(3,2,1) complete without SYMMETRY: every seen-set entry is (reference FP64, check hash, depth, aux key) of one state
    found, in the product build (the hot path's fingerprint and check hash at every state) and in weak16"""
    so = weak_libs[(name, 3, 2, 1)] if name else None
    distinct, depth = in_child(so, "_entries", 3, 2, 1, False, BITS.get(name, 64), 1 << 21, str(tmp_path / "entries.ckpt"))
    assert (distinct, depth) == FULL_321[::2]


@pytest.mark.gpu
@pytest.mark.parametrize("name,R,V,L,sym,depth,worlds,table", [("weak16", 5, 2, 2, True, 7, (2, 4), 1 << 22), ("weak16", 3, 2, 1, False, 0, (2, 4), 1 << 21),
                                                              ("weak0", 2, 2, 2, False, 0, (2,), 4672)])
def test_sharded_under_fingerprint_collisions(weak_libs, name, R, V, L, sym, depth, worlds, table):
    """ranks on one device: the owner inserts records drained from its inbox, recomputing the check hash from the words.
    weak0 gives every state to one rank; the other's frontier stays empty at every level."""
    q, o = tks.oracle(R, V, L, depth, sym)
    for world in worlds:
        r = types.SimpleNamespace(**in_child(weak_libs[(name, R, V, L)], "_multi", R, V, L, sym, depth, world, table, 1 << 20, multi_one_device=True))
        assert r.error_code == 0 and r.rc in (0, 12), (world, r.rc)
        assert r.level_sizes == o.level_sizes, world
        assert r.level_generated[:len(o.level_generated)] == o.level_generated, world
        assert (r.distinct, r.generated, r.depth) == (o.distinct, o.generated, o.depth), world
        assert r.fp_collisions > 0
        if name == "weak16":
            assert r.records_sent > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name,R,V,L,sym,stop,table,table2", [("weak16", 3, 2, 1, False, 17, 1 << 21, (1 << 20) + 8192 + 64),
                                                             ("weak0", 2, 1, 1, True, 7, 128, 192)])
def test_checkpoint_and_recover_under_fingerprint_collisions(weak_libs, tmp_path, name, R, V, L, sym, stop, table, table2):
    """the re-inserted entries (every one new, chains reordered) continue the BFS as if uninterrupted"""
    from test_checkpoint import same_exploration
    whole, part, rest, lb = in_child(weak_libs[(name, R, V, L)], "_recover", R, V, L, sym, stop, table, table2, 1 << 20, BITS[name], str(tmp_path))
    assert whole.complete and not part.complete and part.depth == stop
    same_exploration(rest, whole)
    _, o = tks.oracle(R, V, L, 0, sym)
    assert (whole.distinct, whole.generated, whole.depth) == (o.distinct, o.generated, o.depth)
    assert whole.fp_collisions >= lb > 0 and rest.fp_collisions >= lb
    if name == "weak0":
        for cap in (table, table2):
            assert table_home(cap, 1) + whole.distinct > cap


@pytest.mark.gpu
def test_view_ties_and_collisions_in_one_level(weak_libs):
    """weak16 (3,2,2): tie records and a colliding state share a fingerprint.  The tie reduction is keyed by (fp, check),
    and the patch pass replaces a state only with a tie record of its own check hash."""
    one, two, va, B, vb = in_child(weak_libs[("weak16", 3, 2, 2)], "_ties", 3, 2, 2, 16)
    (n, ties, gen, coll), trace = one
    assert (n, ties, gen) == (2, 2, 4) and coll >= 1
    assert set(trace) == {va[1], B}                # A's smallest variant, and B with its own words ...
    assert trace[va[1]] == (0, 101) and trace[B] == (0, 200)  # ... and trace records
    (n, ties, gen, coll), trace = two
    assert (n, ties, gen) == (2, 3, 5) and coll >= 1
    assert set(trace) == {va[1], vb[1]}
    assert trace[va[1]] == (0, 101) and trace[vb[1]] == (0, 201)


@pytest.mark.gpu
def test_counterexample_under_fingerprint_collisions(weak_libs):
    """weak16 (3,2,1), AcknowledgedWritesExistOnMajority: the violation at the oracle's depth, and a trace that is a
    behaviour of the spec (test_gpu_parity.test_counterexample_is_a_behaviour, run with the weak build)"""
    assert in_child(weak_libs[("weak16", 3, 2, 1)], "_counterexample", 3, 2, 1)
