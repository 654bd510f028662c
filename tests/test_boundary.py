"""The drop-in boundary (SURVEY §8b): TLC's cfg grammar, identity check of the .tla, exported C ABI, struct mirrors,
loud failure without a GPU."""
import ctypes as C
import os
import re
import subprocess

import pytest

import vsr_stub
from conftest import REF_CFG, ROOT

HDR = os.path.join(ROOT, "include", "vsr_b200.h")


def test_library_exports_every_declared_symbol(pkg):
    lib = pkg.load_library()
    text = open(HDR).read()
    declared = set(re.findall(r"\b(vsr_[a-z0-9_]+)\s*\(", text))
    assert declared, "no declarations found"
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/vsr_b200.h but not exported"
    assert declared == set(pkg.checker.EXPORTED_SYMBOLS)


def test_struct_mirrors_match_c_sizes(pkg, tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "vsr_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(VsrFlatState), sizeof(VsrMsg),'
                   ' sizeof(VsrModelInfo), sizeof(VsrRunOpts), sizeof(VsrStats), sizeof(VsrLevelInfo), sizeof(VsrSimOpts),'
                   ' sizeof(VsrSimStats)); return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    ck = pkg.checker
    assert sizes == [C.sizeof(ck.VsrFlatState), C.sizeof(ck.VsrMsg), C.sizeof(ck.VsrModelInfo), C.sizeof(ck.VsrRunOpts),
                     C.sizeof(ck.VsrStats), C.sizeof(ck.VsrLevelInfo), C.sizeof(ck.VsrSimOpts), C.sizeof(ck.VsrSimStats)]


def test_shipped_cfg_loads(pkg):
    """the reference's VSR.cfg as it is shipped (comments, commented-out keywords, model values, VIEW, SYMMETRY)"""
    mc = pkg.ModelChecker.from_cfg(REF_CFG)
    i = mc.info
    assert (i.replica_count, i.client_count, i.value_count, i.start_view_on_timer_limit, i.restart_empty_limit) == (3, 1, 2, 2, 0)
    assert (i.symmetry, i.view, i.invariant) == (1, 1, 1)
    assert [bytes(i.value_names[k]).split(b"\0")[0] for k in range(2)] == [b"v1", b"v2"]
    assert i.state_bytes == 48


def test_an_edited_spec_is_refused_not_verified(pkg, tmp_path, monkeypatch):
    """Next and the invariants are hand-lowered, so a .tla whose definitions differ from VSR.tla must not load as "verified":
    a module with VSR.tla's name, VARIABLES, disjunct names and definitions but other bodies is refused; the explicit override
    loads it, loudly, NOT verified, with the action locations read from that file as TLC reports them."""
    text = vsr_stub.module_text(pkg.ACTION_NAMES[1:])
    p = tmp_path / "VSR.tla"
    p.write_text(text)
    with pytest.raises(pkg.VsrError) as ei:
        pkg.ModelChecker.from_cfg(REF_CFG, str(p))
    assert ei.value.rc == 150 and "hand" in str(ei.value)
    monkeypatch.setenv("VSR_B200_ALLOW_EDITED_SPEC", "1")
    mc = pkg.ModelChecker.from_cfg(REF_CFG, str(p))
    assert mc.info.spec_verified == 0
    for a in range(1, len(pkg.ACTION_NAMES)):
        assert mc.action_location(a) == vsr_stub.location(text, pkg.ACTION_NAMES[a])
    assert mc.action_location(0) == "Unknown location"


def test_readme_constants_load(pkg, tmp_path):
    """README.md:13-18 of the reference: the user edits only the constants of the shipped VSR.cfg"""
    cfg = open(REF_CFG).read().replace("Values = {v1, v2}", "Values = {v1, v2, v3}").replace("StartViewOnTimerLimit = 2", "StartViewOnTimerLimit = 3")
    assert "v3" in cfg and "StartViewOnTimerLimit = 3" in cfg
    p = tmp_path / "VSR.cfg"
    p.write_text(cfg)
    mc = pkg.ModelChecker.from_cfg(str(p))
    assert (mc.info.value_count, mc.info.start_view_on_timer_limit, mc.info.state_bytes) == (3, 3, 64)


def test_other_specs_are_refused(pkg, tmp_path):
    """a module other than the VSR.tla whose Next is lowered by hand (here one of the reference's analysis specs by name)"""
    other = tmp_path / "VR_STATE_TRANSFER.tla"
    other.write_text("------------------------------ MODULE VR_STATE_TRANSFER ------------------------------\n"
                     "EXTENDS Naturals, FiniteSets, Sequences, TLC\nVARIABLES replica_status\nInit == replica_status = 0\n"
                     "Next == replica_status' = replica_status\n====\n")
    with pytest.raises(pkg.VsrError) as e:
        pkg.ModelChecker.from_cfg_text(pkg.cfg_text(3, ["v1", "v2"], 2), str(other))
    assert e.value.rc == 150


def test_cfg_grammar(pkg):
    base = pkg.cfg_text(3, ["v1", "v2"], 2)
    mc = pkg.ModelChecker.from_cfg_text(base)
    assert (mc.info.symmetry, mc.info.view, mc.info.invariant) == (1, 1, 1)
    # comments, commented-out keywords, inline comments after invariant names, no trailing newline (VSR.cfg:1,33-39)
    text = "\\* SPECIFICATION\n" + base.rstrip("\n") + "\n\\* PROPERTY\nAcknowledgedWritesExistOnMajority \\* less strict\n\\* NoLogDivergence"
    mc = pkg.ModelChecker.from_cfg_text(text)
    assert mc.info.invariant == 3
    # no SYMMETRY / VIEW lines
    mc = pkg.ModelChecker.from_cfg_text(pkg.cfg_text(3, ["a", "b"], 2, view=False, symmetry=False, invariants=["TestInv"]))
    assert (mc.info.symmetry, mc.info.view, mc.info.invariant) == (0, 0, 8)
    assert bytes(mc.info.value_names[1]).startswith(b"b")
    # a singleton Values has a trivial symmetry group
    assert pkg.ModelChecker.from_cfg_text(pkg.cfg_text(2, ["v1"], 1)).info.symmetry == 0


def test_specification_spec_is_init_next(pkg):
    """VSR.cfg's first line is a commented-out SPECIFICATION; `SPECIFICATION Spec` (VSR.tla:966: Init /\\ [][Next]_vars /\\
    WF_vars(Next)) in place of INIT/NEXT checks the same invariants over the same state graph, as in TLC"""
    base = pkg.cfg_text(3, ["v1", "v2"], 2)
    spec = base.replace("INIT Init\n", "").replace("NEXT Next\n", "SPECIFICATION Spec\n")
    assert "SPECIFICATION Spec" in spec and "INIT" not in spec
    a, b = pkg.ModelChecker.from_cfg_text(base), pkg.ModelChecker.from_cfg_text(spec)
    assert a.successors(a.init_state()) == b.successors(b.init_state())
    with pytest.raises(pkg.VsrError, match="Spec"):
        pkg.ModelChecker.from_cfg_text(spec.replace("SPECIFICATION Spec", "SPECIFICATION LivenessSpec"))


@pytest.mark.parametrize("mut,frag", [
    (lambda t: t.replace("INIT Init", "SPECIFICATION Spec\nINIT Init"), "SPECIFICATION"),
    (lambda t: t + "PROPERTY ViewChangeCompletes\n", "PROPERTY"),
    (lambda t: t + "CONSTRAINT Foo\n", "CONSTRAINT"),
    (lambda t: t.replace("ClientCount = 1", "ClientCount = 2"), "m.commit"),
    (lambda t: t.replace("RestartEmptyLimit = 0", "RestartEmptyLimit = 1"), "RestartEmptyLimit"),
    (lambda t: t.replace("    Nil = Nil\n", ""), "Nil"),
    (lambda t: t.replace("NEXT Next", "NEXT Foo"), "NEXT"),
    (lambda t: t.replace("AcknowledgedWriteNotLost", "NoSuchInvariant"), "NoSuchInvariant"),
    (lambda t: t.replace("ReplicaCount = 3", "ReplicaCount = 8"), "outside the packed encoding's range"),
    (lambda t: t.replace("    StartViewOnTimerLimit = 2\n", ""), "StartViewOnTimerLimit"),
])
def test_cfg_rejections_are_loud(pkg, mut, frag):
    with pytest.raises(pkg.VsrError) as e:
        pkg.ModelChecker.from_cfg_text(mut(pkg.cfg_text(3, ["v1", "v2"], 2)))
    assert e.value.rc == 151 and frag in str(e.value)


def test_no_gpu_means_loud_failure_not_fallback(pkg):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    mc = pkg.ModelChecker.from_constants(2, 1, 1)
    with pytest.raises(pkg.VsrError) as e:
        mc.check()
    assert e.value.rc == 153
    r = subprocess.run([os.path.join(ROOT, "vsr-tlaplus_b200", "vsrmc"), "-config", "/dev/null"], capture_output=True, text=True)
    assert r.returncode == 151


def test_init_has_the_hand_derivable_successors(pkg):
    """SURVEY §8c: Init has (R-1) + V successors, (R-1) + 1 distinct under symmetry"""
    for (R, V, L) in [(2, 1, 1), (3, 2, 2), (3, 3, 3), (5, 2, 2)]:
        mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=True)
        succ = mc.successors(mc.init_state())
        assert sum(m for _, _, m in succ) == (R - 1) + V
        assert len({t for t, _, _ in succ}) == (R - 1) + 1
        mc = pkg.ModelChecker.from_constants(R, V, L, symmetry=False)
        assert len({t for t, _, _ in mc.successors(mc.init_state())}) == (R - 1) + V


def test_check_deadlock_keyword_of_the_cfg_is_honoured(pkg):
    """ADVICE round 1: CHECK_DEADLOCK FALSE in the cfg must switch deadlock checking off (TLC does), not be parsed and dropped."""
    base = pkg.cfg_text(2, ["v1"], 1)
    off = pkg.ModelChecker.from_cfg_text(base + "CHECK_DEADLOCK FALSE\n")
    on = pkg.ModelChecker.from_cfg_text(base + "CHECK_DEADLOCK TRUE\n")
    absent = pkg.ModelChecker.from_cfg_text(base)
    assert (off.info.check_deadlock, on.info.check_deadlock, absent.info.check_deadlock) == (0, 1, -1)
    assert off.run_opts().check_deadlock == 0 and on.run_opts().check_deadlock == 1 and absent.run_opts().check_deadlock == 0
    assert off.run_opts(deadlock=True).check_deadlock == 1  # an explicit argument wins, like TLC's command line over the cfg
