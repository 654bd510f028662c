"""vsr-tlaplus_b200 — H100-native explicit-state model checker for vsr-revisited/paper/VSR.tla.

The product is the C-ABI shared library ``libvsr_b200.so`` (include/vsr_b200.h): hand-written CUDA
(sm_90a) BFS wavefront + a thin C++ host.  This package is only the Python mirror of TLC's
command-line surface for that one path (``ModelChecker`` ~ ``tlc2.TLC -config VSR.cfg VSR.tla``) and
the multi-GPU pump (``dist``), which uses torch.distributed for the all-to-all plumbing.

The directory name carries a hyphen (it is the name the build contract fixes); import it through
``_pkg.load()`` at the repo root, which registers it as ``vsr_tlaplus_b200``.
"""
from .checker import (  # noqa: F401
    LIB_PATH,
    ModelChecker,
    CheckResult,
    VsrError,
    load_library,
    cfg_text,
    ACTION_NAMES,
)
