"""What one recovery reads and where it puts it.  The owner of a fingerprint is its top bits, and every world is a power of
two, so a new rank's share of a checkpoint lies in a few old files: when the world shrinks (or stays) by k, new rank r
takes old files r k ... r k + k - 1 whole, keeping their histories then their frontiers in file order; when it grows by
s, new rank r's share lies in old file r / s.  Checked here on the written-back files and on the verbose line each rank
prints.

Several ranks are threads of one process sharing device 0 (VSR_B200_MULTI_ONE_DEVICE), as in test_checkpoint.py."""
import os
import re

import numpy as np
import pytest

from test_reshard import CAPS, checkpoint, files_of, read_ckpt, run, sorted_entries, vsrmc

pytestmark = pytest.mark.gpu

READ = re.compile(r"recover: rank (\d+) of (\d+) took its share of (\d+) checkpoint files \((\d+) bytes read\)")


@pytest.fixture(autouse=True)
def one_device(monkeypatch):
    monkeypatch.setenv("VSR_B200_MULTI_ONE_DEVICE", "1")


@pytest.fixture(scope="module")
def mc(pkg):
    return pkg.ModelChecker.from_constants(3, 2, 1, symmetry=False)


def sections(path):
    """(header dict, frontier bytes, seen-set entries sorted, trace bytes)"""
    h, frontier, ents = read_ckpt(path)
    raw = open(path, "rb").read()
    at = h["header_bytes"] + 2 * h["stats_bytes"] + h["n_cur"] * h["state_bytes"] + 16 * h["n_entries"]
    assert len(raw) == at + 8 * h["n_trace"]
    return h, b"".join(frontier), sorted_entries(ents), raw[at:]


def write_back(mc, tmp_path, w_a, w_b):
    """a checkpoint of w_a ranks at depth 16, recovered on w_b ranks and written straight back at the same boundary"""
    old, new = str(tmp_path / "old.ckpt"), str(tmp_path / "new.ckpt")
    checkpoint(mc, w_a, old, 16)
    back = run(mc, w_b, recover_path=old, max_depth=16, checkpoint_path=new, checkpoint_seconds=0, **CAPS)
    assert back.depth == 16
    return [sections(p) for p in files_of(old, w_a)], [sections(p) for p in files_of(new, w_b)]


@pytest.mark.parametrize("world", [1, 2])
def test_same_world_keeps_everything(mc, tmp_path, world):
    olds, news = write_back(mc, tmp_path, world, world)
    for (h0, f0, e0, t0), (h1, f1, e1, t1) in zip(olds, news):
        assert h0 == h1
        assert f0 == f1 and t0 == t1
        assert np.array_equal(e0, e1)


@pytest.mark.parametrize("w_a,w_b", [(4, 2), (2, 1)])
def test_shrink_copies_nothing(mc, tmp_path, w_a, w_b):
    olds, news = write_back(mc, tmp_path, w_a, w_b)
    k = w_a // w_b
    for r, (h, frontier, _, _) in enumerate(news):
        src = olds[r * k:(r + 1) * k]
        assert h["cur_base"] == sum(s[0]["cur_base"] for s in src)
        assert h["n_trace"] == sum(s[0]["next_base"] for s in src)
        assert frontier == b"".join(s[1] for s in src)


def test_files_read(pkg, tmp_path):
    """each rank reads the bulk sections of its source files only, and all of them (without a trace the new rank reads
    a source file's frontier and seen-set whole, whichever way the world changes)"""
    metas = {}
    for w_a in (2, 4):
        metas[w_a] = tmp_path / ("states%d" % w_a)
        r = vsrmc(pkg, tmp_path, "-notrace", "-gpus", w_a, "-checkpoint", 0, "-metadir", metas[w_a], "-depth", 11)
        assert r.returncode == 0, r.stderr
    for w_a, w_b, per_rank in ((2, 2, 1), (2, 4, 1), (4, 2, 2)):
        olds = files_of(str(metas[w_a] / "vsr.ckpt"), w_a)
        r = vsrmc(pkg, tmp_path, "-notrace", "-gpus", w_b, "-recover", metas[w_a], "-depth", 11)
        assert r.returncode == 0, r.stderr
        lines = sorted(tuple(int(x) for x in m.groups()) for m in READ.finditer(r.stderr))
        assert [ln[:3] for ln in lines] == [(rank, w_b, per_rank) for rank in range(w_b)], r.stderr
        for rank, _, _, got in lines:
            src = [rank // (w_b // w_a)] if w_b > w_a else range(rank * per_rank, (rank + 1) * per_rank)
            bulk = 0
            for q in src:
                h = read_ckpt(olds[q])[0]
                bulk += os.path.getsize(olds[q]) - h["header_bytes"] - 2 * h["stats_bytes"]
            assert got == bulk, (w_a, w_b, rank)
