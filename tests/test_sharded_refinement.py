"""The host side of sharded steps with the hydrogen refinement, without a GPU: the C ABI exports the batch window, the
recipe length follows the window, and DeviceLangevin.sharded refuses what it cannot run before it creates an engine."""
import os
import re

import numpy as np
import pytest

from ai2bmd_b200 import engine as vengine
from ai2bmd_b200 import parallel
from ai2bmd_b200.fixtures import WEIGHTS, load_fragments, load_protein
from ai2bmd_b200.md import DeviceLangevin
from ai2bmd_b200.nonbonded import synthetic_parameters

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def test_batch_window_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "visnet_b200.h")).read()
    declared = set(re.findall(r"\b(vb_[a-z_0-9]+)\s*\(", header))
    lib = vengine.load_library()
    sym = "vb_set_batch_window"
    assert sym in declared and sym in vengine.EXPORTED_SYMBOLS and hasattr(lib, sym)


@pytest.fixture
def no_engine(monkeypatch):
    """Any engine or shard DeviceLangevin.sharded tried to create fails the test."""
    def refuse(*args, **kwargs):
        raise AssertionError("DeviceLangevin.sharded created an engine before checking its arguments")
    monkeypatch.setattr(parallel, "DeviceShard", refuse)
    monkeypatch.setattr(vengine, "Engine", refuse)


class _NoGroup:
    """A process group that fails the test when it is asked for anything."""
    def __getattr__(self, name):
        raise AssertionError("DeviceLangevin.sharded used the process group before checking its arguments")


def test_sharded_refuses_a_malformed_recipe_before_any_engine(no_engine):
    fd, pm = load_fragments("chig")
    x, z, recipe = load_protein("chig")
    R = type(recipe)
    r, a, q, b = recipe.real, recipe.acc, recipe.rem, recipe.blen
    lo, hi = int(fd.start[0]), int(fd.end[len(fd) // 2 - 1])
    for bad in (R(r[lo:hi], a[lo:hi], q[lo:hi], b[lo:hi]),          # one shard's slice, not the whole batch
                R(r[:-1], a[:-1], q[:-1], b[:-1]),                  # one atom short
                R(r, a, q[:-1], b)):                                # one array short
        with pytest.raises(ValueError, match="recipe arrays"):
            DeviceLangevin.sharded(WEIGHTS, fd, pm, bad, x, z, _NoGroup())


def test_sharded_refuses_malformed_mm_parameters_before_any_engine(no_engine):
    fd, pm = load_fragments("chig")
    x, z, recipe = load_protein("chig")
    qs, sg, ep = synthetic_parameters(z)
    for bad in ((qs[:-1], sg, ep), (qs, sg), (qs, sg, np.append(ep, 1.0))):
        with pytest.raises(ValueError, match="nonbonded"):
            DeviceLangevin.sharded(WEIGHTS, fd, pm, recipe, x, z, _NoGroup(), nonbonded=bad)


def test_recipe_length_follows_the_window():
    """On a windowed engine the recipe has one entry per BATCH atom: the window's own length is refused before the call
    reaches the library, and so is the batch's on an engine without a window."""
    eng = vengine.Engine.__new__(vengine.Engine)
    eng.n_atoms, eng.n_protein = 10, 5

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError(f"the recipe reached the library ({name})")
    eng.lib, eng.h = NoLib(), None
    assert eng.batch_atoms == 10
    with pytest.raises(ValueError, match="one entry per fragment atom"):
        eng.set_fragment_recipe(np.zeros(25), np.zeros(25), np.zeros(25), np.zeros(25))
    eng._window = (25, 10)
    assert eng.batch_atoms == 25
    for call in (lambda *a: eng.set_fragment_recipe(*a), lambda *a: eng.md_setup(np.ones(5), *a, 1.0, 0.0, 0.0, 0, 0)):
        with pytest.raises(ValueError, match="one entry per fragment atom"):
            call(np.zeros(10), np.zeros(10), np.zeros(10), np.zeros(10))


def test_mm_rows_split_the_protein_evenly():
    for n, world in ((166, 2), (166, 3), (304, 4), (7, 8)):
        rows = [parallel.mm_rows(n, r, world) for r in range(world)]
        assert rows[0][0] == 0 and rows[-1][1] == n
        assert all(rows[r][1] == rows[r + 1][0] for r in range(world - 1))
        assert max(hi - lo for lo, hi in rows) - min(hi - lo for lo, hi in rows) <= 1


def test_more_ranks_than_blocks_are_refused():
    fd, _ = load_fragments("chig")
    parallel.check_shardable(fd, 4)
    with pytest.raises(ValueError, match="without a block"):
        parallel.check_shardable(fd, len(fd) + 1)
