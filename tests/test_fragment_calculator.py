"""The whole-calculator entry's host side without a GPU: the C ABI exports it, and FragmentCalculator refuses what it
cannot run before it creates an engine."""
import os
import re

import numpy as np
import pytest

from ai2bmd_b200 import calculator as vcalc
from ai2bmd_b200 import engine as vengine
from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_fragments, load_protein

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
FRAGMENT_SYMBOLS = ("vb_set_fragment_recipe", "vb_forward_fragments", "vb_forward_fragments_host")


def test_fragment_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "visnet_b200.h")).read()
    declared = set(re.findall(r"\b(vb_[a-z_0-9]+)\s*\(", header))
    lib = vengine.load_library()
    for sym in FRAGMENT_SYMBOLS:
        assert sym in declared and sym in vengine.EXPORTED_SYMBOLS and hasattr(lib, sym), sym


@pytest.fixture
def no_engine(monkeypatch):
    """Any engine the calculator tried to create fails the test."""
    def refuse(*args, **kwargs):
        raise AssertionError("FragmentCalculator created an engine before checking its arguments")
    monkeypatch.setattr(vcalc, "Engine", refuse)


def test_pme_is_refused_before_any_engine(no_engine):
    fd, pm = load_fragments("chig")
    _, _, recipe = load_protein("chig")
    with pytest.raises(NotImplementedError, match="pme"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nbcalc_type="pme")
    with pytest.raises(NotImplementedError, match="pme"):
        vcalc.FragmentCalculator.from_protein(WEIGHTS, "", load_capped_protein("chig"), nbcalc_type="pme")
    with pytest.raises(ValueError, match="nbcalc_type"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nbcalc_type="ewald")


def _malformed(recipe):
    """Recipes whose arrays do not give one entry per fragment atom."""
    r, a, q, b = recipe.real, recipe.acc, recipe.rem, recipe.blen
    R = type(recipe)
    return [R(r[:-1], a[:-1], q[:-1], b[:-1]),          # one atom short everywhere
            R(r, a[:-1], q, b),                          # one array short
            R(r, a, q, np.append(b, 1.0)),               # one array long
            R(r.reshape(-1, 1), a.reshape(-1, 1), q.reshape(-1, 1), b.reshape(-1, 1))]   # not 1-D


def test_malformed_recipe_is_refused_before_any_engine(no_engine):
    fd, pm = load_fragments("chig")
    _, _, recipe = load_protein("chig")
    for bad in _malformed(recipe):
        with pytest.raises(ValueError, match="recipe arrays"):
            vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, bad)


def test_malformed_mm_parameters_are_refused_before_any_engine(no_engine):
    fd, pm = load_fragments("chig")
    _, z, recipe = load_protein("chig")
    from ai2bmd_b200.nonbonded import synthetic_parameters
    q, s, e = synthetic_parameters(z)
    with pytest.raises(ValueError, match="nonbonded"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nonbonded=(q[:-1], s, e))
    with pytest.raises(ValueError, match="nonbonded"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nonbonded=(q, s))


def test_engine_recipe_binding_checks_lengths():
    """Engine.set_fragment_recipe refuses arrays of the wrong length before the call reaches the library."""
    eng = vengine.Engine.__new__(vengine.Engine)
    eng.n_atoms, eng.n_protein = 10, 5

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError(f"set_fragment_recipe reached the library ({name})")
    eng.lib, eng.h = NoLib(), None
    with pytest.raises(ValueError, match="one entry per fragment atom"):
        eng.set_fragment_recipe(np.zeros(9), np.zeros(9), np.zeros(9), np.zeros(9))
    with pytest.raises(ValueError, match="one entry per fragment atom"):
        eng.set_fragment_recipe(np.zeros(10), np.zeros(10), np.zeros(9), np.zeros(10))
