"""The energy-only FragmentCalculator call's host side without a GPU: the C ABI exports its four entries, and
FragmentCalculator takes ``derivative`` as the reference's ``load_model`` does and refuses malformed arguments before it
creates an engine."""
import inspect
import os
import re

import pytest

from ai2bmd_b200 import calculator as vcalc
from ai2bmd_b200 import engine as vengine
from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_fragments, load_protein

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
ENERGY_SYMBOLS = ("vb_forward_fragments_energy", "vb_forward_fragments_energy_host",
                  "vb_group_forward_fragments_energy", "vb_group_forward_fragments_energy_host")


def test_energy_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "visnet_b200.h")).read()
    declared = set(re.findall(r"\b(vb_[a-z_0-9]+)\s*\(", header))
    lib = vengine.load_library()
    for sym in ENERGY_SYMBOLS:
        assert sym in declared and sym in vengine.EXPORTED_SYMBOLS and hasattr(lib, sym), sym


def test_python_entries_exist():
    for cls in (vengine.Engine, vengine.EngineGroup):
        for name in ("forward_fragments_energy_host", "forward_fragments_energy_device"):
            assert callable(getattr(cls, name, None)), (cls.__name__, name)


def test_derivative_defaults_to_the_checkpoint():
    for fn in (vcalc.FragmentCalculator.__init__, vcalc.FragmentCalculator.from_protein):
        assert inspect.signature(fn).parameters["derivative"].default is None


@pytest.fixture
def no_engine(monkeypatch):
    """Any engine the calculator tried to create fails the test."""
    def refuse(*args, **kwargs):
        raise AssertionError("FragmentCalculator created an engine before checking its arguments")
    monkeypatch.setattr(vcalc, "Engine", refuse)


@pytest.mark.parametrize("bad", ["no", 0, 1.0, [False]])
def test_malformed_derivative_is_refused_before_any_engine(no_engine, bad):
    fd, pm = load_fragments("chig")
    _, _, recipe = load_protein("chig")
    with pytest.raises(TypeError, match="derivative"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, derivative=bad)
    with pytest.raises(TypeError, match="derivative"):
        vcalc.FragmentCalculator.from_protein(WEIGHTS, "", load_capped_protein("chig"), derivative=bad)


def test_other_refusals_hold_for_an_energy_only_calculator(no_engine):
    fd, pm = load_fragments("chig")
    _, _, recipe = load_protein("chig")
    with pytest.raises(NotImplementedError, match="pme"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nbcalc_type="pme", derivative=False)
    R = type(recipe)
    short = R(recipe.real[:-1], recipe.acc[:-1], recipe.rem[:-1], recipe.blen[:-1])
    with pytest.raises(ValueError, match="recipe arrays"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, short, derivative=False)
    with pytest.raises(ValueError, match="devices"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, devices=[], derivative=False)
    with pytest.raises(RuntimeError, match="CPU"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, devices=["cuda:0", "cpu"], derivative=False)

