"""DeviceLangevin.grouped checks its arguments before any engine is made (no GPU needed); the device step itself is
tests/test_md_group_gpu.py."""
import numpy as np
import pytest

from ai2bmd_b200.fixtures import load_fragments, load_protein
from ai2bmd_b200.md import DeviceLangevin


def _args():
    fd, pm = load_fragments("chig")
    x0, z, recipe = load_protein("chig")
    return fd, pm, recipe, x0, z


@pytest.mark.parametrize("devices", [None, "cuda:0", []])
def test_devices_must_be_a_list(devices):
    fd, pm, recipe, x0, z = _args()
    with pytest.raises(ValueError, match="devices"):
        DeviceLangevin.grouped(None, fd, pm, recipe, x0, z, devices=devices)


def test_refused_before_any_engine():
    fd, pm, recipe, x0, z = _args()
    with pytest.raises(ValueError, match="noise"):
        DeviceLangevin.grouped(None, fd, pm, recipe, x0, z, devices=["cuda:0"] * 2, noise="numpy")
    with pytest.raises(ValueError):                                      # more members than fragment blocks
        DeviceLangevin.grouped(None, fd, pm, recipe, x0, z, devices=["cuda:0"] * (len(fd) + 1))
    short = type(recipe)(recipe.real[:-1], recipe.acc[:-1], recipe.rem[:-1], recipe.blen[:-1])
    with pytest.raises(ValueError):                                      # a recipe of the wrong length
        DeviceLangevin.grouped(None, fd, pm, short, x0, z, devices=["cuda:0"] * 2)
    with pytest.raises(ValueError):                                      # MM parameters of the wrong length
        DeviceLangevin.grouped(None, fd, pm, recipe, x0, z, devices=["cuda:0"] * 2,
                               nonbonded=(np.zeros(3), np.zeros(3), np.zeros(3)))
