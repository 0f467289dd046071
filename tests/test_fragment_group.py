"""The host side of a FragmentCalculator spread over a group of window engines (vb_group_*, ``devices=``), without a GPU:
the C ABI exports the group, ``devices`` is parsed and refused before any engine exists, and the members the calculator
builds hold the blocks, windows and MM rows of the sharded path, tiling the batch and the protein."""
import os
import re
import types

import numpy as np
import pytest

from ai2bmd_b200 import calculator as vcalc
from ai2bmd_b200 import engine as vengine
from ai2bmd_b200 import parallel as vparallel
from ai2bmd_b200.fixtures import WEIGHTS, load_fragments, load_protein
from ai2bmd_b200.nonbonded import synthetic_parameters

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GROUP_SYMBOLS = ("vb_group_create", "vb_group_destroy", "vb_group_last_error", "vb_group_forward_fragments",
                 "vb_group_forward_fragments_host")


def test_group_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "visnet_b200.h")).read()
    declared = set(re.findall(r"\b(vb_[a-z_0-9]+)\s*\(", header))
    lib = vengine.load_library()
    for sym in GROUP_SYMBOLS:
        assert sym in declared and sym in vengine.EXPORTED_SYMBOLS and hasattr(lib, sym), sym


def test_devices_parsing():
    assert vcalc._device_list(None) is None
    assert vcalc._device_list("cuda:1") is None                   # one device: the single-device path
    assert vcalc._device_list(["cuda:0", "cuda:0"]) == ["cuda:0", "cuda:0"]
    assert vcalc._device_list(("cuda:1", "cuda")) == ["cuda:1", "cuda"]
    with pytest.raises(ValueError, match="at least one"):
        vcalc._device_list([])
    with pytest.raises(RuntimeError, match="no CPU path"):
        vcalc._device_list(["cuda:0", "cpu"])
    with pytest.raises(ValueError, match="Unrecognized device"):
        vcalc._device_list(["cuda:0", "tpu:0"])


@pytest.fixture
def no_engine(monkeypatch):
    """Any engine, shard or group the calculators tried to create fails the test."""
    def refuse(*args, **kwargs):
        raise AssertionError("an engine was created before the arguments were checked")
    for mod, name in ((vcalc, "Engine"), (vcalc, "ViSNetModel"), (vengine, "Engine"), (vengine, "EngineGroup"),
                      (vparallel, "DeviceShard")):
        monkeypatch.setattr(mod, name, refuse)


def test_refusals_come_before_any_engine(no_engine):
    fd, pm = load_fragments("chig")
    _, z, recipe = load_protein("chig")
    with pytest.raises(ValueError, match="without a block"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, devices=["cuda:0"] * (len(fd) + 1))
    with pytest.raises(ValueError, match="at least one"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, devices=[])
    with pytest.raises(RuntimeError, match="no CPU path"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, devices=["cuda:0", "cpu"])
    with pytest.raises(ValueError, match="recipe arrays"):
        R = type(recipe)
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, R(recipe.real[:-1], recipe.acc, recipe.rem, recipe.blen),
                                 devices=["cuda:0", "cuda:0"])
    q, s, e = synthetic_parameters(z)
    with pytest.raises(ValueError, match="nonbonded"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nonbonded=(q[:-1], s, e), devices=["cuda:0", "cuda:0"])
    with pytest.raises(NotImplementedError, match="pme"):
        vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nbcalc_type="pme", devices=["cuda:0", "cuda:0"])
    with pytest.raises(ValueError, match="at least one"):
        vcalc.FragmentCalculator.from_protein(WEIGHTS, "", None, devices=[])
    with pytest.raises(ValueError, match="at least one"):
        vcalc.DLBondedCalculator(WEIGHTS, devices=[])


class _RecordedShard:
    """Stands in for DeviceShard: the host plan of the rank, and what set_window was given."""
    made = []

    def __init__(self, state_dict, frags, pm, rank, world_size, device, native_comm=True, chunk_atoms=0):
        self.plan = vparallel.ShardedBondedCalculator(frags, pm, rank, world_size)
        self.device, self.native_comm, self.chunk_atoms = device, native_comm, chunk_atoms
        self.engine = types.SimpleNamespace(rank=rank)
        _RecordedShard.made.append(self)

    def set_window(self, frags, pm, recipe, caph=None, nonbonded=None):
        self.window = (len(frags.z), self.plan.atom_lo, self.plan.atom_hi)
        self.mm = vparallel.mm_rows(pm.n_protein, self.plan.rank, self.plan.world_size) if nonbonded is not None else None


@pytest.mark.parametrize("name", ["chig", "trpcage"])
@pytest.mark.parametrize("k", [2, 3, 4])
def test_members_tile_the_batch_and_the_protein(monkeypatch, name, k):
    fd, pm = load_fragments(name)
    _, z, recipe = load_protein(name)
    groups = []
    monkeypatch.setattr(vparallel, "DeviceShard", _RecordedShard)
    monkeypatch.setattr(vengine, "EngineGroup", lambda engines: groups.append(engines) or types.SimpleNamespace())
    _RecordedShard.made = []
    devices = [f"cuda:{r % 2}" for r in range(k)]
    vcalc.FragmentCalculator(WEIGHTS, "", fd, pm, recipe, nonbonded=synthetic_parameters(z), devices=devices, chunk_size=60)
    shards = _RecordedShard.made
    assert [sh.plan.rank for sh in shards] == list(range(k)) and all(sh.plan.world_size == k for sh in shards)
    assert [sh.device for sh in shards] == [r % 2 for r in range(k)]
    assert all(not sh.native_comm and sh.chunk_atoms == 60 for sh in shards)
    assert [e.rank for e in groups[0]] == list(range(k))          # the group's rank order is the shards' order
    parts = vparallel.partition_fragments(fd.start, fd.end, k)
    N, P = len(fd.z), pm.n_protein
    atom, row = 0, 0
    for sh, (lo, hi) in zip(shards, parts):
        assert (sh.plan.lo, sh.plan.hi) == (lo, hi) and hi > lo
        assert sh.window == (N, int(fd.start[lo]), int(fd.end[hi - 1]))
        assert sh.window[1] == atom                               # the windows tile the batch in rank order
        atom = sh.window[2]
        assert sh.mm == vparallel.mm_rows(P, sh.plan.rank, k)
        assert sh.mm[0] == row                                    # ... and the MM rows the protein
        row = sh.mm[1]
    assert atom == N and row == P
