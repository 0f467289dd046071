"""The reference's un-fragmented ``--mode visnet`` input, host side: the golden of tests/golden/make_visnet_mode.py (the
reference's own model source on whole Chignolin, whole Trp-cage, a three-residue ACE-ALA-NME input, whole WW and whole ABD,
each ONE graph),
``pdbfrag.whole_input``, the masses of every element the model accepts, and the hint ``fragment_protein`` gives for
inputs it cannot fragment."""
import os

import numpy as np
import pytest
import torch

from ai2bmd_b200 import elements
from ai2bmd_b200.fixtures import load_capped_protein, load_protein
from ai2bmd_b200.pdbfrag import CappedProtein, fragment_protein, whole_input
from oracle import visnet_ref as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ("chig", "trpcage", "c1", "ww", "abd")
PROTEINS = ("chig", "trpcage", "ww", "abd")
N_ATOMS = {"chig": 175, "trpcage": 281, "c1": 22, "ww": 571, "abd": 746}


@pytest.fixture(scope="module")
def gold():
    """Both golden files as one mapping: whole WW and ABD are in reference_visnet_mode_large.npz."""
    out = {}
    for name in ("reference_visnet_mode.npz", "reference_visnet_mode_large.npz"):
        with np.load(os.path.join(GOLDEN, name)) as g:
            out.update({k: g[k] for k in g.files})
    return out


def c1_protein(gold):
    return CappedProtein([str(x) for x in gold["c1_names"]], [str(x) for x in gold["c1_resnames"]],
                         gold["c1_resnums"].astype(np.int64), [str(x) for x in gold["c1_elements"]],
                         gold["c1_pos"].astype(np.float64))


def test_golden_loads(gold):
    for key in CASES:
        n = N_ATOMS[key]
        assert gold[f"{key}_z"].shape == (n,) and gold[f"{key}_pos"].shape == (n, 3)
        assert (gold[f"{key}_batch"] == 0).all()
        assert gold[f"{key}_ref_e"].shape == (1, 1) and gold[f"{key}_e64"].shape == (1, 1)
        assert gold[f"{key}_ref_f"].shape == (n, 3) and gold[f"{key}_f64"].shape == (n, 3)
        assert gold[f"{key}_slots"].shape == (n, 32) and gold[f"{key}_deg"].shape == (n,)
        assert np.isfinite(gold[f"{key}_ref_f"]).all() and np.isfinite(gold[f"{key}_f64"]).all()


@pytest.mark.parametrize("key", CASES)
def test_slots_of_the_c_oracle_equal_the_reference(gold, key):
    """oracle/radius_graph.c, its numpy twin and the slots the reference's model consumed agree; whole proteins truncate."""
    pos, batch = gold[f"{key}_pos"], gold[f"{key}_batch"]
    s1, d1 = O.radius_graph_canonical(pos, batch)
    s2, d2 = O.radius_graph_numpy(pos, batch)
    assert np.array_equal(s1, gold[f"{key}_slots"]) and np.array_equal(d1, gold[f"{key}_deg"])
    assert np.array_equal(s2, s1) and np.array_equal(d2, d1)
    p = pos.astype(np.float32)
    n_cand = (((p[:, None, :] - p[None, :, :]) ** 2).sum(-1) < np.float32(25.0)).sum(1)
    assert np.array_equal(d1, np.minimum(n_cand, 32))
    if key == "c1":
        assert n_cand.max() <= 32
    else:                                   # the first-32-by-index cap drops neighbours of most interior atoms
        assert (n_cand > 32).sum() > len(p) // 3


@pytest.mark.parametrize("key", PROTEINS)
def test_whole_input_is_one_graph_in_file_order(gold, key):
    prot = load_capped_protein(key)
    fd = whole_input(prot)
    prot_pos, prot_z, _ = load_protein(key)
    assert len(fd) == 1 and list(fd.start) == [0] and list(fd.end) == [len(prot)]
    assert (fd.batch == 0).all() and fd.z.dtype == np.int64
    assert np.array_equal(fd.z, prot_z) and np.array_equal(fd.pos, prot_pos.astype(np.float32))
    assert np.array_equal(fd.z, gold[f"{key}_z"]) and np.array_equal(fd.pos, gold[f"{key}_pos"])


def test_three_residue_input_is_refused_with_the_hint(gold):
    prot = c1_protein(gold)
    assert prot.resnames[0] == "ACE" and prot.resnames[-1] == "NME" and int(prot.resnums.max()) == 3
    with pytest.raises(NotImplementedError, match=r"whole_input.*DeviceLangevin\.unfragmented"):
        fragment_protein(prot)
    fd = whole_input(prot)
    assert np.array_equal(fd.z, gold["c1_z"]) and np.array_equal(fd.pos, gold["c1_pos"])


def test_masses_cover_every_element_and_keep_the_old_values():
    old = {1: 1.008, 6: 12.011, 7: 14.007, 8: 15.999, 16: 32.06}       # the table the MD code used before
    from ai2bmd_b200.md import MASSES
    assert MASSES is elements.MASSES and set(MASSES) == set(range(1, 100))
    for z, m in old.items():
        assert MASSES[z] == m and np.float64(MASSES[z]).tobytes() == np.float64(m).tobytes()
    m = np.array([MASSES[z] for z in range(1, 100)])
    assert (m > 0).all() and (np.diff(m[:17]) > 0).all()                # increasing through the light elements
    assert np.array_equal(elements.masses_of([1, 6, 7, 8, 16]), np.array(list(old.values())))
    for bad in ([0], [100], [6, 118]):
        with pytest.raises(ValueError, match="atomic number"):
            elements.masses_of(bad)
    assert elements.atomic_number("C") == 6 and elements.atomic_number("CL") == 17 and elements.atomic_number("Se") == 34
    with pytest.raises(ValueError):
        elements.atomic_number("Qq")


@pytest.mark.parametrize("key", ["c1", "chig", "abd"])
def test_oracle_matches_the_reference_on_one_graph(real_weights, gold, key):
    """The fp32 oracle against the reference's own model source, with the neighbour cap truncating (chig, abd)."""
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in real_weights.items()}
    e, f = O.OracleViSNet(sd, torch.float32).energy_and_forces(gold[f"{key}_z"], gold[f"{key}_pos"], gold[f"{key}_batch"])
    ref_e, ref_f = gold[f"{key}_ref_e"], gold[f"{key}_ref_f"]
    assert np.abs(e.numpy() - ref_e).max() <= 4 * np.spacing(np.float32(np.abs(ref_e).max()))
    assert np.abs(f.numpy() - ref_f).max() <= 2e-5 * max(1.0, np.abs(ref_f).max())
