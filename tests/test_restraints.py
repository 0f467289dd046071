"""Host side of the restraint protocol (no GPU): the hydrogen bond pairs against the reference's own
``PDBAnalyzer.find_bonded_atoms`` (tests/golden/reference_hbond_pairs.json), the Hookean checker against its own gradient,
and the unit constant."""
import json
import os
import types

import numpy as np
import pytest

from ai2bmd_b200.fixtures import load_capped_protein
from ai2bmd_b200.restraints import HBOND_K, KCALMOL_EV, PREEQ_SCHEDULE, hydrogen_bond_springs
from oracle.hookean_ref import hookean, hookean_terms

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_hbond_pairs.json")))


def _assert_pairs(springs, gold_pairs):
    ij, k, rt = springs
    assert len(ij) == len(gold_pairs)
    g = np.asarray(gold_pairs, dtype=np.float64)
    assert (ij[:, 0] == g[:, 0]).all() and (ij[:, 1] == g[:, 1]).all()
    assert (rt == g[:, 2]).all()                     # same float expression as the reference: bitwise
    assert (k == g[:, 3]).all() and (k == HBOND_K).all()


@pytest.mark.parametrize("name", sorted(GOLD))
def test_hydrogen_bond_springs_equal_the_reference(name):
    g = GOLD[name]
    prot = types.SimpleNamespace(names=g["names"], positions=np.asarray(g["positions"]))
    springs = hydrogen_bond_springs(prot)
    _assert_pairs(springs, g["pairs"])
    n_h = sum(n.startswith("H") for n in g["names"])
    assert len(springs[0]) == n_h                    # one partner per hydrogen


@pytest.mark.parametrize("name", ["chig", "trpcage", "ww", "abd"])
def test_hydrogen_bond_springs_of_the_fixture_proteins(name):
    """The packaged proteins have the reference PDB's atom order, so their pairs are the reference's."""
    prot = load_capped_protein(name)
    g = GOLD[name]
    assert list(prot.names) == g["names"]
    assert np.abs(np.asarray(prot.positions) - np.asarray(g["positions"])).max() <= 1e-9
    _assert_pairs(hydrogen_bond_springs(prot), g["pairs"])


def test_hydrogen_bond_springs_reject_a_stray_hydrogen():
    g = GOLD["chig"]
    pos = np.asarray(g["positions"]).copy()
    h = g["names"].index("HA")
    pos[h] += 5.0                                    # no partner left
    with pytest.raises(ValueError):
        hydrogen_bond_springs(types.SimpleNamespace(names=g["names"], positions=pos))


def test_unit_constant_and_schedule():
    # ASE 3.22: units.kcal / units.mol / units.eV with CODATA 2014 (e = 1.6021766208e-19 C, N_A = 6.022140857e23)
    assert KCALMOL_EV == pytest.approx(0.0433641039, abs=1e-10)
    assert abs(KCALMOL_EV - 4.184e3 / 1.6021766208e-19 / 6.022140857e23) <= 1e-16
    assert tuple(PREEQ_SCHEDULE) == (10, 5, 1, 0.5, 0.1)


def _random_terms(rng, n, rt_scale):
    x = rng.normal(scale=2.0, size=(n, 3))
    anchors = x + rng.normal(scale=0.3, size=x.shape)
    ij = np.array([(i, (i + 1 + rng.integers(n - 1)) % n) for i in range(n)])
    d = np.linalg.norm(x[ij[:, 1]] - x[ij[:, 0]], axis=1)
    rt = d * rng.uniform(1.0 - rt_scale, 1.0 + rt_scale, size=n)     # about half the springs active
    return x, hookean_terms(np.arange(0, n, 2), anchors, 0.7, (ij, rng.uniform(0.5, 20.0, size=n), rt))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_hookean_forces_are_minus_the_gradient(seed):
    rng = np.random.default_rng(seed)
    x, terms = _random_terms(rng, 12, 0.3)
    e, f = hookean(x, terms)
    assert e > 0.0
    h = 1e-6
    num = np.zeros_like(x)
    for a in range(len(x)):
        for c in range(3):
            xp, xm = x.copy(), x.copy()
            xp[a, c] += h
            xm[a, c] -= h
            num[a, c] = -(hookean(xp, terms)[0] - hookean(xm, terms)[0]) / (2 * h)
    assert np.abs(f - num).max() <= 1e-6 * max(1.0, np.abs(f).max())
    # both sides of rt are exercised
    active = [t for t in terms if t[0] == "two atoms" and np.linalg.norm(x[t[2]] - x[t[1]]) > t[4]]
    assert 0 < len(active) < sum(t[0] == "two atoms" for t in terms)


def test_hookean_inside_rt_and_at_zero_length():
    x = np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0]])
    e, f = hookean(x, [("two atoms", 0, 1, 15.0, 1.0)])                  # shorter than rt: nothing
    assert e == 0.0 and not f.any()
    e, f = hookean(x, hookean_terms([0, 1], x, 10.0 * KCALMOL_EV))       # on the anchor: L = 0
    assert e == 0.0 and not f.any() and np.isfinite(f).all()
    e, f = hookean(x, [("two atoms", 0, 1, 2.0, 0.0)])
    assert e == pytest.approx(0.25) and f[0, 0] == pytest.approx(1.0) and f[1, 0] == pytest.approx(-1.0)
