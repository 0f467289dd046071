"""Host side of the reference's restraint protocol (device evaluation: ``csrc/k_md.cuh`` ``MdRestraints``).

* Pre-equilibration (``src/AIMD/simulator.py:139-166``): five stages of ``--preeq-steps`` steps each (default 2000,
  ``src/AIMD/arguments.py``) with every protein atom tethered to where it stood at the start of the stage, at
  :data:`PREEQ_SCHEDULE` kcal/mol/A^2 (ASE ``Hookean(a1=idx, a2=pos, k=restraint * kcalmol2ev, rt=0)``).
* ``--constraints`` (``simulator.py:168-180``): a spring between every hydrogen and the atom it is bonded to, for the
  production phase, from ``PDBAnalyzer.find_bonded_atoms("H")`` (``src/utils/utils.py:184-221``), restated by
  :func:`hydrogen_bond_springs`.

``md.DeviceLangevin.set_restraints`` / ``preequilibrate`` run both inside the device step.
"""
from __future__ import annotations

import numpy as np

# (units.kcal / units.mol) / units.eV of ASE 3.22 (CODATA 2014, the constants vb_set_nonbonded uses)
KCALMOL_EV = 4184.0 / (1.6021766208e-19 * 6.022140857e23)
PREEQ_SCHEDULE = (10, 5, 1, 0.5, 0.1)          # kcal/mol/A^2, simulator.py:142
HBOND_K = 15                                    # eV/A^2, utils.py:218
COVALENT_RADII = {"H": 0.31, "C": 0.76, "N": 0.71, "O": 0.66, "P": 1.07, "S": 1.05}   # A, utils.py:186-193


def hydrogen_bond_springs(protein):
    """``(ij [n,2] int32, k [n] eV/A^2, rt [n] A)`` for ``protein`` (anything with ``names`` and ``positions``, e.g. a
    :class:`ai2bmd_b200.pdbfrag.CappedProtein`), as ``find_bonded_atoms("H")`` builds them: for every atom whose name
    starts with "H", in atom order, every other atom within ``r_cov(H) + r_cov(partner) + 0.2`` A, the partner's radius
    taken from the first letter of its name (0 for an unknown letter); rt is that bound, k = 15.  Raises ``ValueError``
    when the pair count differs from the hydrogen count (the reference asserts it)."""
    names = [str(n) for n in protein.names]
    pos = np.asarray(protein.positions, dtype=np.float64)
    r_h = COVALENT_RADII["H"]
    radii = np.array([COVALENT_RADII.get(n[0], 0) for n in names], dtype=np.float64)
    hyd = [i for i, n in enumerate(names) if n.startswith("H")]
    ij, rt = [], []
    bound = (r_h + radii) + 0.2
    for i1 in hyd:
        dist = np.sqrt(((pos[i1] - pos) ** 2).sum(1))
        for i2 in np.flatnonzero(dist <= bound):
            if i2 != i1:
                ij.append((i1, int(i2)))
                rt.append(float(bound[i2]))
    if len(ij) != len(hyd):
        raise ValueError(f"hydrogen bond constraints: {len(ij)} bonded pairs for {len(hyd)} hydrogens")
    return (np.asarray(ij, dtype=np.int32).reshape(-1, 2), np.full(len(ij), float(HBOND_K)), np.asarray(rt, dtype=np.float64))
