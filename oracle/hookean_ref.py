"""fp64 numpy restatement of ASE's ``Hookean`` constraint (ASE 3.22 ``ase/constraints.py``, recalled: ASE is not in the
image) -- the checker of the device restraint evaluation (``ai2bmd_b200/csrc/k_md.cuh`` ``md_restraint_cta``).

Two of its types are used by the reference (``src/AIMD/simulator.py:139-180``):

* ``("point", a, p0, k, rt)``: d = p0 - x[a];
* ``("two atoms", i, j, k, rt)``: d = x[j] - x[i].

With L = |d|, a term with L > rt adds k (L - rt) d / L to the force on a (on i; the opposite to j) and k (L - rt)^2 / 2
to the energy (``adjust_forces`` / ``adjust_potential_energy``).  No minimum image (the reference's cell is far larger than
any displacement a restraint sees).  Terms are applied in list order, each atom's force summed in that order.
"""
from __future__ import annotations

import numpy as np


def hookean_terms(tether_atoms=(), anchors=None, tether_k=0.0, springs=None):
    """Term list: tethers of ``tether_atoms`` to ``anchors[n_atoms_total, 3]`` (rows picked by atom) with ``tether_k`` and
    rt = 0, then ``springs = (ij [n,2], k [n], rt [n])`` in order."""
    terms = [("point", int(a), np.array(anchors[int(a)], dtype=np.float64), float(tether_k), 0.0) for a in tether_atoms]
    if springs is not None:
        ij, k, rt = springs
        terms += [("two atoms", int(i), int(j), float(kk), float(r)) for (i, j), kk, r in zip(np.asarray(ij), k, rt)]
    return terms


def hookean(x, terms):
    """(E [eV], F [n, 3] eV/A) of the terms at positions ``x [n, 3]``."""
    x = np.asarray(x, dtype=np.float64)
    f = np.zeros_like(x)
    e = 0.0
    for kind, a, b, k, rt in terms:
        d = (b - x[a]) if kind == "point" else (x[b] - x[a])
        L = float(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]))
        if L > rt:
            g = d / L * (k * (L - rt))
            f[a] += g
            if kind != "point":
                f[b] -= g
            e += 0.5 * k * ((L - rt) * (L - rt))
    return e, f
