"""Element symbols and standard atomic masses for every atomic number the model accepts (1 <= z < 100).

The reference takes its masses from ASE (``Atoms.get_masses()``, i.e. ``ase.data.atomic_masses``, which in ASE 3.22 is
the IUPAC 2016 table of standard atomic weights, with the mass of the longest-lived isotope for elements that have no
standard weight).  ASE is not a dependency here, so the table below restates those values from memory: it is not pinned
against ASE by any test.  Only the five values the protein runs use (H, C, N, O, S) are checked, and they equal the
values this project used before the table existed, bit for bit.
"""
from __future__ import annotations

import numpy as np

# index z -> symbol; index 0 is the placeholder "X", as in ase.data.chemical_symbols
SYMBOLS = (
    "X",
    "H", "He",
    "Li", "Be", "B", "C", "N", "O", "F", "Ne",
    "Na", "Mg", "Al", "Si", "P", "S", "Cl", "Ar",
    "K", "Ca", "Sc", "Ti", "V", "Cr", "Mn", "Fe", "Co", "Ni", "Cu", "Zn", "Ga", "Ge", "As", "Se", "Br", "Kr",
    "Rb", "Sr", "Y", "Zr", "Nb", "Mo", "Tc", "Ru", "Rh", "Pd", "Ag", "Cd", "In", "Sn", "Sb", "Te", "I", "Xe",
    "Cs", "Ba", "La", "Ce", "Pr", "Nd", "Pm", "Sm", "Eu", "Gd", "Tb", "Dy", "Ho", "Er", "Tm", "Yb", "Lu",
    "Hf", "Ta", "W", "Re", "Os", "Ir", "Pt", "Au", "Hg", "Tl", "Pb", "Bi", "Po", "At", "Rn",
    "Fr", "Ra", "Ac", "Th", "Pa", "U", "Np", "Pu", "Am", "Cm", "Bk", "Cf", "Es",
)

# index z -> mass in amu (IUPAC 2016 standard atomic weights, abridged where IUPAC gives an interval; radioactive
# elements without a standard weight: the longest-lived isotope)
_MASS = (
    None,
    1.008, 4.002602,
    6.94, 9.0121831, 10.81, 12.011, 14.007, 15.999, 18.998403163, 20.1797,
    22.98976928, 24.305, 26.9815385, 28.085, 30.973761998, 32.06, 35.45, 39.948,
    39.0983, 40.078, 44.955908, 47.867, 50.9415, 51.9961, 54.938044, 55.845, 58.933194, 58.6934, 63.546, 65.38,
    69.723, 72.630, 74.921595, 78.971, 79.904, 83.798,
    85.4678, 87.62, 88.90584, 91.224, 92.90637, 95.95, 97.90721, 101.07, 102.90550, 106.42, 107.8682, 112.414,
    114.818, 118.710, 121.760, 127.60, 126.90447, 131.293,
    132.90545196, 137.327, 138.90547, 140.116, 140.90766, 144.242, 144.91276, 150.36, 151.964, 157.25, 158.92535,
    162.500, 164.93033, 167.259, 168.93422, 173.054, 174.9668,
    178.49, 180.94788, 183.84, 186.207, 190.23, 192.217, 195.084, 196.966569, 200.592, 204.38, 207.2, 208.98040,
    208.98243, 209.98715, 222.01758,
    223.01974, 226.02541, 227.02775, 232.0377, 231.03588, 238.02891, 237.04817, 244.06421, 243.06138, 247.07035,
    247.07031, 251.07959, 252.0830,
)

MAX_Z = 99                      # the model's atom embedding has 100 rows (z < 100)
assert len(SYMBOLS) == len(_MASS) == MAX_Z + 1

MASSES = {z: _MASS[z] for z in range(1, MAX_Z + 1)}
Z_OF = {s: z for z, s in enumerate(SYMBOLS) if z}


def masses_of(numbers) -> np.ndarray:
    """float64 masses [n] of the atomic numbers ``numbers``; ValueError for a number outside 1..99."""
    z = np.asarray(numbers).reshape(-1)
    bad = [int(x) for x in z if int(x) not in MASSES]
    if bad:
        raise ValueError(f"no mass for atomic number(s) {sorted(set(bad))}: the model accepts 1 <= z <= {MAX_Z}")
    return np.array([MASSES[int(x)] for x in z], dtype=np.float64)


def atomic_number(symbol: str) -> int:
    """Atomic number of an element symbol (case as in a PDB element column: "C", "CL" or "Cl"); ValueError if unknown."""
    s = symbol.strip()
    z = Z_OF.get(s[:1].upper() + s[1:].lower())
    if z is None:
        raise ValueError(f"unknown element symbol {symbol!r}")
    return z
