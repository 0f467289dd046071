"""ctypes front end of oracle/caph_ref.c (fp32 C restatement of the hydrogen refinement) -- TEST INFRASTRUCTURE ONLY.

``flatten(problems)`` turns the per-dipeptide inputs of ``oracle/caph_ref.py`` into the flat arrays a device kernel will
consume: one position buffer for all dipeptides, terms with global atom indices and their own parameters."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import caph_ref as CR

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


class _Problem(C.Structure):
    _fields_ = [("n_atoms", C.c_int64), ("n_h", C.c_int64), ("h_idx", C.c_void_p),
                ("n_bonds", C.c_int64), ("bond_ij", C.c_void_p), ("bond_k", C.c_void_p), ("bond_r0", C.c_void_p),
                ("n_angles", C.c_int64), ("angle_ijk", C.c_void_p), ("angle_k", C.c_void_p), ("angle_t0", C.c_void_p),
                ("n_dih", C.c_int64), ("dih_ijkl", C.c_void_p), ("dih_k", C.c_void_p), ("dih_n", C.c_void_p), ("dih_p", C.c_void_p),
                ("n_pairs", C.c_int64), ("pair_ij", C.c_void_p), ("pair_a", C.c_void_p), ("pair_b", C.c_void_p), ("pair_qq", C.c_void_p),
                ("scnb", C.c_float), ("scee", C.c_float)]


def build(force: bool = False) -> str:
    out_dir = os.path.join(_HERE, "_build")
    so, src = os.path.join(out_dir, "libcaph_ref.so"), os.path.join(_HERE, "caph_ref.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src, "-lm"])
    return so


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        lib.caph_energy_grad.restype = C.c_float
        lib.caph_energy_grad.argtypes = [C.POINTER(_Problem), C.c_void_p, C.c_void_p]
        lib.caph_relax.restype = C.c_int
        lib.caph_relax.argtypes = [C.POINTER(_Problem), C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float]
        _lib = lib
    return _lib


def flatten(problems):
    """[(pos, table, atom_idx)] -> dict of flat arrays (positions float32 [N,3], int64 indices, float32 parameters)."""
    pos, h_idx = [], []
    acc = {k: [] for k in ("bond_ij", "bond_k", "bond_r0", "angle_ijk", "angle_k", "angle_t0", "dih_ijkl", "dih_k", "dih_n",
                           "dih_p", "pair_ij", "pair_a", "pair_b", "pair_qq")}
    off = 0
    for p, t, atom_idx in problems:
        atom_idx = np.asarray(atom_idx, dtype=np.int64)
        terms = CR.hydrogen_terms(t, atom_idx)
        b, a, d, pr, lj = terms["bonds"], terms["angles"], terms["dihedrals"], terms["pairs"], terms["lj_idx"]
        pos.append(np.asarray(p, dtype=np.float32))
        h_idx.append(atom_idx + off)
        acc["bond_ij"].append(b[:, :2] + off); acc["bond_k"].append(t["bond_force_constant"][b[:, 2]]); acc["bond_r0"].append(t["bond_equil_value"][b[:, 2]])
        acc["angle_ijk"].append(a[:, :3] + off); acc["angle_k"].append(t["angle_force_constant"][a[:, 3]]); acc["angle_t0"].append(t["angle_equil_value"][a[:, 3]])
        acc["dih_ijkl"].append(d[:, :4] + off); acc["dih_k"].append(t["dihedral_force_constant"][d[:, 4]])
        acc["dih_n"].append(t["dihedral_periodicity"][d[:, 4]]); acc["dih_p"].append(t["dihedral_phase"][d[:, 4]])
        acc["pair_ij"].append(pr + off); acc["pair_a"].append(t["lennard_jones_acoef"][lj]); acc["pair_b"].append(t["lennard_jones_bcoef"][lj])
        q = t["charge"].astype(np.float32)
        acc["pair_qq"].append(q[pr[:, 0]] * q[pr[:, 1]])
        off += len(p)
    out = {"pos": np.ascontiguousarray(np.concatenate(pos), dtype=np.float32), "h_idx": np.ascontiguousarray(np.concatenate(h_idx), dtype=np.int64)}
    for k, v in acc.items():
        arr = np.concatenate(v)
        out[k] = np.ascontiguousarray(arr, dtype=np.int64 if k.endswith(("ij", "ijk", "ijkl")) else np.float32)
    return out


def _struct(f):
    p = _Problem()
    p.n_atoms, p.n_h, p.h_idx = len(f["pos"]), len(f["h_idx"]), f["h_idx"].ctypes.data
    p.n_bonds, p.n_angles, p.n_dih, p.n_pairs = len(f["bond_k"]), len(f["angle_k"]), len(f["dih_k"]), len(f["pair_a"])
    for k in ("bond_ij", "bond_k", "bond_r0", "angle_ijk", "angle_k", "angle_t0", "dih_ijkl", "dih_k", "dih_n", "dih_p",
              "pair_ij", "pair_a", "pair_b", "pair_qq"):
        setattr(p, k, f[k].ctypes.data)
    p.scnb, p.scee = CR.SCNB, CR.SCEE
    return p


def energy_grad(f, pos=None):
    """(energy, gradient [N,3]) of the flat problem at ``pos`` (default: its own positions)."""
    x = np.ascontiguousarray(f["pos"] if pos is None else pos, dtype=np.float32)
    g = np.zeros_like(x)
    e = _load().caph_energy_grad(C.byref(_struct(f)), x.ctypes.data, g.ctypes.data)
    return float(e), g


def relax(f, max_iter=10, lr=0.1, tolerance_grad=0.1, tolerance_change=0.01):
    """Relaxed copy of the flat position buffer and the number of energy evaluations."""
    x = f["pos"].copy()
    evals = _load().caph_relax(C.byref(_struct(f)), x.ctypes.data, int(max_iter), lr, tolerance_grad, tolerance_change)
    return x, int(evals)


def relax_problem(pr, pos, **lbfgs):
    """``relax`` on the flat arrays of an :class:`ai2bmd_b200.caph.CapHProblem` at packed positions ``pos``, with the
    ACE-NME mirror copies re-applied afterwards as the device kernel does: (positions, energy evaluations)."""
    flat = {"pos": np.ascontiguousarray(pos, dtype=np.float32).copy(), "h_idx": pr.h_idx.astype(np.int64)}
    for key in ("bond_ij", "angle_ijk", "dih_ijkl", "pair_ij"):
        flat[key] = np.ascontiguousarray(getattr(pr, key), dtype=np.int64)
    for key in ("bond_k", "bond_r0", "angle_k", "angle_t0", "dih_k", "dih_n", "dih_p", "pair_a", "pair_b", "pair_qq"):
        flat[key] = np.ascontiguousarray(getattr(pr, key), dtype=np.float32)
    x, evals = relax(flat, **lbfgs)
    x[pr.mirror_dst] = x[pr.mirror_src]
    return x, evals
