"""The kernels of the device MD step (csrc/k_md.cuh, k_caph.cuh, k_nonbonded.cuh, k_comm.cuh) against fp64 host
restatements, at the sizes where their loops wrap: every kernel here is one CTA (or a warp per atom) whose loops run a
second pass only beyond Chignolin's 175 protein atoms / 35 cap hydrogens.

A. Integrator phases, fp64 against fp64, no ViSNet in the loop.  A bare MD handle (Chignolin's fragment topology, an empty
   protein map, so the evaluation writes exactly 0 to ef) at P protein atoms; the test writes the forces into ef and
   compares kick1 / kick2 with md.Langevin.first_half / second_half at P = 1, 175, 341, 342, 343 (kick1's second pass
   starts at 3P > 1023), 1024, 1025 (kick2's momentum loop wraps) and 14000, at friction 0 and 0.01/fs, Philox and
   pool normals, start steps 0, 5 and 2^32 + 3, a seed with a non-zero high word, with and without restraints.
   The only differences are the centre-of-mass summation order, sincospi against cos(2 pi u) and FMA contraction.
B. Placement (vb_debug_read "pos") for the four example proteins, and the restraint CTA at P = 255, 256, 257, 571, 746,
   5000 and behind fragment batches of 512 and 513 atoms (its block index on both sides of a multiple of 256).
C. Non-bonded term, both instances: <float> at ww / abd against the oracle and at ~5000 atoms against a vectorised fp64
   restatement (rows in chunks), shard slices with lo > 0 and hi - lo not a multiple of 8; <double> inside md_eval.
D. Cap-hydrogen LBFGS with 3 n_h > 1024: K replicas of a protein's problem in one packed batch.
E. Trajectories at real sizes: ww / abd with restraints and the non-bonded term, trpcage with the hydrogen refinement, the
   512-fragment batch with an identity protein map.
F. The peer-memory all-reduce with world = 1: standalone calls at every grid-stride boundary, and inside the step graph.

Measured on one H100 80GB HBM3 at a 400 W power limit (the whole file: ~26 s of test time):
   A  |dx| 2.1e-13 A and |dv| 3.4e-12 max|v0|, both at P = 14000 (bars PX_TOL, PV_REL: ~10x); step and history exact.
   B  placement 0 ulp (bit-equal, caps included); restraints 5.1e-16 relative (bar 1e-12).
   C  <float> |dF| 0.031 and |dE| 0.0076 of their bars (worst of ww / abd / synthetic); <double> |dF| 0.021, |dE| 0.004.
   D  reference tolerances: bit-equal (chig x12 and trpcage x5), evaluation counts equal; tightened: 1.1e-5 A (chig x12)
      and 9.5e-6 A (trpcage x5) against 5e-4, ten evaluations each.  With the LBFGS dot products cut to their first pass
      the tightened cases miss by 1.3e-3 and 6.9e-4 A.
   E  |dx| up to 2.6e-6 (ww), 2.0e-6 (abd), 1.9e-6 (trpcage + refinement), 3.4e-7 (512 fragments) against X_TOL, over
      two runs.
   F  bit-exact; every size meets both window parities; comm_seq advances by one per replay of the step graph.
"""
import dataclasses

import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.fragment_data import FragmentData
from ai2bmd_b200.md import FS, KB, MASSES, BondedForceField, DeviceLangevin, Langevin, philox_normals
from ai2bmd_b200.nonbonded import MMNonBondedCalculator, dipeptide_atom_sets, exclusion_table, synthetic_parameters
from ai2bmd_b200.pdbfrag import FragmentRecipe, ProteinMap
from ai2bmd_b200.restraints import KCALMOL_EV, hydrogen_bond_springs
from ai2bmd_b200.synth import synthetic_batch
from oracle import nonbonded_ref as R
from oracle.caph_c import relax_problem
from oracle.hookean_ref import hookean, hookean_terms

gpu = pytest.mark.gpu

# as tests/test_md_gpu.py: fp32 force rounding amplified by the dynamics
X_TOL, V_TOL = 2e-5, 2e-4
# phases fed identical inputs (A)
PX_TOL, PV_REL = 2e-12, 3e-11
RTOL = 1e-12
SEED = (0xA5A5A5A5 << 32) | 0x1234567
KT = 300.0 * KB


def _measured(what, value):
    print(f"measured {what}: {value:.3e}")


def _lattice(n, rng, spacing=1.5, jitter=0.2):
    """n points of a cubic lattice with jitter: no two closer than spacing - 2 sqrt(3) jitter."""
    side = int(np.ceil(n ** (1 / 3)))
    g = np.stack(np.meshgrid(*(np.arange(side),) * 3, indexing="ij"), -1).reshape(-1, 3)[:n]
    return g * spacing + rng.uniform(-jitter, jitter, size=(n, 3))


def _masses(n, rng):
    z = rng.choice([1, 6, 7, 8, 16], size=n, p=[0.5, 0.3, 0.08, 0.1, 0.02])
    return z, np.array([MASSES[int(a)] for a in z])


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bare(real_weights, P, fd=None):
    """Engine with a fragment topology and an empty protein map of P atoms: the evaluation writes 0 to ef."""
    fd = load_fragments("chig")[0] if fd is None else fd
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    eng.set_protein_map(P, [], [], [], np.zeros(len(fd), np.float32))
    eng.forward_host(np.asarray(fd.pos, dtype=np.float32))
    ef = torch.zeros(3 * P + 1, dtype=torch.float32, device="cuda")
    return eng, ef, len(fd.z)


def _md_setup(eng, ef, n_frag_atoms, masses, fr, seed=SEED):
    P = len(masses)
    n = n_frag_atoms
    zero = np.zeros(n, np.int32)
    eng.md_setup(masses, np.arange(n) % P, zero, zero, np.zeros(n, np.float32), FS, KT, fr / FS, seed, ef.data_ptr())


# ---- A. integrator phases -----------------------------------------------------------------------------------------
def _phases(eng, ef, z, m, fr, start, pool, restrain, rng, worst):
    P = len(m)
    x0 = _lattice(P, rng)
    v0 = rng.normal(size=(P, 3)) * np.sqrt(KT / m)[:, None] + 0.01           # net momentum: the COM terms are not zero
    eng.md_set_state(x0, v0, start)
    rf = np.zeros(3 * P + 1)
    if restrain:
        ns = min(2000, P * (P - 1) // 2)
        ij = np.array([rng.choice(P, 2, replace=False) for _ in range(ns)], dtype=np.int32).reshape(-1, 2)
        eng.md_set_restraints(np.arange(P), 0.3, ij, np.full(ns, 0.05), np.zeros(ns))
        rf = eng.md_restraint_forces()
        assert P == 1 or np.abs(rf[:-1]).max() > 0
    if fr == 0:
        xi = eta = 0.0
    elif pool is not None:
        xi, eta = pool[start % len(pool)]
    else:
        xi, eta = (a.reshape(P, 3) for a in philox_normals(SEED, start, 3 * P))
    f1 = (rng.normal(size=3 * P + 1)).astype(np.float32)
    ef.copy_(torch.from_numpy(f1))
    # the kicks use ef + rf, summed in fp64 in that order
    f1_64 = f1[:-1].reshape(P, 3).astype(np.float64) + rf[:-1].reshape(P, 3)
    host = Langevin(x0, z, lambda x: (0.0, f1_64), dt_fs=1.0, temperature_K=300.0, friction_per_fs=fr)
    host.v = v0.copy()
    eng.md_kick1(_stream())
    x, v, step, _ = eng.md_get_state()
    host.first_half(xi, eta)
    vscale = np.abs(v0).max()             # (at P = 1 with friction the COM removal leaves v = 0)
    dx, dv = np.abs(x - host.x).max(), np.abs(v - host.v).max() / vscale
    assert step == start and dx <= PX_TOL and dv <= PV_REL, (dx, dv)
    if fr > 0:                           # the centre of mass stays where it was
        com = lambda p: (m[:, None] * p).sum(0) / m.sum()      # noqa: E731
        assert np.abs(com(x) - com(x0)).max() <= PX_TOL
    f2 = (rng.normal(size=3 * P + 1)).astype(np.float32)
    ef.copy_(torch.from_numpy(f2))
    host.f = f2[:-1].reshape(P, 3).astype(np.float64) + rf[:-1].reshape(P, 3)
    eng.md_kick2(_stream())
    _, v, step, hist = eng.md_get_state(n_hist=1)
    host.second_half(xi, eta)
    dv2 = np.abs(v - host.v).max() / vscale
    assert dv2 <= PV_REL, dv2
    assert step == start + 1 and hist[0] == float(f2[-1]) + rf[-1]
    if restrain:
        eng.md_set_restraints()
    worst["x"], worst["v"] = max(worst["x"], dx), max(worst["v"], dv, dv2)


@gpu
@pytest.mark.parametrize("P", [1, 175, 341, 342, 343, 1024, 1025, 14000])
def test_kick_phases_equal_the_host_halves(real_weights, P):
    rng = np.random.default_rng(P)
    z, m = _masses(P, rng)
    eng, ef, n = _bare(real_weights, P)
    pool = np.stack([np.stack([rng.normal(size=(P, 3)), rng.normal(size=(P, 3))]) for _ in range(3)])
    worst = {"x": 0.0, "v": 0.0}
    for fr in (0.0, 0.01):
        _md_setup(eng, ef, n, m, fr)
        for use_pool in (False, True):
            dev_pool = None
            if use_pool:
                dev_pool = torch.as_tensor(pool.reshape(3, 2, 3 * P)).cuda()
                eng.md_set_normals(dev_pool.data_ptr(), 3)
            for start in (0, 5, 2 ** 32 + 3):
                _phases(eng, ef, z, m, fr, start, pool if use_pool else None, False, rng, worst)
            if use_pool:
                eng.md_set_normals(0, 0)
        _phases(eng, ef, z, m, fr, 2 ** 32 + 3, None, True, rng, worst)
    _measured(f"A P={P} |dx|", worst["x"])
    _measured(f"A P={P} |dv|/max|v|", worst["v"])


def test_langevin_halves_compose_to_the_step():
    """CPU: step() is normals + first_half + force + second_half, and friction 0 draws no random numbers."""
    rng = np.random.default_rng(0)
    z, m = _masses(50, rng)
    f = rng.normal(size=(50, 3))
    x0 = _lattice(50, rng)
    a = Langevin(x0, z, lambda x: (1.0, f * np.cos(x)), friction_per_fs=0.01, seed=4)
    b = Langevin(x0, z, lambda x: (1.0, f * np.cos(x)), friction_per_fs=0.01, seed=4)
    for _ in range(3):
        a.step()
        xi, eta = b.normals()
        b.first_half(xi, eta)
        b.energy, b.f = b.force_fn(b.x)
        b.second_half(xi, eta)
    assert np.array_equal(a.x, b.x) and np.array_equal(a.v, b.v) and a.nsteps == b.nsteps == 3


# ---- B. placement and the restraint CTA ---------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", ["chig", "trpcage", "ww", "abd"])
def test_placement_equals_the_recipe(real_weights, name):
    fd, pm = load_fragments(name)
    prot_pos, prot_z, recipe = load_protein(name)
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
    eng.forward_host(np.asarray(fd.pos, dtype=np.float32))
    ef = torch.zeros(3 * pm.n_protein + 1, dtype=torch.float32, device="cuda")
    masses = np.array([MASSES[int(a)] for a in prot_z])
    eng.md_setup(masses, recipe.real, recipe.acc, recipe.rem, recipe.blen, FS, KT, 0.0, 0, ef.data_ptr())
    x = prot_pos + np.random.default_rng(1).normal(scale=0.05, size=prot_pos.shape)
    eng.md_set_state(x, np.zeros_like(x), 0)
    eng.md_eval(_stream())
    pos = eng.debug_read("pos", 0, (len(fd.z), 3))
    ref = recipe.positions(x)
    real = recipe.real >= 0
    assert np.array_equal(pos[real], ref[real])                             # real atoms: a copy
    assert (np.abs(pos - ref) <= np.spacing(np.abs(ref))).all()             # cap hydrogens: within 1 ulp
    _measured(f"B {name} cap |dpos| ulps", float((np.abs(pos - ref) / np.spacing(np.abs(ref))).max()))


def _restraint_case(eng, P, x0, springs, rng):
    atoms = np.arange(P)
    eng.md_set_state(x0, np.zeros_like(x0), 0)
    ij, k, rt = springs
    eng.md_set_restraints(atoms, 0.2, ij, k, rt)
    x1 = x0 + rng.normal(scale=0.1, size=x0.shape)
    eng.md_set_state(x1, np.zeros_like(x1), 0)
    eng.md_eval(_stream())
    rf = eng.md_restraint_forces()
    e, f = hookean(x1, hookean_terms(atoms, x0, 0.2, springs))
    err = np.abs(rf[:-1] - f.reshape(-1)).max() / np.abs(f).max()
    assert err <= RTOL and abs(rf[-1] - e) <= RTOL * e
    assert np.count_nonzero(np.abs(rf[:-1].reshape(-1, 3)).sum(1)) == P
    return err


def _random_springs(P, rng, n):
    ij = np.array([rng.choice(P, 2, replace=False) for _ in range(n)], dtype=np.int32)
    return ij, rng.uniform(0.1, 1.0, n), rng.uniform(0.0, 1.0, n)


@gpu
@pytest.mark.parametrize("P", [255, 256, 257, 571, 746, 5000])
def test_restraint_cta_at_size(real_weights, P):
    rng = np.random.default_rng(P)
    _, m = _masses(P, rng)
    eng, ef, n = _bare(real_weights, P)
    _md_setup(eng, ef, n, m, 0.0)
    if P in (571, 746):                  # ww, abd: the reference's hydrogen bond springs
        name = "ww" if P == 571 else "abd"
        x0 = load_protein(name)[0].astype(np.float64)
        assert len(x0) == P
        springs = hydrogen_bond_springs(load_capped_protein(name))
        ij, k, _ = springs
        springs = (ij, k, np.linalg.norm(x0[ij[:, 1]] - x0[ij[:, 0]], axis=1) - 0.05)
    else:
        x0 = _lattice(P, rng)
        springs = _random_springs(P, rng, P // 2)
    _measured(f"B restraints P={P} rel", _restraint_case(eng, P, x0, springs, rng))


def _cut_batch(n_atoms):
    """A synthetic fragment batch of exactly n_atoms: the last fragment cut short."""
    fd = synthetic_batch(40, seed=5)
    assert len(fd.z) > n_atoms
    G = int(fd.batch[n_atoms - 1]) + 1
    start = np.asarray(fd.start[:G])
    end = np.minimum(np.asarray(fd.end[:G]), n_atoms)
    return FragmentData(fd.z[:n_atoms], fd.pos[:n_atoms], start, end, fd.batch[:n_atoms])


@gpu
@pytest.mark.parametrize("N", [512, 513])
def test_restraint_cta_behind_fragment_batches(real_weights, N):
    """The restraint CTA is block N/256 rounded up: block 2 for 512 fragment atoms, 3 for 513.  Placement and
    restraints both checked."""
    P = 300
    rng = np.random.default_rng(N)
    _, m = _masses(P, rng)
    fd = _cut_batch(N)
    eng, ef, n = _bare(real_weights, P, fd)
    assert n == N
    _md_setup(eng, ef, n, m, 0.0)
    x0 = _lattice(P, rng)
    _restraint_case(eng, P, x0, _random_springs(P, rng, 200), rng)
    x, _, _, _ = eng.md_get_state()
    assert np.array_equal(eng.debug_read("pos", 0, (N, 3)), x[np.arange(N) % P].astype(np.float32))


# ---- C. non-bonded term -------------------------------------------------------------------------------------------
def nonbonded_np(pos, q, sg, ep, rowptr, col, lo=0, hi=None, chunk=256):
    """fp64 numpy restatement of nonbonded.py:34-63 for the destination rows [lo, hi): all sources j != i outside the
    exclusion table, rows processed in chunks.  Returns (E [eV] of those rows, halved; F [n,3] eV/A, zero elsewhere)."""
    pos = np.asarray(pos, dtype=np.float64)
    q, sg, ep = (np.asarray(a, dtype=np.float64) for a in (q, sg, ep))
    n = len(pos)
    hi = n if hi is None else hi
    k = 1 / (4 * R.pi * R._eps0) * 10e6 * R.mol * R.C ** (-2)
    f = np.zeros((n, 3))
    e = 0.0
    for a in range(lo, hi, chunk):
        b = min(hi, a + chunk)
        rows = np.arange(a, b)
        vec = pos[rows, None, :] - pos[None, :, :]
        keep = np.ones((b - a, n), dtype=bool)
        keep[rows - a, rows] = False
        for r in rows:
            keep[r - a, col[rowptr[r]:rowptr[r + 1]]] = False
        d2 = np.where(keep, (vec * vec).sum(-1), 1.0)
        d = np.sqrt(d2)
        sij = 0.5 * (sg[None, :] + sg[rows, None]) * R.nm
        eij = np.sqrt(ep[None, :] * ep[rows, None])
        c6 = (sij ** 2 / d2) ** 3
        c12 = c6 ** 2
        e_lj = 4 * eij * (c12 - c6)
        e_c = k * q[None, :] * q[rows, None] / d
        fmag = np.where(keep, 24 * eij * (2 * c12 - c6) / d2 + e_c / d2, 0.0)
        f[rows] = (fmag[..., None] * vec).sum(1)
        e += float(np.where(keep, e_lj + e_c, 0.0).sum())
    return e * (R.kJ / R.mol) / 2, f * (R.kJ / R.mol)


def test_vectorised_nonbonded_reference_equals_the_oracle():
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    n = len(prot_z)
    groups = dipeptide_atom_sets(fd, recipe, pm)
    rowptr, col = exclusion_table(n, groups)
    q, sg, ep = synthetic_parameters(prot_z, seed=2)
    src, dst = R.pair_list(n, R.exclude_pairs_from_groups(groups))
    e64, f64 = R.nonbonded(prot_pos, q, sg, ep, src, dst, torch.float64)
    e, f = nonbonded_np(prot_pos, q, sg, ep, rowptr, col, chunk=37)
    assert abs(e - e64) <= 1e-11 * abs(e64) and np.abs(f - f64).max() <= 1e-11 * np.abs(f64).max()
    es, fs = nonbonded_np(prot_pos, q, sg, ep, rowptr, col, lo=13, hi=101, chunk=16)
    assert np.array_equal(fs[13:101], f[13:101]) and not fs[:13].any() and not fs[101:].any()
    own = (dst >= 13) & (dst < 101)                                 # the oracle over the pairs whose destination is owned
    es64, _ = R.nonbonded(prot_pos, q, sg, ep, src[own], dst[own], torch.float64)
    assert abs(es - es64) <= 1e-11 * abs(es64)


def _nb_problem(name):
    fd, pm = load_fragments(name)
    prot_pos, prot_z, recipe = load_protein(name)
    groups = dipeptide_atom_sets(fd, recipe, pm)
    q, sg, ep = synthetic_parameters(prot_z, seed=2)
    return prot_pos, q, sg, ep, exclusion_table(len(prot_z), groups)


def _synthetic_protein(n_atoms=5000):
    """Synthetic-batch fragments translated onto a cubic grid (each fragment one exclusion group): the grid spacing
    is the smallest whole number of A that keeps every non-excluded pair at least 1 A apart."""
    fd = synthetic_batch(200, seed=7)
    G = int(np.searchsorted(np.asarray(fd.end), n_atoms)) + 1
    z, pos, batch = fd.z[:fd.end[G - 1]], fd.pos[:fd.end[G - 1]].astype(np.float64), fd.batch[:fd.end[G - 1]]
    side = int(np.ceil(G ** (1 / 3)))
    cell = np.stack(np.meshgrid(*(np.arange(side),) * 3, indexing="ij"), -1).reshape(-1, 3)[:G]
    groups = [np.arange(fd.start[g], fd.end[g]) for g in range(G)]
    for spacing in range(8, 30):
        p = pos + cell[batch] * spacing
        p32 = p.astype(np.float32).astype(np.float64)
        ok = True
        for a in range(0, len(p), 512):
            d2 = ((p32[a:a + 512, None] - p32[None]) ** 2).sum(-1)
            d2[batch[a:a + 512, None] == batch[None]] = np.inf
            if d2.min() < 1.0:
                ok = False
                break
        if ok:
            return p, z, groups
    raise AssertionError("no grid spacing separates the fragments")


def _nb_bars(e, f, e64, f64):
    ftol = 2e-5 * np.abs(f64).max() + 1e-6
    df, de = np.abs(f - f64).max(), abs(e - e64)
    assert df <= ftol and de <= 2e-5 * abs(e64) + 1e-4, (df, ftol, de)
    return df / ftol, de / (2e-5 * abs(e64) + 1e-4)


@gpu
@pytest.mark.parametrize("name", ["ww", "abd", "synthetic5000"])
def test_nonbonded_float_at_size(real_weights, name):
    if name == "synthetic5000":
        prot_pos, z, groups = _synthetic_protein()
        q, sg, ep = synthetic_parameters(z, seed=2)
        rowptr, col = exclusion_table(len(z), groups)
    else:
        prot_pos, q, sg, ep, (rowptr, col) = _nb_problem(name)
    n = len(q)
    p32 = prot_pos.astype(np.float32)
    e64, f64 = nonbonded_np(p32, q, sg, ep, rowptr, col)
    if name != "synthetic5000":                   # the oracle's own pair list as well
        groups = [col[rowptr[i]:rowptr[i + 1]] for i in range(n)]
        ex = {(i, int(j)) for i in range(n) for j in groups[i]}
        src, dst = R.pair_list(n, ex)
        eo, fo = R.nonbonded(p32, q, sg, ep, src, dst, torch.float64)
        assert abs(eo - e64) <= 1e-11 * abs(eo) and np.abs(fo - f64).max() <= 1e-11 * np.abs(fo).max()
    calc = MMNonBondedCalculator(Engine(real_weights, 0))
    calc.set_parameters(q, sg, ep, rowptr, col)
    e, f = calc(prot_pos)
    rf_, re_ = _nb_bars(e, f, e64, f64)
    _measured(f"C float {name} |dF|/bar", rf_)
    _measured(f"C float {name} |dE|/bar", re_)
    # shard slices: lo > 0, hi - lo not a multiple of 8; the owned rows are the whole evaluation's rows
    for lo, hi in ((37, 37 + 203), (n // 2 + 5, n)):
        calc.set_parameters(q, sg, ep, rowptr, col, lo, hi)
        es, fs = calc(prot_pos)
        assert np.array_equal(fs[lo:hi], f[lo:hi]) and not fs[:lo].any() and not fs[hi:].any()
        e64s, _ = nonbonded_np(p32, q, sg, ep, rowptr, col, lo, hi)
        assert abs(es - e64s) <= 2e-5 * abs(e64) + 1e-4


@gpu
@pytest.mark.parametrize("name", ["ww", "abd"])
def test_nonbonded_double_inside_md_eval(real_weights, name):
    """With the bare handle the whole-protein buffer after md_eval is the non-bonded term at the fp64 positions."""
    prot_pos, q, sg, ep, (rowptr, col) = _nb_problem(name)
    n = len(q)
    rng = np.random.default_rng(3)
    _, m = _masses(n, rng)
    eng, ef, nf = _bare(real_weights, n)
    _md_setup(eng, ef, nf, m, 0.0)
    eng.set_nonbonded(q, sg, ep, rowptr, col)
    x = prot_pos + rng.normal(scale=0.02, size=prot_pos.shape)
    eng.md_set_state(x, np.zeros_like(x), 0)
    eng.md_eval(_stream())
    out = ef.cpu().numpy()
    e64, f64 = nonbonded_np(x.astype(np.float32), q, sg, ep, rowptr, col)
    rf_, re_ = _nb_bars(float(out[-1]), out[:-1].reshape(-1, 3), e64, f64)
    _measured(f"C double {name} |dF|/bar", rf_)
    _measured(f"C double {name} |dE|/bar", re_)


# ---- D. cap-hydrogen LBFGS beyond one pass ------------------------------------------------------------------------
def _problem(name):
    fd, pm = load_fragments(name)
    _, _, recipe = load_protein(name)
    tables, _ = load_caph_tables(name)
    return fd, caph.build_problem(load_capped_protein(name), fd, recipe, tables)


def tile_problem(pr, N, K):
    """K replicas of a cap-hydrogen problem over N packed atoms in one batch of K N atoms (indices offset by replica N)."""
    def cat(a, off):
        a = np.asarray(a)
        return np.concatenate([a + k * N * off for k in range(K)]).astype(a.dtype)
    fields = {}
    for f in dataclasses.fields(pr):
        v = getattr(pr, f.name)
        if f.name == "table_to_frag":
            fields[f.name] = [np.asarray(t) + k * N for k in range(K) for t in v]
        elif isinstance(v, np.ndarray):
            idx = f.name in ("h_idx", "mirror_dst", "mirror_src") or f.name.endswith(("_ij", "_ijk", "_ijkl"))
            fields[f.name] = cat(v, 1 if idx else 0)
    return dataclasses.replace(pr, **fields)


def test_one_replica_tiling_is_the_problem():
    fd, pr = _problem("chig")
    t = tile_problem(pr, len(fd.z), 1)
    for f in dataclasses.fields(pr):
        a, b = getattr(pr, f.name), getattr(t, f.name)
        if f.name == "table_to_frag":
            assert all(np.array_equal(x, y) for x, y in zip(a, b)) and len(a) == len(b)
        elif isinstance(a, np.ndarray):
            assert a.dtype == b.dtype and np.array_equal(a, b), f.name
        else:
            assert a == b, f.name
    t3 = tile_problem(pr, len(fd.z), 3)
    assert len(t3.h_idx) == 3 * len(pr.h_idx) and np.array_equal(t3.bond_ij[-len(pr.bond_ij):], pr.bond_ij + 2 * len(fd.z))


@gpu
@pytest.mark.parametrize("name,K", [("chig", 12), ("trpcage", 5)])
def test_caph_relax_beyond_one_pass(real_weights, name, K):
    fd, pr = _problem(name)
    N = len(fd.z)
    t = tile_problem(pr, N, K)
    assert 3 * len(t.h_idx) > 1024
    rng = np.random.default_rng(K)
    # Replicas 40 A apart on a grid centred at the origin (the terms are indexed, so replicas never interact through
    # their geometry; the distance only keeps them apart in space).  Ten tight fp32 LBFGS steps amplify one ulp of the
    # start: the C restatement itself moves by up to 4e-5 A here (1e-3 A with the grid 100 A apart, 7e-3 A with the
    # replicas strung out to 1,100 A), so 5e-4 A is a bar with a margin of ten.
    cell = np.stack(np.meshgrid(*(np.arange(3),) * 3, indexing="ij"), -1).reshape(-1, 3)[:K].astype(np.float64)
    off = 40.0 * (cell - cell.mean(0)) - fd.pos.mean(0)
    start = np.concatenate([fd.pos + off[k] for k in range(K)]).astype(np.float32)
    start[t.h_idx] += rng.normal(scale=0.1, size=(len(t.h_idx), 3)).astype(np.float32)
    start[t.mirror_dst] = start[t.mirror_src]
    eng = Engine(real_weights, 0)
    eng.set_topology(np.tile(fd.z, K), np.concatenate([fd.batch + k * len(fd) for k in range(K)]), n_graphs=K * len(fd))
    for tight in (False, True):
        p = dataclasses.replace(t, tol_grad=1e-12, tol_change=1e-12) if tight else t
        eng.set_caph(p)
        pos = torch.from_numpy(start.copy()).cuda()
        eng.caph_relax(pos.data_ptr(), _stream())
        out = pos.cpu().numpy()
        lb = dict(tolerance_grad=1e-12, tolerance_change=1e-12) if tight else {}
        x_c, evals_c = relax_problem(p, start, **lb)
        evals = eng.get_option("caph_evals")
        dx = np.abs(out - x_c).max()
        _measured(f"D {name} K={K} tight={tight} |dx| (evals {evals} / {evals_c})", dx)
        assert evals == evals_c
        assert dx <= (5e-4 if tight else 4e-6)
        if tight:
            assert evals_c == p.max_iter and np.abs(x_c - start).max() > 5e-3        # every iteration ran
        assert np.array_equal(out[t.mirror_dst], out[t.mirror_src])


# ---- E. trajectories at real sizes --------------------------------------------------------------------------------
def _normals(seed, n):
    return lambda s: tuple(a.reshape(n, 3) for a in philox_normals(seed, s, 3 * n))


@gpu
@pytest.mark.parametrize("name", ["ww", "abd"])
def test_restrained_nonbonded_trajectory_at_size(real_weights, name):
    fd, pm = load_fragments(name)
    prot_pos, prot_z, recipe = load_protein(name)
    n = len(prot_z)
    seed, fr = 17, 0.01
    rowptr, col = exclusion_table(n, dipeptide_atom_sets(fd, recipe, pm))
    q, sg, ep = synthetic_parameters(prot_z, seed=3)
    q *= 0.25                                                   # as test_nonbonded.py: keep the toy system gentle
    ij, k, _ = hydrogen_bond_springs(load_capped_protein(name))
    springs = (ij, k, np.linalg.norm(prot_pos[ij[:, 1]] - prot_pos[ij[:, 0]], axis=1) - 0.02)
    heavy = np.flatnonzero(prot_z > 1)
    terms = hookean_terms(heavy, prot_pos, 10 * KCALMOL_EV, springs)
    ff = BondedForceField(real_weights, fd, pm, recipe)
    nb = MMNonBondedCalculator(ff.engine)
    nb.set_parameters(q, sg, ep, rowptr, col)

    def force_fn(x):
        eb, fb = ff(x)
        en, fn = nb(x)
        eh, fh = hookean(x, terms)
        return eb + en + eh, fb + fn + fh

    host = Langevin(prot_pos, prot_z, force_fn, dt_fs=1.0, friction_per_fs=fr, seed=seed, normal_source=_normals(seed, n))
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, dt_fs=1.0, friction_per_fs=fr, seed=seed,
                         velocities=host.v.copy())
    dev.engine.set_nonbonded(q, sg, ep, rowptr, col)
    dev._eval()
    dev.set_restraints(tether_atoms=heavy, tether_k_kcal=10, springs=springs)
    for _ in range(20):
        host.step()
    dev.run(20)
    x, v, step, _ = dev.state()
    dx, dv = np.abs(x - host.x).max(), np.abs(v - host.v).max()
    _measured(f"E {name} |dx|", dx)
    assert step == 20 and dx <= X_TOL and dv <= V_TOL


@gpu
def test_trpcage_md_with_refinement_matches_host_loop(real_weights):
    fd, pm = load_fragments("trpcage")
    prot_pos, prot_z, recipe = load_protein("trpcage")
    tables, _ = load_caph_tables("trpcage")
    pr = caph.build_problem(load_capped_protein("trpcage"), fd, recipe, tables)
    seed, n = 11, pm.n_protein
    ff = BondedForceField(real_weights, fd, pm, recipe, refine=lambda p: relax_problem(pr, p)[0])
    host = Langevin(prot_pos, prot_z, ff, dt_fs=1.0, friction_per_fs=0.001, seed=seed, normal_source=_normals(seed, n))
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, dt_fs=1.0, friction_per_fs=0.001, seed=seed,
                         velocities=host.v.copy(), caph=pr)
    host.run(25)
    dev.run(25)
    x, v, step, _ = dev.state()
    dx, dv = np.abs(x - host.x).max(), np.abs(v - host.v).max()
    _measured("E trpcage+caph |dx|", dx)
    assert step == 25 and dx <= X_TOL and dv <= V_TOL


@gpu
def test_512_fragment_batch_identity_map_trajectory(real_weights):
    fd = synthetic_batch(512, seed=0)
    n = len(fd.z)
    idx = np.arange(n, dtype=np.int32)
    pm = ProteinMap(n, idx, idx, np.ones(n, np.float32), np.ones(len(fd), np.float32))
    recipe = FragmentRecipe(idx, np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32))
    pos = fd.pos.astype(np.float64)
    seed = 23
    ff = BondedForceField(real_weights, fd, pm, recipe)
    host = Langevin(pos, fd.z, ff, dt_fs=1.0, friction_per_fs=0.001, seed=seed, normal_source=_normals(seed, n))
    dev = DeviceLangevin(real_weights, fd, pm, recipe, pos, fd.z, dt_fs=1.0, friction_per_fs=0.001, seed=seed,
                         velocities=host.v.copy())
    host.run(5)
    dev.run(5)
    x, v, step, _ = dev.state()
    dx, dv = np.abs(x - host.x).max(), np.abs(v - host.v).max()
    _measured(f"E 512-fragment (P = {n}) |dx|", dx)
    assert step == 5 and dx <= X_TOL and dv <= V_TOL


# ---- F. the all-reduce with world = 1 -----------------------------------------------------------------------------
COMM_SIZES = [1, 511, 512, 513, 16383, 16384, 16385, 40000]


def _comm_engine(real_weights, eng=None):
    eng = Engine(real_weights, 0) if eng is None else eng
    eng.comm_connect([eng.comm_init(0, 1, 40000)])
    return eng


def _awkward(n, rng):
    """float32 data with -0.0, denormals, infinities and extremes among ordinary values."""
    x = rng.normal(size=n).astype(np.float32)
    special = np.array([-0.0, 0.0, 1e-45, -1e-45, 1e-40, -3e-39, np.inf, -np.inf, 3.4028235e38, -3.4028235e38,
                        1.1754944e-38, 6e-8], dtype=np.float32)
    at = rng.choice(n, size=min(n, len(special)), replace=False)
    x[at] = special[:len(at)]
    return x


def _allreduce_rounds(eng, rng, rounds=2):
    """Every size three times in a row, the sizes interleaved, fresh data each call (a slot left stale by the last call
    shows); the window parity of a call is that of comm_seq + 1, and every size must meet both."""
    parities = {n: set() for n in COMM_SIZES}
    for _ in range(rounds):
        for n in COMM_SIZES:
            for _ in range(3):
                seq = eng.get_option("comm_seq")
                x = _awkward(n, rng)
                buf = torch.from_numpy(x.copy()).cuda()
                eng.comm_allreduce(buf.data_ptr(), n, _stream())
                out = buf.cpu().numpy()
                # the fixed-order sum starts at +0.0f: -0.0 comes out as +0.0, everything else unchanged
                assert np.array_equal(out.view(np.uint32), (np.float32(0) + x).view(np.uint32)), n
                assert eng.get_option("comm_seq") == seq + 1
                parities[n].add((seq + 1) & 1)
    assert all(p == {0, 1} for p in parities.values()), parities


@gpu
def test_allreduce_one_rank_is_plus_zero_plus_x(real_weights):
    eng = _comm_engine(real_weights)
    _allreduce_rounds(eng, np.random.default_rng(0))
    buf = torch.zeros(40001, dtype=torch.float32, device="cuda")
    with pytest.raises(RuntimeError, match="exceeds the window"):
        eng.comm_allreduce(buf.data_ptr(), 40001, _stream())
    assert eng.get_option("comm_timeouts") == 0


@gpu
def test_allreduce_inside_the_step_graph(real_weights):
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    seed, n = 29, pm.n_protein
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
    eng.forward_host(np.asarray(fd.pos, dtype=np.float32))
    eng.set_option("calibrate", 1)
    _comm_engine(real_weights, eng)
    assert eng.get_option("comm_ready") == 1 and eng.get_option("comm_auto") == 1
    ff = BondedForceField(real_weights, fd, pm, recipe)
    host = Langevin(prot_pos, prot_z, ff, dt_fs=1.0, friction_per_fs=0.001, seed=seed, normal_source=_normals(seed, n))
    dev = DeviceLangevin(None, fd, pm, recipe, prot_pos, prot_z, dt_fs=1.0, friction_per_fs=0.001, seed=seed,
                         velocities=host.v.copy(), engine=eng)
    seq = eng.get_option("comm_seq")
    assert seq == 1                                              # the evaluation at the start
    host.run(30)
    dev.run(30)                                                  # one graph replay per step, the all-reduce inside
    x, v, step, _ = dev.state()
    assert step == 30 and np.abs(x - host.x).max() <= X_TOL and np.abs(v - host.v).max() <= V_TOL
    assert eng.get_option("comm_seq") == seq + 30                # ... one all-reduce per replay
    _allreduce_rounds(eng, np.random.default_rng(1), rounds=2)      # the sequence number carried across the replays
    assert eng.get_option("comm_timeouts") == 0
