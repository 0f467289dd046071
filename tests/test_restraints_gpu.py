"""Hookean restraints inside the device MD step (csrc/k_md.cuh MdRestraints, vb_md_set_restraints): the reference's
pre-equilibration tethers and hydrogen bond springs (src/AIMD/simulator.py:139-180), checked against the fp64 numpy
restatement of ASE's Hookean (oracle/hookean_ref.py) and against the host integrator driven by bonded + Hookean forces."""
import os
import socket

import numpy as np
import pytest
import torch

from ai2bmd_b200.fixtures import load_capped_protein, load_fragments, load_protein
from ai2bmd_b200.md import BondedForceField, DeviceLangevin, Langevin, philox_normals
from ai2bmd_b200.restraints import KCALMOL_EV, PREEQ_SCHEDULE, hydrogen_bond_springs
from oracle.hookean_ref import hookean, hookean_terms

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
# as tests/test_md_gpu.py: fp32 force rounding amplified by the dynamics; whole-protein energy is an fp32 sum
X_TOL, V_TOL, E_TOL = 2e-5, 2e-4, 2e-2
RTOL = 1e-12


def _chig():
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    return fd, pm, prot_pos, prot_z, recipe


def _springs():
    return hydrogen_bond_springs(load_capped_protein("chig"))


def _pulled(x, springs, which=0, by=0.5):
    """x with the hydrogen of spring `which` moved `by` A outwards along its bond (that spring is then active)."""
    ij = springs[0]
    h, p = int(ij[which, 0]), int(ij[which, 1])
    x = np.array(x, dtype=np.float64)
    d = x[h] - x[p]
    x[h] += by * d / np.linalg.norm(d)
    return x


def _assert_rf(rf, x, terms):
    e, f = hookean(x, terms)
    assert np.isfinite(rf).all()
    assert np.abs(rf[:-1] - f.reshape(-1)).max() <= RTOL * max(np.abs(f).max(), 1e-300)
    assert abs(rf[-1] - e) <= RTOL * e


def test_rf_equals_the_hookean_checker(real_weights):
    fd, pm, prot_pos, prot_z, recipe = _chig()
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, seed=2)
    atoms = np.arange(dev.n)
    dev.run(3)
    x0, v0, s0, _ = dev.state()
    dev.set_restraints(tether_atoms=atoms, tether_k_kcal=10)
    assert not dev.engine.md_restraint_forces().any()                # anchored where the atoms stand: L = 0, no NaN
    dev.run(6)                                                         # tethers after some steps
    x1, _, _, _ = dev.state()
    tk = 10 * KCALMOL_EV
    _assert_rf(dev.engine.md_restraint_forces(), x1, hookean_terms(atoms, x0, tk))
    # springs, one hydrogen pulled 0.5 A out, together with tethers to the pulled geometry (an atom with both kinds)
    springs = _springs()
    xp = _pulled(x1, springs)
    dev.engine.md_set_state(xp, v0, s0)
    dev.set_restraints(tether_atoms=atoms[::3], tether_k_kcal=1, springs=springs)
    rf_set = dev.engine.md_restraint_forces()
    terms = hookean_terms(atoms[::3], xp, 1 * KCALMOL_EV, springs)
    _assert_rf(rf_set, xp, terms)
    assert np.abs(rf_set[:-1]).max() > 0.1                             # the pulled spring pulls
    # only the springs: rt keeps every other spring slack
    dev.set_restraints(springs=springs)
    rf = dev.engine.md_restraint_forces()
    _assert_rf(rf, xp, hookean_terms(springs=springs))
    assert np.count_nonzero(np.abs(rf[:-1].reshape(-1, 3)).sum(1)) == 2
    # reproducible: the evaluation of the same state gives the same bits, at set time and in every later evaluation
    dev.set_restraints(tether_atoms=atoms[::3], tether_k_kcal=1, springs=springs)
    sp = torch.cuda.current_stream().cuda_stream
    dev.engine.md_eval(sp)
    rf_a = dev.engine.md_restraint_forces()
    dev.engine.md_eval(sp)
    rf_b = dev.engine.md_restraint_forces()
    assert np.array_equal(rf_a, rf_set) and np.array_equal(rf_a, rf_b)


def _host_pair(real_weights, fr, seed, x_start):
    """(host integrator, device integrator) from the same start; the host's force is bonded + the terms in `holder`."""
    fd, pm, prot_pos, prot_z, recipe = _chig()
    n = len(prot_z)
    ff = BondedForceField(real_weights, fd, pm, recipe)
    holder = {"terms": []}

    def force_fn(x):
        e, f = ff(x)
        eh, fh = hookean(x, holder["terms"])
        return e + eh, f + fh

    def src(step):
        xi, eta = philox_normals(seed, step, 3 * n)
        return xi.reshape(n, 3), eta.reshape(n, 3)

    host = Langevin(x_start, prot_z, force_fn, dt_fs=1.0, temperature_K=300.0, friction_per_fs=fr, seed=seed,
                    normal_source=src)
    dev = DeviceLangevin(real_weights, fd, pm, recipe, x_start, prot_z, dt_fs=1.0, temperature_K=300.0,
                         friction_per_fs=fr, seed=seed, velocities=host.v.copy())

    def host_terms(terms):            # ASE: the next get_forces() is the cached calculator result + the new constraints
        holder["terms"] = terms
        host.energy, host.f = force_fn(host.x)
    return host, dev, host_terms


@pytest.mark.parametrize("fr", [0.0, 0.01])
def test_restrained_trajectory_equals_host_integrator(real_weights, fr):
    """Every spring's rt 0.02 A below its bond length at the start: all springs pull gently, and as the bonds vibrate
    they cross rt both ways (a hydrogen pulled far out instead makes one bond so hot that fp32 force rounding alone
    drifts past X_TOL in 40 steps)."""
    _, _, x_start, _, _ = _chig()
    ij, k, _ = _springs()
    springs = (ij, k, np.linalg.norm(x_start[ij[:, 1]] - x_start[ij[:, 0]], axis=1) - 0.02)
    host, dev, host_terms = _host_pair(real_weights, fr, 7, x_start)
    atoms = np.arange(dev.n)
    dev.set_restraints(tether_atoms=atoms, tether_k_kcal=10, springs=springs)
    host_terms(hookean_terms(atoms, x_start, 10 * KCALMOL_EV, springs))
    n = 40
    host_e = [host.step() for _ in range(n)]
    dev.run(n)
    x, v, step, hist = dev.state(n_hist=n)
    assert step == n
    assert np.abs(x - host.x).max() <= X_TOL and np.abs(v - host.v).max() <= V_TOL
    assert np.abs(hist - np.asarray(host_e)).max() <= E_TOL                # restrained E_pot, as ASE prints it
    e_hook, _ = hookean(x, hookean_terms(atoms, x_start, 10 * KCALMOL_EV, springs))
    assert e_hook > 1e-3                                                   # the restraints did work


def test_preequilibration_schedule_then_springs_equals_host(real_weights):
    _, _, prot_pos, _, _ = _chig()
    seed, fr = 13, 0.001
    host, dev, host_terms = _host_pair(real_weights, fr, seed, prot_pos)
    atoms = np.arange(dev.n)
    seen = []
    dev.preequilibrate(8, record_per_steps=4, observer=lambda step, x, v, epot, ekin: seen.append((step, epot)))
    host_e = []
    for k in PREEQ_SCHEDULE:
        host_terms(hookean_terms(atoms, host.x.copy(), k * KCALMOL_EV))    # re-anchored at the start of every stage
        host_e += [host.step() for _ in range(8)]
        host_terms([])
    springs = _springs()
    dev.set_restraints(springs=springs)
    dev.run(10)
    host_terms(hookean_terms(springs=springs))
    for _ in range(10):
        host.step()
    x, v, step, _ = dev.state()
    assert step == 5 * 8 + 10
    assert np.abs(x - host.x).max() <= X_TOL and np.abs(v - host.v).max() <= V_TOL
    assert [s for s, _ in seen] == list(range(4, 41, 4))
    assert np.abs(np.array([e for _, e in seen]) - np.array(host_e)[3::4]).max() <= E_TOL


def test_restrained_energy_is_conserved(real_weights, reference_outputs):
    """friction = 0 with every atom tethered at 10 kcal/mol/A^2, dt 0.5 fs, 300 steps: restrained E_pot + E_kin stays
    within the bound of test_md_gpu.py's conservation test.  One unfragmented graph (the 22-atom dipeptide of that test),
    so the potential is exactly conservative and any drift would come from the restraint forces."""
    from ai2bmd_b200.pdbfrag import FragmentRecipe, ProteinMap, single_graph
    r = reference_outputs
    z, pos = r["c1_ala_z"], r["c1_ala_pos"].astype(np.float64)
    n = len(z)
    fd = single_graph(z, pos.astype(np.float32))
    idx = np.arange(n, dtype=np.int32)
    pm = ProteinMap(n, idx, idx, np.ones(n, np.float32), np.ones(1, np.float32))
    rec = FragmentRecipe(idx, np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32))
    dev = DeviceLangevin(real_weights, fd, pm, rec, pos, z, dt_fs=0.5, temperature_K=300.0, friction_per_fs=0.0, seed=1)
    dev.set_restraints(tether_atoms=np.arange(n), tether_k_kcal=10)
    m = dev.masses[:, None]
    e0 = dev.energy + 0.5 * float((m * dev.state()[1] ** 2).sum())       # rf = 0 at the anchors
    tot, ehook = [], 0.0
    for _ in range(30):
        dev.run(10)
        x, v, _, hist = dev.state(n_hist=10)
        tot.append(hist[-1] + 0.5 * float((m * v * v).sum()))
        ehook = max(ehook, dev.engine.md_restraint_forces()[-1])
    tot = np.asarray(tot)
    assert np.abs(tot - e0).max() < 2e-2
    assert abs(tot[-5:].mean() - tot[:5].mean()) < 1e-2
    assert ehook > 1e-3 and dev.kinetic_energy() > 0.1                     # the tethers are stretched, the system moves


def test_phases_equal_the_whole_step_with_restraints(real_weights):
    fd, pm, prot_pos, prot_z, recipe = _chig()
    springs = _springs()
    x_start = _pulled(prot_pos, springs, which=2, by=0.3)
    a = DeviceLangevin(real_weights, fd, pm, recipe, x_start, prot_z, friction_per_fs=0.002, seed=5)
    b = DeviceLangevin(real_weights, fd, pm, recipe, x_start, prot_z, friction_per_fs=0.002, seed=5)
    for d in (a, b):
        d.set_restraints(tether_atoms=np.arange(d.n), tether_k_kcal=5, springs=springs)
    a.run(8)
    sp = torch.cuda.current_stream().cuda_stream
    for _ in range(8):
        b.engine.md_kick1(sp)
        b.engine.md_eval(sp)
        b.engine.md_kick2(sp)
    xa, va, sa, ha = a.state(n_hist=8)
    xb, vb, sb, hb = b.state(n_hist=8)
    assert sa == sb == 8 and np.abs(xa - xb).max() <= X_TOL and np.abs(va - vb).max() <= V_TOL
    assert np.abs(ha - hb).max() <= E_TOL


def test_removed_restraints_leave_the_plain_step(real_weights):
    fd, pm, prot_pos, prot_z, recipe = _chig()
    a = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, seed=9)
    b = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, seed=9)
    a.set_restraints(tether_atoms=np.arange(a.n), tether_k_kcal=10, springs=_springs())
    a.run(2)
    a.engine.md_set_state(*b.state()[:2], 0)             # back to the start ...
    a.set_restraints()                                    # ... and no restraints
    a.engine.md_eval(torch.cuda.current_stream().cuda_stream)
    with pytest.raises(RuntimeError):
        a.engine.md_restraint_forces()                    # no rf buffer any more
    a.run(20)
    b.run(20)
    xa, va, sa, ha = a.state(n_hist=20)
    xb, vb, sb, hb = b.state(n_hist=20)
    assert sa == sb == 20 and np.abs(xa - xb).max() <= X_TOL and np.abs(va - vb).max() <= V_TOL
    assert np.abs(ha - hb).max() <= E_TOL


def test_set_restraints_validates_its_arguments(real_weights):
    from ai2bmd_b200.engine import Engine
    with pytest.raises(RuntimeError, match="vb_md_setup"):
        Engine(real_weights).md_set_restraints([0], 1.0)
    fd, pm, prot_pos, prot_z, recipe = _chig()
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, seed=0)
    eng, n = dev.engine, dev.n
    bad = [
        dict(tether_atoms=[n], tether_k=1.0),
        dict(tether_atoms=[-1], tether_k=1.0),
        dict(tether_atoms=[3, 4, 3], tether_k=1.0),
        dict(tether_atoms=[0], tether_k=-1.0),
        dict(tether_atoms=[0], tether_k=float("nan")),
        dict(spring_ij=[[0, n]], spring_k=[1.0], spring_rt=[1.0]),
        dict(spring_ij=[[2, 2]], spring_k=[1.0], spring_rt=[1.0]),
        dict(spring_ij=[[0, 1]], spring_k=[-1.0], spring_rt=[1.0]),
        dict(spring_ij=[[0, 1]], spring_k=[1.0], spring_rt=[-0.1]),
        dict(spring_ij=[[0, 1]], spring_k=[float("inf")], spring_rt=[1.0]),
        dict(spring_ij=[[0, 1]], spring_k=[1.0], spring_rt=[float("nan")]),
    ]
    for kw in bad:
        with pytest.raises(RuntimeError, match="vb_md_set_restraints"):
            eng.md_set_restraints(**kw)
    eng.md_set_restraints(tether_atoms=[0, 1], tether_k=0.0)             # k = 0 is allowed
    assert not eng.md_restraint_forces().any()


# ---- several GPUs -------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out):
    import torch.distributed as dist
    from ai2bmd_b200.parallel import DeviceShard
    from ai2bmd_b200.pdbfrag import FragmentRecipe
    from ai2bmd_b200.weights import load_state_dict
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    sd = load_state_dict(os.path.join(ROOT, "tests", "golden", "weights_2ef43f29.npz"))
    fd, pm, prot_pos, prot_z, recipe = _chig()
    sh = DeviceShard(sd, fd, pm, rank, world, rank, native_comm=True)
    lo, hi = sh.plan.atom_lo, sh.plan.atom_hi
    rec = FragmentRecipe(recipe.real[lo:hi], recipe.acc[lo:hi], recipe.rem[lo:hi], recipe.blen[lo:hi])
    md = DeviceLangevin(None, None, pm, rec, prot_pos, prot_z, dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.001, seed=0,
                        device=rank, group=dist.group.WORLD, engine=sh.engine)
    md.set_restraints(tether_atoms=np.arange(md.n), tether_k_kcal=10, springs=_springs())
    md.run(20)
    x, v, step, _ = md.state()
    xs = torch.from_numpy(np.concatenate([x.reshape(-1), v.reshape(-1)])).to(torch.device("cuda", rank))
    gathered = [torch.empty_like(xs) for _ in range(world)]
    dist.all_gather(gathered, xs)
    if rank == 0:
        np.savez(out, x=x, step=step, identical=all(bool((g == xs).all()) for g in gathered))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs")
def test_sharded_restrained_run_equals_one_gpu(tmp_path, real_weights):
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 8)
    out = str(tmp_path / "ranks.npz")
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    r = np.load(out)
    assert int(r["step"]) == 20 and bool(r["identical"])
    fd, pm, prot_pos, prot_z, recipe = _chig()
    one = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.001,
                         seed=0, device=0)
    one.set_restraints(tether_atoms=np.arange(one.n), tether_k_kcal=10, springs=_springs())
    one.run(20)
    assert np.abs(r["x"] - one.state()[0]).max() <= X_TOL
