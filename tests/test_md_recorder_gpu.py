"""The device frame recorder (csrc/k_md.cuh MdRecorder, vb_md_set_recorder / vb_md_read_frames) and the observed run on
top of it (DeviceLangevin.run_observed): the reference's MDObserver protocol (src/utils/utils.py:114-166) -- frames every
record_per_steps steps, restrained Epot, Ekin, TemperatureRunawayError above 1.5 T0 -- with the frames and the runaway
decision made on the device."""
import os
import socket

import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.fixtures import load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.md import KB, BondedForceField, DeviceLangevin, Langevin, TemperatureRunawayError, philox_normals
from ai2bmd_b200.nonbonded import dipeptide_atom_sets, exclusion_table, synthetic_parameters
from ai2bmd_b200.restraints import hydrogen_bond_springs

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
# as tests/test_restraints_gpu.py: fp32 force rounding amplified by the dynamics; whole-protein energy is an fp32 sum
X_TOL, V_TOL, E_TOL = 2e-5, 2e-4, 2e-2


def _chig():
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    return fd, pm, prot_pos, prot_z, recipe


def _ekin(masses, v):
    return 0.5 * float((masses[:, None] * v * v).sum())


def _hot_velocities(masses, shape, temperature_K, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(shape) * np.sqrt(temperature_K * KB / masses[:, None])


def _full_step(real_weights, seed=3):
    """Chignolin with every part of the device step set: hydrogen refinement, non-bonded term, tethers and springs."""
    fd, pm, prot_pos, prot_z, recipe = _chig()
    tables, _ = load_caph_tables("chig")
    pr = caph.build_problem(load_capped_protein("chig"), fd, recipe, tables)
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, friction_per_fs=0.01, seed=seed, caph=pr)
    n = dev.n
    rowptr, col = exclusion_table(n, dipeptide_atom_sets(fd, recipe, pm))
    q, sg, ep = synthetic_parameters(prot_z, seed=3)
    dev.engine.set_nonbonded(q * 0.25, sg, ep, rowptr, col)
    dev._eval()
    ij, k, _ = hydrogen_bond_springs(load_capped_protein("chig"))
    springs = (ij, k, np.linalg.norm(prot_pos[ij[:, 1]] - prot_pos[ij[:, 0]], axis=1) - 0.02)
    dev.set_restraints(tether_atoms=np.flatnonzero(prot_z > 1), tether_k_kcal=10, springs=springs)
    return dev


@pytest.mark.parametrize("every", [1, 4])
def test_frames_are_the_state(real_weights, every):
    dev = _full_step(real_weights)
    eng = dev.engine
    eng.md_set_recorder(every, 64, 0.0)
    assert eng.get_option("md_frames") == 0 and eng.get_option("md_halt_step") == -1
    assert eng.get_option("caph_ready") == 1 and dev.engine.md_restraint_forces()[-1] != 0.0
    seen = 0
    for chunk in (every, 2 * every, 3 * every):               # every chunk ends at a record step
        dev.run(chunk)
        x, v, step, hist = dev.state(n_hist=chunk)
        nf = eng.get_option("md_frames")
        assert nf == step // every
        fr = eng.md_read_frames(0, nf)
        assert list(fr["step"]) == [every * (i + 1) for i in range(nf)]
        assert not fr["halted"].any()
        assert np.array_equal(fr["x"][-1], x) and np.array_equal(fr["v"][-1], v) and fr["step"][-1] == step
        for i in range(seen, nf):                             # the frames of this chunk against the energy history
            s = int(fr["step"][i])
            assert fr["epot"][i] == hist[s - 1 - step + chunk]
            ek = _ekin(dev.masses, fr["v"][i])
            assert abs(fr["ekin"][i] - ek) <= 1e-12 * ek
        seen = nf


def test_ring_wraps_and_refuses_frames_it_does_not_hold(real_weights):
    fd, pm, prot_pos, prot_z, recipe = _chig()
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, seed=4)
    eng = dev.engine
    eng.md_set_recorder(1, 4, 0.0)
    steps = []
    for i in range(10):                                       # 20 frames through a ring of 4
        dev.run(2)
        fr = eng.md_read_frames(2 * i, 2)
        steps += list(fr["step"])
        x, v, step, _ = dev.state()
        assert np.array_equal(fr["x"][-1], x) and np.array_equal(fr["v"][-1], v) and step == fr["step"][-1]
    assert steps == list(range(1, 21)) and eng.get_option("md_frames") == 20
    assert eng.md_read_frames(16, 4)["step"].tolist() == [17, 18, 19, 20]
    for first, n in ((15, 1), (20, 1), (18, 3), (-1, 1)):       # overwritten, not yet written, past the end, negative
        with pytest.raises(RuntimeError, match="vb_md_read_frames"):
            eng.md_read_frames(first, n)
    eng.md_set_recorder(0)
    with pytest.raises(RuntimeError, match="recorder is off"):
        eng.md_read_frames(0, 0)
    assert eng.get_option("md_frames") == 0 and eng.get_option("md_halt_step") == -1
    with pytest.raises(RuntimeError, match="vb_md_set_recorder"):
        eng.md_set_recorder(1, 0)
    with pytest.raises(RuntimeError, match="vb_md_set_recorder"):
        eng.md_set_recorder(1, 4, float("nan"))


def _host_pair(real_weights, seed, fr=0.001):
    fd, pm, prot_pos, prot_z, recipe = _chig()
    n = len(prot_z)
    ff = BondedForceField(real_weights, fd, pm, recipe)

    def src(step):
        xi, eta = philox_normals(seed, step, 3 * n)
        return xi.reshape(n, 3), eta.reshape(n, 3)

    host = Langevin(prot_pos, prot_z, ff, dt_fs=1.0, temperature_K=300.0, friction_per_fs=fr, seed=seed, normal_source=src)
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, dt_fs=1.0, temperature_K=300.0,
                         friction_per_fs=fr, seed=seed, velocities=host.v.copy())
    return host, dev


@pytest.mark.parametrize("k,use_graph,n_steps", [(1, 1, 80), (4, 1, 80), (4, 0, 24)])
def test_run_observed_keeps_its_contract(real_weights, k, use_graph, n_steps):
    """Started at step 3 (not a record step), against the host integrator driven by the device's normals."""
    host, dev = _host_pair(real_weights, seed=21)
    if not use_graph:
        dev.engine.set_option("use_graph", 0)
    dev.run(3)
    host.run(3)
    want = {}
    for _ in range(n_steps):
        e = host.step()
        if host.nsteps % k == 0:
            want[host.nsteps] = (host.x.copy(), host.v.copy(), e)
    seen = []

    def obs(step, x, v, epot, ekin):
        seen.append((step, x, v, epot, ekin))

    dev.run_observed(n_steps, k, obs)
    assert [s for s, *_ in seen] == sorted(want) == list(range(k * (3 // k + 1), 3 + n_steps + 1, k))
    for step, x, v, epot, ekin in seen:
        hx, hv, he = want[step]
        assert np.abs(x - hx).max() <= X_TOL and np.abs(v - hv).max() <= V_TOL and abs(epot - he) <= E_TOL
        assert ekin == _ekin(dev.masses, v)
    x, v, step, _ = dev.state()
    assert step == 3 + n_steps
    if step % k == 0:                                             # the last step was observed: the frame is the state
        assert np.array_equal(x, seen[-1][1]) and np.array_equal(v, seen[-1][2])
    else:                                                         # steps after the last record step still ran
        assert np.abs(x - host.x).max() <= X_TOL and np.abs(v - host.v).max() <= V_TOL
    assert dev.engine.get_option("md_frames") == 0                # the recorder is off again after the run


def test_runaway_halts_on_the_device(real_weights):
    fd, pm, prot_pos, prot_z, recipe = _chig()
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, temperature_K=300.0, seed=6)
    v_hot = _hot_velocities(dev.masses, prot_pos.shape, 1000.0, seed=6)
    dev.engine.md_set_state(prot_pos, v_hot, 0)
    dev._eval()
    seen = []
    with pytest.raises(TemperatureRunawayError) as err:
        dev.run_observed(200, 5, lambda step, x, v, epot, ekin: seen.append(step))
    eng = dev.engine
    halt, nf = eng.get_option("md_halt_step"), eng.get_option("md_frames")
    fr = eng.md_read_frames(0, nf)
    temps = 2.0 * fr["ekin"] / (3 * dev.n) / KB
    # the first record step above 1.5 T0 = 450 K, and no frame after it
    assert halt == fr["step"][-1] == 5 * nf and f"at step {halt}:" in str(err.value)
    assert temps[-1] > 450.0 and (temps[:-1] <= 450.0).all() and fr["halted"].tolist() == [0] * (nf - 1) + [1]
    assert seen == list(fr["step"][:-1])                          # the halting frame is not observed
    x, v, step, _ = dev.state()
    assert step == halt and np.array_equal(x, fr["x"][-1]) and np.array_equal(v, fr["v"][-1])
    dev.run(7)                                                    # halted: nothing moves
    x2, v2, step2, _ = dev.state()
    assert step2 == halt and np.array_equal(x2, x) and np.array_equal(v2, v) and eng.get_option("md_frames") == nf
    eng.md_set_state(x, v * 0.5, step)                            # a new state lifts the halt
    assert eng.get_option("md_halt_step") == -1
    dev._eval()
    dev.run(3)
    x3, _, step3, _ = dev.state()
    assert step3 == halt + 3 and np.abs(x3 - x).max() > 0.0


def test_restart_from_a_frame(real_weights):
    fd, pm, prot_pos, prot_z, recipe = _chig()
    k = 10
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, friction_per_fs=0.001, seed=8)
    frames = {}
    dev.run_observed(2 * k, k, lambda step, x, v, epot, ekin: frames.__setitem__(step, (x, v)))
    assert sorted(frames) == [k, 2 * k]
    x_k, v_k = frames[k]
    again = DeviceLangevin(real_weights, fd, pm, recipe, x_k, prot_z, friction_per_fs=0.001, seed=8, velocities=v_k, step=k)
    again.run(k)
    x, v, step, _ = again.state()
    x_2k, v_2k = frames[2 * k]
    assert step == 2 * k
    assert np.abs(x - x_2k).max() <= X_TOL and np.abs(v - v_2k).max() <= V_TOL
    # the random stream of steps k..2k matters: from step 0 the same start gives another trajectory
    other = DeviceLangevin(real_weights, fd, pm, recipe, x_k, prot_z, friction_per_fs=0.001, seed=8, velocities=v_k)
    other.run(k)
    assert np.abs(other.state()[1] - v_2k).max() > 10 * V_TOL


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
    eng = md.engine
    eng.md_set_recorder(2, 16, 0.0)
    md.run(12)
    fr = eng.md_read_frames(0, 6)
    blob = np.concatenate([fr["step"].astype(np.float64), fr["x"].reshape(-1), fr["v"].reshape(-1), fr["epot"], fr["ekin"]])
    # the runaway guard: a hot start, the same on every rank
    eng.md_set_state(prot_pos, _hot_velocities(md.masses, prot_pos.shape, 1000.0, seed=1), 0)
    eng.md_set_recorder(3, 8, 1.5)
    md._eval()
    md.run(12)
    halt = eng.get_option("md_halt_step")
    blob = np.concatenate([blob, [float(halt), float(md.state()[2])]])
    t = torch.from_numpy(blob).to(torch.device("cuda", rank))
    gathered = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(gathered, t)
    if rank == 0:
        np.savez(out, identical=all(bool((g == t).all()) for g in gathered), halt=halt, step=md.state()[2],
                 native=md._native_comm)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs")
def test_frames_and_halt_identical_on_all_ranks(tmp_path):
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 8)
    out = str(tmp_path / "ranks.npz")
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    r = np.load(out)
    assert bool(r["native"]) and bool(r["identical"])               # frames, halt step and state step on every rank
    halt = int(r["halt"])
    assert halt > 0 and halt % 3 == 0 and int(r["step"]) == halt
