"""The reference's un-fragmented ``--mode visnet`` on the device: the whole input is ONE ViSNet graph inside the device
MD step (``vb_md_setup`` with no placement recipe, ``DeviceLangevin.unfragmented``).

a. whole Chignolin, whole Trp-cage and a three-residue ACE-ALA-NME input (tests/golden/reference_visnet_mode.npz, the
   reference's own model source): neighbour lists bit-exact, energy and forces against the reference and the fp64 oracle.
   Energy bars: 4 ulp(E) against the reference and max(4e-3, 2 ulp) against fp64 for the 22-atom input (as for a
   fragment); for the whole proteins (|E| ~ 1.3e5 .. 2e5 eV) the relative bar 2e-6 |E| + 4e-3 that test_engine_gpu.py
   sets for larger energies.  Forces 5e-5 + 2e-5 max|F| against the fp64 hand adjoint on the VecLayerNorm(max_min)
   branch the evaluating handle took (oracle/vecln_branch.py), for the engine and for the ViSNetModel path alike.  In
   whole Chignolin atom 130 sits on an argmax tie in layer 4 (top-two channel norms 8.8e-7 apart, relative, in the fp64
   oracle): the engine takes the other channel, 2.1e-2 eV/A from the natural fp64 forces and 2.0e-5 (0.16 of the bar)
   from the fp64 forces on its own branch (measured on one H100 80GB HBM3 at 700 W).  The reference's fp32 forces took a
   branch nothing records, so against them whole Chignolin keeps only the bound of the jump, 5e-2 eV/A.
b. every launch of the G = 1 plans of whole Chignolin and whole Trp-cage against the fp64 hand adjoint on the branch the
   engine took, stage by stage (tools/stage_check.py), on a clean workspace and after a dense and a NaN decoy geometry;
   bars of test_stages_gpu.py (2e-3 of the buffer's largest entry) and the per-fragment bars of
   test_kernel_variants_gpu.py, on every stage.  The branch is read from a handle with the same plan; the stage run's
   own handle must have taken it too.
c. device MD == the host integrator (md.Langevin) driven by ViSNetCalculator's evaluation of the same graph, over 200
   steps at the 200-step trajectory bars of test_refnoise_gpu.py, on the ACE-ALA-NME input; Verlet energy conservation;
   the reference noise stream.  Whole proteins are not compared step for step: the truncated neighbour lists make their
   forces discontinuous (an atom crossing 5 A evicts a kept neighbour), so two trajectories that differ by fp32 rounding
   part at the first such crossing between them (whole Chignolin, measured: 10.6 A apart after 200 steps).
d. the run protocol in this mode (restraints against oracle/hookean_ref.py, recorder frames, runaway guard) and the
   loud refusals.
e. fragment mode did not move: the launch list and the MD step's kernel count of Chignolin equal those recorded from the
   engine before the un-fragmented step existed (tests/golden/chig_fragment_plan.json).
"""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

from ai2bmd_b200.calculator import ViSNetModel
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import load_capped_protein, load_fragments, load_protein
from ai2bmd_b200.md import KB, DeviceLangevin, Langevin, TemperatureRunawayError
from ai2bmd_b200.pdbfrag import single_graph
from ai2bmd_b200.restraints import KCALMOL_EV, hydrogen_bond_springs
from oracle.hookean_ref import hookean, hookean_terms

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tools"))

X_TOL, V_TOL = 2e-5, 2e-4                     # tests/test_md_gpu.py
X_TOL_200, V_TOL_200 = 4 * X_TOL, 4 * V_TOL   # tests/test_refnoise_gpu.py: the same bars over 200 steps
CASES = ("chig", "trpcage", "c1")


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "reference_visnet_mode.npz"))


def _zp(gold, key):
    return gold[f"{key}_z"], gold[f"{key}_pos"]


def _engine(real_weights, z, pos=None):
    eng = Engine(real_weights, 0)
    eng.set_topology(z, np.zeros(len(z), dtype=np.int64), n_graphs=1)
    if pos is not None:
        eng.forward_host(np.asarray(pos, dtype=np.float32))
    return eng


def e_bar(e, key):
    e = np.abs(np.asarray(e, dtype=np.float64))
    return np.maximum(4e-3, 2 * np.spacing(e.astype(np.float32))) if key == "c1" else 2e-6 * e + 4e-3


def f_bar(f):
    return 5e-5 + 2e-5 * np.abs(f).max()


def traj_e_bar(e):
    """Two fp32 energies of one O(1e4 .. 1e5 eV) graph at positions that differ by the trajectory bars."""
    return max(2e-2, 4 * float(np.spacing(np.float32(abs(e)))))


# ---- a. one graph against the reference ------------------------------------------------------------------------------
@pytest.mark.parametrize("key", CASES)
def test_neighbour_lists_bit_exact(real_weights, gold, key):
    z, pos = _zp(gold, key)
    eng = _engine(real_weights, z, pos)
    slots, deg = eng.get_edges()
    assert np.array_equal(deg, gold[f"{key}_deg"]) and np.array_equal(slots, gold[f"{key}_slots"])
    if key != "c1":
        assert deg.max() == 32


def _own_branch(real_weights, eng, z, pos, f):
    """fp64 energy and forces of the one graph on the VecLayerNorm branch the handle's last evaluation took
    (oracle/vecln_branch.py), the branch closest to f where the engine's norms leave more than one open."""
    from oracle.vecln_branch import Candidates, best_branch, engine_vectors
    return best_branch(real_weights, Candidates(engine_vectors(eng)), z, pos, 0, len(z), f)


@pytest.mark.parametrize("key", CASES)
def test_energy_and_forces(real_weights, gold, key):
    z, pos = _zp(gold, key)
    eng = _engine(real_weights, z)
    e, f = eng.forward_host(pos)
    ref_e, ref_f, e64, f64 = (gold[f"{key}_{s}"].astype(np.float64) for s in ("ref_e", "ref_f", "e64", "f64"))
    e = e.astype(np.float64)
    e_own, f_own, n_br = _own_branch(real_weights, eng, z, pos, f)
    print(f"{key}: |E - ref| {abs(e[0] - ref_e[0, 0]):.3e} |E - e64| {abs(e[0] - e64[0, 0]):.3e} "
          f"|F - ref| {np.abs(f - ref_f).max():.3e} |F - f64| {np.abs(f - f64).max():.3e} "
          f"|F - f64 on its branch| {np.abs(f - f_own).max():.3e} = {np.abs(f - f_own).max() / f_bar(f_own):.2f} of "
          f"the bar ({n_br} branch(es) open)")
    ref_bar = 4 * np.spacing(np.float32(abs(ref_e[0, 0]))) if key == "c1" else e_bar(ref_e[0, 0], key)
    assert abs(e[0] - ref_e[0, 0]) <= max(4e-3, ref_bar)
    assert abs(e[0] - e64[0, 0]) <= e_bar(e64[0, 0], key) and abs(e[0] - e_own) <= e_bar(e_own, key)
    assert np.abs(f - f_own).max() <= f_bar(f_own)
    if key == "chig":
        # the layer-4 VecLayerNorm tie at atom 130: the engine sees it, and the reference's fp32 forces, whose branch is
        # unknown, are held only to the jump between the two branches
        assert 130 in eng.vecln_near_ties()
        assert np.abs(f - ref_f).max() <= 5e-2
    else:
        assert np.abs(f - ref_f).max() <= f_bar(ref_f) and np.abs(f - f64).max() <= f_bar(f64)
    # the reference's calculator path (ViSNetModel.dl_potential_loader of one graph) is the same evaluation, held to
    # fp64 on the branch its own handle took
    model = ViSNetModel(real_weights, device="cuda:0")
    e2, f2 = model.dl_potential_loader(single_graph(z, pos))
    assert abs(float(e2[0, 0]) - e[0]) <= e_bar(e64[0, 0], key)
    e2_own, f2_own, _ = _own_branch(real_weights, model.engine, z, pos, f2)
    assert abs(float(e2[0, 0]) - e2_own) <= e_bar(e2_own, key)
    assert np.abs(f2 - f2_own).max() <= f_bar(f2_own)


# ---- b. every launch of the G = 1 plans ------------------------------------------------------------------------------
@pytest.mark.parametrize("decoy", [None, "dense", "nan"])
@pytest.mark.parametrize("key", ["chig", "trpcage"])
def test_every_launch_of_the_one_graph_plan(real_weights, gold, key, decoy):
    from stage_check import stage_report
    from test_kernel_variants_gpu import frag_bar
    from oracle.vecln_branch import Candidates, engine_vectors
    z, pos = _zp(gold, key)
    n = len(z)
    probe = _engine(real_weights, z, pos)           # the plan stage_report runs: calibrated on the geometry itself
    probe.set_option("calibrate", 1)
    probe.forward_host(pos)
    failures = []
    for pins in Candidates(engine_vectors(probe)).branches(0, n):
        detail = {}
        lines, worst = stage_report((z, pos, np.zeros(n, dtype=np.int64)), calibrate=True, detail=detail, decoy=decoy,
                                    pins=pins)
        print("\n".join(lines))
        bad = [(s, w, r) for s, w, r in worst if not r <= 2e-3]
        bad += [(s, w, r) for s, w, r, _ in detail["fragments"] if not r <= frag_bar(w)]
        assert Candidates(detail["vectors"]).contains(pins, 0, n), "the stage run took a branch the probe did not see"
        if not bad:
            break
        failures.append(bad)
    else:
        raise AssertionError(f"no branch the engine may have taken holds every stage: {failures}")
    assert detail["max_degree"] == 32 and detail["n_atoms"] == n
    assert {"nbr_build", "head", "embed_node_bwd", "finalize", "edge_bwd0"} <= {s for s, _, _ in worst}


# ---- c. device MD == host MD -----------------------------------------------------------------------------------------
def _host_force(real_weights, z):
    """ViSNetCalculator's evaluation (one graph through ViSNetModel.dl_potential_loader) as md.Langevin's force_fn."""
    model = ViSNetModel(real_weights, device="cuda:0")

    def force_fn(x):
        e, f = model.dl_potential_loader(single_graph(z, x.astype(np.float32)))
        return float(e[0, 0]), f.astype(np.float64)
    return force_fn


def test_device_md_equals_host_md_verlet(real_weights, gold):
    key = "c1"
    z, pos = _zp(gold, key)
    pos = pos.astype(np.float64)
    host = Langevin(pos, z, _host_force(real_weights, z), dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.0, seed=3)
    dev = DeviceLangevin.unfragmented(real_weights, z, pos, dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.0, seed=3,
                                      velocities=host.v.copy())
    assert dev.engine.get_option("md_unfragmented") == 1 and dev.n == len(z)
    assert abs(dev.energy - host.energy) <= traj_e_bar(host.energy)
    n = 200
    host_e = [host.step() for _ in range(n)]
    dev.run(n)
    x, v, step, hist = dev.state(n_hist=n)
    print(f"{key}: |dx| {np.abs(x - host.x).max():.2e} |dv| {np.abs(v - host.v).max():.2e} "
          f"|dE| {np.abs(hist - np.asarray(host_e)).max():.2e} after {n} steps")
    assert step == n
    assert np.abs(x - host.x).max() <= X_TOL_200 and np.abs(v - host.v).max() <= V_TOL_200
    assert np.abs(hist - np.asarray(host_e)).max() <= traj_e_bar(host_e[0])


def test_device_md_equals_host_md_langevin_shared_pool(real_weights, gold):
    z, pos = _zp(gold, "c1")
    pos, n_at, n = pos.astype(np.float64), len(z), 200
    g = np.random.default_rng(17)
    pool = g.standard_normal((n, 2, n_at, 3))
    host = Langevin(pos, z, _host_force(real_weights, z), dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.01, seed=17,
                    normal_source=lambda s: (pool[s, 0], pool[s, 1]))
    dev = DeviceLangevin.unfragmented(real_weights, z, pos, dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.01, seed=17,
                                      velocities=host.v.copy())
    dev.set_normals(pool)                       # step s reads row s % 200
    host.run(n)
    dev.run(n)
    x, v, step, _ = dev.state()
    print(f"c1, friction 0.01: |dx| {np.abs(x - host.x).max():.2e} |dv| {np.abs(v - host.v).max():.2e} after {n} steps")
    assert step == n
    assert np.abs(x - host.x).max() <= X_TOL_200 and np.abs(v - host.v).max() <= V_TOL_200
    m = dev.masses[:, None]
    assert np.abs((m * v).sum(0)).max() <= 1e-9
    assert np.abs((m * x).sum(0) / m.sum() - (m * pos).sum(0) / m.sum()).max() <= 1e-9


@pytest.mark.parametrize("key", ["c1", "chig"])
def test_verlet_energy_drift_is_bounded(real_weights, gold, key):
    """friction = 0, dt = 0.5 fs, 300 steps, E_pot + E_kin of every step from the frame recorder (no runaway guard).  The
    22-atom input has no truncated neighbour list, so its potential is smooth and the bar is test_md_gpu.py's.  In whole
    Chignolin the first-32-by-index cap truncates the lists of 100 of 175 atoms: an atom crossing 5 A of such an atom with
    a lower index than its last kept neighbour evicts that neighbour, which sits inside the cutoff, so the potential
    itself jumps (in the reference as here; the fp32 oracle on the CPU shows the same 0.1 eV change of the total energy
    in the first step).  So whole Chignolin does not conserve energy in this mode: measured on one H100 80GB HBM3 at
    700 W, the total energy rose by 22 eV in 300 steps (1.25 eV in one step) and the temperature reached 815-1,033 K in two
    runs.  Only
    a stability bound applies there: finite, and below 50 eV."""
    z, pos = _zp(gold, key)
    dev = DeviceLangevin.unfragmented(real_weights, z, pos.astype(np.float64), dt_fs=0.5, temperature_K=300.0,
                                      friction_per_fs=0.0, seed=1)
    e0 = dev.energy + dev.kinetic_energy()
    dev.engine.md_set_recorder(1, 300, 0.0)
    dev.run(300)
    fr = dev.engine.md_read_frames(0, 300)
    dev.engine.md_set_recorder(0)
    tot = fr["epot"] + fr["ekin"] - e0
    drift = abs(tot[-50:].mean() - tot[:50].mean())
    print(f"{key}: max |E_tot - E_0| {np.abs(tot).max():.3e} eV, drift first/last 50 steps {drift:.3e} eV, "
          f"T {dev.temperature():.1f} K")
    assert len(tot) == 300 and np.isfinite(tot).all()
    if key == "c1":
        assert np.abs(tot).max() < 2e-2 and drift < 1e-2
        assert 50.0 < dev.temperature() < 450.0
    else:
        assert np.abs(tot).max() < 50.0


def test_reference_noise_stream(real_weights, gold):
    z, pos = _zp(gold, "c1")
    seed, n = 7, len(z)
    g = np.random.default_rng(seed)
    for _ in range(64):
        xi, eta = g.standard_normal((n, 3)), g.standard_normal((n, 3))
    dev = DeviceLangevin.unfragmented(real_weights, z, pos.astype(np.float64), seed=seed, noise="reference")
    _, v0, _, _ = dev.state()
    assert np.array_equal(v0, Langevin(pos, z, lambda x: (0.0, np.zeros_like(x)), seed=seed, noise="reference").v)
    dev.run(64)
    assert dev.noise_state() == int(g.bit_generator.state["state"]["state"])
    dxi, deta = dev.engine.md_get_noise()
    assert np.array_equal(dxi, xi) and np.array_equal(deta, eta)


# ---- d. the run protocol and the refusals ----------------------------------------------------------------------------
def _assert_rf(rf, x, terms):
    e, f = hookean(x, terms)
    assert np.isfinite(rf).all()
    assert np.abs(rf[:-1] - f.reshape(-1)).max() <= 1e-12 * max(np.abs(f).max(), 1e-300)
    assert abs(rf[-1] - e) <= 1e-12 * e


def test_preequilibration_and_hydrogen_springs(real_weights, gold):
    z, pos = _zp(gold, "chig")
    dev = DeviceLangevin.unfragmented(real_weights, z, pos.astype(np.float64), seed=2)
    atoms = np.arange(dev.n)
    seen = []
    dev.preequilibrate(4, schedule=(10.0, 5.0), record_per_steps=2, observer=lambda s, *a: seen.append(s))
    x0, v0, s0, _ = dev.state()
    assert s0 == 8 and seen == [2, 4, 6, 8] and np.isfinite(x0).all()
    dev.set_restraints(tether_atoms=atoms, tether_k_kcal=10)         # a stage's tethers, after some steps
    assert not dev.engine.md_restraint_forces().any()
    dev.run(6)
    x1, _, _, _ = dev.state()
    _assert_rf(dev.engine.md_restraint_forces(), x1, hookean_terms(atoms, x0, 10 * KCALMOL_EV))
    # the reference's --constraints springs, protein atom indices = the one graph's atom indices
    springs = hydrogen_bond_springs(load_capped_protein("chig"))
    h, p = int(springs[0][0, 0]), int(springs[0][0, 1])
    xp = np.array(x1)
    xp[h] += 0.5 * (xp[h] - xp[p]) / np.linalg.norm(xp[h] - xp[p])
    dev.engine.md_set_state(xp, v0, s0)
    dev.set_restraints(tether_atoms=atoms[::3], tether_k_kcal=1, springs=springs)
    rf = dev.engine.md_restraint_forces()
    _assert_rf(rf, xp, hookean_terms(atoms[::3], xp, 1 * KCALMOL_EV, springs))
    assert np.abs(rf[:-1]).max() > 0.1
    dev.set_restraints(springs=springs)
    dev.run(5)
    x2, _, s2, _ = dev.state()
    _assert_rf(dev.engine.md_restraint_forces(), x2, hookean_terms(springs=springs))
    assert s2 == s0 + 5


def test_recorder_frames_are_the_state(real_weights, gold):
    z, pos = _zp(gold, "c1")
    dev = DeviceLangevin.unfragmented(real_weights, z, pos.astype(np.float64), friction_per_fs=0.01, seed=4)
    eng = dev.engine
    eng.md_set_recorder(4, 16, 0.0)
    for chunk in (4, 8, 12):
        dev.run(chunk)
        x, v, step, hist = dev.state(n_hist=chunk)
        nf = eng.get_option("md_frames")
        assert nf == step // 4
        fr = eng.md_read_frames(0, nf)
        assert list(fr["step"]) == [4 * (i + 1) for i in range(nf)] and not fr["halted"].any()
        assert np.array_equal(fr["x"][-1], x) and np.array_equal(fr["v"][-1], v) and fr["epot"][-1] == hist[-1]
        assert abs(fr["ekin"][-1] - 0.5 * float((dev.masses[:, None] * v * v).sum())) <= 1e-12 * fr["ekin"][-1]
    eng.md_set_recorder(0)
    seen = []
    dev.run_observed(20, 5, lambda step, x, v, epot, ekin: seen.append((step, x, v)))
    x, v, step, _ = dev.state()
    assert [s for s, _, _ in seen] == [25, 30, 35, 40] and step == 44
    assert eng.get_option("md_frames") == 0


def test_runaway_guard_halts(real_weights, gold):
    z, pos = _zp(gold, "chig")
    pos = pos.astype(np.float64)
    dev = DeviceLangevin.unfragmented(real_weights, z, pos, temperature_K=300.0, seed=6)
    v_hot = np.random.default_rng(6).standard_normal(pos.shape) * np.sqrt(1000.0 * KB / dev.masses[:, None])
    dev.engine.md_set_state(pos, v_hot, 0)
    dev._eval()
    with pytest.raises(TemperatureRunawayError):
        dev.run_observed(200, 5)
    eng = dev.engine
    halt, nf = eng.get_option("md_halt_step"), eng.get_option("md_frames")
    assert halt > 0 and halt == 5 * nf
    x, v, step, _ = dev.state()
    dev.run(7)
    x2, v2, step2, _ = dev.state()
    assert step == step2 == halt and np.array_equal(x2, x) and np.array_equal(v2, v)


def _empty_caph():
    e2, e3, e4 = np.zeros((0, 2)), np.zeros((0, 3)), np.zeros((0, 4))
    return types.SimpleNamespace(h_idx=[], bond_ij=e2, bond_k=[], bond_r0=[], angle_ijk=e3, angle_k=[], angle_t0=[],
                                 dih_ijkl=e4, dih_k=[], dih_n=[], dih_p=[], pair_ij=e2, pair_a=[], pair_b=[], pair_qq=[],
                                 mirror_dst=[], mirror_src=[], scnb=1.2, scee=2.0, max_iter=10, lr=0.1, tol_grad=0.1,
                                 tol_change=0.01)


def test_loud_refusals(real_weights, gold):
    z, pos = _zp(gold, "c1")
    n = len(z)
    m = np.ones(n)
    ef = torch.zeros(3 * n + 1, device="cuda")
    with pytest.raises(ValueError, match="sharded"):
        DeviceLangevin.unfragmented(real_weights, z, pos, group=object())
    eng = Engine(real_weights, 0)
    eng.set_topology(np.concatenate([z, z]), np.repeat([0, 1], n), n_graphs=2)      # two graphs
    with pytest.raises(RuntimeError, match="ONE graph"):
        eng.md_setup_unfragmented(np.ones(2 * n), 0.1, 0.025, 0.0, 0, ef.data_ptr())
    eng = _engine(real_weights, z, pos)
    with pytest.raises(RuntimeError, match="must equal the topology's atom count"):
        eng.md_setup_unfragmented(m[:-1], 0.1, 0.025, 0.0, 0, ef.data_ptr())
    eng.md_setup_unfragmented(m, 0.1, 0.025, 0.0, 0, ef.data_ptr())
    assert eng.get_option("md_unfragmented") == 1
    with pytest.raises(RuntimeError, match="vb_set_caph: .*un-fragmented"):
        eng.set_caph(_empty_caph())
    with pytest.raises(RuntimeError, match="vb_set_protein_map: .*un-fragmented"):
        eng.set_protein_map(n, np.arange(n), np.arange(n), np.ones(n), np.ones(1))
    h = eng.comm_init(0, 2, 3 * n + 1)
    with pytest.raises(RuntimeError, match="vb_comm_connect: .*cannot be sharded"):
        eng.comm_connect([h, h])
    # a new topology ends the mode: the fragment path works again on the same handle
    eng.set_topology(z, np.zeros(n, dtype=np.int64), n_graphs=1)
    assert eng.get_option("md_unfragmented") == 0
    eng.set_protein_map(n, np.arange(n), np.arange(n), np.ones(n), np.ones(1))
    with pytest.raises(RuntimeError, match="protein map is set"):
        eng.md_setup_unfragmented(m, 0.1, 0.025, 0.0, 0, ef.data_ptr())


# ---- e. fragment mode did not move -----------------------------------------------------------------------------------
def _md_step_kernels(dev):
    """CUDA kernels one direct (uncaptured) MD step launches, counted by torch.profiler over two steps: the kernels after
    the first step's md_kick2_kernel, which ends a step.  Late in a long test process the profiler has lost the first
    kernels of a session (7 of a whole-WW step's 38, the same count again with 50 ms of idle time before the step; a
    second session right after counted all 38), so the first step only marks where the counted one begins."""
    from torch.profiler import ProfilerActivity, profile
    dev.engine.set_option("use_graph", 0)
    dev.run(1)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev.run(2)
        torch.cuda.synchronize()
    dev.engine.set_option("use_graph", 1)
    ks = sorted((e.time_range.start, e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    ends = [i for i, (_, name) in enumerate(ks) if "md_kick2_kernel" in name]
    assert len(ends) == 2 and ends[1] == len(ks) - 1, [name for _, name in ks]
    return ends[1] - ends[0]


def fragment_plan(real_weights):
    """Chignolin in fragment mode: the evaluation's launch list (stage, kernel, grid), its launch count and the kernels
    of one MD step; plus the un-fragmented step's kernel count and launch count of whole Chignolin."""
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, seed=1)
    out = dict(sm_count=torch.cuda.get_device_properties(0).multi_processor_count,
               stage_kernels=[list(k) for k in dev.engine.stage_kernels()],
               launches_per_forward=dev.engine.launches_per_forward, md_step_kernels=_md_step_kernels(dev))
    return out, dev


def test_fragment_mode_did_not_move(real_weights):
    with open(os.path.join(GOLDEN, "chig_fragment_plan.json")) as fh:
        want = json.load(fh)
    got, _ = fragment_plan(real_weights)
    assert [(s, k) for s, k, _ in got["stage_kernels"]] == [(s, k) for s, k, _ in want["stage_kernels"]]
    if got["sm_count"] == want["sm_count"]:
        assert got["stage_kernels"] == want["stage_kernels"]
    assert got["launches_per_forward"] == want["launches_per_forward"]
    assert got["md_step_kernels"] == want["md_step_kernels"] == want["launches_per_forward"] + 3
    # the un-fragmented step of whole Chignolin has the same shape: kick1, the placement (a cast), the plan, kick2
    prot_pos, prot_z, _ = load_protein("chig")
    dev = DeviceLangevin.unfragmented(real_weights, prot_z, prot_pos, seed=1)
    assert _md_step_kernels(dev) == dev.engine.launches_per_forward + 3
