"""The whole FragmentCalculator call on the device (vb_forward_fragments*, calculator.FragmentCalculator): protein
positions in, bonded + non-bonded energy and forces out, with the placement, the hydrogen refinement and the MM term in
the same graph replay.

Checked against (1) the host composition of the same call -- recipe.positions, the C restatement of the refinement,
forward_host, DipeptideBondedCombiner and the fp32 restatement of MMNonBondedCalculator -- at the PDB geometry and a
seeded perturbation; (2) the fragment positions the reference's own HydrogenOptimizer produced (golden); (3) the MD
step's evaluation at the same positions; and for isolation from the MD state, stale workspaces, the variants (no
refinement, no MM, chunks, no graph), the graph cache, the reference's loop shape and every refusal."""
import types

import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.calculator import DipeptideBondedCombiner, FragmentCalculator
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.md import DeviceLangevin, Langevin
from ai2bmd_b200.nonbonded import dipeptide_atom_sets, synthetic_parameters
from oracle import nonbonded_ref
from oracle.caph_c import relax_problem

pytestmark = pytest.mark.gpu

NAMES = ["chig", "trpcage"]
F_TIE = 5e-2          # forces of protein atoms fed by a fragment on a VecLayerNorm tie: bounded jump only (DESIGN §2)


def e_tol(e, ulps=2):
    return np.maximum(4e-3, ulps * np.spacing(np.abs(e).astype(np.float32)))


def f_tol(f):
    return 5e-5 + 2e-5 * np.abs(f).max()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Case:
    def __init__(self, name):
        self.name = name
        self.fd, self.pm = load_fragments(name)
        self.x0, self.z, self.recipe = load_protein(name)
        self.prot = load_capped_protein(name)
        tables, self.golden = load_caph_tables(name)
        self.pr = caph.build_problem(self.prot, self.fd, self.recipe, tables)
        self.nb = synthetic_parameters(self.z, seed=1)
        self.geoms = {"pdb": self.x0,
                      "perturbed": self.x0 + 0.03 * np.random.default_rng(5).standard_normal(self.x0.shape)}

    def calc(self, refine=True, mm=True, **kw):
        return FragmentCalculator(WEIGHTS, "", self.fd, self.pm, self.recipe, caph=self.pr if refine else None,
                                  nonbonded=self.nb if mm else None, **kw)


_CASES = {}


def _case(name):
    if name not in _CASES:
        _CASES[name] = _Case(name)
    return _CASES[name]


def _host_composition(c, x, real_weights, refine=True, mm=True):
    """(energy, forces [P,3], refined fragment positions, fragment energies, tie mask over protein atoms) of the
    reference's call restated on the host around the engine's plain fragment evaluation."""
    pos = c.recipe.positions(x)
    if refine:
        pos = relax_problem(c.pr, pos)[0]
    eng = Engine(real_weights, 0)
    eng.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd))
    e, f = eng.forward_host(pos)
    dip_g, an_g = c.fd.scalar_split()
    dip_a, an_a = c.fd.vector_split()
    # the concatenation [dipeptide atoms, ACE-NME atoms] the combiner selects from, and where each packed atom lands in it
    at = np.empty(len(c.fd.z), dtype=np.int64)
    at[dip_a] = np.arange(dip_a.sum())
    at[an_a] = dip_a.sum() + np.arange(an_a.sum())
    E = float(DipeptideBondedCombiner.energy_combine(e[dip_g], e[an_g]))
    F = DipeptideBondedCombiner.forces_combine(c.pm.n_protein, f[dip_a], f[an_a], at[c.pm.src_atom], c.pm.dst_atom)
    F = F.astype(np.float64)
    if mm:
        ex = nonbonded_ref.exclude_pairs_from_groups(dipeptide_atom_sets(c.fd, c.recipe, c.pm))
        src, dst = nonbonded_ref.pair_list(c.pm.n_protein, ex)
        e_mm, f_mm = nonbonded_ref.nonbonded(x, *c.nb, src, dst)
        E, F = E + e_mm, F + f_mm
    tie_frag = np.unique(c.fd.batch[eng.vecln_near_ties()])
    tie_atoms = np.isin(c.fd.batch, tie_frag)
    tied = np.zeros(c.pm.n_protein, bool)
    tied[c.pm.dst_atom[tie_atoms[c.pm.src_atom]]] = True
    return E, F, pos, e, tied


def _check_against_host(c, calc, x, real_weights, refine=True, mm=True, label=""):
    E, F = calc.engine.forward_fragments_host(x)
    E_h, F_h, pos_h, e_frag, tied = _host_composition(c, x, real_weights, refine, mm)
    pos_d = calc.engine.debug_read("pos", 0, (len(c.fd.z), 3))
    dpos = np.abs(pos_d - pos_h).max()
    df = np.abs(F - F_h).max(1)
    print(f"\n{c.name} {label}: |dpos| {dpos:.2e} A, |dE| {abs(E - E_h):.2e} eV (bar {np.sum(e_tol(e_frag)):.2e}), "
          f"|dF| {df[~tied].max():.2e} eV/A (bar {f_tol(F_h):.2e}), {tied.sum()} tie atoms")
    assert np.isfinite(F).all() and np.isfinite(E)
    assert dpos <= 1e-5
    assert abs(E - E_h) <= float(np.sum(e_tol(e_frag)))
    assert df[~tied].max() <= f_tol(F_h)
    assert (df[tied] <= F_TIE).all()
    return E, F


# ---- 1. against the host composition ---------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", ["pdb", "perturbed"])
@pytest.mark.parametrize("name", NAMES)
def test_matches_the_host_composition(real_weights, name, geom):
    c = _case(name)
    calc = c.calc()
    _check_against_host(c, calc, c.geoms[geom], real_weights, label=geom)
    # the ASE surface returns the same values (the forces are fp32 sums in no fixed order: to the bar), and caches them
    # while the positions stay
    atoms = types.SimpleNamespace(numbers=c.z, positions=c.geoms[geom].copy())
    E, F = calc.engine.forward_fragments_host(atoms.positions)
    assert calc.get_potential_energy(atoms) == E and np.abs(calc.get_forces(atoms) - F).max() <= f_tol(F)
    assert calc.get_forces(atoms) is calc.results["forces"] and calc.get_potential_energy(atoms) == E


# ---- 2. against the reference's own refinement output -----------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_fragment_positions_match_the_reference_optimizer(name):
    c = _case(name)
    calc = c.calc()
    calc.engine.forward_fragments_host(c.x0)
    pos = calc.engine.debug_read("pos", 0, (len(c.fd.z), 3))
    off = 0
    for t2f in c.pr.table_to_frag:
        assert np.abs(pos[t2f] - c.golden["pos1"][off:off + len(t2f)]).max() <= 1e-5
        off += len(t2f)
    assert off == len(c.golden["pos1"])


# ---- 3. against the MD step ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_equals_the_md_evaluation(name):
    c = _case(name)
    calc = c.calc()
    eng = calc.engine
    x = c.geoms["perturbed"]
    ef = torch.zeros(3 * c.pm.n_protein + 1, device="cuda")
    eng.md_setup(np.ones(c.pm.n_protein), c.recipe.real, c.recipe.acc, c.recipe.rem, c.recipe.blen, 0.1, 0.025, 0.0, 0,
                 ef.data_ptr())
    eng.md_set_state(x, np.zeros_like(x), 0)
    md = []
    for _ in range(6):
        eng.md_eval(_stream())
        md.append(ef.cpu().numpy().copy())
    fr = []
    for _ in range(2):
        E, F = eng.forward_fragments_host(x)
        fr.append(np.r_[F.reshape(-1), E])
    spread_md = max(np.abs(a[:-1] - b[:-1]).max() for a in md for b in md)
    spread_fr = np.abs(fr[0][:-1] - fr[1][:-1]).max()
    diff = max(np.abs(f[:-1] - m[:-1]).max() for f in fr for m in md)
    print(f"\n{name}: md_eval run-to-run force spread {spread_md:.2e}, entry spread {spread_fr:.2e}, entry vs md_eval {diff:.2e} eV/A")
    assert all(np.float32(f[-1]) == m[-1] for f in fr for m in md)           # energies bit-identical
    # the same launches: the forces differ only by the order of their fp32 atomic sums.  The spread of a few calls is
    # itself a sample of that order (measured: one float32 ulp of the largest forces more or less), hence the factor 2
    assert diff <= 2 * max(spread_md, spread_fr)


# ---- 4. the MD state stays as it was -----------------------------------------------------------------------------------
def test_leaves_the_md_state_alone(real_weights):
    c = _case("chig")
    dev = DeviceLangevin(real_weights, c.fd, c.pm, c.recipe, c.x0, c.z, seed=3, caph=c.pr, noise="reference")
    eng = dev.engine
    dev.set_restraints(tether_atoms=np.arange(0, c.pm.n_protein, 3), tether_k_kcal=1.0)
    eng.md_set_recorder(4, 8, 0.0)
    dev.run(10)

    def snapshot():
        x, v, step, hist = dev.state(n_hist=10)
        return dict(x=x, v=v, step=step, hist=hist, rf=eng.md_restraint_forces(), noise=dev.noise_state(),
                    frames=eng.get_option("md_frames"), ef=dev.ef.cpu().numpy().copy())

    before = snapshot()
    other = c.geoms["perturbed"]
    E, F = eng.forward_fragments_host(other)
    xd = torch.from_numpy(np.ascontiguousarray(other)).cuda()
    out = torch.zeros(3 * c.pm.n_protein + 1, device="cuda")
    eng.forward_fragments_device(xd.data_ptr(), out.data_ptr(), _stream())
    torch.cuda.synchronize()
    after = snapshot()
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    assert np.isfinite(out.cpu().numpy()).all() and abs(float(out[-1]) - E) <= 1e-2
    dev.run(5)
    x, _, step, _ = dev.state()
    assert step == 15 and np.isfinite(x).all() and eng.get_option("md_frames") == 3


def test_host_call_right_after_unsynchronised_md_steps(real_weights):
    """The host entry on an engine whose MD steps are still running on the caller's stream (``run`` only enqueues): it
    shares their workspace, so it waits for them.  The MD trajectory and its own result equal those of a twin run that
    synchronised before the call: energies bit for bit, forces and trajectory to the device-vs-host bars."""
    c = _case("chig")
    other = c.geoms["perturbed"]
    out = []
    for sync in (False, True):
        dev = DeviceLangevin(real_weights, c.fd, c.pm, c.recipe, c.x0, c.z, seed=3, caph=c.pr)
        eng = dev.engine
        eng.forward_fragments_host(c.x0)              # graph captures of both paths before the overlap under test
        dev.run(5)
        dev.state()
        dev.run(40)                                   # about 40 ms of steps enqueued on the caller's stream
        if sync:
            torch.cuda.synchronize()
        E, F = eng.forward_fragments_host(other)
        dev.run(5)
        x, v, step, _ = dev.state()
        out.append((E, F, x, v, step))
    (E0, F0, x0, v0, s0), (E1, F1, x1, v1, s1) = out
    print(f"\nunsynchronised vs synchronised: |dF| {np.abs(F0 - F1).max():.2e} eV/A, |dx| {np.abs(x0 - x1).max():.2e} A, "
          f"|dv| {np.abs(v0 - v1).max():.2e}")
    assert s0 == s1 == 50
    assert E0 == E1 and np.abs(F0 - F1).max() <= f_tol(F1)
    assert np.abs(x0 - x1).max() <= X_TOL and np.abs(v0 - v1).max() <= V_TOL


# ---- 5. a workspace that holds another geometry's poison ---------------------------------------------------------------
def _nan_decoy(c):
    """Another protein geometry with, in every residue, the first HA atom on its CA: every fragment of two or more atoms
    holds such a pair, so r = 0 reaches the edge geometry and NaN every buffer after it.  The cap hydrogens are placed
    on rays that do not start or end at an HA, so the coordinates stay finite."""
    x = c.x0 + 0.2 * np.random.default_rng(9).standard_normal(c.x0.shape)
    for r in np.unique(c.prot.resnums):
        at = [i for i in range(len(c.prot)) if c.prot.resnums[i] == r]
        ca = [i for i in at if c.prot.names[i] == "CA"]
        ha = [i for i in at if c.prot.names[i].startswith("HA")]
        if ca and ha:
            x[ha[0]] = x[ca[0]]
    return x


@pytest.mark.parametrize("name", NAMES)
def test_stale_workspace(name):
    c = _case(name)
    poisoned, clean = c.calc(), c.calc()
    E_decoy, _ = poisoned.engine.forward_fragments_host(_nan_decoy(c))
    assert not np.isfinite(E_decoy)
    for geom in ("pdb", "perturbed"):
        E_p, F_p = poisoned.engine.forward_fragments_host(c.geoms[geom])
        E_c, F_c = clean.engine.forward_fragments_host(c.geoms[geom])
        assert np.isfinite(F_p).all() and E_p == E_c, geom


# ---- 6. variants ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["no_refinement", "no_mm", "chunks", "no_graph"])
@pytest.mark.parametrize("name", NAMES)
def test_variants(real_weights, name, variant):
    c = _case(name)
    refine, mm = variant != "no_refinement", variant != "no_mm"
    calc = c.calc(refine=refine, mm=mm, chunk_size=250 if variant == "chunks" else None)
    if variant == "chunks":
        assert calc.engine.get_option("chunks") >= 2
    if variant == "no_graph":
        calc.engine.set_option("use_graph", 0)
    _check_against_host(c, calc, c.geoms["perturbed"], real_weights, refine, mm, label=variant)


# ---- 7. graph cache ---------------------------------------------------------------------------------------------------
def test_graph_cache():
    c = _case("chig")
    eng = c.calc().engine
    eng.forward_fragments_host(c.x0)
    n0 = eng.get_option("graph_captures")
    for g in ("perturbed", "pdb", "perturbed"):
        eng.forward_fragments_host(c.geoms[g])
    assert eng.get_option("graph_captures") == n0
    xd = torch.from_numpy(np.ascontiguousarray(c.x0)).cuda()
    out = [torch.zeros(3 * c.pm.n_protein + 1, device="cuda") for _ in range(2)]
    eng.forward_fragments_device(xd.data_ptr(), out[0].data_ptr(), _stream())
    assert eng.get_option("graph_captures") == n0 + 1
    eng.forward_fragments_device(xd.data_ptr(), out[0].data_ptr(), _stream())
    assert eng.get_option("graph_captures") == n0 + 1
    eng.forward_fragments_device(xd.data_ptr(), out[1].data_ptr(), _stream())
    assert eng.get_option("graph_captures") == n0 + 2
    torch.cuda.synchronize()
    E, _ = eng.forward_fragments_host(c.x0)
    assert float(out[0][-1]) == float(out[1][-1]) == np.float32(E)


# ---- 8. the reference's loop shape --------------------------------------------------------------------------------------
X_TOL, V_TOL = 2e-5, 2e-4          # tests/test_md_gpu.py: device vs host integrator


def test_host_loop_with_the_calculator_follows_the_device_step(real_weights):
    """ASE's loop shape -- the integrator on the host, the calculator asked for energy and forces once per step -- against
    the device step with the same normals.  The synthetic charges are scaled by 0.25 as in tests/test_md_loop_gpu.py:
    at full strength they pull the unrestrained protein apart within 200 steps, and two diverging runs say nothing.
    Two host runs of the same start differ only by the order of the fp32 force sums; over 200 steps the dynamics
    amplifies that, so the bar is the larger of test_md_gpu's and twice that host-vs-host spread (printed)."""
    c = _case("chig")
    n, steps, seed = c.pm.n_protein, 200, 17
    pool = np.random.default_rng(seed).standard_normal((steps, 2, n, 3))
    q, sg, ep = c.nb
    nb = (0.25 * q, sg, ep)
    calc = FragmentCalculator(WEIGHTS, "", c.fd, c.pm, c.recipe, caph=c.pr, nonbonded=nb)
    atoms = types.SimpleNamespace(numbers=c.z, positions=None)

    def force_fn(x):
        atoms.positions = x
        return float(calc.get_potential_energy(atoms)), np.asarray(calc.get_forces(atoms), dtype=np.float64)

    runs = []
    for _ in range(2):             # two host runs: the run-to-run spread of the forces, amplified over the steps
        host = Langevin(c.x0, c.z, force_fn, friction_per_fs=0.001, seed=seed, normal_source=lambda s: tuple(pool[s]))
        v0 = host.v.copy()
        host.run(steps)
        runs.append(host)
    twin = FragmentCalculator(WEIGHTS, "", c.fd, c.pm, c.recipe, caph=c.pr, nonbonded=nb)
    dev = DeviceLangevin(None, c.fd, c.pm, c.recipe, c.x0, c.z, friction_per_fs=0.001, seed=seed, velocities=v0,
                         engine=twin.engine)
    dev.set_normals(pool)
    dev.run(steps)
    x, v, step, _ = dev.state()
    host = runs[0]
    dx, dv = np.abs(x - host.x).max(), np.abs(v - host.v).max()
    sx, sv = np.abs(runs[1].x - host.x).max(), np.abs(runs[1].v - host.v).max()
    print(f"\nchig {steps} steps: device vs host |dx| {dx:.2e} A, |dv| {dv:.2e}; host vs host |dx| {sx:.2e} A, "
          f"|dv| {sv:.2e}; T {host.temperature():.0f} K, max displacement {np.abs(host.x - c.x0).max():.2f} A")
    assert step == steps
    assert host.temperature() < 1.5 * 300 + 150 and np.abs(host.x - c.x0).max() < 2.0      # nothing flew apart (test_md_gpu)
    assert dx <= max(X_TOL, 2 * sx) and dv <= max(V_TOL, 2 * sv)


# ---- 9. refusals -----------------------------------------------------------------------------------------------------
def _rc(eng, fn, *args):
    rc = getattr(eng.lib, fn)(eng.h, *args)
    return rc, eng.lib.vb_last_error(eng.h).decode()


def test_refusals(real_weights):
    c = _case("chig")
    P, N = c.pm.n_protein, len(c.fd.z)
    x = np.ascontiguousarray(c.x0)
    ef = np.zeros(3 * P + 1, np.float32)
    r = c.recipe
    args = (r.real.ctypes.data, r.acc.ctypes.data, r.rem.ctypes.data, r.blen.ctypes.data)

    def host(eng):
        return _rc(eng, "vb_forward_fragments_host", x.ctypes.data, ef.ctypes.data)

    eng = Engine(real_weights, 0)
    rc, msg = host(eng)
    assert rc == -3 and "vb_set_topology" in msg                               # no topology
    assert _rc(eng, "vb_set_fragment_recipe", P, *args)[0] == -3
    eng.set_topology(c.fd.z, c.fd.batch)
    rc, msg = host(eng)
    assert rc == -3 and "protein map" in msg and "recipe" not in msg            # no map
    assert _rc(eng, "vb_set_fragment_recipe", P, *args)[0] == -3
    eng.set_protein_map(P, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)
    rc, msg = host(eng)
    assert rc == -3 and "placement recipe" in msg                               # no recipe
    assert _rc(eng, "vb_set_fragment_recipe", P + 1, *args)[0] == -1           # another protein
    assert _rc(eng, "vb_set_fragment_recipe", P, None, *args[1:])[0] == -1     # null array
    bad = r.real.copy()
    bad[0] = P
    rc, msg = _rc(eng, "vb_set_fragment_recipe", P, bad.ctypes.data, *args[1:])
    assert rc == -1 and "recipe index" in msg
    eng.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
    assert host(eng)[0] == 0
    assert _rc(eng, "vb_forward_fragments_host", None, ef.ctypes.data)[0] == -1          # null buffers
    assert _rc(eng, "vb_forward_fragments_host", x.ctypes.data, None)[0] == -1
    xd = torch.from_numpy(x).cuda()
    efd = torch.zeros(3 * P + 1, device="cuda")
    for pos_ptr, ef_ptr in ((None, None), (None, efd.data_ptr()), (xd.data_ptr(), None)):
        rc, msg = _rc(eng, "vb_forward_fragments", pos_ptr, ef_ptr, None)
        assert rc == -1 and "null buffer" in msg
    assert _rc(eng, "vb_forward_fragments", xd.data_ptr(), efd.data_ptr(), None)[0] == 0
    torch.cuda.synchronize()
    eng.set_protein_map(P, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)     # a new map drops the recipe
    rc, msg = host(eng)
    assert rc == -3 and "placement recipe" in msg
    eng.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
    eng.set_topology(c.fd.z, c.fd.batch)                                                 # ... and so does a topology,
    eng.set_protein_map(P, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)     # with the map set again
    rc, msg = host(eng)
    assert rc == -3 and "placement recipe" in msg
    # Not tested here: the refusal after an all-reduce flag wait timed out (comm_check, option comm_timeouts).  A wait
    # only times out when a peer rank never signals, which one GPU cannot produce; the refusal is the same comm_check
    # every vb_md_* call makes, and test_allreduce_of_a_connected_handle runs the entry through a connected handle.
    # a forward-only handle
    en = Engine(real_weights, 0, derivative=False)
    en.set_topology(c.fd.z, c.fd.batch)
    en.set_protein_map(P, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)
    en.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
    rc, msg = host(en)
    assert rc == -3 and "derivative" in msg
    # an un-fragmented MD handle
    un = DeviceLangevin.unfragmented(real_weights, c.z, c.x0, seed=1)
    rc, msg = host(un.engine)
    assert rc == -3 and "un-fragmented" in msg
    with pytest.raises(RuntimeError, match="un-fragmented"):
        un.engine.forward_fragments_device(0, 0)


def test_allreduce_of_a_connected_handle():
    """A handle connected through vb_comm_* (one rank here) all-reduces the call's buffer as its last launch."""
    c = _case("chig")
    calc = c.calc()
    eng = calc.engine
    E0, F0 = eng.forward_fragments_host(c.x0)
    eng.comm_connect([eng.comm_init(0, 1, 4 * c.pm.n_protein)])
    seq = eng.get_option("comm_seq")
    E1, F1 = eng.forward_fragments_host(c.x0)
    assert eng.get_option("comm_seq") == seq + 1
    assert E1 == E0 and np.abs(F1 - F0).max() <= f_tol(F0)
