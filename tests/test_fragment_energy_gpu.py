"""The whole FragmentCalculator call without forces (vb_forward_fragments_energy*, vb_group_forward_fragments_energy*,
``FragmentCalculator(derivative=False)``): protein positions in, bonded + MM energy out, on the energy plan.

Checked on Chignolin and Trp-cage at the PDB geometry and a seeded perturbation: (1) bit for bit against slot 3P of
vb_forward_fragments on the same derivative = 1 handle, with and without refinement and MM, in chunks and without
graphs; (2) bit for bit on a derivative = 0 handle, whose workspace is at most a quarter of the full one; (3) against the
host composition of the same call; (4) the energy-only MM kernel against the full one and the fp64 restatement; (5) a
group's energy entry against its force entry, its members' partials and the single handle; (6) the calculator surface;
(7) stale workspaces, the graph cache, MD work still running, refusals and an edge overflow."""
import types

import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.calculator import DipeptideBondedCombiner, FragmentCalculator
from ai2bmd_b200.engine import Engine, EngineGroup
from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.md import DeviceLangevin
from ai2bmd_b200.nonbonded import dipeptide_atom_sets, synthetic_parameters
from oracle import nonbonded_ref
from oracle.caph_c import relax_problem

pytestmark = pytest.mark.gpu

NAMES = ["chig", "trpcage"]
GEOMS = ["pdb", "perturbed"]
X_TOL, V_TOL = 2e-5, 2e-4          # tests/test_md_gpu.py: device vs host integrator


def e_tol(e, ulps=2):
    return np.maximum(4e-3, ulps * np.spacing(np.abs(e).astype(np.float32)))


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(e):
    return np.float32(e).view(np.uint32)


class _Case:
    def __init__(self, name):
        self.name = name
        self.fd, self.pm = load_fragments(name)
        self.x0, self.z, self.recipe = load_protein(name)
        self.prot = load_capped_protein(name)
        tables, _ = load_caph_tables(name)
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


def _device_energy(eng, x):
    xd = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()
    e = torch.full((1,), float("nan"), device="cuda")
    eng.forward_fragments_energy_device(xd.data_ptr(), e.data_ptr(), _stream())
    torch.cuda.synchronize()
    return float(e.item())


def _mm_energy(c, x):
    ex = nonbonded_ref.exclude_pairs_from_groups(dipeptide_atom_sets(c.fd, c.recipe, c.pm))
    src, dst = nonbonded_ref.pair_list(c.pm.n_protein, ex)
    return float(nonbonded_ref.nonbonded(x, *c.nb, src, dst)[0])


def _host_energy(c, x, real_weights, refine=True, mm=True):
    """(energy, fragment energies) of the reference's call restated on the host around the engine's plain fragment
    evaluation: recipe.positions, the C restatement of the refinement, forward_host, DipeptideBondedCombiner and the
    restatement of MMNonBondedCalculator."""
    pos = c.recipe.positions(x)
    if refine:
        pos = relax_problem(c.pr, pos)[0]
    eng = Engine(real_weights, 0)
    eng.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd))
    e, _ = eng.forward_host(pos)
    dip_g, an_g = c.fd.scalar_split()
    E = float(DipeptideBondedCombiner.energy_combine(e[dip_g], e[an_g]))
    if mm:
        E += _mm_energy(c, x)
    return E, e


# ---- 1. bit identity on the same derivative = 1 handle -----------------------------------------------------------------
@pytest.mark.parametrize("variant", ["full", "no_refinement", "no_mm", "chunks", "no_graph"])
@pytest.mark.parametrize("name", NAMES)
def test_equals_the_force_entry_bit_for_bit(name, variant):
    c = _case(name)
    calc = c.calc(variant != "no_refinement", variant != "no_mm", chunk_size=250 if variant == "chunks" else None)
    eng = calc.engine
    if variant == "chunks":
        assert eng.get_option("chunks") >= 2
    if variant == "no_graph":
        eng.set_option("use_graph", 0)
    for geom in GEOMS:
        x = c.geoms[geom]
        E, _ = eng.forward_fragments_host(x)
        e_host = eng.forward_fragments_energy_host(x)
        e_dev = _device_energy(eng, x)
        print(f"\n{name} {variant} {geom}: E {E:.6f} eV, energy entry {e_host:.6f}, device entry {e_dev:.6f}")
        assert np.isfinite(E)
        assert _bits(e_host) == _bits(E) and _bits(e_dev) == _bits(E), geom


# ---- 2. bit identity on a derivative = 0 handle, and its workspace ----------------------------------------------------
@pytest.mark.parametrize("variant", ["full", "no_refinement", "no_mm", "chunks"])
@pytest.mark.parametrize("name", NAMES)
def test_forward_only_handle(name, variant):
    c = _case(name)
    kw = dict(refine=variant != "no_refinement", mm=variant != "no_mm", chunk_size=250 if variant == "chunks" else None)
    full, fwd = c.calc(**kw), c.calc(derivative=False, **kw)
    assert not fwd.engine.derivative and fwd.implemented_properties == ["energy"]
    a_full, a_fwd = full.engine.get_option("arena_bytes"), fwd.engine.get_option("arena_bytes")
    print(f"\n{name} {variant}: arena {a_fwd} B energy-only vs {a_full} B full ({a_fwd / a_full:.3f})")
    assert a_fwd <= a_full // 4
    for geom in GEOMS:
        x = c.geoms[geom]
        E, _ = full.engine.forward_fragments_host(x)
        assert _bits(fwd.engine.forward_fragments_energy_host(x)) == _bits(E), geom
        assert _bits(_device_energy(fwd.engine, x)) == _bits(E), geom


# ---- 3. against the host composition ------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("name", NAMES)
def test_matches_the_host_composition(real_weights, name, geom):
    c = _case(name)
    x = c.geoms[geom]
    e = c.calc(derivative=False).engine.forward_fragments_energy_host(x)
    E_h, e_frag = _host_energy(c, x, real_weights)
    bar = float(np.sum(e_tol(e_frag)))
    print(f"\n{name} {geom}: |dE| {abs(e - E_h):.2e} eV (bar {bar:.2e})")
    assert abs(e - E_h) <= bar


# ---- 4. the energy-only MM kernel -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_mm_energy(name):
    """With the bonded part bit-identical (test 1 without MM), the energy entry with MM equals the force entry's slot
    bit for bit only if the energy-only MM kernel's energy equals the full kernel's; the MM part itself against the fp64
    restatement within test_nonbonded.py's bar plus the fp32 rounding of the two totals."""
    c = _case(name)
    with_mm, without = c.calc(), c.calc(mm=False)
    for geom in GEOMS:
        x = c.geoms[geom]
        e_mm, e_no = with_mm.engine.forward_fragments_energy_host(x), without.engine.forward_fragments_energy_host(x)
        assert _bits(e_mm) == _bits(with_mm.engine.forward_fragments_host(x)[0]), geom
        ref = _mm_energy(c, x)
        bar = 4 * float(np.spacing(np.float32(abs(e_mm)))) + 1e-3 * abs(ref) + 1e-3      # test_nonbonded.py's bar
        print(f"\n{name} {geom}: MM {e_mm - e_no:.6f} eV vs {ref:.6f} (|d| {abs(e_mm - e_no - ref):.2e}, bar {bar:.2e})")
        assert abs((e_mm - e_no) - ref) <= bar


# ---- 5. a group ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("name", NAMES)
def test_group(name, k):
    c = _case(name)
    devices = ["cuda:0"] * k
    group = c.calc(devices=devices)
    single = c.calc(derivative=False)
    energy_calc = c.calc(devices=devices, derivative=False)
    assert energy_calc.implemented_properties == ["energy"]
    P = c.pm.n_protein
    for geom in GEOMS:
        x = c.geoms[geom]
        E_f, _ = group.group.forward_fragments_host(x)
        e = group.group.forward_fragments_energy_host(x)
        assert _bits(e) == _bits(E_f), geom                                        # the force call's slot
        parts = [np.float32(sh.engine.debug_read("ef", 0, (3 * P + 1,))[-1]) for sh in group.shards]
        s = np.float32(0.0)
        for p in parts:
            s = np.float32(s + p)
        assert _bits(s) == _bits(e), geom                                          # the rank-order sum of the partials
        xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
        out = torch.full((1,), float("nan"), device="cuda")
        group.group.forward_fragments_energy_device(xd.data_ptr(), out.data_ptr(), _stream())
        torch.cuda.synchronize()
        assert _bits(float(out.item())) == _bits(e), geom                          # the device entry
        e1 = single.engine.forward_fragments_energy_host(x)
        bar = 4e-3 * len(c.fd)
        print(f"\n{name} k={k} {geom}: group {e:.6f} eV, single {e1:.6f} (|dE| {abs(e - e1):.2e}, bar {bar:.2e})")
        assert abs(e - e1) <= bar                                                  # the single handle
        atoms = types.SimpleNamespace(numbers=c.z, positions=x.copy())
        assert _bits(energy_calc.get_potential_energy(atoms)) == _bits(e), geom  # the calculator


def test_group_refusals(real_weights):
    """Group members stay full handles: vb_group_create still refuses a derivative = 0 member."""
    c = _case("chig")
    fwd = c.calc(derivative=False)
    with pytest.raises(RuntimeError, match="derivative"):
        EngineGroup([fwd.engine])
    g = c.calc(devices=["cuda:0"] * 2).group
    rc = g.lib.vb_group_forward_fragments_energy_host(g.g, None, None)
    assert rc == -1 and "null buffer" in g.last_error()


# ---- 6. the calculator ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_calculator(name):
    c = _case(name)
    full, fwd = c.calc(), c.calc(derivative=False)
    assert full.implemented_properties == ["energy", "forces"] and full.derivative
    for geom in GEOMS:
        x = c.geoms[geom]
        atoms = types.SimpleNamespace(numbers=c.z, positions=x.copy())
        E, F = full.engine.forward_fragments_host(x)
        assert _bits(fwd.get_potential_energy(atoms)) == _bits(E), geom
        with pytest.raises(NotImplementedError):
            fwd.get_forces(atoms)
        # the derivative = True calculator: energy and forces of every calculate, as before
        assert full.get_potential_energy(atoms) == E
        assert full.get_forces(atoms) is full.results["forces"] and set(full.results) == {"energy", "forces"}
    prot = FragmentCalculator.from_protein(WEIGHTS, "", c.prot, nonbonded=c.nb, derivative=False)
    assert prot.implemented_properties == ["energy"] and not prot.engine.derivative
    assert np.isfinite(prot.get_potential_energy(types.SimpleNamespace(numbers=c.z, positions=c.x0.copy())))


# ---- 7. robustness ------------------------------------------------------------------------------------------------------
def _nan_decoy(c):
    """Another geometry with, in every residue, the first HA atom on its CA: r = 0 reaches the edge geometry of every
    fragment of two or more atoms and NaNs every buffer after it (test_fragment_calculator_gpu.py)."""
    x = c.x0 + 0.2 * np.random.default_rng(9).standard_normal(c.x0.shape)
    for r in np.unique(c.prot.resnums):
        at = [i for i in range(len(c.prot)) if c.prot.resnums[i] == r]
        ca = [i for i in at if c.prot.names[i] == "CA"]
        ha = [i for i in at if c.prot.names[i].startswith("HA")]
        if ca and ha:
            x[ha[0]] = x[ca[0]]
    return x


@pytest.mark.parametrize("derivative", [True, False])
@pytest.mark.parametrize("name", NAMES)
def test_stale_workspace(name, derivative):
    c = _case(name)
    poisoned, clean = c.calc(derivative=derivative), c.calc(derivative=derivative)
    assert not np.isfinite(poisoned.engine.forward_fragments_energy_host(_nan_decoy(c)))
    for geom in GEOMS:
        e_p = poisoned.engine.forward_fragments_energy_host(c.geoms[geom])
        assert np.isfinite(e_p) and _bits(e_p) == _bits(clean.engine.forward_fragments_energy_host(c.geoms[geom])), geom


def test_both_graphs_stay_cached():
    c = _case("chig")
    eng = c.calc().engine
    eng.forward_fragments_host(c.x0)
    eng.forward_fragments_energy_host(c.x0)
    n0 = eng.get_option("graph_captures")
    for g in ("perturbed", "pdb", "perturbed", "pdb"):
        E, _ = eng.forward_fragments_host(c.geoms[g])
        assert _bits(eng.forward_fragments_energy_host(c.geoms[g])) == _bits(E), g
    assert eng.get_option("graph_captures") == n0
    xd = torch.from_numpy(np.ascontiguousarray(c.x0)).cuda()
    out = [torch.zeros(1, device="cuda") for _ in range(2)]
    for o in (out[0], out[0], out[1]):
        eng.forward_fragments_energy_device(xd.data_ptr(), o.data_ptr(), _stream())
    assert eng.get_option("graph_captures") == n0 + 2                 # one graph per buffer pair
    torch.cuda.synchronize()
    E, _ = eng.forward_fragments_host(c.x0)
    assert float(out[0]) == float(out[1]) == np.float32(E)


def test_host_call_right_after_unsynchronised_md_steps(real_weights):
    """The energy host entry on an engine whose MD steps still run on the caller's stream waits for them: the MD
    trajectory and the energy equal those of a twin run that synchronised first, and the MD state is left alone."""
    c = _case("chig")
    other = c.geoms["perturbed"]
    out = []
    for sync in (False, True):
        dev = DeviceLangevin(real_weights, c.fd, c.pm, c.recipe, c.x0, c.z, seed=3, caph=c.pr)
        eng = dev.engine
        eng.forward_fragments_energy_host(c.x0)       # graph capture before the overlap under test
        dev.run(5)
        dev.state()
        dev.run(40)
        if sync:
            torch.cuda.synchronize()
        e = eng.forward_fragments_energy_host(other)
        before = dev.state(n_hist=10)
        ef_before = dev.ef.cpu().numpy().copy()
        assert _bits(eng.forward_fragments_energy_host(other)) == _bits(e)
        after = dev.state(n_hist=10)
        for a, b in zip(before, after):
            assert np.array_equal(a, b)
        assert np.array_equal(ef_before, dev.ef.cpu().numpy())
        dev.run(5)
        x, v, step, _ = dev.state()
        out.append((e, x, v, step))
    (e0, x0, v0, s0), (e1, x1, v1, s1) = out
    assert s0 == s1 == 50
    assert _bits(e0) == _bits(e1)
    assert np.abs(x0 - x1).max() <= X_TOL and np.abs(v0 - v1).max() <= V_TOL


def _rc(eng, fn, *args):
    rc = getattr(eng.lib, fn)(eng.h, *args)
    return rc, eng.lib.vb_last_error(eng.h).decode()


def test_refusals(real_weights):
    c = _case("chig")
    P = c.pm.n_protein
    x = np.ascontiguousarray(c.x0)
    e = np.zeros(1, np.float32)
    ef = np.zeros(3 * P + 1, np.float32)
    r = c.recipe

    def host(eng):
        return _rc(eng, "vb_forward_fragments_energy_host", x.ctypes.data, e.ctypes.data)

    for derivative in (True, False):
        eng = Engine(real_weights, 0, derivative=derivative)
        rc, msg = host(eng)
        assert rc == -3 and "vb_set_topology" in msg                                # no topology
        eng.set_topology(c.fd.z, c.fd.batch)
        rc, msg = host(eng)
        assert rc == -3 and "protein map" in msg                                    # no map
        eng.set_protein_map(P, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)
        rc, msg = host(eng)
        assert rc == -3 and "placement recipe" in msg                               # no recipe
        eng.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
        assert host(eng)[0] == 0
        assert _rc(eng, "vb_forward_fragments_energy_host", None, e.ctypes.data)[0] == -1     # null buffers
        assert _rc(eng, "vb_forward_fragments_energy_host", x.ctypes.data, None)[0] == -1
        xd = torch.from_numpy(x).cuda()
        ed = torch.zeros(1, device="cuda")
        for pos_ptr, e_ptr in ((None, None), (None, ed.data_ptr()), (xd.data_ptr(), None)):
            rc, msg = _rc(eng, "vb_forward_fragments_energy", pos_ptr, e_ptr, None)
            assert rc == -1 and "null buffer" in msg
        # the force entries still refuse a forward-only handle
        rc, msg = _rc(eng, "vb_forward_fragments_host", x.ctypes.data, ef.ctypes.data)
        assert (rc == 0) if derivative else (rc == -3 and "derivative" in msg)
    un = DeviceLangevin.unfragmented(real_weights, c.z, c.x0, seed=1)              # an un-fragmented MD handle
    rc, msg = host(un.engine)
    assert rc == -3 and "un-fragmented" in msg
    with pytest.raises(RuntimeError, match="un-fragmented"):
        un.engine.forward_fragments_energy_device(0, 0)


@pytest.mark.parametrize("derivative", [True, False])
def test_edge_overflow_is_reported(real_weights, derivative):
    c = _case("chig")
    r = c.recipe
    eng = Engine(real_weights, 0, derivative=derivative)
    eng.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd), max_edges=len(c.fd.z) * 4)
    eng.set_protein_map(c.pm.n_protein, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)
    eng.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
    with pytest.raises(RuntimeError, match="vb_forward_fragments_energy_host.*max_edges"):
        eng.forward_fragments_energy_host(c.x0)
    if derivative:
        with pytest.raises(RuntimeError, match="vb_forward_fragments_host.*max_edges"):
            eng.forward_fragments_host(c.x0)
