"""The device MD step over a group of window engines in one process (vb_group_md_run / vb_group_md_eval,
EngineGroup.md_run, DeviceLangevin.grouped): the members evaluate their fragment blocks, member 0 integrates.

Cases run with k = 2 and 3 members on cuda:0 and again on k distinct GPUs when that many are visible (skipped otherwise):

1. the step's evaluation: the leader's buffer is the rank-order float32 sum of the members' partials bit for bit, and
   equals the group's FragmentCalculator call at the same positions -- the energy bit for bit, the forces to the bar
   (fp32 atomic sums in no fixed order differ in the last bits between two evaluations) -- with and without refinement
   and MM, and with chunked members;
2. step structure: every recorded frame of 200 Chignolin steps is one host Langevin step, driven by the group
   calculator, from the frame before, and its Epot is a fresh group call at that frame;
3. the trajectory, the reference noise stream, restraints (applied once) against the single-handle DeviceLangevin;
4. the runaway guard freezes the state; the graph cache and the per-member replay path; stale NaN partials;
5. every refusal, including run_segment and the device loop on the leader."""
import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.calculator import FragmentCalculator
from ai2bmd_b200.engine import Engine, EngineGroup
from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.md import FS, KB, DeviceLangevin, Langevin, TemperatureRunawayError, masses_of, philox_normals
from ai2bmd_b200.nonbonded import synthetic_parameters
from ai2bmd_b200.parallel import DeviceShard
from ai2bmd_b200.restraints import hydrogen_bond_springs

pytestmark = pytest.mark.gpu

X_TOL, V_TOL = 2e-5, 2e-4          # tests/test_md_gpu.py: fp32 force rounding amplified by the dynamics
X_SHARDED = 2e-5                   # tests/test_multigpu.py: sharded MD against single-GPU MD after 20 steps


def f_tol(f):
    return 5e-5 + 2e-5 * np.abs(f).max()


class _Case:
    def __init__(self, name):
        self.fd, self.pm = load_fragments(name)
        self.x0, self.z, self.recipe = load_protein(name)
        tables, _ = load_caph_tables(name)
        self.prot = load_capped_protein(name)
        self.pr = caph.build_problem(self.prot, self.fd, self.recipe, tables)
        self.nb = synthetic_parameters(self.z, seed=1)
        self.perturbed = self.x0 + 0.03 * np.random.default_rng(5).standard_normal(self.x0.shape)


_CASES = {}


def _case(name="chig"):
    if name not in _CASES:
        _CASES[name] = _Case(name)
    return _CASES[name]


def _layouts(ks=(2, 3)):
    out = []
    for k in ks:
        out.append(pytest.param(["cuda:0"] * k, id=f"k{k}-cuda0"))
        out.append(pytest.param([f"cuda:{i}" for i in range(k)], id=f"k{k}-distinct",
                                marks=pytest.mark.skipif(torch.cuda.device_count() < k,
                                                         reason=f"{k} distinct GPUs are not visible")))
    return out


LAYOUTS = _layouts()


def _grouped(sd, c, devices, refine=True, mm=False, chunk=0, **kw):
    return DeviceLangevin.grouped(sd, c.fd, c.pm, c.recipe, c.x0, c.z, devices=devices, caph=c.pr if refine else None,
                                  nonbonded=c.nb if mm else None, chunk_atoms=chunk, **kw)


def _single(sd, c, **kw):
    return DeviceLangevin(sd, c.fd, c.pm, c.recipe, c.x0, c.z, caph=c.pr, **kw)


def _partials(md):
    return [sh.engine.debug_read("ef", 0, (3 * md.n + 1,)) for sh in md.shards]


def _rank_sum(parts):
    s = np.zeros_like(parts[0])                       # +0.0f
    for p in parts:
        s = (s + p).astype(np.float32)
    return s


def _ef(md):
    md.stream.synchronize()
    return md.ef.cpu().numpy()


def _eval_at(md, x, v=None):
    md.engine.md_set_state(x, np.zeros_like(x) if v is None else v, 0)
    md._eval()
    return _ef(md)


# ---- 1. the step's evaluation -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,variant", [("chig", "full"), ("chig", "no_refinement"), ("chig", "no_mm"),
                                          ("chig", "chunks"), ("trpcage", "full")])
@pytest.mark.parametrize("devices", LAYOUTS)
def test_eval_equals_the_group_call(real_weights, name, variant, devices):
    c = _case(name)
    md = _grouped(real_weights, c, devices, refine=variant != "no_refinement", mm=variant != "no_mm",
                  chunk=60 if variant == "chunks" else 0)
    if variant == "chunks":
        assert all(sh.engine.get_option("chunks") >= 2 for sh in md.shards)
    ef = _eval_at(md, c.perturbed)
    assert np.array_equal(_rank_sum(_partials(md)).view(np.uint32), ef.view(np.uint32))      # the join, bitwise
    E, F = md.engine_group.forward_fragments_host(c.perturbed)
    assert np.isfinite(ef).all()
    assert np.float32(E) == ef[-1]
    assert np.abs(ef[:-1] - F.reshape(-1)).max() <= f_tol(F)


# ---- 2. step structure and the recorder -------------------------------------------------------------------------------
def test_every_step_is_one_host_step_around_a_group_call(real_weights):
    c = _case()
    devices = ["cuda:0"] * 2
    seed, n = 4, 200
    md = _grouped(real_weights, c, devices, seed=seed)
    calc = FragmentCalculator(WEIGHTS, "", c.fd, c.pm, c.recipe, caph=c.pr, devices=devices)
    x0, v0, s0, _ = md.state()
    md.engine.md_set_recorder(1, n)
    md.run(n)
    fr = md.engine.md_read_frames(0, n)
    assert fr["step"].tolist() == list(range(1, n + 1)) and not fr["halted"].any()
    P = md.n

    def force(x):
        E, F = calc.group.forward_fragments_host(x)
        return E, F.astype(np.float64)

    def src(step):
        xi, eta = philox_normals(seed, step, 3 * P)
        return xi.reshape(P, 3), eta.reshape(P, 3)

    xs, vs = [x0] + list(fr["x"]), [v0] + list(fr["v"])
    for f in range(n):
        host = Langevin(xs[f], c.z, force, seed=seed, normal_source=src)
        host.v, host.nsteps = vs[f].copy(), f
        host.step()
        assert np.abs(host.x - xs[f + 1]).max() <= X_TOL and np.abs(host.v - vs[f + 1]).max() <= V_TOL, f
        assert fr["epot"][f] == np.float64(np.float32(force(xs[f + 1])[0])), f   # the Epot is a fresh group call there
    md.engine.md_set_recorder(0)


# ---- 3. against the single-handle step --------------------------------------------------------------------------------
@pytest.mark.parametrize("devices", LAYOUTS)
def test_trajectory_equals_single_gpu_md(real_weights, devices):
    c = _case()
    one, grp = _single(real_weights, c, seed=0), _grouped(real_weights, c, devices, seed=0)
    one.run(20)
    grp.run(20)
    x1, v1, s1, _ = one.state()
    x, v, s, _ = grp.state()
    assert s == s1 == 20
    assert np.abs(x - x1).max() <= X_SHARDED and np.abs(v - v1).max() <= V_TOL


@pytest.mark.parametrize("devices", _layouts((2,)))
def test_reference_noise_stream(real_weights, devices):
    c = _case()
    one = _single(real_weights, c, seed=9, noise="reference")
    grp = _grouped(real_weights, c, devices, seed=9, noise="reference")
    for n in (7, 5):
        one.run(n)
        grp.run(n)
        assert grp.noise_state() == one.noise_state()
    assert np.abs(grp.state()[0] - one.state()[0]).max() <= X_TOL


@pytest.mark.parametrize("devices", _layouts((2, 3)))
def test_restraints_apply_once(real_weights, devices):
    c = _case()
    ij, k, rt = hydrogen_bond_springs(c.prot)
    h, p = int(ij[0, 0]), int(ij[0, 1])
    x = np.array(c.x0)
    x[h] += 0.5 * (x[h] - x[p]) / np.linalg.norm(x[h] - x[p])          # one spring stretched: active from step 0
    runs = []
    for md in (_single(real_weights, c, seed=2), _grouped(real_weights, c, devices, seed=2)):
        md.engine.md_set_state(x, md.state()[1], 0)
        md.set_restraints(tether_atoms=np.arange(0, md.n, 3), tether_k_kcal=2.0, springs=(ij, k, rt))
        md._eval()
        rf0 = md.engine.md_restraint_forces()
        md.run(15)
        runs.append((md, rf0))
    (one, rf_one), (grp, rf_grp) = runs
    assert rf_grp[-1] > 0 and np.array_equal(rf_grp, rf_one)        # the leader's restraint CTA at the same positions
    ef = _ef(grp)
    assert np.array_equal(_rank_sum(_partials(grp)).view(np.uint32), ef.view(np.uint32))   # no member adds rf to ef
    x1, v1, _, hist1 = one.state(15)
    xg, vg, _, histg = grp.state(15)
    assert np.abs(xg - x1).max() <= X_TOL and np.abs(vg - v1).max() <= V_TOL
    assert np.abs(histg - hist1).max() <= 2e-2                       # restrained Epot: the restraint energy once
    # the preequilibration protocol runs on the group as on one GPU
    grp.preequilibrate(5, schedule=(1.0, 0.5))
    assert grp.state()[2] == 25


# ---- 4. halt, graph cache, replays, stale partials --------------------------------------------------------------------
@pytest.mark.parametrize("devices", _layouts((2,)))
def test_runaway_halt_freezes_the_group_step(real_weights, devices):
    c = _case()
    md = _grouped(real_weights, c, devices, seed=6)
    v_hot = np.random.default_rng(6).standard_normal(c.x0.shape) * np.sqrt(1000.0 * KB / md.masses[:, None])
    md.engine.md_set_state(c.x0, v_hot, 0)
    md._eval()
    with pytest.raises(TemperatureRunawayError):
        md.run_observed(200, 5)
    eng = md.engine
    halt, nf = eng.get_option("md_halt_step"), eng.get_option("md_frames")
    x, v, step, _ = md.state()
    assert step == halt > 0
    md.run(7)
    x2, v2, step2, _ = md.state()
    assert step2 == halt and np.array_equal(x2, x) and np.array_equal(v2, v) and eng.get_option("md_frames") == nf
    E, _ = md.engine_group.forward_fragments_host(x)
    assert _ef(md)[-1] == np.float32(E)                # what the members evaluated behind the halt is the halted state


@pytest.mark.parametrize("devices", LAYOUTS)
def test_graph_cache_and_per_member_replays(real_weights, devices):
    c = _case()
    md = _grouped(real_weights, c, devices, seed=1)
    eng = md.engine
    md.run(2)
    captures = eng.get_option("graph_captures")
    assert eng.get_option("md_group_graph") in (0, 1)
    if len(set(devices)) == 1:
        assert eng.get_option("md_group_graph") == 1     # one GPU: the step is one graph
    md.run(3)
    md.run(1)
    assert eng.get_option("graph_captures") == captures   # repeated runs replay the cached step graph
    md.set_restraints(tether_atoms=np.arange(md.n), tether_k_kcal=1.0)
    md.run(2)
    md.set_restraints()
    md.run(2)
    assert md.state()[2] == 10
    # use_graph = 0 on the leader: kick1, every member's launches, the join and kick2 enqueued one by one
    shards = [DeviceShard(real_weights, c.fd, c.pm, r, len(devices), torch.device(d).index or 0, native_comm=False)
              for r, d in enumerate(devices)]
    for sh in shards:
        sh.set_window(c.fd, c.pm, c.recipe, caph=c.pr)
    lead = shards[0].engine
    lead.set_option("use_graph", 0)
    ref = _grouped(real_weights, c, devices, seed=1)
    x0, v0, _, _ = ref.state()
    ef = torch.zeros(3 * md.n + 1, dtype=torch.float32, device=devices[0])
    lead.md_setup(masses_of(c.z), c.recipe.real, c.recipe.acc, c.recipe.rem, c.recipe.blen, 1.0 * FS, 300.0 * KB,
                  0.001 / FS, 1, ef.data_ptr())
    g = EngineGroup([sh.engine for sh in shards])
    lead.md_set_state(x0, v0, 0)
    stream = torch.cuda.current_stream(torch.device(devices[0])).cuda_stream
    g.md_eval(stream)
    g.md_run(10, stream)
    ref.run(10)
    assert lead.get_option("md_group_graph") == 0
    x, v, s, _ = lead.md_get_state()
    assert s == 10 and np.abs(x - ref.state()[0]).max() <= X_TOL


def _nan_decoy(c):
    """test_fragment_group_gpu.py's decoy: the first HA atom of every residue on its CA."""
    x = c.x0 + 0.2 * np.random.default_rng(9).standard_normal(c.x0.shape)
    for r in np.unique(c.prot.resnums):
        at = [i for i in range(len(c.prot)) if c.prot.resnums[i] == r]
        ca = [i for i in at if c.prot.names[i] == "CA"]
        ha = [i for i in at if c.prot.names[i].startswith("HA")]
        if ca and ha:
            x[ha[0]] = x[ca[0]]
    return x


@pytest.mark.parametrize("devices", _layouts((2,)))
def test_stale_nan_partials(real_weights, devices):
    c = _case()
    clean = _grouped(real_weights, c, devices, seed=3)
    md = _grouped(real_weights, c, devices, seed=3)
    x0, v0, _, _ = md.state()
    e0 = _ef(md)[-1]
    for sh in md.shards:
        sh.engine.forward_fragments_host(_nan_decoy(c))
    assert all(not np.isfinite(p).all() for p in _partials(md))
    ef = _eval_at(md, x0, v0)
    assert np.isfinite(ef).all() and ef[-1] == e0
    md.run(5)
    clean.run(5)
    assert np.abs(md.state()[0] - clean.state()[0]).max() <= X_TOL


# ---- 5. refusals ------------------------------------------------------------------------------------------------------
def _windows(sd, c, k=2):
    shards = [DeviceShard(sd, c.fd, c.pm, r, k, 0, native_comm=False) for r in range(k)]
    for sh in shards:
        sh.set_window(c.fd, c.pm, c.recipe, caph=c.pr)
    return shards


def _md_setup(eng, c, ef):
    eng.md_setup(masses_of(c.z), c.recipe.real, c.recipe.acc, c.recipe.rem, c.recipe.blen, FS, 300.0 * KB, 0.001 / FS, 1,
                 ef.data_ptr())


def test_refusals(real_weights):
    c = _case()
    P = c.pm.n_protein
    ef = torch.zeros(3 * P + 1, dtype=torch.float32, device="cuda:0")
    # a leader without MD state
    g = EngineGroup([sh.engine for sh in _windows(real_weights, c)])
    with pytest.raises(RuntimeError, match="member 0 leads the step and has no MD state"):
        g.md_run(1)
    with pytest.raises(RuntimeError, match="no MD state"):
        g.md_eval()
    # a leader set up un-fragmented
    w = _windows(real_weights, c)
    g = EngineGroup([sh.engine for sh in w])
    w[0].engine.set_topology(c.z, np.zeros(P, dtype=np.int64), n_graphs=1)
    w[0].engine.md_setup_unfragmented(masses_of(c.z), FS, 300.0 * KB, 0.0, 1, ef.data_ptr())
    with pytest.raises(RuntimeError, match="un-fragmented"):
        g.md_run(1)
    # a member with derivative = 0, a member reconfigured, a negative step count
    for change in ("derivative", "option", "md_setup"):
        w = _windows(real_weights, c)
        _md_setup(w[0].engine, c, ef)
        g = EngineGroup([sh.engine for sh in w])
        g.md_run(1)
        if change == "derivative":
            w[1].engine.set_option("derivative", 0)
            with pytest.raises(RuntimeError, match="member 1 has option derivative = 0"):
                g.md_run(1)
        elif change == "option":
            w[1].engine.set_option("calibrate", 1)
            with pytest.raises(RuntimeError, match="member 1 was reconfigured"):
                g.md_run(1)
        else:
            _md_setup(w[0].engine, c, ef)
            with pytest.raises(RuntimeError, match="member 0 was reconfigured"):
                g.md_eval()
    w = _windows(real_weights, c)
    _md_setup(w[0].engine, c, ef)
    g = EngineGroup([sh.engine for sh in w])
    with pytest.raises(RuntimeError, match="negative step count"):
        g.md_run(-1)
    # the device loop on the leader, and run_segment
    md = _grouped(real_weights, c, ["cuda:0"] * 2, seed=1)
    with pytest.raises(RuntimeError, match="leads a group"):
        md.engine.md_run_loop(3)
    with pytest.raises(ValueError, match="run_observed"):
        md.run_segment(3)
    assert md.state()[2] == 0
    # a single handle keeps its device loop
    one = Engine(real_weights, 0)
    assert one.get_option("md_group_graph") == -1
