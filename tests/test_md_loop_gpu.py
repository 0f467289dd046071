"""The device loop (vb_md_run_loop, DeviceLangevin.run_segment): a segment of the MD run as ONE launch of a graph whose
WHILE conditional node repeats the step graph until the step count is reached, the recorder's runaway guard halts, or
the host asks it to stop.

a. the same trajectory as ``run(n)``: Chignolin's full fragment step (hydrogen refinement, restraints, non-bonded term)
   and the un-fragmented ACE-ALA-NME step, both noise streams;
b. a runaway halt ends the launch at the halting step, with no step evaluated behind it;
c. a stop request ends it at the next step boundary, from the same thread or through a KeyboardInterrupt;
d. the loop graph is captured once per handle and I/O binding, whatever the step count, and again exactly when the
   per-step graph is;
e. the refusals: the torch.distributed all-reduce between the kicks, a stop request on a sharded handle;
f. on two or more GPUs, the ranks of a sharded run leave the loop at the same halting step with identical state."""
import os
import socket
import threading
import _thread

import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.fixtures import load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.md import KB, DeviceLangevin, TemperatureRunawayError
from ai2bmd_b200.nonbonded import dipeptide_atom_sets, exclusion_table, synthetic_parameters
from ai2bmd_b200.restraints import hydrogen_bond_springs

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden")
# tests/test_restraints_gpu.py and test_md_recorder_gpu.py, over 200 steps as tests/test_refnoise_gpu.py: the evaluation's
# red.add sums are not run-to-run deterministic, and the dynamics amplify their last-bit differences
X_TOL, V_TOL, E_TOL = 4 * 2e-5, 4 * 2e-4, 2e-2
# Chignolin's full step (tethers at 10 kcal/mol/A^2, springs, refinement, MM term) spreads faster: two plain runs of the
# same start differed in x by up to 1.6e-4 A within 200 steps (a recorded frame, one H100 80GB HBM3); the test prints
# that run-to-run spread beside the run / run_segment difference
X_TOL_FULL = 5 * X_TOL
VB_ERR_STATE = -3
LONG = 200_000          # a segment the stop request ends after about 500 steps; bounded, so a failure cannot run for hours


def _chig_full(real_weights, noise, seed=3):
    """Chignolin with every part of the fragment step set: hydrogen refinement, non-bonded term, tethers and springs."""
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    tables, _ = load_caph_tables("chig")
    pr = caph.build_problem(load_capped_protein("chig"), fd, recipe, tables)
    dev = DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, friction_per_fs=0.01, seed=seed, caph=pr,
                         noise=noise)
    rowptr, col = exclusion_table(dev.n, dipeptide_atom_sets(fd, recipe, pm))
    q, sg, ep = synthetic_parameters(prot_z, seed=3)
    dev.engine.set_nonbonded(q * 0.25, sg, ep, rowptr, col)
    dev._eval()
    ij, k, _ = hydrogen_bond_springs(load_capped_protein("chig"))
    springs = (ij, k, np.linalg.norm(prot_pos[ij[:, 1]] - prot_pos[ij[:, 0]], axis=1) - 0.02)
    dev.set_restraints(tether_atoms=np.flatnonzero(prot_z > 1), tether_k_kcal=10, springs=springs)
    return dev


def _ace(real_weights, noise, seed=3):
    g = np.load(os.path.join(GOLDEN, "reference_visnet_mode.npz"))
    return DeviceLangevin.unfragmented(real_weights, g["c1_z"], g["c1_pos"].astype(np.float64), friction_per_fs=0.01,
                                       seed=seed, noise=noise)


def _chig(real_weights, seed=6, **kw):
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    return DeviceLangevin(real_weights, fd, pm, recipe, prot_pos, prot_z, seed=seed, **kw)


def _hot(dev, seed=6):
    """A 1000 K start at 300 K: the recorder's guard (1.5 T0) fires on an early record step."""
    x, _, _, _ = dev.state()
    v = np.random.default_rng(seed).standard_normal(x.shape) * np.sqrt(1000.0 * KB / dev.masses[:, None])
    dev.engine.md_set_state(x, v, 0)
    dev._eval()
    return x, v


# ---- a. the same trajectory ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("noise", ["philox", "reference"])
@pytest.mark.parametrize("system", ["chig_full", "ace_unfragmented"])
def test_segment_equals_run(real_weights, system, noise):
    make = _chig_full if system == "chig_full" else _ace
    n, every = 200, 10
    a, b, c = make(real_weights, noise), make(real_weights, noise), make(real_weights, noise)
    for dev in (a, b, c):
        dev.engine.md_set_recorder(every, 32, 0.0)
    a.run(n)
    ran = b.run_segment(n)
    c.run(n)                                    # a second plain run: the spread the evaluation's atomics alone give
    xa, va, sa, ha = a.state(n_hist=n)
    xb, vb, sb, hb = b.state(n_hist=n)
    xc, vc, _, _ = c.state()
    assert ran == n == b.engine.md_loop_iterations() and sa == sb == n
    if noise == "reference":
        assert a.noise_state() == b.noise_state()
    nf = n // every
    assert a.engine.get_option("md_frames") == b.engine.get_option("md_frames") == nf
    fa, fb = a.engine.md_read_frames(0, nf), b.engine.md_read_frames(0, nf)
    assert fa["step"].tolist() == fb["step"].tolist() == [every * (i + 1) for i in range(nf)]
    fc = c.engine.md_read_frames(0, nf)
    print(f"{system} {noise}: run vs run_segment |dx| {np.abs(xa - xb).max():.2e} (frames {np.abs(fa['x'] - fb['x']).max():.2e}) "
          f"|dv| {np.abs(va - vb).max():.2e} |dE| {np.abs(ha - hb).max():.2e}; run vs run |dx| {np.abs(xa - xc).max():.2e} "
          f"(frames {np.abs(fa['x'] - fc['x']).max():.2e}) |dv| {np.abs(va - vc).max():.2e} after {n} steps")
    x_tol = X_TOL_FULL if system == "chig_full" else X_TOL
    e_tol = E_TOL if system == "chig_full" else max(E_TOL, 4 * float(np.spacing(np.float32(abs(ha[0])))))
    assert np.abs(xa - xb).max() <= x_tol and np.abs(va - vb).max() <= V_TOL
    assert np.abs(ha - hb).max() <= e_tol
    assert np.abs(fa["x"] - fb["x"]).max() <= x_tol and np.abs(fa["v"] - fb["v"]).max() <= V_TOL
    # a plain run continues from where the segment stopped
    a.run(5)
    b.run(5)
    assert a.state()[2] == b.state()[2] == n + 5


# ---- b. a runaway halt ends the launch -----------------------------------------------------------------------------
def test_halt_ends_the_loop_without_dead_steps(real_weights):
    dev = _chig(real_weights, temperature_K=300.0)
    x0, v0 = _hot(dev)
    eng = dev.engine
    eng.md_set_recorder(5, 64, 1.5)
    with pytest.raises(TemperatureRunawayError) as err:
        dev.run_segment(10_000)
    halt, nf = eng.get_option("md_halt_step"), eng.get_option("md_frames")
    fr = eng.md_read_frames(0, nf)
    assert halt > 0 and halt == fr["step"][-1] == 5 * nf and fr["halted"].tolist() == [0] * (nf - 1) + [1]
    assert f"at step {halt}:" in str(err.value)
    assert eng.md_loop_iterations() == halt - 0             # every iteration ran a step up to the halting one, no more
    x, v, step, _ = dev.state()
    assert step == halt and np.array_equal(x, fr["x"][-1]) and np.array_equal(v, fr["v"][-1])
    # halted: the next launch runs no iteration and raises again
    with pytest.raises(TemperatureRunawayError):
        dev.run_segment(50)
    assert eng.md_loop_iterations() == 0
    x2, v2, step2, _ = dev.state()
    assert step2 == halt and np.array_equal(x2, x) and np.array_equal(v2, v)
    # a new state lifts the halt
    eng.md_set_state(x, v * 0.5, step)
    dev._eval()
    assert dev.run_segment(4) == 4 and dev.state()[2] == halt + 4


def test_halt_step_matches_run_observed(real_weights):
    """The loop halts at the step run_observed reports for the same start."""
    a, b = _chig(real_weights), _chig(real_weights)
    _hot(a)
    _hot(b)
    with pytest.raises(TemperatureRunawayError):
        a.run_observed(400, 5)
    b.engine.md_set_recorder(5, 128, 1.5)
    with pytest.raises(TemperatureRunawayError):
        b.run_segment(400)
    assert a.engine.get_option("md_halt_step") == b.engine.get_option("md_halt_step") == b.state()[2]


# ---- c. a stop request ends the launch -----------------------------------------------------------------------------
def test_stop_request(real_weights):
    dev = _chig(real_weights)
    eng, sp = dev.engine, dev.stream.cuda_stream
    assert dev.run_segment(0) == 0 and dev.state()[2] == 0          # max_steps = 0 runs nothing
    start = dev.state()[2]
    eng.md_run_loop(LONG, sp)
    threading.Event().wait(0.5)
    dev.request_stop()
    done = torch.cuda.Event()
    done.record(dev.stream)
    for _ in range(600):                                            # returns within a step or so of the request
        if done.query():
            break
        threading.Event().wait(0.1)
    assert done.query(), "the loop did not stop"
    ran = eng.md_loop_iterations()
    x, v, step, _ = dev.state()
    assert 0 < ran < LONG and step == start + ran
    dev.run(5)                                                      # a plain run continues from that step
    assert dev.state()[2] == step + 5
    # a request made before a launch does not stop it
    dev.request_stop()
    assert dev.run_segment(6) == 6 and dev.state()[2] == step + 11


def test_keyboard_interrupt_stops_at_a_step_boundary(real_weights):
    dev = _chig(real_weights)
    assert dev.run_segment(1) == 1                                  # the loop graph is captured here, not under the timer
    start = dev.state()[2]
    timer = threading.Timer(0.5, _thread.interrupt_main)
    timer.start()
    try:
        with pytest.raises(KeyboardInterrupt):
            dev.run_segment(LONG)
    finally:
        timer.cancel()
    ran = dev.engine.md_loop_iterations()
    _, _, step, _ = dev.state()
    assert 0 < ran < LONG and step == start + ran
    dev.run(3)
    assert dev.state()[2] == step + 3


# ---- d. graph captures ---------------------------------------------------------------------------------------------
def test_loop_graph_is_captured_once_per_binding(real_weights):
    dev = _chig(real_weights)
    eng = dev.engine
    x, v, _, _ = dev.state()

    def captures(fn):
        c0 = eng.get_option("graph_captures")
        fn()
        dev.state()
        return eng.get_option("graph_captures") - c0

    assert captures(lambda: dev.run_segment(3)) == 1
    for n in (7, 0, 1, 12):                                         # the step count is not part of the graph
        assert captures(lambda: dev.run_segment(n)) == 0
    assert captures(lambda: dev.run(2)) == 1 and captures(lambda: dev.run(2)) == 0
    # md_set_state: neither graph is captured again
    eng.md_set_state(x, v, 100)
    assert captures(lambda: dev.run(1)) == 0 and captures(lambda: dev.run_segment(2)) == 0
    assert dev.state()[2] == 103
    # restraints, recorder on, recorder off: each drops both graphs, and each is captured again once
    for change in (lambda: dev.set_restraints(tether_atoms=np.arange(dev.n), tether_k_kcal=1.0),
                   lambda: eng.md_set_recorder(4, 8, 0.0), lambda: eng.md_set_recorder(0)):
        change()
        assert captures(lambda: dev.run(1)) == 1 and captures(lambda: dev.run_segment(3)) == 1
        assert captures(lambda: dev.run(1)) == 0 and captures(lambda: dev.run_segment(3)) == 0
    assert eng.get_option("use_pdl") == 0 and eng.get_option("md_loop_pdl") == 0     # the default body has no PDL edges


def test_loop_with_pdl_option(real_weights):
    """With option use_pdl the conditional body accepts programmatic edges on the H100 (DESIGN section 7): the loop
    graph is captured with them (md_loop_pdl = 1, no fallback capture), and runs the same steps."""
    a, b = _chig(real_weights, friction_per_fs=0.01), _chig(real_weights, friction_per_fs=0.01)
    assert b.run_segment(1) == 1 and b.engine.get_option("md_loop_pdl") == 0
    c0 = b.engine.get_option("graph_captures")
    b.engine.set_option("use_pdl", 1)                   # drops the cached graphs: the next loop is captured again
    a.run(1)
    assert b.run_segment(40) == 40
    assert b.engine.get_option("graph_captures") == c0 + 1
    assert b.engine.get_option("use_pdl") == 1 and b.engine.get_option("md_loop_pdl") == 1
    a.run(40)
    xa, va, sa, _ = a.state()
    xb, vb, sb, _ = b.state()
    assert sa == sb == 41 and np.abs(xa - xb).max() <= X_TOL and np.abs(va - vb).max() <= V_TOL


# ---- e. refusals ---------------------------------------------------------------------------------------------------
def test_refusals(real_weights):
    dev = _chig(real_weights)
    eng = dev.engine
    with pytest.raises(ValueError, match="n_steps"):
        dev.run_segment(-1)
    with pytest.raises(RuntimeError, match="negative step count"):
        eng.md_run_loop(-1)
    # the torch.distributed path (a group without the engine's all-reduce) all-reduces between the kicks
    dev.group = object()
    with pytest.raises(ValueError, match="torch.distributed"):
        dev.run_segment(5)
    dev.group = None
    # the caller's all-reduce (comm_auto = 0) refused by the library too
    h = eng.comm_init(0, 1, 3 * dev.n + 1)
    eng.comm_connect([h])
    eng.set_option("comm_auto", 0)
    with pytest.raises(RuntimeError, match="comm_auto = 0"):
        eng.md_run_loop(5)
    eng.set_option("comm_auto", 1)
    # a stop request on one rank of several
    eng.comm_init(0, 2, 3 * dev.n + 1)
    rc = eng.lib.vb_md_request_stop(eng.h)
    assert rc == VB_ERR_STATE and "different steps" in eng.lib.vb_last_error(eng.h).decode()
    with pytest.raises(RuntimeError, match="vb_md_request_stop"):
        dev.request_stop()


# ---- f. several GPUs -----------------------------------------------------------------------------------------------
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
    sd = load_state_dict(os.path.join(GOLDEN, "weights_2ef43f29.npz"))
    fd, pm = load_fragments("chig")
    prot_pos, prot_z, recipe = load_protein("chig")
    sh = DeviceShard(sd, fd, pm, rank, world, rank, native_comm=True)
    lo, hi = sh.plan.atom_lo, sh.plan.atom_hi
    rec = FragmentRecipe(recipe.real[lo:hi], recipe.acc[lo:hi], recipe.rem[lo:hi], recipe.blen[lo:hi])
    md = DeviceLangevin(None, None, pm, rec, prot_pos, prot_z, dt_fs=1.0, temperature_K=300.0, friction_per_fs=0.001, seed=0,
                        device=rank, group=dist.group.WORLD, engine=sh.engine)
    eng = md.engine
    ran_plain = md.run_segment(8)
    v_hot = np.random.default_rng(1).standard_normal(prot_pos.shape) * np.sqrt(1000.0 * KB / md.masses[:, None])
    eng.md_set_state(prot_pos, v_hot, 0)
    eng.md_set_recorder(3, 64, 1.5)
    md._eval()
    raised = False
    try:
        md.run_segment(10_000)
    except TemperatureRunawayError:
        raised = True
    halt, iters = eng.get_option("md_halt_step"), eng.md_loop_iterations()
    x, v, step, _ = md.state()
    stop_rc = eng.lib.vb_md_request_stop(eng.h)
    blob = np.concatenate([[float(halt), float(iters), float(step)], x.reshape(-1), v.reshape(-1)])
    t = torch.from_numpy(blob).to(torch.device("cuda", rank))
    gathered = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(gathered, t)
    if rank == 0:
        np.savez(out, identical=all(bool((g == t).all()) for g in gathered), halt=halt, iters=iters, step=step,
                 raised=raised, ran_plain=ran_plain, native=md._native_comm, stop_rc=stop_rc)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs")
def test_ranks_leave_the_loop_together(tmp_path):
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 8)
    out = str(tmp_path / "ranks.npz")
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    r = np.load(out)
    assert bool(r["native"]) and int(r["ran_plain"]) == 8
    assert bool(r["raised"]) and bool(r["identical"])               # halt step, iterations and state on every rank
    halt = int(r["halt"])
    assert halt > 0 and halt % 3 == 0 and int(r["step"]) == halt == int(r["iters"])
    assert int(r["stop_rc"]) == VB_ERR_STATE
