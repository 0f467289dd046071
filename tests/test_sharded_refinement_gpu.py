"""Sharded steps with the per-step hydrogen refinement (vb_set_batch_window, DeviceShard.set_window,
DeviceLangevin.sharded): every rank places and refines the WHOLE fragment batch, then evaluates its own block of it.

On one GPU, several window handles in one process stand in for the ranks and the test does their all-reduce:

1. every window's placed and refined batch is bit-identical to the unwindowed handle's, and the sum of the window
   buffers matches the unwindowed buffer within test_multigpu.py's bars (also in chunks and without graphs);
2. a W = 2 MD run through the phase API stays bit-identical on both handles and follows the unsharded run;
3. a window adds no launch and no kernel, and the (N, 0) window leaves the Chignolin plan as it was;
4. every refusal.

With two or more GPUs a spawned run checks DeviceLangevin.sharded with the engine's own all-reduce."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from ai2bmd_b200 import caph
from ai2bmd_b200.calculator import FragmentCalculator
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import WEIGHTS, load_capped_protein, load_caph_tables, load_fragments, load_protein
from ai2bmd_b200.md import DeviceLangevin
from ai2bmd_b200.nonbonded import synthetic_parameters
from ai2bmd_b200.parallel import DeviceShard

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NAMES = ["chig", "trpcage"]
F_TIE = 5e-2          # forces of protein atoms fed by a fragment on a VecLayerNorm tie: bounded jump only (DESIGN §2)
X_TOL = 2e-5          # tests/test_multigpu.py: sharded vs single-GPU MD after 20 steps
SEED, STEPS = 4, 20


class _Case:
    def __init__(self, name):
        self.name = name
        self.fd, self.pm = load_fragments(name)
        self.x0, self.z, self.recipe = load_protein(name)
        tables, _ = load_caph_tables(name)
        self.pr = caph.build_problem(load_capped_protein(name), self.fd, self.recipe, tables)
        self.nb = synthetic_parameters(self.z, seed=1)
        self.geoms = {"pdb": self.x0,
                      "perturbed": self.x0 + 0.03 * np.random.default_rng(5).standard_normal(self.x0.shape)}


_CASES = {}


def _case(name):
    if name not in _CASES:
        _CASES[name] = _Case(name)
    return _CASES[name]


def _full(c, chunk_atoms=0):
    """The unwindowed handle: the whole batch with the refinement and the whole MM term."""
    return FragmentCalculator(WEIGHTS, "", c.fd, c.pm, c.recipe, caph=c.pr, nonbonded=c.nb, chunk_size=chunk_atoms).engine


def _windows(c, sd, world, chunk_atoms=0):
    """One window handle per rank of `world`, all on this GPU, with the whole recipe, refinement and its MM rows."""
    shards = [DeviceShard(sd, c.fd, c.pm, r, world, 0, native_comm=False, chunk_atoms=chunk_atoms) for r in range(world)]
    for sh in shards:
        sh.set_window(c.fd, c.pm, c.recipe, caph=c.pr, nonbonded=c.nb)
    return shards


def _tied_atoms(c, sd, pos):
    """Protein atoms fed by a fragment on a VecLayerNorm tie at the placed positions `pos` (an unchunked evaluation)."""
    eng = Engine(sd, 0)
    eng.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd))
    eng.forward_host(pos)
    tie_frag = np.unique(c.fd.batch[eng.vecln_near_ties()])
    tie_atoms = np.isin(c.fd.batch, tie_frag)
    tied = np.zeros(c.pm.n_protein, bool)
    tied[c.pm.dst_atom[tie_atoms[c.pm.src_atom]]] = True
    return tied


# ---- 1. the placed batch and the combined buffer ----------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["graph", "chunks", "no_graph"])
@pytest.mark.parametrize("name", NAMES)
def test_windows_place_the_batch_bit_for_bit(real_weights, name, variant):
    c = _case(name)
    N = len(c.fd.z)
    chunk = 60 if variant == "chunks" else 0
    full = _full(c, chunk)
    for world in (2, 3, 4):
        shards = _windows(c, real_weights, world, chunk)
        engines = [full] + [sh.engine for sh in shards]
        if variant == "chunks":
            assert all(e.get_option("chunks") >= 2 for e in engines)
        if variant == "no_graph":
            for e in engines:
                e.set_option("use_graph", 0)
        for sh in shards:
            assert sh.engine.get_option("batch_atoms") == N
            assert sh.engine.get_option("batch_first_atom") == sh.plan.atom_lo
        for geom, x in c.geoms.items():
            E, F = full.forward_fragments_host(x)
            pos = full.debug_read("pos", 0, (N, 3))
            Es, Fs = 0.0, np.zeros_like(F, dtype=np.float64)
            for sh in shards:
                e, f = sh.engine.forward_fragments_host(x)
                assert np.array_equal(sh.engine.debug_read("pos", 0, (N, 3)), pos), (world, geom, sh.plan.rank)
                Es, Fs = Es + e, Fs + f
            tied = _tied_atoms(c, real_weights, pos)
            df = np.abs(Fs - F).max(1)
            print(f"\n{name} {variant} W={world} {geom}: |dE| {abs(Es - E):.2e} eV, |dF| {df[~tied].max():.2e} eV/A "
                  f"(bar {5e-5 + 2e-5 * np.abs(F).max():.2e}), {tied.sum()} tie atoms")
            assert np.isfinite(Fs).all()
            assert abs(Es - E) <= 4e-3 * len(c.fd)
            assert df[~tied].max() <= 5e-5 + 2e-5 * np.abs(F).max()
            assert (df[tied] <= F_TIE).all()
        del shards


# ---- 2. sharded MD through the phase API ------------------------------------------------------------------------------
def _unsharded_run(c):
    dev = DeviceLangevin(None, c.fd, c.pm, c.recipe, c.x0, c.z, friction_per_fs=0.001, seed=SEED, engine=_full(c))
    dev.run(STEPS)
    x, v, step, _ = dev.state()
    assert step == STEPS
    return x, v


def test_sharded_md_through_the_phase_api(real_weights):
    c = _case("chig")
    shards = _windows(c, real_weights, 2)
    devs = [DeviceLangevin(None, None, c.pm, c.recipe, c.x0, c.z, friction_per_fs=0.001, seed=SEED, engine=sh.engine)
            for sh in shards]
    sp = torch.cuda.current_stream().cuda_stream

    def all_reduce():
        total = devs[0].ef + devs[1].ef
        for d in devs:
            d.ef.copy_(total)

    all_reduce()                                      # the start forces: each constructor evaluated its own block
    for _ in range(STEPS):
        for d in devs:
            d.engine.md_kick1(sp)
        for d in devs:
            d.engine.md_eval(sp)
        all_reduce()
        for d in devs:
            d.engine.md_kick2(sp)
    (x0, v0, s0, _), (x1, v1, s1, _) = (d.state() for d in devs)
    assert s0 == s1 == STEPS
    assert np.array_equal(x0, x1) and np.array_equal(v0, v1)
    xa, _ = _unsharded_run(c)
    xb, _ = _unsharded_run(c)
    spread = np.abs(xa - xb).max()
    bar = max(X_TOL, 2 * spread)
    dx = np.abs(x0 - xa).max()
    print(f"\nchig W=2, {STEPS} steps: sharded vs unsharded |dx| {dx:.2e} A; unsharded run-to-run {spread:.2e} A; bar {bar:.2e} A")
    assert np.isfinite(x0).all() and dx <= bar


# ---- 3. launches ------------------------------------------------------------------------------------------------------
# The kernels of one MD step are counted with torch.profiler, in a child process: once the profiler has attached CUPTI to
# a process it stays attached, and the tests that run after these in the same process (the launch counts and timing-
# sensitive trajectories of test_visnet_mode_gpu.py among them) must see the process as they would without them.
def _md_step_kernels(dev):
    """Names of the CUDA kernels one direct (uncaptured) MD step launches, in order, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    dev.engine.set_option("use_graph", 0)
    dev.run(1)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dev.run(1)
        torch.cuda.synchronize()
    dev.engine.set_option("use_graph", 1)
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _profile_md_steps():
    """Run in the child process: the MD-step kernels of a W = 2 window handle with refinement and MM, of the same block
    without a window (the existing sharded path: a sliced recipe, no refinement), of the unwindowed whole batch, and of
    the Chignolin handle with the whole-batch window (N, 0); printed as one JSON line."""
    from ai2bmd_b200.nonbonded import dipeptide_atom_sets, exclusion_table
    from ai2bmd_b200.parallel import mm_rows
    from ai2bmd_b200.pdbfrag import FragmentRecipe
    from ai2bmd_b200.weights import load_state_dict
    sd = load_state_dict(WEIGHTS)
    c = _case("chig")
    r = c.recipe
    sh = DeviceShard(sd, c.fd, c.pm, 0, 2, 0, native_comm=False)
    sh.set_window(c.fd, c.pm, c.recipe, caph=c.pr, nonbonded=c.nb)
    win = DeviceLangevin(None, None, c.pm, c.recipe, c.x0, c.z, seed=SEED, engine=sh.engine)
    ref = DeviceShard(sd, c.fd, c.pm, 0, 2, 0, native_comm=False)
    lo, hi = ref.plan.atom_lo, ref.plan.atom_hi
    ref.engine.set_nonbonded(*c.nb, *exclusion_table(c.pm.n_protein, dipeptide_atom_sets(c.fd, c.recipe, c.pm)),
                             *mm_rows(c.pm.n_protein, 0, 2))
    blk = DeviceLangevin(None, None, c.pm, FragmentRecipe(r.real[lo:hi], r.acc[lo:hi], r.rem[lo:hi], r.blen[lo:hi]),
                         c.x0, c.z, seed=SEED, engine=ref.engine)
    one = DeviceLangevin(None, c.fd, c.pm, c.recipe, c.x0, c.z, seed=SEED, engine=_full(c))
    n0 = DeviceLangevin(None, c.fd, c.pm, c.recipe, c.x0, c.z, seed=1, engine=_whole_batch_window(c, sd))
    out = {k: {"kernels": _md_step_kernels(d), "launches_per_forward": d.engine.launches_per_forward}
           for k, d in (("window", win), ("block", blk), ("whole", one), ("whole_window", n0))}
    print(json.dumps(out))


_PROFILED = {}


def _profiled():
    """The MD-step kernel lists of _profile_md_steps, from one child process per test session."""
    if not _PROFILED:
        code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.dirname(os.path.abspath(__file__))!r}]; "
                "import test_sharded_refinement_gpu as t; t._profile_md_steps()")
        args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
        res = subprocess.run(args, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert res.returncode == 0, res.stderr[-4000:]
        _PROFILED.update(json.loads(res.stdout.strip().splitlines()[-1]))
    return _PROFILED


def test_a_window_adds_no_launch(real_weights):
    """A window handle's evaluation plan is its block's, and its MD step launches what the block's step without a window
    launches plus the one refinement CTA."""
    from collections import Counter
    c = _case("chig")
    sh = DeviceShard(real_weights, c.fd, c.pm, 0, 2, 0, native_comm=False)
    plan = sh.engine.stage_kernels(), sh.engine.launches_per_forward
    sh.set_window(c.fd, c.pm, c.recipe, caph=c.pr, nonbonded=c.nb)
    assert (sh.engine.stage_kernels(), sh.engine.launches_per_forward) == plan
    p = _profiled()
    kw, kb = p["window"]["kernels"], p["block"]["kernels"]
    extra = Counter(kw) - Counter(kb)
    assert not Counter(kb) - Counter(kw) and sum(extra.values()) == 1 and "caph_relax_kernel" in next(iter(extra))
    # placement, refinement, the evaluation, the MM term (two launches) and the two kicks, as on the whole batch
    for k in ("window", "whole"):
        assert len(p[k]["kernels"]) - p[k]["launches_per_forward"] == 6, k


def _whole_batch_window(c, sd):
    """Chignolin's handle as DeviceLangevin makes it, with the window (N, 0) of the whole batch set before the recipe."""
    eng = Engine(sd, 0)
    eng.set_topology(c.fd.z, c.fd.batch, n_graphs=len(c.fd))
    eng.set_protein_map(c.pm.n_protein, c.pm.src_atom, c.pm.dst_atom, c.pm.sign, c.pm.frag_sign)
    eng.forward_host(np.asarray(c.fd.pos, dtype=np.float32))
    eng.set_option("calibrate", 1)
    eng.set_batch_window(len(c.fd.z), 0)
    return eng


def test_the_whole_batch_window_keeps_the_chignolin_plan(real_weights):
    with open(os.path.join(ROOT, "tests", "golden", "chig_fragment_plan.json")) as fh:
        want = json.load(fh)
    c = _case("chig")
    eng = _whole_batch_window(c, real_weights)
    assert eng.get_option("batch_atoms") == len(c.fd.z) and eng.get_option("batch_first_atom") == 0
    DeviceLangevin(None, c.fd, c.pm, c.recipe, c.x0, c.z, seed=1, engine=eng)
    got = [list(k) for k in eng.stage_kernels()]
    assert [(s, k) for s, k, _ in got] == [(s, k) for s, k, _ in want["stage_kernels"]]
    if torch.cuda.get_device_properties(0).multi_processor_count == want["sm_count"]:
        assert got == want["stage_kernels"]
    assert eng.launches_per_forward == want["launches_per_forward"]
    assert len(_profiled()["whole_window"]["kernels"]) == want["md_step_kernels"]


# ---- 4. refusals ------------------------------------------------------------------------------------------------------
def _rc(eng, *args):
    rc = eng.lib.vb_set_batch_window(eng.h, *args)
    return rc, eng.lib.vb_last_error(eng.h).decode()


def test_refusals(real_weights):
    c = _case("chig")
    P, N = c.pm.n_protein, len(c.fd.z)
    sh = DeviceShard(real_weights, c.fd, c.pm, 1, 2, 0, native_comm=False)
    eng, n, a0 = sh.engine, sh.engine.n_atoms, sh.plan.atom_lo
    fresh = Engine(real_weights, 0)
    rc, msg = _rc(fresh, N, 0)
    assert rc == -3 and "vb_set_topology" in msg                                  # no topology
    for bad in ((N, a0 + 1), (N, -1), (n - 1, 0), (N, N)):
        rc, msg = _rc(eng, *bad)
        assert rc == -1 and "do not lie in a batch" in msg, bad                 # a window outside the batch
    with pytest.raises(RuntimeError, match="is not a fragment atom"):
        eng.set_caph(c.pr)                                                       # the whole problem needs the window
    eng.set_batch_window(N, a0)
    assert (eng.get_option("batch_atoms"), eng.get_option("batch_first_atom")) == (N, a0)
    eng.set_batch_window(N, a0)                                                  # may be set again while nothing uses it
    r = c.recipe
    # after the recipe, the refinement or vb_md_setup
    eng.set_fragment_recipe(r.real, r.acc, r.rem, r.blen)
    rc, msg = _rc(eng, N, a0)
    assert rc == -3 and "set the window first" in msg
    eng.set_topology(sh.plan.local_fragments(c.fd).z, sh.plan.local_fragments(c.fd).batch)   # drops the window
    assert (eng.get_option("batch_atoms"), eng.get_option("batch_first_atom")) == (n, 0)
    m = sh.plan.local_map
    eng.set_protein_map(P, m.src_atom, m.dst_atom, m.sign, m.frag_sign)
    eng.set_batch_window(N, a0)
    eng.set_caph(c.pr)
    rc, msg = _rc(eng, N, a0)
    assert rc == -3 and "set the window first" in msg
    eng.set_topology(sh.plan.local_fragments(c.fd).z, sh.plan.local_fragments(c.fd).batch)
    eng.set_protein_map(P, m.src_atom, m.dst_atom, m.sign, m.frag_sign)
    eng.set_batch_window(N, a0)
    ef = torch.zeros(3 * P + 1, device="cuda")
    eng.md_setup(np.ones(P), r.real, r.acc, r.rem, r.blen, 0.1, 0.025, 0.0, 0, ef.data_ptr())
    rc, msg = _rc(eng, N, a0)
    assert rc == -3 and "set the window first" in msg
    # the (n, 0) window is no window; a window refuses the un-fragmented step, and an un-fragmented handle a window
    eng.set_topology(c.z, np.zeros(P, np.int64), n_graphs=1)
    eng.set_batch_window(P + 5, 5)
    assert eng.get_option("batch_atoms") == P + 5
    with pytest.raises(RuntimeError, match="batch window"):
        eng.md_setup_unfragmented(np.ones(P), 0.1, 0.025, 0.0, 0, ef.data_ptr())
    eng.set_batch_window(P, 0)
    assert (eng.get_option("batch_atoms"), eng.get_option("batch_first_atom")) == (P, 0)
    eng.md_setup_unfragmented(np.ones(P), 0.1, 0.025, 0.0, 0, ef.data_ptr())
    rc, msg = _rc(eng, P + 5, 5)
    assert rc == -3 and "un-fragmented" in msg


# ---- two or more GPUs: DeviceLangevin.sharded with the engine's own all-reduce ----------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out):
    import torch.distributed as dist
    from ai2bmd_b200.weights import load_state_dict
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    sd = load_state_dict(WEIGHTS)
    c = _Case("chig")
    md = DeviceLangevin.sharded(sd, c.fd, c.pm, c.recipe, c.x0, c.z, dist.group.WORLD, caph=c.pr, nonbonded=c.nb,
                                device=rank, friction_per_fs=0.001, seed=SEED)
    md.run(STEPS)
    x, v, step, _ = md.state()
    xs = [torch.empty(x.size, dtype=torch.float64, device="cuda") for _ in range(world)]
    vs = [torch.empty(v.size, dtype=torch.float64, device="cuda") for _ in range(world)]
    dist.all_gather(xs, torch.from_numpy(x.reshape(-1)).cuda())
    dist.all_gather(vs, torch.from_numpy(v.reshape(-1)).cuda())
    if rank == 0:
        np.savez(out, x=x, step=step, native=md._native_comm,
                 identical=all(bool((a == xs[0]).all()) for a in xs) and all(bool((a == vs[0]).all()) for a in vs))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs")
def test_sharded_langevin_on_several_gpus(tmp_path):
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 4)
    out = str(tmp_path / "ranks.npz")
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    r = np.load(out)
    assert bool(r["native"]) and bool(r["identical"]) and int(r["step"]) == STEPS
    c = _case("chig")
    xa, _ = _unsharded_run(c)
    xb, _ = _unsharded_run(c)
    bar = max(X_TOL, 2 * np.abs(xa - xb).max())
    dx = np.abs(r["x"] - xa).max()
    print(f"\nchig W={world}, {STEPS} steps: sharded vs single GPU |dx| {dx:.2e} A, bar {bar:.2e} A")
    assert dx <= bar
