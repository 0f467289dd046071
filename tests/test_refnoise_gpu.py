"""The reference's noise stream generated inside the device MD step (``DeviceLangevin(noise="reference")``, k_md.cuh
``md_refnoise_cta``): the PCG64 state and the normals against numpy, trajectories against a numpy-drawn pool and the
host integrator, and the stream's continuity through pre-equilibration, a recorder halt, a restart and ranks."""
import os

import numpy as np
import pytest
import torch

from ai2bmd_b200 import refnoise as R
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import load_fragments, load_protein
from ai2bmd_b200.md import FS, KB, MASSES, BondedForceField, DeviceLangevin, Langevin, TemperatureRunawayError
from ai2bmd_b200.synth import synthetic_batch, synthetic_protein_map

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_rngpool.npz")
X_TOL, V_TOL = 2e-5, 2e-4          # tests/test_md_gpu.py: fp32 force rounding amplified by the dynamics
# Over 200 steps that amplification alone reaches the bars above: the same handle run twice from the same start with
# bit-identical normals differed by 2.0e-5 A after 200 steps (0 after one), so the 200-step comparisons allow 4x.
X_TOL_200, V_TOL_200 = 4 * X_TOL, 4 * V_TOL
KT = 300.0 * KB


def _numpy_states(seed, n, steps):
    """numpy's default_rng(seed) drawn in RNGPool order: the state after each step, and the last step's (xi, eta)."""
    g = np.random.default_rng(seed)
    states = []
    for _ in range(steps):
        xi, eta = g.standard_normal((n, 3)), g.standard_normal((n, 3))
        states.append(int(g.bit_generator.state["state"]["state"]))
    return states, np.stack([xi, eta])


def _bare(real_weights, P, seed, fr=0.001 / FS):
    """An engine with Chignolin's fragments and an empty protein map of P atoms (ef = 0), MD set up on P atoms."""
    fd = load_fragments("chig")[0]
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    eng.set_protein_map(P, [], [], [], np.zeros(len(fd), np.float32))
    eng.forward_host(np.asarray(fd.pos, dtype=np.float32))
    ef = torch.zeros(3 * P + 1, dtype=torch.float32, device="cuda")
    n = len(fd.z)
    zero = np.zeros(n, np.int32)
    rng = np.random.default_rng(1)
    m = np.array([MASSES[int(a)] for a in rng.choice([1, 6, 7, 8, 16], size=P)])
    eng.md_setup(m, np.arange(n) % P, zero, zero, np.zeros(n, np.float32), FS, KT, fr, seed, ef.data_ptr())
    eng.md_set_state(rng.normal(size=(P, 3)) * 10, rng.normal(size=(P, 3)) * 0.01, 0)
    s0, inc = R.pcg_state(seed)
    eng.md_set_noise(1, s0, inc, R.tables())
    return eng, ef


def _check_normals(got, want, what):
    """Bit-identical except values of the idx-0 tail (|v| > r), within 2 ulp there (the device's log1p)."""
    diff = got != want
    tail = np.abs(want) > R.tables()["r"]
    assert not (diff & ~tail).any(), what
    ulps = np.abs(got.view(np.int64) - want.view(np.int64))
    assert (ulps[diff] <= 2).all(), what
    print(f"measured {what}: {int(tail.sum())} tail values, {int(diff.sum())} differ (max {int(ulps.max())} ulp)")


def _c4_20k_atoms():
    return synthetic_protein_map(synthetic_batch(512, seed=0, min_atoms=20000)).n_protein


@pytest.mark.parametrize("name", ["chig", "trpcage", "c4_20k"])
def test_stream_state_and_normals_equal_numpy(real_weights, name):
    seed = 2**31 - 1 if name == "trpcage" else 0
    P = _c4_20k_atoms() if name == "c4_20k" else len(load_protein(name)[0])
    eng, ef = _bare(real_weights, P, seed)
    want, last = _numpy_states(seed, P, 1000)
    if name != "c4_20k":        # numpy's draws in RNGPool order are the reference's own pool (tests/test_refnoise.py)
        g = np.load(GOLDEN)
        hist = [(int(h) << 64) | int(lo) for h, lo in g[f"state_{P}_{seed}"]]
        assert want == hist[:1000]
    st = torch.cuda.current_stream().cuda_stream
    for k in range(64):
        eng.md_run(1, st)
        assert eng.md_get_noise_state() == want[k], (name, k + 1)
        if k == 0:
            xi, eta = eng.md_get_noise()
            _check_normals(np.stack([xi, eta]), _numpy_states(seed, P, 1)[1], f"{name} step 1 normals")
    eng.md_run(1000 - 64, st)
    assert eng.md_get_noise_state() == want[-1]
    xi, eta = eng.md_get_noise()
    _check_normals(np.stack([xi, eta]), last, f"{name} step 1000 normals")
    _, _, step, _ = eng.md_get_state()
    assert step == 1000


def test_stream_advances_at_friction_zero_and_excludes_a_pool(real_weights):
    eng, ef = _bare(real_weights, 166, 3, fr=0.0)
    eng.md_run(5, torch.cuda.current_stream().cuda_stream)
    assert eng.md_get_noise_state() == _numpy_states(3, 166, 5)[0][-1]
    pool = torch.zeros(2 * 2 * 166 * 3, dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError):
        eng.md_set_normals(pool.data_ptr(), 2)
    eng.md_set_noise(0)
    with pytest.raises(RuntimeError):
        eng.md_get_noise_state()
    eng.md_set_normals(pool.data_ptr(), 2)
    with pytest.raises(RuntimeError):
        eng.md_set_noise(1, *R.pcg_state(3), R.tables())
    eng.md_set_normals(0, 0)


def _chig():
    fd, pm = load_fragments("chig")
    pos, z, recipe = load_protein("chig")
    return fd, pm, pos, z, recipe


def test_trajectory_equals_a_numpy_pool_and_the_host(real_weights):
    fd, pm, pos, z, recipe = _chig()
    seed, n = 0, len(pos)
    ref = DeviceLangevin(real_weights, fd, pm, recipe, pos, z, seed=seed, noise="reference")
    x0, v0, _, _ = ref.state()
    ef0 = ref.ef.clone()
    assert np.array_equal(v0, Langevin(pos, z, lambda x: (0.0, np.zeros_like(x)), seed=seed, noise="reference").v)
    g = np.random.default_rng(seed)
    pool = np.stack([np.stack([g.standard_normal((n, 3)), g.standard_normal((n, 3))]) for _ in range(200)])
    ref.run(1)
    xa1 = ref.state()[0]
    ref.run(199)
    xa, va, _, _ = ref.state()
    # the same handle from the same start, fed numpy's draws as a pool
    ref.engine.md_set_noise(0)
    ref.set_normals(pool)
    ref.engine.md_set_state(x0, v0, 0)
    ref.ef.copy_(ef0)            # the start forces as the first run had them: step 1 then differs only by the normals
    ref.run(1)
    dx1 = np.abs(xa1 - ref.state()[0]).max()
    assert dx1 <= 1e-9, dx1
    ref.run(199)
    xb, vb, _, _ = ref.state()
    print(f"measured against the numpy pool: |dx| {dx1:.2e} after 1 step, {np.abs(xa - xb).max():.2e} after 200")
    assert np.abs(xa - xb).max() <= X_TOL_200 and np.abs(va - vb).max() <= V_TOL_200
    # the host integrator drawing from numpy in RNGPool order
    host = Langevin(pos, z, BondedForceField(real_weights, fd, pm, recipe), seed=seed, noise="reference")
    for _ in range(200):
        host.step()
    print(f"measured against the host: |dx| {np.abs(xa - host.x).max():.2e}, |dv| {np.abs(va - host.v).max():.2e}")
    assert np.abs(xa - host.x).max() <= X_TOL_200 and np.abs(va - host.v).max() <= V_TOL_200


def test_stream_continuity(real_weights):
    fd, pm, pos, z, recipe = _chig()
    n = len(pos)
    want = _numpy_states(5, n, 60)[0]
    md = DeviceLangevin(real_weights, fd, pm, recipe, pos, z, seed=5, noise="reference")
    md.preequilibrate(4, schedule=(10.0, 5.0, 2.0, 1.0, 0.5))
    assert md.noise_state() == want[20 - 1]
    # a noise_state hand-over continues the stream: 20 + 10 + 10 steps equal 20 + 20 unbroken
    x, v, step, _ = md.state()
    saved = md.noise_state()
    md.run(20)
    xa, va, _, _ = md.state()
    assert md.noise_state() == want[40 - 1]
    cont = DeviceLangevin(real_weights, fd, pm, recipe, x, z, seed=5, noise="reference", noise_state=saved,
                          velocities=v, step=step)
    cont.run(10)
    cont2 = DeviceLangevin(real_weights, fd, pm, recipe, cont.state()[0], z, seed=5, noise="reference",
                           noise_state=cont.noise_state(), velocities=cont.state()[1], step=step + 10)
    cont2.run(10)
    xb, vb, _, _ = cont2.state()
    assert cont2.noise_state() == want[40 - 1]
    assert np.abs(xa - xb).max() <= X_TOL and np.abs(va - vb).max() <= V_TOL
    # without noise_state a restart reseeds, as the reference's --restart does
    fresh = DeviceLangevin(real_weights, fd, pm, recipe, x, z, seed=5, noise="reference", velocities=v, step=step)
    fresh.run(1)
    assert fresh.noise_state() == want[0]
    # a recorder halt stops the stream at the halting step
    hot = DeviceLangevin(real_weights, fd, pm, recipe, pos, z, seed=5, noise="reference", velocities=md.state()[1] * 3.0)
    with pytest.raises(TemperatureRunawayError):
        hot.run_observed(50, 5)
    halt = hot.engine.get_option("md_halt_step")
    assert 0 < halt <= 50 and hot.noise_state() == want[halt - 1]
    hot.run(3)
    assert hot.noise_state() == want[halt - 1]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_ranks_generate_the_same_stream(real_weights):
    states = []
    for dev in range(2):
        with torch.cuda.device(dev):
            fd = load_fragments("chig")[0]
            eng = Engine(real_weights, dev)
            eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
            eng.set_protein_map(166, [], [], [], np.zeros(len(fd), np.float32))
            eng.forward_host(np.asarray(fd.pos, dtype=np.float32))
            ef = torch.zeros(3 * 166 + 1, dtype=torch.float32, device=f"cuda:{dev}")
            n = len(fd.z)
            zero = np.zeros(n, np.int32)
            eng.md_setup(np.full(166, 12.011), np.arange(n) % 166, zero, zero, np.zeros(n, np.float32), FS, KT, 0.001 / FS,
                         9, ef.data_ptr())
            eng.md_set_state(np.arange(498.0).reshape(166, 3), np.zeros((166, 3)), 0)
            eng.md_set_noise(1, *R.pcg_state(9), R.tables())
            eng.md_run(100, torch.cuda.current_stream(dev).cuda_stream)
            states.append(eng.md_get_noise_state())
    assert states[0] == states[1] == _numpy_states(9, 166, 100)[0][-1]
