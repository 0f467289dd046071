"""The reference's noise stream on the host: numpy's ziggurat tables recovered through the public API, the sequential
restatement of ``random_standard_normal``, the device kernel's window scheme, PCG64 jump-ahead, and the reference's own
``RNGPool`` order (golden ``reference_rngpool.npz``, made by ``tests/golden/make_rngpool.py``)."""
import os

import numpy as np
import pytest

from ai2bmd_b200 import refnoise as R
from ai2bmd_b200.md import Langevin

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_rngpool.npz")
SEEDS = (0, 1, 2, 7, 42, 12345, 2**31 - 1, 2**63 + 11)


def test_sequential_restatement_equals_numpy_over_1e7_normals():
    n = 1_250_000
    tails = slows = 0
    for seed in SEEDS:
        s, inc = R.pcg_state(seed)
        raw, _ = R.pcg_raw(s, inc, n + n // 20 + 1000)
        out, used = R.normals_from_raw(raw, n)
        g = np.random.default_rng(seed)
        want = g.standard_normal(n)
        assert np.array_equal(out.view(np.uint64), want.view(np.uint64)), seed
        assert R.pcg_advance(s, inc, used) == int(g.bit_generator.state["state"]["state"]), seed
        cost, val = R.attempts(raw[:used])
        starts = R.attempt_starts(cost, val)
        tails += int((cost[starts] >= 3).sum())
        slows += int((cost[starts] == 2).sum())
    print(f"measured {len(SEEDS) * n} normals: {tails} from the idx-0 tail, {slows} slow-path attempts")
    assert tails >= 100


def test_jump_ahead_equals_pcg64_advance():
    rng = np.random.default_rng(3)
    for seed in SEEDS[:4]:
        s, inc = R.pcg_state(seed)
        for k in [0, 1, 2, 31, 32768, 2**40 + 5] + [int(v) for v in rng.integers(0, 2**62, 4)]:
            bg = np.random.PCG64(seed)
            bg.advance(k)
            assert R.pcg_advance(s, inc, k) == int(bg.state["state"]["state"]), (seed, k)
    s, inc = R.pcg_state(5)
    raw, after = R.pcg_raw(s, inc, 10)
    assert after == R.pcg_advance(s, inc, 10) and int(raw[0]) == R.pcg_output(R.pcg_advance(s, inc, 1))


def _raw_for(tab, rng, kind, idx=None):
    """A raw draw whose attempt is fast, slow (idx > 0, rabs >= ki) or an idx-0 tail start."""
    if kind == "fast":
        i = int(rng.integers(2, 256)) if idx is None else idx
        rabs = int(rng.integers(0, max(int(tab["ki"][i]), 1)))
    else:
        i = (int(rng.integers(1, 256)) if idx is None else idx) if kind == "slow" else 0
        rabs = int(rng.integers(int(tab["ki"][i]), 1 << 52))
    return np.uint64(i | (int(rng.integers(0, 2)) << 8) | (rabs << 9))


def _forced_stream(m, rng, plant):
    """A real PCG64 stream with planted attempts: plant(raw, W, T, C) edits it in place."""
    s, inc = R.pcg_state(int(rng.integers(0, 2**31)))
    raw, _ = R.pcg_raw(s, inc, 4 * m + 40000)
    W = R.window_size(m)
    T = min(R.WIN_THREADS, -(-W // R.WIN_MIN_CHUNK))
    plant(raw, W, T, -(-W // T))
    return raw


@pytest.mark.parametrize("m", [996, 1824, 60000])
def test_window_scheme_equals_the_sequential_stream(m):
    tab = R.tables()
    rng = np.random.default_rng(m)
    U1 = np.uint64((1 << 64) - 1)           # u ~ 1: a long tail round never accepts with the next u tiny
    U0 = np.uint64(5)                        # u = 0

    def boundaries(raw, W, T, C):            # slow and tail attempts on chunk boundaries and at the window end
        for t in range(1, T):
            raw[t * C - 1] = _raw_for(tab, rng, "slow")
            raw[t * C] = _raw_for(tab, rng, "tail" if t % 3 == 0 else "slow")
        raw[W - 1] = _raw_for(tab, rng, "tail")
        raw[W - 2] = _raw_for(tab, rng, "slow")

    def runs(raw, W, T, C):                  # runs of consecutive slow draws, and a long tail loop
        for p in range(10, 40):
            raw[p] = _raw_for(tab, rng, "slow")
        raw[100] = _raw_for(tab, rng, "tail")
        for k in range(12):                  # 12 rejected tail rounds: xx large, yy = 0
            raw[101 + 2 * k], raw[102 + 2 * k] = U1, U0

    def short(raw, W, T, C):                 # so many slow rejections and tails that the window falls short
        for p in range(0, min(W, 3000), 2):
            raw[p] = _raw_for(tab, rng, "slow", idx=255)    # outer layer at rabs ~ max: mostly rejected
            raw[p + 1] = U1

    def crowded(raw, W, T, C):               # more non-fast positions than one window's list holds
        for p in range(0, min(W, 4 * R.WIN_LIST), 3):
            raw[p] = _raw_for(tab, rng, "slow")

    for plant in (boundaries, runs, short, crowded):
        raw = _forced_stream(m, rng, plant)
        want, used = R.normals_from_raw(raw, m)
        got, used_w = R.window_normals(raw, m)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), plant.__name__
        assert used_w == used, plant.__name__
    # the short window really ran a second window
    raw = _forced_stream(m, rng, short)
    assert R.normals_from_raw(raw, m)[1] > R.window_size(m)


def test_host_reference_draws_reproduce_the_golden_rngpool():
    g = np.load(GOLDEN)
    assert str(g["numpy_version"]) == np.__version__ or pytest.skip(f"golden made with numpy {g['numpy_version']}")
    keys = sorted(k[len("state_"):] for k in g.files if k.startswith("state_"))
    assert len(keys) == 4
    for key in keys:
        n, seed = (int(v) for v in key.split("_"))
        hist = [(int(h) << 64) | int(lo) for h, lo in g[f"state_{key}"]]
        inc = (int(g[f"inc_{key}"][0]) << 64) | int(g[f"inc_{key}"][1])
        md = Langevin(np.zeros((n, 3)), np.full(n, 6), lambda x: (0.0, np.zeros_like(x)), seed=seed, noise="reference")
        assert R.pcg_state(seed)[1] == inc
        drawn = []
        for step in range(1, 1001):
            xi, eta = md.normals()
            md.nsteps += 1
            if step <= 4:
                drawn.append(np.stack([xi, eta]))
            # the pool runs two arrays ahead: after step k its generator is where the device is after k + 1 steps
            assert int(md.rng.bit_generator.state["state"]["state"]) == hist[step - 1], (key, step)
        assert np.array_equal(np.stack(drawn), g[f"normals_{key}"]), key
        # the window scheme, step by step from the seed's state, consumes what the pool's generator did
        s, _ = R.pcg_state(seed)
        for step in range(1, 65):
            raw, _ = R.pcg_raw(s, inc, 2 * 3 * n + 400)
            _, used = R.window_normals(raw, 2 * 3 * n)
            s = R.pcg_advance(s, inc, used)
            assert s == hist[step - 1], (key, step)


def test_reference_velocities_are_the_legacy_generator():
    from ai2bmd_b200.md import KB, reference_velocities
    m = np.array([1.008, 12.011, 15.999])
    v = reference_velocities(4, m, 300 * KB)
    assert np.array_equal(v, np.random.RandomState(4).standard_normal((3, 3)) * np.sqrt(300 * KB / m[:, None]))
