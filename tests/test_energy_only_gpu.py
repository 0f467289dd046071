"""Energies without forces: the energy plan (vb_forward_energy / vb_forward_energy_host) and the forward-only workspace
of option "derivative" = 0, the reference's ``ViSNet(derivative=False)`` (``src/ViSNet/model/visnet.py:135-166``).

The energy plan runs the full plan's forward launches with the same kernel choices, so its energies must equal
vb_forward's bit for bit.  That rests on the full plan being bit-reproducible itself: every per-target sum of an edge
stage is either stored or, for a target cut across two tiles, two atomic adds onto zero (which commute).  Each case
checks that premise first; were it to fail, the case's bar becomes the full plan's own run-to-run spread (printed).
"""
import os

import numpy as np
import pytest
import torch

from ai2bmd_b200.calculator import ViSNetCalculator, ViSNetModel
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import load_fragments
from ai2bmd_b200.fragment_data import FragmentData
from ai2bmd_b200.synth import synthetic_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
WEIGHTS = os.path.join(ROOT, "tests", "golden", "weights_2ef43f29.npz")
ADJOINT_MARKS = ("_bwd", "node_tc_kernel<2>", "node_tc_kernel<3>", "node_norm_bwd")   # node_tc_kernel<NT_BWDA / NT_BWDB>
ENERGY_LAUNCHES = {0: 20, 1: 32}     # 5 graph/embedding + 6 x (node, edge) + node 6 + head + finalize; node_tc: 3-launch node stages


def _fd(name):
    if name[0] == "c" and name[1:].isdigit():
        return synthetic_batch(int(name[1:]), seed=5)
    return load_fragments(name)[0]


def _opts(eng, opts):
    for kv in filter(None, opts.split(",")):
        k, v = kv.split("=")
        eng.set_option(k, int(v))


def _handle(weights, fd, derivative, opts=""):
    """An engine on fd with opts, calibrated from one evaluation as the host entry points are."""
    eng = Engine(weights, 0, derivative=derivative)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    _opts(eng, opts)
    if derivative:
        eng.forward_host(fd.pos)
    else:
        eng.energy_host(fd.pos)
    if "tc_rows" not in opts:
        eng.set_option("calibrate", 1)
    return eng


def _plan(eng):
    return [k for _, k, _ in eng.stage_kernels()], eng.get_option("tile_rows"), eng.get_option("tc_rows")


CASES = {
    "chig-default": ("chig", ""),
    "chig-simt-edge": ("chig", "edge_tc=0"),
    "chig-rows32": ("chig", "tc_rows=32"),
    "trpcage-default": ("trpcage", ""),
    "abd-default": ("abd", ""),
    "c160-npw1": ("c160", "npw=1"),
    "c160-default": ("c160", ""),
}


@pytest.mark.parametrize("case", list(CASES))
def test_energies_bit_identical_to_the_full_plan(real_weights, case):
    name, opts = CASES[case]
    fd = _fd(name)
    full = _handle(real_weights, fd, True, opts)
    fwd_only = _handle(real_weights, fd, False, opts)
    e_ref, _ = full.forward_host(fd.pos)
    reps = [full.forward_host(fd.pos)[0] for _ in range(2)]
    premise = all(np.array_equal(e_ref, r) for r in reps)
    spread = max(np.abs(r - e_ref).max() for r in reps)
    # the energy plan makes the full plan's choices: its forward launches are the full plan's first ones
    k_full, k_energy = _plan(full)[0], _plan(fwd_only)[0]
    assert k_energy[:-1] == k_full[:len(k_energy) - 1] and "finalize_kernel" in k_energy[-1]
    assert _plan(full)[1:] == _plan(fwd_only)[1:]
    got = {"energy_host (derivative=1)": full.energy_host(fd.pos), "energy_host (derivative=0)": fwd_only.energy_host(fd.pos)}
    pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
    for label, eng in (("energy_device (derivative=1)", full), ("energy_device (derivative=0)", fwd_only)):
        e = torch.empty(len(fd), device="cuda")
        eng.energy_device(pos.data_ptr(), e.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        got[label] = e.cpu().numpy()
    if premise:
        for label, e in got.items():
            assert np.array_equal(e, e_ref), f"{case}: {label} differs from vb_forward by up to {np.abs(e - e_ref).max():.3e} eV"
    else:
        print(f"{case}: two vb_forward runs differ by up to {spread:.3e} eV; bar = that spread")
        for label, e in got.items():
            assert np.abs(e - e_ref).max() <= spread, label


@pytest.mark.parametrize("key", ["c1_ala", "chig", "trpcage"])
def test_derivative_false_model_against_golden_vectors(reference_outputs, key):
    r = reference_outputs
    z, pos, batch = r[f"{key}_z"], r[f"{key}_pos"], r[f"{key}_batch"]
    g = int(batch.max()) + 1
    fd = FragmentData(z, pos, np.searchsorted(batch, np.arange(g)), np.searchsorted(batch, np.arange(g), side="right"), batch)
    model = ViSNetModel.from_file(model_path=WEIGHTS, device="cuda:0", derivative=False)
    assert model.engine.get_option("derivative") == 0
    e, f = model.dl_potential_loader(fd)
    assert f is None and e.dtype == np.float32 and e.shape == r[f"{key}_ref_e"].shape
    tol = np.maximum(4e-3, 4 * np.spacing(np.abs(r[f"{key}_ref_e"]).astype(np.float32)))   # the golden parity bar
    assert (np.abs(e - r[f"{key}_ref_e"]) <= tol).all()


@pytest.mark.parametrize("node_tc", [0, 1])
def test_energy_plan_has_no_adjoint_launch(real_weights, chig, node_tc):
    fd, _ = chig
    eng = Engine(real_weights, 0, derivative=False)
    eng.set_option("node_tc", node_tc)
    eng.set_topology(fd.z, fd.batch)
    ks = eng.stage_kernels()
    assert not [k for _, k, _ in ks if any(m in k for m in ADJOINT_MARKS)], ks
    assert len(ks) == eng.launches_per_forward == ENERGY_LAUNCHES[node_tc]
    assert [s for s, _, _ in ks][-2:] == ["head", "finalize"]
    # the diagnostics run the energy plan
    pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
    prof = eng.profile_stages(pos.data_ptr(), n_iter=2)
    assert len(prof) == ENERGY_LAUNCHES[node_tc] and all(ms >= 0 for _, ms in prof)
    eng.debug_run(pos.data_ptr(), -1)
    assert np.array_equal(eng.debug_read("energy", 0, (len(fd),)), eng.energy_host(fd.pos))


@pytest.mark.parametrize("name", ["chig", "c512"])
def test_forward_only_arena_is_at_most_a_quarter(real_weights, name):
    fd = synthetic_batch(512, seed=0) if name == "c512" else _fd(name)
    sizes = {}
    for derivative in (True, False):
        eng = Engine(real_weights, 0, derivative=derivative)
        assert eng.get_option("arena_bytes") == 0
        eng.set_topology(fd.z, fd.batch)
        sizes[derivative] = eng.get_option("arena_bytes")
        del eng
    ratio = sizes[False] / sizes[True]
    print(f"{name}: N={len(fd.z)} arena derivative=1 {sizes[True] / 2**20:.1f} MiB, derivative=0 {sizes[False] / 2**20:.1f} MiB, "
          f"ratio {ratio:.3f}")
    assert ratio <= 0.25


def test_refusals_and_errors(real_weights, chig):
    fd, _ = chig
    n, g = len(fd.z), len(fd)
    pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
    e = torch.empty(g, device="cuda")
    f = torch.empty(n, 3, device="cuda")
    eng = Engine(real_weights, 0, derivative=False)
    lib, h = eng.lib, eng.h
    assert lib.vb_forward_energy(h, pos.data_ptr(), e.data_ptr(), None) == -3                # before vb_set_topology
    assert lib.vb_forward_energy_host(h, fd.pos.ctypes.data, np.empty(g, np.float32).ctypes.data) == -3
    eng.set_topology(fd.z, fd.batch)
    assert eng.get_option("derivative") == 0
    assert lib.vb_forward_energy(h, None, e.data_ptr(), None) == -1
    assert lib.vb_forward_energy(h, pos.data_ptr(), None, None) == -1
    assert lib.vb_forward_energy_host(h, None, np.empty(g, np.float32).ctypes.data) == -1
    assert lib.vb_forward_energy_host(h, fd.pos.ctypes.data, None) == -1
    # entries that need forces or the adjoint's buffers
    assert lib.vb_forward(h, pos.data_ptr(), e.data_ptr(), f.data_ptr(), None) == -3
    assert b"derivative" in lib.vb_last_error(h)
    assert lib.vb_forward_host(h, fd.pos.ctypes.data, np.empty(g, np.float32).ctypes.data, np.empty((n, 3), np.float32).ctypes.data) == -3
    assert b"derivative" in lib.vb_last_error(h)
    eng.set_protein_map(n, np.arange(n), np.arange(n), np.ones(n), np.ones(g))
    ef = torch.empty(3 * n + 1, device="cuda")
    assert lib.vb_forward_protein(h, pos.data_ptr(), ef.data_ptr(), None) == -3
    assert b"derivative" in lib.vb_last_error(h)
    with pytest.raises(RuntimeError, match="derivative"):
        eng.md_setup(np.ones(n), np.arange(n), np.zeros(n), np.zeros(n), np.zeros(n), 1.0, 0.0, 0.0, 0, ef.data_ptr())
    for buf in ("P1", "SP", "ATT", "GX", "GVEC", "GF", "GXA", "GQKV", "GVNMSG", "GTU", "eacc", "grbf", "forces"):
        with pytest.raises(RuntimeError, match="derivative"):
            eng.debug_read(buf, 1, (1,))
    eng.energy_host(fd.pos)
    eng.debug_read("X", 6, (n, 128))                       # the last layer of each slot stays readable
    with pytest.raises(RuntimeError, match="derivative"):
        eng.debug_read("X", 2, (n, 128))                   # layer 2's slot now holds layer 6
    # a changed "derivative" drops the topology
    eng.set_option("derivative", 1)
    assert eng.get_option("derivative") == 1 and eng.get_option("arena_bytes") == 0 and eng.launches_per_forward == 0
    assert lib.vb_forward(h, pos.data_ptr(), e.data_ptr(), f.data_ptr(), None) == -3
    assert lib.vb_forward_energy(h, pos.data_ptr(), e.data_ptr(), None) == -3
    eng.set_topology(fd.z, fd.batch)
    eng.forward_host(fd.pos)


def test_trimmed_max_edges_fails_the_energy_entry_like_the_forward_entry(real_weights, chig):
    fd, _ = chig
    few = len(fd.z) * 4                                    # far fewer directed edges than the fragments have
    for derivative in (True, False):
        eng = Engine(real_weights, 0, derivative=derivative)
        eng.set_topology(fd.z, fd.batch, max_edges=few)
        with pytest.raises(RuntimeError, match="max_edges"):
            eng.energy_host(fd.pos)
        if derivative:
            with pytest.raises(RuntimeError, match="max_edges"):
                eng.forward_host(fd.pos)


def test_interleaved_with_the_full_plan(real_weights, chig):
    fd, _ = chig
    n, g = len(fd.z), len(fd)
    ref = _handle(real_weights, fd, True)
    e0, f0 = ref.forward_host(fd.pos)
    fbar = 5e-5 + 2e-5 * np.abs(f0).max()
    pos = torch.from_numpy(np.ascontiguousarray(fd.pos, dtype=np.float32)).cuda()
    st = torch.cuda.current_stream().cuda_stream
    results = {}
    for use_graph in (1, 0):
        eng = _handle(real_weights, fd, True)
        eng.set_option("use_graph", use_graph)
        for it in range(3):
            e, f, ee = torch.empty(g, device="cuda"), torch.empty(n, 3, device="cuda"), torch.empty(g, device="cuda")
            eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), st)
            eng.energy_device(pos.data_ptr(), ee.data_ptr(), st)
            torch.cuda.synchronize()
            e, f, ee = e.cpu().numpy(), f.cpu().numpy(), ee.cpu().numpy()
            assert np.array_equal(e, e0) and np.array_equal(ee, e0), (use_graph, it)
            assert np.abs(f - f0).max() <= fbar, (use_graph, it)
            eh = eng.energy_host(fd.pos)
            e_host, f_host = eng.forward_host(fd.pos)
            assert np.array_equal(eh, e0) and np.array_equal(e_host, e0)
            assert np.abs(f_host - f0).max() <= fbar
        results[use_graph] = (eng.energy_host(fd.pos), eng.forward_host(fd.pos)[0])
    assert all(np.array_equal(a, b) for a, b in zip(results[0], results[1]))


class _Atoms:
    def __init__(self, numbers, positions):
        self.numbers, self.positions = numbers, positions


def test_calculator_without_forces(chig):
    fd, _ = chig
    s, t = int(fd.start[0]), int(fd.end[0])
    atoms = _Atoms(np.asarray(fd.z[s:t]), np.asarray(fd.pos[s:t], dtype=np.float64))
    with_f = ViSNetCalculator(WEIGHTS, "", device="cuda:0", derivative=True)
    without = ViSNetCalculator(WEIGHTS, "", device="cuda:0", derivative=False)
    assert without.model.engine.get_option("derivative") == 0 and with_f.model.engine.get_option("derivative") == 1
    e1, e0 = with_f.get_potential_energy(atoms), without.get_potential_energy(atoms)
    assert e0.dtype == np.float32 and np.array_equal(e0, e1)
    assert with_f.get_forces(atoms).shape == (t - s, 3)
    with pytest.raises(NotImplementedError):
        without.get_forces(atoms)
