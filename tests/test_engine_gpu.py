"""Parity of the CUDA engine (through the C ABI) with the oracle and the committed golden vectors.

Stated tolerances (fp32 end to end; the reference's own scatter atomics are order-nondeterministic at this
level, and the fp32 oracle itself sits 3e-3 eV / 9e-6 eV/A from the fp64 anchor on these inputs):
  neighbour lists  bit-exact
  energy/fragment  |dE| <= max(4e-3 eV, 2 ulp(E)) against the fp64 anchor; 4 ulp(E) against fp32 golden vectors
                   (both sides carry their own fp32 rounding of an O(2e4 eV) sum; 1 ulp = 2e-3 eV there)
  forces           |dF| <= 5e-5 eV/A + 2e-5 * max|F|
"""
import numpy as np
import pytest
import torch

from ai2bmd_b200.calculator import DLBondedCalculator, DipeptideBondedCombiner, ViSNetCalculator, ViSNetModel
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import load_fragments
from ai2bmd_b200.fragment_data import FragmentData
from ai2bmd_b200.parallel import combine_local
from ai2bmd_b200.pdbfrag import single_graph
from ai2bmd_b200.synth import synthetic_batch, synthetic_protein_map
from oracle import visnet_ref as O

pytestmark = pytest.mark.gpu


def e_tol(e, ulps=2):
    return np.maximum(4e-3, ulps * np.spacing(np.abs(e).astype(np.float32)))


def f_tol(f):
    return 5e-5 + 2e-5 * np.abs(f).max()


@pytest.fixture(scope="module")
def model(real_weights):
    return ViSNetModel(real_weights, device="cuda:0")


def _case(r, key):
    z, pos, batch = r[f"{key}_z"], r[f"{key}_pos"], r[f"{key}_batch"]
    g = int(batch.max()) + 1
    start = np.searchsorted(batch, np.arange(g))
    end = np.searchsorted(batch, np.arange(g), side="right")
    return FragmentData(z, pos, start, end, batch)


@pytest.mark.parametrize("name", ["chig", "trpcage", "ww", "abd"])
def test_neighbour_list_bit_exact(model, name):
    fd, _ = load_fragments(name)
    model.dl_potential_loader(fd)
    slots, deg = model.engine.get_edges()
    s_ref, d_ref = O.radius_graph_canonical(fd.pos, fd.batch)
    assert np.array_equal(deg, d_ref)
    assert np.array_equal(slots, s_ref)


def test_neighbour_cap_32_bit_exact(model, reference_outputs):
    fd = _case(reference_outputs, "dense44")
    model.dl_potential_loader(fd)
    slots, deg = model.engine.get_edges()
    assert np.array_equal(slots, reference_outputs["dense44_slots"]) and deg.max() == 32


@pytest.mark.parametrize("key", ["c1_ala", "chig", "trpcage"])
def test_parity_with_reference_golden_vectors(model, reference_outputs, key):
    """Golden vectors were produced by the reference's own model source (tests/golden/make_golden.py)."""
    r = reference_outputs
    e, f = model.dl_potential_loader(_case(r, key))
    assert e.shape == r[f"{key}_ref_e"].shape and f.shape == r[f"{key}_ref_f"].shape
    assert e.dtype == np.float32 and f.dtype == np.float32
    assert (np.abs(e - r[f"{key}_ref_e"]) <= e_tol(r[f"{key}_ref_e"], ulps=4)).all()
    assert np.abs(f - r[f"{key}_ref_f"]).max() <= f_tol(r[f"{key}_ref_f"])
    # and against the fp64 anchor
    assert (np.abs(e - r[f"{key}_e64"]) <= e_tol(r[f"{key}_e64"])).all()
    assert np.abs(f - r[f"{key}_f64"]).max() <= f_tol(r[f"{key}_f64"])


def test_parity_dense_fragment(model, reference_outputs):
    """Over-dense random fragment (deg capped at 32, forces O(1e2)): relative tolerance only."""
    r = reference_outputs
    e, f = model.dl_potential_loader(_case(r, "dense44"))
    assert np.abs(f - r["dense44_f64"]).max() <= 2e-5 * np.abs(r["dense44_f64"]).max() + 5e-5
    assert np.abs(e - r["dense44_e64"]).max() <= 2e-6 * np.abs(r["dense44_e64"]).max() + 4e-3


@pytest.mark.parametrize("edge_tc,tc_rows", [(0, 128), (1, 64), (3, 32), (3, 64), (3, 96), (3, 128)])
@pytest.mark.parametrize("key", ["chig", "dense44"])
def test_parity_every_edge_kernel_variant(real_weights, reference_outputs, key, edge_tc, tc_rows):
    """SIMT and tensor-core (3xTF32) edge stages, every tile length, against the fp64 anchor (same bar as the default)."""
    r = reference_outputs
    fd = _case(r, key)
    eng = Engine(real_weights, 0)
    eng.set_option("edge_tc", edge_tc)
    eng.set_option("tc_rows", tc_rows)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    assert eng.get_option("edge_tc") == edge_tc and eng.get_option("tc_rows") == tc_rows
    e, f = eng.forward_host(fd.pos)
    e64, f64 = r[f"{key}_e64"], r[f"{key}_f64"]
    assert np.abs(f - f64).max() <= 2e-5 * np.abs(f64).max() + 5e-5
    tol = e_tol(e64) if key == "chig" else 2e-6 * np.abs(e64).max() + 4e-3      # same bars as the default-path tests
    assert (np.abs(e.reshape(e64.shape) - e64) <= tol).all()


@pytest.mark.parametrize("key", ["chig", "trpcage", "dense44"])
def test_parity_planned_tile_lengths(real_weights, reference_outputs, key):
    """Default plan: tiles of equal length (a multiple of 16, not necessarily the kernel's compiled capacity) that fill
    whole waves of CTAs (rows dealt to the warps in runs of ceil(nvalid / 16)), first from the 17-edges-per-atom
    estimate, then calibrated to the real edge count."""
    r = reference_outputs
    fd = _case(r, key)
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    e64, f64 = r[f"{key}_e64"], r[f"{key}_f64"]
    seen = []
    for calibrated in (False, True):
        if calibrated:
            eng.set_option("calibrate", 1)
        rows, cap = eng.get_option("tile_rows"), eng.get_option("tc_rows")
        assert 16 <= rows <= cap <= 128 and rows % 16 == 0
        seen.append(rows)
        e, f = eng.forward_host(fd.pos)
        assert np.abs(f - f64).max() <= 2e-5 * np.abs(f64).max() + 5e-5, (calibrated, rows)
        assert (np.abs(e.reshape(e64.shape) - e64) <= 2e-6 * np.abs(e64).max() + 4e-3).all(), (calibrated, rows)
        e2, f2 = eng.forward_host(fd.pos)              # graph replay on re-zeroed accumulators
        assert np.abs(f2 - f).max() <= 2e-5 * max(1.0, np.abs(f2).max()), (calibrated, rows)
    n_edges = int(eng.get_edges()[1].sum())
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert -(-n_edges // seen[1]) <= sms * max(1, -(-n_edges // (sms * 128)))      # the calibrated tiles fill whole waves


@pytest.mark.parametrize("seed", [0, 7])
def test_parity_random_weights(seed, chig):
    fd, _ = chig
    sub = fd[0:6]
    sd = O.random_state_dict(seed)
    oracle = O.OracleViSNet(sd, torch.float64)
    e_ref, f_ref = oracle.energy_and_forces(sub.z, sub.pos, sub.batch)
    m = ViSNetModel({k: v.numpy() for k, v in sd.items()}, device="cuda:0")
    e, f = m.dl_potential_loader(sub)
    assert (np.abs(e - e_ref.numpy()) <= e_tol(e_ref.numpy())).all()
    assert np.abs(f - f_ref.numpy()).max() <= f_tol(f_ref.numpy())


def test_edge_cases_tiny_graphs(real_weights):
    """A single-atom graph (self-loop only), a 3-atom graph, and two atoms beyond the cutoff."""
    z = np.array([8, 8, 1, 1, 6, 6], dtype=np.int64)
    pos = np.array([[0, 0, 0], [10, 0, 0], [10.76, 0.59, 0], [9.24, 0.59, 0], [20, 0, 0], [26, 0, 0]], np.float32)
    batch = np.array([0, 1, 1, 1, 2, 2], dtype=np.int64)
    fd = FragmentData(z, pos, np.array([0, 1, 4]), np.array([1, 4, 6]), batch)
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64)
    e_ref, f_ref = oracle.energy_and_forces(z, pos, batch)
    e, f = ViSNetModel(real_weights, device="cuda:0").dl_potential_loader(fd)
    assert np.isfinite(e).all() and np.isfinite(f).all()
    assert (np.abs(e - e_ref.numpy()) <= e_tol(e_ref.numpy())).all()
    assert np.abs(f - f_ref.numpy()).max() <= f_tol(f_ref.numpy())
    assert np.abs(f[0]).max() == 0 and np.abs(f[4:]).max() == 0      # isolated atoms feel no force


def test_cystine_pair_as_one_graph_with_an_empty_fragment(model, real_weights):
    """Disulfide-bridged dipeptides packed as one (large) graph + the partner's empty slot (distancefrag.py:185-238)."""
    from ai2bmd_b200.fixtures import load_synthetic_cyx
    from ai2bmd_b200.pdbfrag import fragment_protein
    prot, _ = load_synthetic_cyx()
    fd, pm = fragment_protein(prot)
    sizes = fd.end - fd.start
    assert (sizes == 0).any() and sizes.max() > 44
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64)
    e_ref, f_ref = oracle.forward_all(fd) if hasattr(oracle, "forward_all") else oracle.energy_and_forces(fd.z, fd.pos, fd.batch)
    e, f = model.dl_potential_loader(fd)
    assert e.shape == (len(fd), 1)
    er = np.zeros(len(fd)); er[:len(e_ref)] = e_ref.numpy()[:, 0]
    assert (np.abs(e[:, 0] - er) <= e_tol(er)).all() and (e[sizes == 0, 0] == 0).all()
    assert np.abs(f - f_ref.numpy()).max() <= f_tol(f_ref.numpy())
    slots, deg = model.engine.get_edges()
    s_ref, d_ref = O.radius_graph_canonical(fd.pos, fd.batch)
    assert np.array_equal(deg, d_ref) and np.array_equal(slots, s_ref)


def test_batch_composition_independence(model, chig):
    fd, _ = chig
    e_all, f_all = model.dl_potential_loader(fd)
    sub = fd[3:7]
    e_sub, f_sub = model.dl_potential_loader(sub)
    a0, a1 = fd.start[3], fd.end[6]
    assert (np.abs(e_all[3:7] - e_sub) <= e_tol(e_sub)).all()
    assert np.abs(f_all[a0:a1] - f_sub).max() <= 2e-5


def test_graph_replay_equals_eager_and_tile_variants(real_weights, chig):
    fd, _ = chig
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch)
    e0, f0 = eng.forward_host(fd.pos)
    e1, f1 = eng.forward_host(fd.pos)                 # graph replay
    assert np.abs(f0 - f1).max() <= 1e-5 and np.abs(e0 - e1).max() <= 2e-3
    # te_fwd / te_bwd choose the tile length of the SIMT edge kernels, so they follow edge_tc = 0
    for key, val in (("use_graph", 0), ("edge_tc", 0), ("te_fwd", 64), ("te_bwd", 64), ("npw", 2)):
        before = eng.stage_kernels()
        eng.set_option(key, val)
        if key != "use_graph":                        # eager launches instead of a graph replay: the same kernels
            assert eng.stage_kernels() != before, f"{key}={val} changed no kernel"
        e2, f2 = eng.forward_host(fd.pos)
        assert np.abs(f0 - f2).max() <= 2e-5 and (np.abs(e0 - e2) <= e_tol(e0)).all(), key
    assert 15 <= eng.launches_per_forward <= 40


@pytest.mark.parametrize("name", ["ww", "abd"])
def test_parity_ww_abd_against_fp64_oracle(model, real_weights, name):
    """The two larger example proteins (69 / 93 fragments), full energy / force parity against the fp64 oracle."""
    fd, _ = load_fragments(name)
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64)
    e_ref, f_ref = oracle.energy_and_forces(fd.z, fd.pos, fd.batch)
    e, f = model.dl_potential_loader(fd)
    assert (np.abs(e - e_ref.numpy()) <= e_tol(e_ref.numpy())).all()
    assert np.abs(f - f_ref.numpy()).max() <= f_tol(f_ref.numpy())


def test_parity_c5_conformers_against_fp64_oracle(model, real_weights):
    """Config C5 (Protein-Unit conformer batch): 32 of the 2048 conformers against the fp64 oracle."""
    from ai2bmd_b200.synth import conformer_batch
    fd = conformer_batch(32, seed=1)
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64)
    e_ref, f_ref = oracle.energy_and_forces(fd.z, fd.pos, fd.batch)
    e, f = model.dl_potential_loader(fd)
    assert (np.abs(e - e_ref.numpy()) <= e_tol(e_ref.numpy())).all()
    assert np.abs(f - f_ref.numpy()).max() <= f_tol(f_ref.numpy())


@pytest.mark.parametrize("key", ["chig", "trpcage", "dense44"])
def test_tensor_core_node_stage_agrees(real_weights, reference_outputs, key):
    """Node stage as tensor-core GEMM tiles (k_node_tc.cuh, one job per CTA at these sizes) against the fp64 anchor."""
    r = reference_outputs
    fd = _case(r, key)
    eng = Engine(real_weights, 0)
    eng.set_option("node_tc", 1)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    assert eng.get_option("node_tc") == 1
    e, f = eng.forward_host(fd.pos)
    e2, f2 = eng.forward_host(fd.pos)
    assert np.abs(f2 - f).max() <= 2e-5 * max(1.0, np.abs(f).max())
    e64, f64 = r[f"{key}_e64"], r[f"{key}_f64"]
    assert np.abs(f - f64).max() <= 2e-5 * np.abs(f64).max() + 5e-5
    assert (np.abs(e.reshape(e64.shape) - e64) <= 2e-6 * np.abs(e64).max() + 4e-3).all()


def test_tensor_core_node_stage_all_chunks_per_cta(real_weights):
    """A batch large enough that every CTA runs all column chunks of its row tile on one staged A operand (default plan
    of the 512-fragment config) against the SIMT node stage."""
    fd = synthetic_batch(160, seed=5)
    outs = []
    for node_tc in (0, 1):
        eng = Engine(real_weights, 0)
        eng.set_option("node_tc", node_tc)
        eng.set_topology(fd.z, fd.batch)
        outs.append(eng.forward_host(fd.pos))
    (e0, f0), (e1, f1) = outs
    assert np.isfinite(e1).all() and np.isfinite(f1).all()
    assert (np.abs(e1 - e0) <= e_tol(e0)).all()
    assert np.abs(f1 - f0).max() <= f_tol(f0)            # two fp32-level evaluations of jittered conformers (|F| up to tens of eV/A)


def test_trimmed_edge_capacity_overflow_is_reported(real_weights, chig):
    fd, _ = chig
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch, max_edges=1000)            # Chignolin has ~6.7k edges
    with pytest.raises(RuntimeError, match="max_edges"):
        eng.forward_host(fd.pos)
    assert eng.get_option("edge_overflow") == 1
    eng.set_topology(fd.z, fd.batch)                             # full capacity: fine again, flag cleared
    e, f = eng.forward_host(fd.pos)
    assert np.isfinite(f).all() and eng.get_option("edge_overflow") == 0


def test_protein_map_change_invalidates_md_state(real_weights, chig):
    """vb_set_protein_map after vb_md_setup drops the captured step and the MD state (sized by the old map)."""
    from ai2bmd_b200.fixtures import load_protein
    fd, pm = chig
    prot_pos, prot_z, recipe = load_protein("chig")
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch)
    eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
    ef = torch.zeros(3 * pm.n_protein + 1, device="cuda")
    eng.md_setup(np.ones(pm.n_protein), recipe.real, recipe.acc, recipe.rem, recipe.blen, 0.1, 0.025, 0.0, 0, ef.data_ptr())
    eng.md_set_state(prot_pos, np.zeros_like(prot_pos), 0)
    eng.md_eval()
    eng.md_run(2)
    torch.cuda.synchronize()
    eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
    with pytest.raises(RuntimeError, match="vb_md_setup first"):
        eng.md_run(1)
    eng.set_topology(fd.z, fd.batch)                             # ... and a new topology drops the map itself
    pos = torch.from_numpy(fd.pos).cuda()
    with pytest.raises(RuntimeError, match="protein map"):
        eng.forward_protein_device(pos.data_ptr(), ef.data_ptr())


def test_device_pointer_entry_point(real_weights, chig):
    fd, pm = chig
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch)
    e_h, f_h = eng.forward_host(fd.pos)
    pos = torch.from_numpy(fd.pos).cuda()
    e = torch.empty(len(fd), device="cuda")
    f = torch.empty(len(fd.z), 3, device="cuda")
    eng.forward_device(pos.data_ptr(), e.data_ptr(), f.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.abs(e.cpu().numpy() - e_h).max() <= 2e-3 and np.abs(f.cpu().numpy() - f_h).max() <= 1e-5
    # whole-protein reduction on the device == host restatement of the reference combiner
    eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
    ef = torch.empty(3 * pm.n_protein + 1, device="cuda")
    eng.forward_protein_device(pos.data_ptr(), ef.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = combine_local(pm, e_h, f_h)
    assert np.abs(ef.cpu().numpy()[:-1] - ref[:-1]).max() <= 2e-5
    assert abs(float(ef[-1]) - float(ref[-1])) <= 2e-2


def test_bonded_calculator_surface(real_weights, chig, golden_dir):
    import os
    fd, pm = chig
    calc = DLBondedCalculator(os.path.join(golden_dir, "weights_2ef43f29.npz"))
    dip_e, dip_f, an_e, an_f = calc.calculate(fd)
    assert dip_e.shape == (10, 1) and an_e.shape == (9, 1) and dip_f.shape[0] + an_f.shape[0] == 391
    vd, va = fd.vector_split()
    order = np.concatenate([np.flatnonzero(vd), np.flatnonzero(va)])
    inv = np.empty_like(order)
    inv[order] = np.arange(len(order))
    F = DipeptideBondedCombiner.forces_combine(pm.n_protein, dip_f, an_f, inv[pm.src_atom], pm.dst_atom)
    assert F.shape == (175, 3) and np.isfinite(F).all()
    # (the net force is NOT zero: like the reference, the forces on the added cap hydrogens are dropped)
    e_h, f_h = calc.models[0].dl_potential_loader(fd)
    assert np.abs(F - combine_local(pm, e_h, f_h)[:-1].reshape(-1, 3)).max() <= 2e-5


def test_unfragmented_calculator_ase_semantics(real_weights, reference_outputs, golden_dir):
    import os
    r = reference_outputs

    class Atoms:
        numbers = r["c1_ala_z"]
        positions = r["c1_ala_pos"].astype(np.float64)

    calc = ViSNetCalculator(os.path.join(golden_dir, "weights_2ef43f29.npz"), "", device="cuda:0")
    e = calc.get_potential_energy(Atoms)
    f = calc.get_forces(Atoms)                       # second property: served from the cache
    assert e.shape == (1, 1) and f.shape == (22, 3)
    assert np.abs(f - r["c1_ala_ref_f"]).max() <= f_tol(r["c1_ala_ref_f"])


def test_errors_are_loud(real_weights, chig):
    fd, _ = chig
    eng = Engine(real_weights, 0)
    buf = np.zeros((len(fd.z), 3), np.float32)
    with pytest.raises(RuntimeError, match="vb_set_topology"):
        eng._check(eng.lib.vb_forward_host(eng.h, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data), "vb_forward_host")
    with pytest.raises(RuntimeError, match="sorted"):
        eng.set_topology(fd.z, fd.batch[::-1].copy())
    eng.set_topology(fd.z, fd.batch)
    with pytest.raises(ValueError):
        eng.forward_host(fd.pos[:-1])


def test_md_and_nonbonded_errors_are_loud(real_weights, chig):
    from ai2bmd_b200.fixtures import load_protein
    fd, pm = chig
    _, _, recipe = load_protein("chig")
    n = pm.n_protein
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch)
    ef = torch.zeros(3 * n + 1, device="cuda")
    masses = np.ones(n)
    args = (recipe.real, recipe.acc, recipe.rem, recipe.blen, 0.1, 0.025, 0.0, 0, ef.data_ptr())
    with pytest.raises(RuntimeError, match="protein map"):
        eng.md_setup(masses, *args)
    with pytest.raises(RuntimeError, match="vb_md_setup first"):
        eng.md_run(1)
    eng.set_protein_map(n, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
    bad = recipe.real.copy()
    bad[0] = n
    with pytest.raises(RuntimeError, match="recipe index"):
        eng.md_setup(masses, bad, *args[1:])
    with pytest.raises(RuntimeError, match="mass"):
        eng.md_setup(np.zeros(n), *args)
    with pytest.raises(RuntimeError, match="n_protein"):
        eng.md_setup(np.ones(n + 1), *args)
    with pytest.raises(RuntimeError, match="vb_set_nonbonded first"):
        eng.nonbonded_device(ef.data_ptr(), ef.data_ptr())
    q = np.zeros(n, np.float32)
    rowptr = np.zeros(n + 1, np.int32)
    rowptr[1:] = 2
    with pytest.raises(RuntimeError, match="ascending"):
        eng.set_nonbonded(q, q, q, rowptr, np.array([1, 1], np.int32))
    with pytest.raises(RuntimeError, match="protein map"):
        eng.set_nonbonded(np.zeros(n + 1, np.float32), np.zeros(n + 1, np.float32), np.zeros(n + 1, np.float32),
                          np.zeros(n + 2, np.int32), np.zeros(0, np.int32))
    with pytest.raises(RuntimeError, match="unknown key"):
        eng.set_option("tc_rows", 48)


# ---- full-size properties (config C4: 512 fragments, ~14k atoms): no oracle needed -------------------
@pytest.fixture(scope="module")
def c4(real_weights):
    fd = synthetic_batch(512, seed=0)
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch)
    e, f = eng.forward_host(fd.pos)
    return fd, eng, e, f


def test_fullsize_forces_sum_to_zero_per_fragment(c4):
    fd, eng, e, f = c4
    assert np.isfinite(e).all() and np.isfinite(f).all()
    net = np.zeros((len(fd), 3))
    np.add.at(net, fd.batch, f.astype(np.float64))
    assert np.abs(net).max() <= 1e-3                  # translation invariance of every fragment energy
    tq = np.zeros((len(fd), 3))
    np.add.at(tq, fd.batch, np.cross(fd.pos.astype(np.float64), f.astype(np.float64)))
    assert np.abs(tq).max() <= 1e-2                   # rotation invariance (no net torque)


def assert_kinks_on_own_branch(eng, fd, pos, e, f, kink, real_weights):
    """The fragments ``kink`` of the engine's last evaluation (at pos, giving e, f) against the fp64 oracle pinned to the
    VecLayerNorm branch the engine took there (oracle/vecln_branch.py), at the full bars."""
    from oracle.vecln_branch import Candidates, best_branch, engine_vectors
    cand = Candidates(engine_vectors(eng))
    for g in kink:
        s, t = int(fd.start[g]), int(fd.end[g])
        er, fr, _ = best_branch(real_weights, cand, fd.z, pos, s, t, f)
        assert abs(float(e[g]) - er) <= e_tol(er), (g, float(e[g]), er)
        assert np.abs(f[s:t] - fr).max() <= f_tol(fr), (g, np.abs(f[s:t] - fr).max(), f_tol(fr))


def test_fullsize_rigid_motion_equivariance(c4, real_weights):
    fd, eng, e, f = c4
    rng = np.random.default_rng(5)
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if np.linalg.det(q) < 0:
        q[:, 0] *= -1
    pos2 = (fd.pos.astype(np.float64) @ q.T + np.array([3.0, -2.0, 1.0])).astype(np.float32)
    e2, f2 = eng.forward_host(pos2)
    ties2 = eng.vecln_near_ties()
    e1, f1 = eng.forward_host(fd.pos)
    kink = np.union1d(fd.batch[ties2], fd.batch[eng.vecln_near_ties()])   # fragments on a VecLayerNorm argmax/argmin tie
    assert len(kink) <= len(fd) // 20
    keep = ~np.isin(fd.batch, kink)
    assert (np.abs(e2 - e) <= 3 * e_tol(e)).all()
    d = np.abs(f2 - f @ q.T.astype(np.float32)).max(1)
    assert d[keep].max() <= 3e-4                      # fp32 positions re-rounded after the rotation
    # every kink fragment of both inputs, each evaluation on its own branch
    assert_kinks_on_own_branch(eng, fd, fd.pos, e1, f1, kink, real_weights)
    e2, f2 = eng.forward_host(pos2)
    assert_kinks_on_own_branch(eng, fd, pos2, e2, f2, kink, real_weights)
    eng.forward_host(fd.pos)                          # the module's handle ends on the original input, as it started


def test_vecln_tie_is_the_only_plan_dependence(c4, real_weights):
    """Atom 11957 of this batch has two channel norms of its layer-4 vector features equal to 6e-7 relative: the
    VecLayerNorm(max_min) argmax (reference src/ViSNet/model/utils.py:199-215) flips with the rounding order, and with it
    the force on that one fragment.  Every other fragment agrees between the SIMT and the tensor-core node stage to
    3e-4; the tie fragments of each plan match the fp64 oracle pinned to that plan's own branch at the full bars."""
    fd, eng, e, f = c4
    e, f = eng.forward_host(fd.pos)
    ties = eng.vecln_near_ties(rel_gap=5e-6)
    assert 11957 in ties
    eng2 = Engine(real_weights, 0)
    eng2.set_option("node_tc", 0)
    eng2.set_topology(fd.z, fd.batch)
    e2, f2 = eng2.forward_host(fd.pos)
    kink = np.union1d(fd.batch[eng.vecln_near_ties()], fd.batch[eng2.vecln_near_ties()])
    assert fd.batch[11957] in kink
    keep = ~np.isin(fd.batch, kink)
    d = np.abs(f2 - f).max(1)
    assert d[keep].max() <= 3e-4
    assert (np.abs(e2 - e) <= 3 * e_tol(e)).all()
    assert_kinks_on_own_branch(eng, fd, fd.pos, e, f, kink, real_weights)      # tensor-core node stage
    assert_kinks_on_own_branch(eng2, fd, fd.pos, e2, f2, kink, real_weights)   # SIMT node stage


def test_fullsize_fragment_order_independence(c4, real_weights):
    fd, eng, e, f = c4
    perm = np.random.default_rng(6).permutation(len(fd))
    z, pos, batch, sizes = [], [], [], []
    for g_new, g in enumerate(perm):
        s, t = int(fd.start[g]), int(fd.end[g])
        z.append(fd.z[s:t]); pos.append(fd.pos[s:t]); batch.append(np.full(t - s, g_new)); sizes.append(t - s)
    eng2 = Engine(real_weights, 0)
    eng2.set_topology(np.concatenate(z), np.concatenate(batch))
    e2, f2 = eng2.forward_host(np.concatenate(pos))
    assert (np.abs(e2 - e[perm]) <= e_tol(e[perm])).all()
    offs = np.concatenate([[0], np.cumsum(sizes)])
    for g_new, g in enumerate(perm[:64]):
        assert np.abs(f2[offs[g_new]:offs[g_new + 1]] - f[fd.start[g]:fd.end[g]]).max() <= 3e-5


def test_fullsize_subset_matches_oracle(c4, real_weights):
    fd, eng, e, f = c4
    sub = fd[100:104]
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64)
    e_ref, f_ref = oracle.energy_and_forces(sub.z, sub.pos, sub.batch)
    a0, a1 = fd.start[100], fd.end[103]
    assert (np.abs(e[100:104] - e_ref.numpy()[:, 0]) <= e_tol(e_ref.numpy()[:, 0])).all()
    assert np.abs(f[a0:a1] - f_ref.numpy()).max() <= f_tol(f_ref.numpy())


def test_protein_reduction_fullsize(c4):
    fd, eng, e, f = c4
    pm = synthetic_protein_map(fd)
    eng.set_protein_map(pm.n_protein, pm.src_atom, pm.dst_atom, pm.sign, pm.frag_sign)
    pos = torch.from_numpy(fd.pos).cuda()
    ef = torch.empty(3 * pm.n_protein + 1, device="cuda")
    eng.forward_protein_device(pos.data_ptr(), ef.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = combine_local(pm, e, f)
    assert np.abs(ef.cpu().numpy()[:-1] - ref[:-1]).max() <= 5e-5
