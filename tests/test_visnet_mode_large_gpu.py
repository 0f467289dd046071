"""The reference's un-fragmented ``--mode visnet`` on whole proteins above the launch planner's size rules: whole WW and
whole ABD as ONE graph (tests/golden/reference_visnet_mode_large.npz, tests/golden/make_visnet_mode.py: the reference's
own model source in fp32 on the CPU, and the fp64 oracle).  The neighbour truncation is that of the repo's
``radius_graph`` stand-in (the first 32 candidates by index, oracle/radius_graph.c), not ``torch_cluster``'s: that
ordering stays unpinned (DESIGN section 2).  From the generator:

    case  atoms  edges   most candidates within 5 A  truncated lists  max degree
    ww    571    16,580  63                           354              32
    abd   746    21,839  63                           480              32

So nearly every target has 32 edges (29 on average), against about 17 per atom in fragment batches, and every
per-fragment quantity is one sum over hundreds of atoms.

a. The plan each case runs, uncalibrated (the 17 N edge estimate a handle starts from) and calibrated (the real edge
   count; what ``DeviceLangevin.unfragmented`` and ``ViSNetModel`` run after their first evaluation).  Measured on one
   H100 80GB HBM3 (132 SMs), see PLANS:
       ww   SIMT node stage node_fwd2 / node_bwd2 <8>, te_fwd 32, npw 1; 80-row tiles (tc_rows 96) both ways: 16,580
            edges (+3 %) overflow one wave of 128-row tiles on 132 SMs, and two waves of 80 rows is also what the
            estimate gave, so calibration leaves the plan as it was; 208 tiles over 132 CTAs: several tiles per CTA.
       abd  tensor-core node stage (node_tc_kernel<0..3>, node_norm_fwd / bwd), gxa_parts 3, te_fwd 32, npw 1;
            uncalibrated 128-row tiles (171 tiles over 132 CTAs), calibrated 96-row tiles (228 tiles): several tiles
            per CTA both ways, and calibration changes the tile length.
b. Neighbour lists bit-exact against the golden's.
c. Energy and forces, uncalibrated and calibrated, against the reference golden and the fp64 oracle, through the engine
   and through ``ViSNetModel.dl_potential_loader``, at the bars of test_visnet_mode_gpu.py: 2e-6 |E| + 4e-3 for the
   energy, 5e-5 + 2e-5 max|F| for the forces against the fp64 hand adjoint on the VecLayerNorm(max_min) branch the
   handle took.  Each golden geometry holds one near tie in the fp64 oracle (top-two channel norms within 1e-5,
   relative): WW atom 173 at layer 4 (5.0e-6 apart) and ABD atom 376 at layer 2 (3.7e-6 apart), both far outside the
   3-ulp window in which the engine's branch is open; the engine reports them (Engine.vecln_near_ties) and takes the
   natural channel, as the reference's fp32 forces do (9.2e-6 / 1.0e-5 eV/A from the fp64 oracle), so every force is
   held to the normal bar against the reference too.
d. Every launch of the one-graph plan against the fp64 hand adjoint on the branch the engine took, stage by stage
   (tools/stage_check.py), on a clean workspace and after the dense and NaN decoys, uncalibrated and calibrated: 2e-3 of
   the buffer's largest entry, and the per-fragment bars of test_kernel_variants_gpu.py (here the one fragment is the
   whole protein).
e. The energy plan: a derivative = 0 handle's energy and vb_forward_energy on a derivative = 1 handle equal
   forward_host's energy bit for bit (DESIGN section 4), uncalibrated and calibrated.
f. The device MD step on these plans: 20 steps of DeviceLangevin.unfragmented at friction 0, every step recorded.
   Whole proteins are not compared step for step against md.Langevin (the truncated lists make two trajectories part,
   test_visnet_mode_gpu.py); instead every frame's potential energy equals a fresh ViSNetModel evaluation at its x
   within the energy bar, and one host velocity-Verlet step (md.Langevin's half-kick and drift) from each frame's
   (x, v) with that evaluation's forces reaches the next frame's x within X_TOL of test_md_gpu.py.  So the step
   integrates the evaluation of its own positions (md_place_kernel's cast path at N >= 600 included).  The step
   launches the plan + 3 kernels, as for the smaller inputs (DESIGN section 7).

Worst ratio to each bar, measured on one H100 80GB HBM3 at 700 W (uncalibrated / calibrated where they differ):
   c  ww:  |E - ref| 0.039 of e_bar, |E - e64| 0.017; |F - f64| on the engine's branch 0.111 / 0.114 of f_bar, |F - ref|
           0.115 / 0.117; ViSNetModel 0.111 / 0.109.
      abd: |E - ref| 0.096, |E - e64| 0.011; |F - f64| on the engine's branch 0.130 / 0.128, |F - ref| 0.130;
           ViSNetModel 0.133 / 0.126.  One branch open on every atom of every evaluation.
   d  ww:  buffers 3.2e-5 (0.016 of 2e-3, g_vn_msg at edge_bwd3); per fragment 0.105 of its bar (vn at node_fwd5).
      abd: buffers 4.3e-5 / 3.5e-5 (0.021 / 0.018 of 2e-3, gvec_in2 at bnorm2); per fragment 0.190 / 0.202 of its bar
           (vec_in4 at norm4).  The dense and NaN decoys change no number.
   f  frame energies within 1e-3 of e_bar of the fresh evaluation; one host step lands within 1e-3 X_TOL of the next
      frame; in 20 steps atoms moved up to 0.84 A (ww) and 1.70 A (abd).
"""
import os
import sys

import numpy as np
import pytest

from ai2bmd_b200.calculator import ViSNetModel
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.md import DeviceLangevin, Langevin
from ai2bmd_b200.pdbfrag import single_graph

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tools"))

CASES = ("ww", "abd")
TIES = {"ww": 173, "abd": 376}          # the fp64 oracle's near tie in each golden geometry (docstring c)
# (case, calibrated) -> the plan the planner picks, measured on one H100 80GB HBM3 (132 SMs).  "multi": CTAs of the
# edge stages run several tiles (edge tiles of the real edge count > the edge_fwd0 grid).
PLANS = {
    ("ww", False): dict(node_tc=0, node_nb=8, npw=1, te_fwd=32, gxa_parts=1, tile_rows=80, tc_rows=96, multi=True),
    ("ww", True): dict(node_tc=0, node_nb=8, npw=1, te_fwd=32, gxa_parts=1, tile_rows=80, tc_rows=96, multi=True),
    ("abd", False): dict(node_tc=1, npw=1, te_fwd=32, gxa_parts=3, tile_rows=128, tc_rows=128, multi=True),
    ("abd", True): dict(node_tc=1, npw=1, te_fwd=32, gxa_parts=3, tile_rows=96, tc_rows=96, multi=True),
}
NODE_KERNELS = {"ww": ["node_fwd2_kernel<8>", "node_bwd2_kernel<8>"],
                "abd": ["node_tc_kernel<0>", "node_tc_kernel<1>", "node_tc_kernel<2>", "node_tc_kernel<3>",
                        "node_norm_fwd_kernel", "node_norm_bwd_kernel"]}
CALIBRATION_CHANGES_THE_PLAN = {"ww": False, "abd": True}
MD_STEPS, DT_FS = 20, 1.0


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "reference_visnet_mode_large.npz"))


def _zp(gold, key):
    return gold[f"{key}_z"], gold[f"{key}_pos"]


def _engine(real_weights, z, pos, calibrated, derivative=True):
    """One-graph handle on z; calibrated: evaluated once at pos and re-planned from the real edge count."""
    eng = Engine(real_weights, 0, derivative=derivative)
    eng.set_topology(z, np.zeros(len(z), dtype=np.int64), n_graphs=1)
    if calibrated:
        (eng.forward_host if derivative else eng.energy_host)(np.asarray(pos, dtype=np.float32))
        eng.set_option("calibrate", 1)
    return eng


def _multi(kernels, n_edges, tile_rows):
    """check_plan's "multi" of test_kernel_variants_gpu.py: more edge tiles than CTAs in the edge stages' grid."""
    grid = dict((s, g) for s, _, g in kernels)["edge_fwd0"]
    return -(-n_edges // tile_rows) > grid


def check_plan(eng, key, calibrated, n_edges):
    """The plan PLANS records for the case, its node-stage kernels and its edge kernels at the tile capacity."""
    from test_kernel_variants_gpu import _kernel_set
    want = PLANS[(key, calibrated)]
    ks = eng.stage_kernels()
    got = {k: eng.get_option(k) for k in want if k != "multi"}
    got["multi"] = _multi(ks, n_edges, got["tile_rows"])
    assert got == want, f"{key} (calibrated: {calibrated}) runs {got}"
    ran = _kernel_set(ks)
    rows = want["tc_rows"]
    need = set(NODE_KERNELS[key]) | {f"edge_fwd_tc_kernel<{rows}>", f"edge_bwd_tc_kernel<{rows}>"}
    assert need <= ran, f"{key} does not run {sorted(need - ran)}; it runs {sorted(ran)}"
    other = NODE_KERNELS["ww" if key == "abd" else "abd"]
    assert not any(k.split("<")[0] == o.split("<")[0] for k in ran for o in other), sorted(ran)
    return ks


# ---- a. the plan -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", CASES)
def test_plan(real_weights, gold, key):
    z, pos = _zp(gold, key)
    n_edges = int(gold[f"{key}_deg"].sum())
    eng = _engine(real_weights, z, pos, False)
    plans = [check_plan(eng, key, False, n_edges)]
    eng.forward_host(pos)
    eng.set_option("calibrate", 1)
    plans.append(check_plan(eng, key, True, n_edges))
    changed = (plans[0] != plans[1], PLANS[(key, False)] != PLANS[(key, True)])
    assert changed == (CALIBRATION_CHANGES_THE_PLAN[key],) * 2


# ---- b. neighbour lists ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", CASES)
def test_neighbour_lists_bit_exact(real_weights, gold, key):
    z, pos = _zp(gold, key)
    eng = _engine(real_weights, z, pos, True)
    slots, deg = eng.get_edges()
    assert np.array_equal(deg, gold[f"{key}_deg"]) and np.array_equal(slots, gold[f"{key}_slots"])
    assert deg.max() == 32


# ---- c. energy and forces --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("calibrated", [False, True], ids=["uncalibrated", "calibrated"])
@pytest.mark.parametrize("key", CASES)
def test_energy_and_forces(real_weights, gold, key, calibrated):
    from test_visnet_mode_gpu import _own_branch, e_bar, f_bar
    z, pos = _zp(gold, key)
    eng = _engine(real_weights, z, pos, calibrated)
    check_plan(eng, key, calibrated, int(gold[f"{key}_deg"].sum()))
    e, f = eng.forward_host(pos)
    ref_e, ref_f, e64, f64 = (gold[f"{key}_{s}"].astype(np.float64) for s in ("ref_e", "ref_f", "e64", "f64"))
    e = float(e[0])
    e_own, f_own, n_br = _own_branch(real_weights, eng, z, pos, f)
    ties = eng.vecln_near_ties()
    print(f"{key} (calibrated: {calibrated}): |E - ref| / bar {abs(e - ref_e[0, 0]) / e_bar(ref_e[0, 0], key):.3f} "
          f"|E - e64| / bar {abs(e - e64[0, 0]) / e_bar(e64[0, 0], key):.3f} "
          f"|F - ref| / bar {np.abs(f - ref_f).max() / f_bar(ref_f):.3f} |F - f64| / bar {np.abs(f - f64).max() / f_bar(f64):.3f} "
          f"|F - f64 on its branch| / bar {np.abs(f - f_own).max() / f_bar(f_own):.3f} ({n_br} branch(es) open); "
          f"near ties {list(ties)}")
    assert abs(e - ref_e[0, 0]) <= e_bar(ref_e[0, 0], key)
    assert abs(e - e64[0, 0]) <= e_bar(e64[0, 0], key) and abs(e - e_own) <= e_bar(e_own, key)
    assert np.abs(f - f_own).max() <= f_bar(f_own)
    # the fp64 near tie is seen, and the engine took the natural channel there as the reference did
    assert TIES[key] in ties
    assert np.abs(f - ref_f).max() <= f_bar(ref_f) and np.abs(f - f64).max() <= f_bar(f64)
    # the reference's calculator path: the first call runs the uncalibrated plan, the second the calibrated one
    model = ViSNetModel(real_weights, device="cuda:0")
    for _ in range(2 if calibrated else 1):
        e2, f2 = model.dl_potential_loader(single_graph(z, pos))
    e2_own, f2_own, _ = _own_branch(real_weights, model.engine, z, pos, f2)
    print(f"  ViSNetModel: |E - e64| / bar {abs(float(e2[0, 0]) - e64[0, 0]) / e_bar(e64[0, 0], key):.3f} "
          f"|F - f64 on its branch| / bar {np.abs(f2 - f2_own).max() / f_bar(f2_own):.3f}")
    assert abs(float(e2[0, 0]) - e64[0, 0]) <= e_bar(e64[0, 0], key)
    assert abs(float(e2[0, 0]) - e2_own) <= e_bar(e2_own, key)
    assert np.abs(f2 - f2_own).max() <= f_bar(f2_own)


# ---- d. every launch of the one-graph plan ---------------------------------------------------------------------------
@pytest.mark.parametrize("decoy", [None, "dense", "nan"])
@pytest.mark.parametrize("calibrated", [False, True], ids=["uncalibrated", "calibrated"])
@pytest.mark.parametrize("key", CASES)
def test_every_launch_of_the_one_graph_plan(real_weights, gold, key, calibrated, decoy):
    from stage_check import stage_report
    from test_kernel_variants_gpu import frag_bar
    from oracle.vecln_branch import Candidates, engine_vectors
    z, pos = _zp(gold, key)
    n = len(z)
    probe = _engine(real_weights, z, pos, calibrated)      # the plan the stage run runs
    probe.forward_host(pos)
    failures = []
    for pins in Candidates(engine_vectors(probe)).branches(0, n):
        detail = {}
        lines, worst = stage_report((z, pos, np.zeros(n, dtype=np.int64)), calibrate=calibrated, detail=detail,
                                    decoy=decoy, pins=pins)
        print("\n".join(lines))
        bad = [(s, w, r) for s, w, r in worst if not r <= 2e-3]
        bad += [(s, w, r) for s, w, r, _ in detail["fragments"] if not r <= frag_bar(w)]
        assert Candidates(detail["vectors"]).contains(pins, 0, n), "the stage run took a branch the probe did not see"
        if not bad:
            break
        failures.append(bad)
    else:
        raise AssertionError(f"no branch the engine may have taken holds every stage: {failures}")
    want = PLANS[(key, calibrated)]
    opts = detail["options"]
    assert {k: opts[k] for k in ("node_tc", "gxa_parts", "npw", "tile_rows", "tc_rows")} == \
        {k: want[k] for k in ("node_tc", "gxa_parts", "npw", "tile_rows", "tc_rows")}
    assert _multi(detail["kernels"], detail["n_edges"], opts["tile_rows"]) == want["multi"]
    assert detail["max_degree"] == 32 and detail["n_atoms"] == n
    stages = {s for s, _, _ in worst}
    assert {"nbr_build", "head", "embed_node_bwd", "finalize", "edge_bwd0"} <= stages
    if key == "abd":        # bwdA writes K-chunk partials only: their sums are checked at bnorm
        assert {"oproj1", "proj0", "norm1", "bnorm1", "bwdB1"} <= stages
        assert "bwdA1" in {s for s, _, _ in detail["kernels"]}
    worst_frag = max(detail["fragments"], key=lambda r: r[2] / frag_bar(r[1]))
    print(f"{key} (calibrated: {calibrated}, decoy {decoy}): worst buffer {max(r for _, _, r in worst):.2e}; "
          f"worst per-fragment {worst_frag[2]:.2e} ({worst_frag[1]} at {worst_frag[0]}, "
          f"{worst_frag[2] / frag_bar(worst_frag[1]):.3f} of its bar)")


# ---- e. the energy plan ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("calibrated", [False, True], ids=["uncalibrated", "calibrated"])
@pytest.mark.parametrize("key", CASES)
def test_energy_plan_is_bit_identical(real_weights, gold, key, calibrated):
    import torch
    z, pos = _zp(gold, key)
    full = _engine(real_weights, z, pos, calibrated)
    fwd_only = _engine(real_weights, z, pos, calibrated, derivative=False)
    plan = [(e.stage_kernels(), e.get_option("tile_rows"), e.get_option("tc_rows")) for e in (full, fwd_only)]
    k_full, k_energy = [k for _, k, _ in plan[0][0]], [k for _, k, _ in plan[1][0]]
    assert k_energy[:-1] == k_full[:len(k_energy) - 1] and "finalize_kernel" in k_energy[-1]
    assert plan[0][1:] == plan[1][1:] == (PLANS[(key, calibrated)]["tile_rows"], PLANS[(key, calibrated)]["tc_rows"])
    e_ref, _ = full.forward_host(pos)
    # the premise: the full plan's energy is bit-reproducible (every sum of one graph has a fixed order)
    assert all(np.array_equal(full.forward_host(pos)[0], e_ref) for _ in range(2))
    got = {"energy_host (derivative=1)": full.energy_host(pos), "energy_host (derivative=0)": fwd_only.energy_host(pos)}
    dpos = torch.from_numpy(np.ascontiguousarray(pos, dtype=np.float32)).cuda()
    for label, eng in (("energy_device (derivative=1)", full), ("energy_device (derivative=0)", fwd_only)):
        e = torch.empty(1, device="cuda")
        eng.energy_device(dpos.data_ptr(), e.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        got[label] = e.cpu().numpy()
    for label, e in got.items():
        assert np.array_equal(e, e_ref), f"{key}: {label} differs from vb_forward by {np.abs(e - e_ref).max():.3e} eV"


# ---- f. the MD step on these plans -----------------------------------------------------------------------------------
def _drift(z, x, v, f):
    """Positions after md.Langevin's first half step at friction 0 (velocity Verlet: half kick with f, drift)."""
    host = Langevin(x, z, lambda _: (0.0, f), dt_fs=DT_FS, friction_per_fs=0.0)
    host.v = np.array(v, dtype=np.float64)
    host.first_half(0.0, 0.0)
    return host.x


@pytest.mark.parametrize("key", CASES)
def test_md_step_integrates_its_own_evaluation(real_weights, gold, key):
    from test_md_gpu import X_TOL
    from test_visnet_mode_gpu import _md_step_kernels, e_bar
    z, pos = _zp(gold, key)
    dev = DeviceLangevin.unfragmented(real_weights, z, pos.astype(np.float64), dt_fs=DT_FS, temperature_K=300.0,
                                      friction_per_fs=0.0, seed=11)
    eng = dev.engine
    check_plan(eng, key, True, int(gold[f"{key}_deg"].sum()))     # calibrated on the start geometry
    x0, v0, _, _ = dev.state()
    eng.md_set_recorder(1, MD_STEPS, 0.0)
    dev.run(MD_STEPS)
    fr = eng.md_read_frames(0, MD_STEPS)
    eng.md_set_recorder(0)
    assert list(fr["step"]) == list(range(1, MD_STEPS + 1)) and not fr["halted"].any()
    xs, vs = [x0] + list(fr["x"]), [v0] + list(fr["v"])
    model = ViSNetModel(real_weights, device="cuda:0")
    worst_e, worst_x = 0.0, 0.0
    for i in range(MD_STEPS + 1):
        e, f = model.dl_potential_loader(single_graph(z, xs[i].astype(np.float32)))
        e = float(e[0, 0])
        if i >= 1:
            worst_e = max(worst_e, abs(float(fr["epot"][i - 1]) - e) / e_bar(e, key))
            assert abs(float(fr["epot"][i - 1]) - e) <= e_bar(e, key), f"{key}: Epot of step {i}"
        if i < MD_STEPS:
            dx = np.abs(_drift(z, xs[i], vs[i], f.astype(np.float64)) - xs[i + 1]).max()
            worst_x = max(worst_x, dx / X_TOL)
            assert dx <= X_TOL, f"{key}: step {i} -> {i + 1}: |dx| {dx:.2e}"
    moved = np.abs(xs[-1] - xs[0]).max()
    print(f"{key}: worst |dEpot| / e_bar {worst_e:.2e}, worst |dx| / X_TOL {worst_x:.2e}, atoms moved up to {moved:.3f} A")
    assert moved > 100 * X_TOL
    assert _md_step_kernels(dev) == eng.launches_per_forward + 3
