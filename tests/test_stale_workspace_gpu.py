"""Every launch plan on a workspace that holds another geometry's data.

A stage that reads a buffer (or a shared-memory row) before the current evaluation writes it -- a missing grid-dependency
wait, a warp-specialised hand-off read before its producer fills it, an unmasked tile tail, a consumer launched before
its producer -- passes every check that runs on memory already holding the right answer: the stage matrix re-runs
stages 0..k at the positions of the prefix before, and the edge rows past the last edge only ever held zeros.  Here a
decoy geometry (tools/stage_check.decoy_positions) is evaluated before every prefix and between evaluations:
"dense" (more edges than the target by at least one 128-row tile, every neighbour list moved) leaves finite wrong data
in every row, "nan" (two coincident atoms per fragment) leaves NaN in every buffer and shared-memory row it reaches.

a. (no GPU) the decoys are what they claim, on the fp64 oracle.
b. the poison reaches the GPU buffers, and a stage left unrun now shows in the stage checks.
c. the stage matrix of test_kernel_variants_gpu.py (same bars, plan checks and per-fragment metric), the option list of
   test_stages_gpu.py and the programmatic-dependent-launch plans, each with a decoy evaluation before every prefix.
d. the energy plan (derivative = 0, forward-only arena with per-layer slots by parity) stage by stage under the NaN
   decoy, and its layer-0 slots of V / V123 / TU still exactly zero after a NaN evaluation.
e. every plan end to end through the public entries (host and caller buffers, graph replay and direct launches, both
   workspaces) over target -> NaN decoy -> target -> dense decoy -> target, against a handle that saw only the target:
   finite, energies bit-identical, forces within the adjoint's run-to-run jitter.
f. the kernels (c) and (e) run cover every model-evaluation kernel of test_kernel_variants_gpu.KERNELS.

The worst error of each case, measured on one H100 80GB HBM3 at 700 W, is in the docstring of its test.  The whole file
takes about 90 s there.
"""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from stage_check import decoy_positions, fragment_rel                         # noqa: E402
from test_energy_only_gpu import CASES as ENERGY_CASES                        # noqa: E402
from test_kernel_variants_gpu import (E2E_CASES, KERNELS, STAGE_CASES, _kernel_set, check_plan,  # noqa: E402
                                      frag_bar)
from test_stages_gpu import OPTS as STAGE_OPTS                                # noqa: E402

TILE = 128
PDL_STAGE = ["chig-default", "trp-default", "abd-default"]
# kernels whose own tests feed fresh data on every call (MD step, hydrogen refinement, non-bonded term, all-reduce,
# the tensor-core self-test): not part of the model evaluation
NOT_MODEL = re.compile(r"tc_selftest_.*|md_.*|caph_relax_kernel|nonbonded_.*|comm_allreduce_kernel")


def _fixture(name, max_frags=0):
    """(z, pos, batch) of a fixture name: tests/golden fragments, or "c<n>" = synthetic_batch(n, seed=5)."""
    if name[0] == "c" and name[1:].isdigit():
        from ai2bmd_b200.synth import synthetic_batch
        fd = synthetic_batch(int(name[1:]), seed=5)
    else:
        from ai2bmd_b200.fixtures import load_fragments
        fd = load_fragments(name)[0]
    z, pos, batch = np.asarray(fd.z), np.asarray(fd.pos, dtype=np.float32), np.asarray(fd.batch)
    if max_frags:
        keep = batch < max_frags
        z, pos, batch = z[keep], pos[keep], batch[keep]
    return z, pos, batch


def _multi_atom_fragments(batch):
    return np.flatnonzero(np.bincount(batch) >= 2)


# ---- a. the decoys (CPU) --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,max_frags", [("chig", 0), ("chig", 4), ("trpcage", 0), ("abd", 0), ("c160", 0)],
                         ids=["chig", "chig4", "trpcage", "abd", "c160"])
def test_decoys_move_every_edge_row(name, max_frags):
    from oracle import visnet_ref as O
    z, pos, batch = _fixture(name, max_frags)
    slots, deg = O.radius_graph_canonical(pos, batch)
    rowptr = np.concatenate([[0], np.cumsum(deg)])
    for kind in ("dense", "nan"):
        d = decoy_positions(pos, batch, kind)
        assert d.dtype == np.float32 and d.shape == pos.shape and np.isfinite(d).all()
        s2, d2 = O.radius_graph_canonical(d, batch)
        rp2 = np.concatenate([[0], np.cumsum(d2)])
        assert d2.sum() >= deg.sum() + TILE, (kind, deg.sum(), d2.sum())
        moved = (s2 != slots).any(1) | (rp2[:-1] != rowptr[:-1])
        assert moved.mean() >= 0.9, (kind, moved.mean())
    assert np.array_equal(decoy_positions(pos, batch, "dense"), decoy_positions(pos, batch, "dense"))   # seeded
    # the NaN decoy: one coincident pair in every fragment of >= 2 atoms, and the two are each other's neighbours
    d = decoy_positions(pos, batch, "nan")
    s2, d2 = O.radius_graph_canonical(d, batch)
    for g in _multi_atom_fragments(batch):
        idx = np.flatnonzero(batch == g)
        p = d[idx].astype(np.float64)
        same = (p[:, None, :] == p[None, :, :]).all(-1) & ~np.eye(len(idx), dtype=bool)
        assert same.sum() == 2, (g, same.sum())
        a, b = idx[np.argwhere(same)[0]]
        assert b in s2[a, :d2[a]] and a in s2[b, :d2[b]]


def test_nan_decoy_poisons_the_fp64_oracle(real_weights):
    import torch
    from oracle import visnet_ref as O
    z, pos, batch = _fixture("chig", 4)
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64)
    e_ref, _ = oracle.energy_and_forces(z, pos, batch)
    assert np.isfinite(e_ref.numpy()).all()
    e, _ = oracle.energy_and_forces(z, decoy_positions(pos, batch, "nan"), batch)
    e = e.numpy()[:, 0]
    assert not np.isfinite(e[_multi_atom_fragments(batch)]).any(), e


# ---- b. the poison reaches the GPU; an unrun stage shows ----------------------------------------------------------
@pytest.mark.gpu
def test_nan_decoy_reaches_the_buffers_and_an_unrun_stage_fails(real_weights):
    import torch
    from ai2bmd_b200.engine import Engine
    from oracle import visnet_ref as O
    from stage_check import _oracle
    from test_kernel_variants_gpu import FRAG_BAR
    z, pos, batch = _fixture("chig")
    N, G = len(z), int(batch.max()) + 1
    eng = Engine(real_weights, 0)
    eng.set_topology(z, batch, n_graphs=G)
    e0, _ = eng.forward_host(pos)
    assert np.isfinite(e0).all()
    e, _ = eng.forward_host(decoy_positions(pos, batch, "nan"))
    x_out = eng.debug_read("X", 6, (N, 128))
    bad_rows = ~np.isfinite(x_out).all(1)
    assert bad_rows.mean() >= 0.99, bad_rows.mean()
    assert not np.isfinite(e[_multi_atom_fragments(batch)]).any()
    # the target up to, not including, node_fwd1: X[1] still holds the decoy's
    sd = O.load_state_dict(os.path.join(ROOT, "tests", "golden", "weights_2ef43f29.npz"))
    slots, deg = O.radius_graph_canonical(pos, batch)
    S, _ = _oracle(("chig", 0, "real"), sd, z, pos, batch, torch.from_numpy(O.slots_to_edge_index(slots, deg)))
    names = eng.stage_names()
    dpos = torch.from_numpy(pos).cuda()
    eng.debug_run(dpos.data_ptr(), names.index("node_fwd1"))
    got, ref = eng.debug_read("X", 1, (N, 128)).astype(np.float64), S["x_in1"]
    row_err = np.abs(got - ref).max(1)
    stale = ~(row_err <= 100 * FRAG_BAR * np.abs(ref).max())
    assert stale.mean() >= 0.99, stale.mean()
    rel, _ = fragment_rel(got, ref, batch, G)
    assert not rel <= 100 * FRAG_BAR
    eng.debug_run(dpos.data_ptr(), names.index("node_fwd1") + 1)       # ... and the stage itself rewrites it
    got = eng.debug_read("X", 1, (N, 128)).astype(np.float64)
    assert fragment_rel(got, ref, batch, G)[0] <= FRAG_BAR


# ---- c. the stage matrix under decoys -------------------------------------------------------------------------------
def _stage_cases():
    out = []
    for case in STAGE_CASES:
        for decoy in ("nan", "dense"):
            out.append(pytest.param(case, "", decoy, id=f"{case}-{decoy}"))
    for case in PDL_STAGE:
        out.append(pytest.param(case, "use_pdl=1", "nan", id=f"{case}-pdl-nan"))
    return out


def _check_bars(lines, worst, detail, label):
    bad = [(s, w, r) for s, w, r in worst if not r <= 2e-3]
    assert not bad, "buffer bar:\n" + "\n".join(lines)
    bad = [(s, w, r, g) for s, w, r, g in detail["fragments"] if not r <= frag_bar(w)]
    assert not bad, f"per-fragment bar: {bad[:8]}\n" + "\n".join(lines)
    s, w, r, g = max(detail["fragments"], key=lambda t: t[2] / frag_bar(t[1]))
    print(f"\n{label}: worst per-fragment {r:.1e} ({w} @ {s}, fragment {g}; bar {frag_bar(w):.0e})")


@pytest.mark.gpu
@pytest.mark.parametrize("case,extra,decoy", _stage_cases())
def test_stage_matrix_after_a_decoy(case, extra, decoy):
    """Bars of test_stage_matrix_against_the_fp64_adjoint_oracle, a decoy evaluation before every prefix.
    Worst per-fragment error relative to its bar (buffer, fragment), measured on one H100 80GB HBM3 at 700 W; the NaN
    and the dense decoy give the same numbers except where noted:
        chig-default 5.7e-6 (va, 0)      chig-tc32 5.4e-6 (va, 0)      chig-simt-te64 1.3e-5 (g_qkv, 7; dense 1.2e-5)
        chig-npw2 5.4e-6 (va, 0)         chig-knobs 5.2e-6 (va, 18)    trp-default 1.1e-5 (va, 4)
        trp-tc64 1.0e-5 (va, 4)          abd-default 1.1e-5 (va, 42)   abd-simt 6.3e-6 (va, 42)
        use_pdl=1: chig-default 5.7e-6, trp-default 1.1e-5, abd-default 1.1e-5 (va), PDL kept through graph capture.
    test_stage_options_after_a_nan_decoy (chig[:4]): at most 1.0e-5 (va, node_tc=1); edge_tc 0 / 2 1.7e-6 (f_in4)."""
    from stage_check import stage_report
    fixture, opts, calibrate, _, _ = STAGE_CASES[case]
    opts = ",".join(filter(None, [opts, extra]))
    detail = {}
    lines, worst = stage_report(fixture, "real", opts=opts, calibrate=calibrate, detail=detail, decoy=decoy)
    check_plan(case, detail)
    if "use_pdl=1" in opts:                   # the debug runs launched with the attribute, the graph capture kept it
        assert detail["options"]["use_pdl"] == 1 and detail["options"]["use_pdl_after"] == 1
    _check_bars(lines, worst, detail, f"{case} {extra} {decoy}")
    assert {"head", "embed_node_bwd", "finalize", "edge_bwd0"} <= {s for s, _, _ in worst}


@pytest.mark.gpu
@pytest.mark.parametrize("opts", STAGE_OPTS, ids=lambda o: o or "default")
def test_stage_options_after_a_nan_decoy(opts):
    from stage_check import stage_report
    detail = {}
    lines, worst = stage_report("chig", "real", max_frags=4, opts=opts, detail=detail, decoy="nan")
    _check_bars(lines, worst, detail, f"chig[:4] {opts or 'default'} nan")
    stages = {s for s, _, _ in worst}
    assert {"head", "embed_node_bwd", "finalize"} <= stages
    assert ("proj3" in stages and "bwdB2" in stages) == ("node_tc=1" in opts)


# ---- d. the energy plan stage by stage ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(STAGE_CASES))
def test_energy_plan_stages_after_a_nan_decoy(case):
    """The forward checks of the stage matrix on a derivative = 0 handle, a NaN evaluation before every prefix.
    Worst per-fragment error relative to its bar, measured on one H100 80GB HBM3 at 700 W: chig-default 5.7e-6,
    chig-tc32 5.4e-6, chig-simt-te64 1.8e-6 (vn), chig-npw2 5.4e-6, chig-knobs 5.2e-6, trp-default 1.1e-5,
    trp-tc64 1.0e-5, abd-default 1.1e-5, abd-simt 6.3e-6 (va unless noted)."""
    from stage_check import stage_report
    fixture, opts, calibrate, _, _ = STAGE_CASES[case]
    detail = {}
    lines, worst = stage_report(fixture, "real", opts=opts, calibrate=calibrate, detail=detail, decoy="nan",
                                derivative=False)
    check_plan(case, detail, forward_only=True)
    _check_bars(lines, worst, detail, f"{case} energy plan nan")
    stages = {s for s, _, _ in worst}
    assert {"head", "finalize", "edge_fwd5"} <= stages and not any("bwd" in s for s in stages)


@pytest.mark.gpu
@pytest.mark.parametrize("node_tc", [0, 1])
def test_energy_plan_layer0_slots_stay_zero_after_a_nan_decoy(real_weights, node_tc):
    from ai2bmd_b200.engine import Engine
    z, pos, batch = _fixture("chig")
    N = len(z)
    eng = Engine(real_weights, 0, derivative=False)
    eng.set_option("node_tc", node_tc)
    eng.set_topology(z, batch)
    e = eng.energy_host(decoy_positions(pos, batch, "nan"))
    assert not np.isfinite(e).any()
    assert not np.isfinite(eng.debug_read("X", 6, (N, 128))).all()          # the slots of the later layers are poisoned
    for name, width in (("V", 128), ("V123", 3 * 128), ("TU", 2 * 128)):
        v = eng.debug_read(name, 0, (N, 3, width))
        assert not np.any(v), f"{name}[0]: {np.count_nonzero(v)} non-zero entries ({np.isnan(v).sum()} NaN)"
    assert np.isfinite(eng.energy_host(pos)).all()


# ---- e. every plan end to end over a sequence of geometries -----------------------------------------------------------
def _e2e_table():
    """id -> (fixture, options, calibrate): the cases of (b)-(d), the end-to-end and energy-plan cases, the PDL plans."""
    t = {f"stage:{c}": (fx, o, cal) for c, (fx, o, cal, _, _) in STAGE_CASES.items()}
    t.update({f"e2e:{c}": (f"c{n}" if seed == 5 else f"c{n}s{seed}", o, True) for c, (n, seed, o, _) in E2E_CASES.items()})
    t.update({f"energy:{c}": (name, o, "tc_rows" not in o) for c, (name, o) in ENERGY_CASES.items()})
    t.update({f"pdl:{fx}": (fx, "use_pdl=1", True) for fx in ("chig", "trpcage", "c160")})
    return t


E2E_TABLE = _e2e_table()


def _fd(name):
    from ai2bmd_b200.fixtures import load_fragments
    from ai2bmd_b200.synth import synthetic_batch
    m = re.fullmatch(r"c(\d+)(?:s(\d+))?", name)
    if m:
        return synthetic_batch(int(m.group(1)), seed=int(m.group(2) or 5))
    return load_fragments(name)[0]


def _set_opts(eng, opts):
    for kv in filter(None, opts.split(",")):
        k, v = kv.split("=")
        eng.set_option(k, int(v))


def _handle(weights, fd, derivative, opts, calibrate):
    from ai2bmd_b200.engine import Engine
    eng = Engine(weights, 0, derivative=derivative)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    _set_opts(eng, opts)
    (eng.forward_host if derivative else eng.energy_host)(fd.pos)
    if calibrate:
        eng.set_option("calibrate", 1)
    return eng


class _Caller:
    """Evaluations of one handle through one entry: "host" (the handle's own buffers) or "device" (caller buffers, the
    same ones on every call, new positions copied in, as an MD loop does)."""

    def __init__(self, eng, entry, n, g):
        import torch
        self.eng, self.entry = eng, entry
        self.pos = torch.empty(n, 3, device="cuda")
        self.e = torch.empty(g, device="cuda")
        self.f = torch.empty(n, 3, device="cuda")

    def __call__(self, pos):
        import torch
        eng = self.eng
        if self.entry == "host":
            if eng.derivative:
                return eng.forward_host(pos)
            return eng.energy_host(pos), None
        self.pos.copy_(torch.from_numpy(np.ascontiguousarray(pos, dtype=np.float32)))
        self.e.fill_(-1.0)
        self.f.fill_(-1.0)
        st = torch.cuda.current_stream().cuda_stream
        if eng.derivative:
            eng.forward_device(self.pos.data_ptr(), self.e.data_ptr(), self.f.data_ptr(), st)
        else:
            eng.energy_device(self.pos.data_ptr(), self.e.data_ptr(), st)
        torch.cuda.synchronize()
        return self.e.cpu().numpy(), (self.f.cpu().numpy() if eng.derivative else None)


@pytest.mark.gpu
@pytest.mark.parametrize("derivative", [1, 0])
@pytest.mark.parametrize("case", list(E2E_TABLE))
def test_sequence_of_geometries_matches_a_handle_that_saw_only_the_target(real_weights, case, derivative):
    """Measured on one H100 80GB HBM3 at 700 W: every target energy bit-identical to handle B's (premise held in every
    case: B's three evaluations agree bit for bit); forces within 1.4e-6 .. 1.9e-6 eV/A on the fixtures and up to
    5.7e-6 (c160) and 7.6e-6 eV/A (c512); use_pdl stayed 1 through every capture."""
    fixture, opts, calibrate = E2E_TABLE[case]
    fd = _fd(fixture)
    n, g = len(fd.z), len(fd)
    target = np.ascontiguousarray(fd.pos, dtype=np.float32)
    seq = [target, decoy_positions(target, fd.batch, "nan"), target, decoy_positions(target, fd.batch, "dense"), target]
    a = _handle(real_weights, fd, derivative, opts, calibrate)
    b = _handle(real_weights, fd, derivative, opts, calibrate)
    worst_e, worst_f = 0.0, 0.0
    for entry in ("host", "device"):
        for use_graph in (0, 1):
            for eng in (a, b):
                eng.set_option("use_graph", use_graph)
            run_a, run_b = _Caller(a, entry, n, g), _Caller(b, entry, n, g)
            got = [run_a(p) for p in seq]
            ref = [run_b(target) for _ in range(3)]
            label = f"{case} derivative={derivative} {entry} use_graph={use_graph}"
            nan_e = got[1][0]
            assert not np.isfinite(nan_e[np.bincount(fd.batch) >= 2]).any(), f"{label}: the NaN decoy did not poison"
            targets = [got[0], got[2], got[4]]
            for i, (e, f) in enumerate(targets + ref):
                assert np.isfinite(e).all() and (f is None or np.isfinite(f).all()), f"{label}: evaluation {i} not finite"
            e_b = ref[0][0]
            spread = max(np.abs(r[0] - e_b).max() for r in ref)
            if spread == 0:
                for i, (e, _) in enumerate(targets):
                    assert np.array_equal(e, e_b), \
                        f"{label}: target {i} after decoys differs by {np.abs(e - e_b).max():.3e} eV"
            else:
                print(f"{label}: three evaluations of the target differ by up to {spread:.3e} eV; bar = that spread")
                for i, (e, _) in enumerate(targets):
                    assert np.abs(e - e_b).max() <= spread, label
            worst_e = max(worst_e, max(np.abs(e - e_b).max() for e, _ in targets))
            if derivative:
                f_b = ref[0][1]
                ties = np.isin(fd.batch, np.unique(fd.batch[b.vecln_near_ties()]))
                bar = 1e-5 + 1e-6 * np.abs(f_b).max()
                for i, (_, f) in enumerate(targets):
                    df = np.abs(f - f_b).max(1)
                    bad = np.flatnonzero(~ties & (df > bar))
                    assert not len(bad), f"{label}: target {i}, atoms {bad[:8]} off by {df[bad[:8]]} (bar {bar:.1e})"
                    assert df.max() <= 5e-2, label
                    worst_f = max(worst_f, df[~ties].max(initial=0.0))
    if "use_pdl=1" in opts:
        assert a.get_option("use_pdl") == 1 and b.get_option("use_pdl") == 1, "graph capture dropped use_pdl"
    print(f"\n{case} derivative={derivative}: |dE| {worst_e:.1e} eV, |dF| {worst_f:.1e} eV/A"
          f"{', use_pdl stayed 1' if 'use_pdl=1' in opts else ''}")


# ---- f. coverage --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_decoy_cases_run_every_model_kernel(real_weights):
    from ai2bmd_b200.engine import Engine
    ran = set()

    def plan(z, pos, batch, opts, calibrate, derivative=True):
        eng = Engine(real_weights, 0, derivative=derivative)
        eng.set_topology(z, batch)
        _set_opts(eng, opts)
        if calibrate:                        # the tile plan (and so the kernel variant) the case runs
            (eng.forward_host if derivative else eng.energy_host)(pos)
            eng.set_option("calibrate", 1)
        ran.update(_kernel_set(eng.stage_kernels()))

    for fixture, opts, calibrate, _, _ in STAGE_CASES.values():
        z, pos, batch = _fixture(fixture)
        for derivative in (True, False):
            plan(z, pos, batch, opts, calibrate, derivative)
    z, pos, batch = _fixture("chig", 4)
    for opts in STAGE_OPTS:
        plan(z, pos, batch, opts, False)
    for fixture, opts, calibrate in E2E_TABLE.values():
        fd = _fd(fixture)
        for derivative in (True, False):
            plan(fd.z, fd.pos, fd.batch, opts, calibrate, derivative)
    from test_kernel_variants_gpu import _demangled
    want = {_demangled(k) for k in KERNELS if not NOT_MODEL.fullmatch(k.split("<")[0])}
    assert want, KERNELS
    missing = sorted(want - ran)
    assert not missing, f"model kernels no decoy case runs: {missing}"
