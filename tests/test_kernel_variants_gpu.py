"""Every kernel variant the launch planner can choose, run at the problem sizes and options that select it and checked
against the fp64 oracle.

a. Inventory (no GPU): every ``__global__`` kernel of ai2bmd_b200/csrc, and every template instance engine.cu names, is
   listed in KERNELS with the test that runs it.  A kernel added without parity coverage fails here on any machine.
b. Stage matrix: the evaluation one launch at a time against the fp64 hand-adjoint oracle (tools/stage_check.py) at
   production sizes: CTAs that run several edge tiles (persistent loop, weight ring wrapping across tiles), tile
   capacities 32..128, both modes of the tensor-core node stage, the batched embedding kernels, NB = 8 / 16 SIMT node
   kernels.  Each case asserts what it runs (the dry-run kernel list of Engine.stage_kernels(), the tile plan,
   "gxa_parts") and two bars on every buffer of every stage: 2e-3 of the buffer's largest reference entry (as
   test_stages_gpu.py) and a per-fragment bar (stage_check.fragment_rel: the error over a fragment's rows relative to
   that fragment's largest entry), so that a fault confined to one tile, one fragment or the rows of cut targets is
   not diluted by the largest entry of the whole buffer.
   Worst per-fragment error of each case, measured on one H100 80GB HBM3 at 700 W (buffer, fragment):
       chig-default 4.5e-5 (gvec_in3, 17)      chig-tc32 3.9e-5 (gvec_in2, 2)      chig-tc32 seed 3 5.7e-5 (gvec_in2, 11)
       chig-simt-te64 1.8e-5 (gvec_in4, 5)     chig-npw2 4.8e-5 (gvec_in3, 17)     chig-knobs 4.3e-5 (gvec_in2, 2)
       trp-default 7.4e-5 (gvec_in2, 11)       trp-tc64 7.0e-5 (gvec_in2, 11)      abd-simt 4.5e-5 (gvec_out, 51)
       abd-default 1.5e-4 (gvec_in2, 17)       abd-default seed 3 3.3e-4 (g_vn_msg, 13)
   The bars per buffer are at FRAG_BAR below.
c. End to end per fragment above 4,096 atoms, where the stage oracle is too large for one CPU process: every fragment's
   energy and forces against the fp64 oracle on the VecLayerNorm(max_min) branch the engine took (DESIGN section 2,
   oracle/vecln_branch.py): the natural oracle (run on the GPU in chunks of 64 fragments) where the engine's channel
   norms leave one branch and it is the oracle's own, else the CPU hand adjoint pinned to each branch they leave open,
   the best of them.  Bars, for every fragment: energy e_tol, forces 5e-5 + 2e-5 max|F_fragment|.  Measured on the same
   card: |dE| up to 0.30 e_tol (c160) and 0.32 e_tol (c512); |dF| up to 0.40 of its bar (c160, tensor-core node stage),
   0.17 (c160, SIMT) and 0.59 (c512).  No fragment of either batch needed a pinned evaluation: the 2 of 160 and 8 of
   512 fragments with channel norms within 1e-5 of each other (Engine.vecln_near_ties) leave the engine one branch
   each, and it is the fp64 oracle's.  That is measured, not assumed: a fragment where it is not is checked pinned.
d. Every option a case sets changes the dry-run kernel list (or the tile plan / gxa_parts) against the same case
   without it; "krot" and "use_pdl" change kernel arguments and launch attributes only and are exempt.
"""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tools"))
CSRC = os.path.join(ROOT, "ai2bmd_b200", "csrc")

# ---- a. inventory -------------------------------------------------------------------------------------------------
# kernel (template instance where the kernel is a template) -> the test that runs it: "stage:<id>" / "e2e:<id>" are
# cases of this file (whose dry-run kernel list must contain the kernel), otherwise a test file of this directory.
KERNELS = {
    "nbr_build_kernel": "stage:chig-default",
    "rowptr_scan_kernel": "stage:chig-default",
    "edge_geom_kernel": "stage:chig-default",
    "embed_node_small_kernel": "stage:chig-default",
    "embed_node_kernel<8>": "stage:abd-default",
    "embed_edge_kernel": "stage:chig-default",
    "embed_edge_bwd_kernel": "stage:chig-default",
    "embed_node_bwd_kernel": "stage:chig-default",
    "finalize_kernel": "stage:chig-default",
    "head2_kernel": "stage:chig-default",
    "head_kernel<1>": "e2e:c160-npw1",
    "head_kernel<2>": "e2e:c160-default",
    "node_fwd2_kernel<1>": "test_stages_gpu.py",          # node_nb = 1 .. 4 at chig[:4]
    "node_fwd2_kernel<2>": "test_stages_gpu.py",
    "node_fwd2_kernel<3>": "stage:chig-default",
    "node_fwd2_kernel<4>": "test_stages_gpu.py",
    "node_fwd2_kernel<8>": "stage:abd-simt",
    "node_fwd2_kernel<16>": "stage:chig-npw2",
    "node_bwd2_kernel<1>": "test_stages_gpu.py",
    "node_bwd2_kernel<2>": "test_stages_gpu.py",
    "node_bwd2_kernel<3>": "stage:chig-default",
    "node_bwd2_kernel<4>": "test_stages_gpu.py",
    "node_bwd2_kernel<8>": "stage:abd-simt",
    "edge_fwd_kernel<32,8>": "test_stages_gpu.py",        # edge_tc = 0, 2
    "edge_fwd_kernel<64,8>": "stage:chig-simt-te64",
    "edge_bwd_kernel<32,8>": "test_stages_gpu.py",        # edge_tc = 0, 1
    "edge_bwd_kernel<64,8>": "stage:chig-simt-te64",
    "edge_fwd_tc_kernel<32>": "stage:chig-tc32",
    "edge_fwd_tc_kernel<64>": "stage:chig-default",
    "edge_fwd_tc_kernel<96>": "stage:trp-default",
    "edge_fwd_tc_kernel<128>": "stage:abd-default",
    "edge_bwd_tc_kernel<32>": "stage:chig-tc32",
    "edge_bwd_tc_kernel<64>": "stage:chig-default",
    "edge_bwd_tc_kernel<96>": "stage:trp-default",
    "edge_bwd_tc_kernel<128>": "stage:abd-default",
    "node_tc_kernel<NT_OPROJ>": "stage:trp-default",
    "node_tc_kernel<NT_PROJ>": "stage:trp-default",
    "node_tc_kernel<NT_BWDA>": "stage:trp-default",
    "node_tc_kernel<NT_BWDB>": "stage:trp-default",
    "node_norm_fwd_kernel": "stage:trp-default",
    "node_norm_bwd_kernel": "stage:trp-default",
    "tc_selftest_kernel<32>": "test_tc_selftest_gpu.py",
    "tc_selftest_kernel<64>": "test_tc_selftest_gpu.py",
    "tc_selftest_kernel<TC_TE>": "test_tc_selftest_gpu.py",
    "md_kick1_kernel": "test_md_kernels_gpu.py",
    "md_place_kernel": "test_md_kernels_gpu.py",
    "md_kick2_kernel": "test_md_kernels_gpu.py",
    "caph_relax_kernel": "test_md_kernels_gpu.py",
    "nonbonded_kernel": "test_md_kernels_gpu.py",
    "nonbonded_energy_kernel": "test_md_kernels_gpu.py",
    "comm_allreduce_kernel": "test_md_kernels_gpu.py",    # world = 1 here; test_multigpu.py runs world > 1
}
_NT = {"NT_OPROJ": "0", "NT_PROJ": "1", "NT_BWDA": "2", "NT_BWDB": "3"}


def kernel_inventory():
    """Names of every __global__ kernel of csrc; a template is listed by the instances engine.cu names instead."""
    src = {f: open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))}
    bases = set()
    for text in src.values():
        bases |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", text))
    inst = set()
    for name, args in re.findall(r"\b(\w+_kernel)<([\w\s,]+)>", src["engine.cu"]):
        args = re.sub(r"\s+", "", args)
        if name in bases and re.fullmatch(r"(\d+|NT_[A-Z]+|TC_TE)(,\d+)*", args):
            inst.add(f"{name}<{args}>")
    templated = {i.split("<")[0] for i in inst}
    return (bases - templated) | inst


def test_every_kernel_is_pinned_by_a_test():
    found = kernel_inventory()
    missing = sorted(found - set(KERNELS))
    assert not missing, f"kernels without a parity test (add a case and an entry in KERNELS): {missing}"
    stale = sorted(set(KERNELS) - found)
    assert not stale, f"KERNELS lists kernels the sources no longer have: {stale}"
    for k, where in KERNELS.items():
        if where.startswith("stage:"):
            assert where[6:] in STAGE_CASES, (k, where)
        elif where.startswith("e2e:"):
            assert where[4:] in E2E_CASES, (k, where)
        else:
            assert os.path.exists(os.path.join(ROOT, "tests", where)), (k, where)


def _demangled(k):
    """KERNELS key -> the form Engine.stage_kernels() reports: "vb::edge_fwd_kernel<64,8>" (spaces dropped)."""
    for a, b in _NT.items():
        k = k.replace(a, b)
    return k


def _pinned(case):
    return sorted(_demangled(k) for k, w in KERNELS.items() if w == case)


def _kernel_set(kernels):
    return {re.sub(r"\s+", "", re.sub(r"\(\.\.\.\)$", "", k)).replace("vb::", "").replace("(anonymousnamespace)::", "")
            for _, k, _ in kernels}


# ---- b. stage matrix ----------------------------------------------------------------------------------------------
# id -> (fixture, options, calibrate, kernels the case must run besides those KERNELS pins to it, plan checks)
STAGE_CASES = {
    "chig-default": ("chig", "", True, ["edge_bwd_tc_kernel<64>"], dict(node_tc=0, node_nb=3, tile_rows=64, multi=False)),
    "chig-tc32": ("chig", "tc_rows=32", False, [], dict(tile_rows=32, multi=True)),
    "chig-simt-te64": ("chig", "edge_tc=0,te_fwd=64,te_bwd=64", False, [], dict(edge_tc=0)),
    "chig-npw2": ("chig", "npw=2", False, ["node_bwd2_kernel<3>"], dict(npw=2, node_tc=0)),
    "chig-knobs": ("chig", "embed_batch=3,krot=0,use_pdl=1", False, ["embed_node_kernel<8>"], dict(node_tc=0)),
    "trp-default": ("trpcage", "", True, [], dict(node_tc=1, gxa_parts=3, tile_rows=96, multi=False)),
    "trp-tc64": ("trpcage", "tc_rows=64", False, ["edge_fwd_tc_kernel<64>", "edge_bwd_tc_kernel<64>"],
                 dict(node_tc=1, gxa_parts=3, tile_rows=64, multi=True)),
    "abd-default": ("abd", "", True, ["node_tc_kernel<3>", "embed_node_kernel<8>"],
                    dict(node_tc=1, gxa_parts=1, tile_rows=128, multi=True, max_degree=32)),
    "abd-simt": ("abd", "node_tc=0", False, [], dict(node_tc=0, node_nb=8)),
}
STAGE_PARAMS = [pytest.param(c, "real", id=f"{c}-real") for c in STAGE_CASES] + \
               [pytest.param(c, "3", id=f"{c}-seed3") for c in ("chig-tc32", "abd-default")]

# Per-fragment bar: the first entry of FRAG_BAR_BUFFER whose pattern matches the buffer, else FRAG_BAR (forward
# buffers).  Worst measured over the matrix (H100 80GB HBM3, 700 W): forward buffers 1.1e-5 (va, xa), the adjoint
# 5.7e-5 (g_qkv), the vector adjoint through VecLayerNorm(max_min) 3.3e-4 (g_vn_msg, gvec_out, gvec_in, abd-default
# with seed-3 weights).  Each bar is 4-6x its worst case and none is looser than the buffer bar.
FRAG_BAR = 5e-5
FRAG_BAR_BUFFER = {r"g_vn_msg|gvec_out|gvec_in\d": 2e-3, r"g_\w+|g\w+_\w+|forces": 3e-4}


def frag_bar(what):
    for pat, bar in FRAG_BAR_BUFFER.items():
        if re.fullmatch(pat, what):
            return bar
    return FRAG_BAR


def check_plan(case, detail, forward_only=False):
    """What the case claims to run: kernels (template arguments included), tile plan, node-stage mode.  forward_only:
    the energy plan of a derivative = 0 handle, which runs the case's kernels but no adjoint ones."""
    _, _, _, extra, plan = STAGE_CASES[case]
    ran = _kernel_set(detail["kernels"])
    want = set(_pinned(f"stage:{case}")) | set(extra)
    if forward_only:
        want = {k for k in want if not re.search(r"_bwd|node_tc_kernel<[23]>", k)}
    assert want <= ran, f"{case} does not run {sorted(want - ran)}; it runs {sorted(ran)}"
    opts = detail["options"]
    for k, v in plan.items():
        if k == "multi":
            grid = dict((s, g) for s, _, g in detail["kernels"])["edge_fwd0"]
            tiles = -(-detail["n_edges"] // opts["tile_rows"])
            assert (tiles > grid) == v, f"{case}: {tiles} edge tiles over {grid} CTAs"
        elif k == "max_degree":
            assert detail["max_degree"] == v
        else:
            assert opts[k] == v, f"{case}: {k} = {opts[k]}, expected {v}"


@pytest.mark.gpu
@pytest.mark.parametrize("case,weights", STAGE_PARAMS)
def test_stage_matrix_against_the_fp64_adjoint_oracle(case, weights):
    from stage_check import stage_report
    fixture, opts, calibrate, _, _ = STAGE_CASES[case]
    detail = {}
    lines, worst = stage_report(fixture, weights, opts=opts, calibrate=calibrate, detail=detail)
    check_plan(case, detail)
    bad = [(s, w, r) for s, w, r in worst if not r <= 2e-3]
    assert not bad, "buffer bar:\n" + "\n".join(lines)
    bad = [(s, w, r, g) for s, w, r, g in detail["fragments"] if not r <= frag_bar(w)]
    assert not bad, f"per-fragment bar: {bad[:8]}\n" + "\n".join(lines)
    stages = {s for s, _, _ in worst}
    assert {"head", "embed_node_bwd", "finalize", "edge_bwd0"} <= stages


# ---- c. end to end per fragment -----------------------------------------------------------------------------------
# id -> (fragments, seed of synthetic_batch, options, plan checks)
E2E_CASES = {
    "c160-npw1": (160, 5, "npw=1", dict(node_tc=1, gxa_parts=1)),
    "c160-default": (160, 5, "", dict(node_tc=1, gxa_parts=1, npw=2)),
    "c160-simt": (160, 5, "node_tc=0", dict(node_tc=0, node_nb=8, npw=2)),
    "c512-default": (512, 0, "", dict(node_tc=1, gxa_parts=1, npw=2, tile_rows=128)),
}
E2E_EXTRA = {"c160-simt": ["node_fwd2_kernel<16>", "node_bwd2_kernel<8>"],
             "c512-default": ["head_kernel<2>", "node_tc_kernel<3>", "edge_fwd_tc_kernel<128>", "edge_bwd_tc_kernel<128>"]}


def e_tol(e, ulps=2):
    return np.maximum(4e-3, ulps * np.spacing(np.abs(e).astype(np.float32)))


def _set_opts(eng, opts):
    for kv in filter(None, opts.split(",")):
        k, v = kv.split("=")
        eng.set_option(k, int(v))


def e2e_errors(real_weights, case):
    """Engine vs fp64 oracle per fragment for one E2E case, on the VecLayerNorm branch the engine took: (fd, eng, dE [G],
    dF [G], F bar [G], pinned, off_natural).  A fragment is checked against the natural oracle (run on the GPU in chunks
    of 64 fragments) when the engine's branch there is one branch and is the oracle's own; otherwise against the pinned
    CPU hand adjoint (oracle/vecln_branch.py) on each branch the engine may have taken, keeping the best.  pinned: the
    fragments that needed that; off_natural: those of them whose best branch is not the natural one."""
    import torch
    from ai2bmd_b200.engine import Engine
    from ai2bmd_b200.synth import synthetic_batch
    from oracle import visnet_ref as O
    from oracle.vecln_branch import Candidates, best_branch, engine_vectors, natural_branch
    n, seed, opts, _ = E2E_CASES[case]
    fd = synthetic_batch(n, seed=seed)
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch)
    _set_opts(eng, opts)
    eng.forward_host(fd.pos)
    eng.set_option("calibrate", 1)                   # the plan the host entry points run
    e, f = eng.forward_host(fd.pos)
    cand = Candidates(engine_vectors(eng))
    amb = set(np.unique(fd.batch[cand.ambiguous()[:, 1]]).tolist())
    oracle = O.OracleViSNet({k: torch.from_numpy(v) for k, v in real_weights.items()}, torch.float64, device="cuda")
    G = len(fd)
    de, df, fbar = np.zeros(G), np.zeros(G), np.zeros(G)
    pinned, off_natural = [], []

    def score(g, e_ref, f_ref, lo):
        s, t = int(fd.start[g]), int(fd.end[g])
        return (abs(float(e[g]) - e_ref) / e_tol(e_ref), np.abs(f[s:t] - f_ref[s - lo:t - lo]).max(),
                5e-5 + 2e-5 * np.abs(f_ref[s - lo:t - lo]).max())

    for g0 in range(0, G, 64):                       # fragments are independent: bounded oracle memory
        sub = fd[g0:min(G, g0 + 64)]
        cap = {}
        with torch.no_grad():
            oracle.forward(torch.from_numpy(sub.z).cuda(), torch.from_numpy(sub.pos).cuda().double(),
                           torch.from_numpy(sub.batch).cuda(), cap=cap)
        nat = natural_branch([cap[f"vec_in{l}"] for l in range(6)] + [cap["vec_out"]])
        del cap
        e_ref, f_ref = oracle.energy_and_forces(sub.z, sub.pos, sub.batch)
        e_ref, f_ref = e_ref.cpu().numpy()[:, 0], f_ref.cpu().numpy()
        a0 = int(fd.start[g0])
        for j in range(len(sub)):
            g, s, t = g0 + j, int(fd.start[g0 + j]), int(fd.end[g0 + j])
            own = cand.contains({k: (mx[s - a0:t - a0], mn[s - a0:t - a0]) for k, (mx, mn) in nat.items()}, s, t)
            if own and g not in amb:
                de[g], df[g], fbar[g] = score(g, e_ref[j], f_ref, a0)
                continue
            pinned.append(g)
            er, fr, _ = best_branch(real_weights, cand, fd.z, fd.pos, s, t, f)
            de[g], df[g], fbar[g] = score(g, er, fr, s)
            nat_err = score(g, e_ref[j], f_ref, a0)
            if nat_err[1] > nat_err[2]:
                off_natural.append(g)
    del oracle
    torch.cuda.empty_cache()
    return fd, eng, de, df, fbar, pinned, off_natural


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(E2E_CASES))
def test_every_fragment_against_the_fp64_oracle(real_weights, case):
    fd, eng, de, df, fbar, pinned, off_natural = e2e_errors(real_weights, case)
    ran = _kernel_set(eng.stage_kernels())
    want = set(_pinned(f"e2e:{case}")) | set(E2E_EXTRA.get(case, []))
    assert want <= ran, f"{case} does not run {sorted(want - ran)}; it runs {sorted(ran)}"
    assert len(fd.z) > 4096
    for k, v in E2E_CASES[case][3].items():
        assert eng.get_option(k) == v, (case, k)
    print(f"{case}: |dE| / e_tol up to {de.max():.2f}, |dF| / bar up to {(df / fbar).max():.2f}; "
          f"{len(pinned)} fragments checked on a pinned branch (worst |dF| / bar "
          f"{max([df[g] / fbar[g] for g in pinned], default=0):.2f}), {len(off_natural)} off the natural one")
    assert (de <= 1).all(), f"energy: fragments {np.flatnonzero(de > 1)[:8]} (|dE| / e_tol up to {de.max():.2f})"
    bad = np.flatnonzero(df > fbar)
    assert not len(bad), f"forces: fragments {bad[:8]}, |dF| {df[bad[:8]]} over {fbar[bad[:8]]}"


# ---- d. knobs act ---------------------------------------------------------------------------------------------------
EXEMPT = {"krot", "use_pdl"}          # change kernel arguments / launch attributes, not kernels


def _plan(eng):
    return eng.stage_kernels(), eng.get_option("tile_rows"), eng.get_option("gxa_parts")


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(STAGE_CASES) + list(E2E_CASES))
def test_every_option_a_case_sets_changes_the_plan(real_weights, case):
    from ai2bmd_b200.engine import Engine
    from ai2bmd_b200.fixtures import load_fragments
    from ai2bmd_b200.synth import synthetic_batch
    if case in STAGE_CASES:
        fixture, opts, calibrate = STAGE_CASES[case][:3]
        fd, _ = load_fragments(fixture)
    else:
        n, seed, opts, _ = E2E_CASES[case]
        fd = synthetic_batch(n, seed=seed)
    kvs = [kv for kv in opts.split(",") if kv and kv.split("=")[0] not in EXEMPT]
    for kv in kvs:
        plans = []
        for with_it in (False, True):
            eng = Engine(real_weights, 0)
            eng.set_topology(fd.z, fd.batch)
            _set_opts(eng, ",".join(x for x in kvs if x != kv or with_it))
            plans.append(_plan(eng))
        assert plans[0] != plans[1], f"{case}: {kv} changes no kernel, grid or tile plan"


@pytest.mark.gpu
def test_dry_run_lists_every_launch_and_enqueues_nothing(real_weights, chig):
    import torch
    from ai2bmd_b200.engine import Engine
    fd, _ = chig
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch)
    ks = eng.stage_kernels()
    assert len(ks) == eng.launches_per_forward == 35
    assert all(k.startswith("vb::") or "finalize_kernel" in k for _, k, _ in ks) and all(g >= 1 for _, _, g in ks)
    assert [s for s, _, _ in ks] == eng.stage_names()
    eng.forward_host(fd.pos)
    # positions moved by 0.1 A through the first three stages only (neighbours, row pointers, geometry): every later
    # buffer still holds the first evaluation, and would not after a launch of the later stages
    pos2 = torch.from_numpy(fd.pos + np.float32(0.1) * np.sin(np.arange(fd.pos.size, dtype=np.float32)).reshape(-1, 3)).cuda()
    eng.debug_run(pos2.data_ptr(), 3)
    before = [eng.debug_read(n, 1, (len(fd.z), 128)) for n in ("X", "GX")] + [eng.debug_read("forces", 0, (len(fd.z), 3))]
    eng.set_option("node_tc", 1)                      # a dry run of the new plan
    ks1 = eng.stage_kernels()
    torch.cuda.synchronize()
    after = [eng.debug_read(n, 1, (len(fd.z), 128)) for n in ("X", "GX")] + [eng.debug_read("forces", 0, (len(fd.z), 3))]
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert len(ks1) == eng.launches_per_forward == 59
    assert any("node_tc_kernel" in k for _, k, _ in ks1)
    eng.debug_run(pos2.data_ptr(), -1)                # ... whereas launching the stages does change them
    moved = [eng.debug_read(n, 1, (len(fd.z), 128)) for n in ("X", "GX")] + [eng.debug_read("forces", 0, (len(fd.z), 3))]
    assert not any(np.array_equal(a, b) for a, b in zip(before, moved))
