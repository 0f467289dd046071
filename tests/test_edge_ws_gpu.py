"""The <= 64-row tensor-core edge kernels (warp-specialised forward) against the fp64 stage oracle, on the tile
layouts that exercise their edge cases: tiles whose first and last targets are cut by a tile boundary (plain store
vs atomicAdd of the per-target sums), a final tile of fewer than 16 edges (gather warps without rows, MMA rows past
the tile), and 32-row tiles with several tiles per CTA (the weight ring and the hand-offs reused across tiles).
Every buffer that edge_fwd0..5 and edge_bwd0..5 produce is held to the bars of test_kernel_variants_gpu.py."""
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tools"))

# per-fragment bars of test_kernel_variants_gpu.py: forward buffers, the adjoint, the vector adjoint through VecLayerNorm
FRAG_BAR = 5e-5
FRAG_BAR_BUFFER = {r"g_vn_msg": 2e-3, r"g_\w+|g\w+_\w+": 3e-4}


def frag_bar(what):
    return next((bar for pat, bar in FRAG_BAR_BUFFER.items() if re.fullmatch(pat, what)), FRAG_BAR)


def _chig(drop=None):
    """Chignolin's fragments, optionally without fragment `drop` (graph ids renumbered)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "fragments_chig.npz"))
    z, pos, batch = g["z"], g["pos"], g["batch"]
    if drop is not None:
        keep = batch != drop
        z, pos, batch = z[keep], pos[keep], batch[keep] - (batch[keep] > drop)
    return z, pos, batch


def _edges_per_target(pos, batch):
    from oracle import visnet_ref as O
    _, deg = O.radius_graph_canonical(pos, batch)
    return np.asarray(deg)


def _short_tail_drop(rows):
    """The first chig fragment whose removal leaves a final tile of 1..15 edges."""
    _, pos, batch = _chig()
    for k in range(int(batch.max()) + 1):
        keep = batch != k
        if 0 < int(_edges_per_target(pos[keep], batch[keep]).sum()) % rows < 16:
            return k
    raise AssertionError("no chig subset leaves a short final tile")


def _has_tile_cut_at_both_ends(deg, rows):
    rowptr = np.concatenate([[0], np.cumsum(deg)])
    for e0 in range(0, int(rowptr[-1]), rows):
        e1 = min(e0 + rows, int(rowptr[-1]))
        first = np.searchsorted(rowptr, e0, side="right") - 1
        last = np.searchsorted(rowptr, e1 - 1, side="right") - 1
        if rowptr[first] < e0 and rowptr[last + 1] > e1:
            return True
    return False


CASES = {   # id -> (fragment to drop or None, options, calibrate, tile rows)
    "chig-default-64": (None, "", True, 64),
    "chig-short-tail-64": ("short", "tc_rows=64", False, 64),
    "chig-tc32": (None, "tc_rows=32", False, 32),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_small_tile_edge_stages_against_the_fp64_oracle(case):
    from stage_check import stage_report
    n, opts, calibrate, rows = CASES[case]
    if n == "short":
        n = _short_tail_drop(rows)
    z, pos, batch = _chig(n)
    deg = _edges_per_target(pos, batch)
    E = int(deg.sum())
    if case == "chig-default-64":
        assert _has_tile_cut_at_both_ends(deg, rows)
    else:
        assert 0 < E % rows < 16
    detail = {}
    lines, worst = stage_report((z, pos, batch), "real", opts=opts, calibrate=calibrate, detail=detail)
    assert detail["options"]["tile_rows"] == rows and detail["options"]["edge_tc"] == 3
    ran = {k for _, k, _ in detail["kernels"]}
    for d in ("fwd", "bwd"):
        assert any(re.search(rf"edge_{d}_tc_kernel<{rows}>", k) for k in ran), f"{case}: no edge_{d}_tc_kernel<{rows}> in {ran}"
    edge = [(s, w, r) for s, w, r in worst if s.startswith(("edge_fwd", "edge_bwd"))]
    assert {s for s, _, _ in edge} == {f"edge_{d}{l}" for d in ("fwd", "bwd") for l in range(6)}
    bad = [(s, w, r) for s, w, r in edge if not r <= 2e-3]
    assert not bad, f"buffer bar: {bad}\n" + "\n".join(lines)
    bad = [(s, w, r, g) for s, w, r, g in detail["fragments"] if s.startswith(("edge_fwd", "edge_bwd"))
           and not r <= frag_bar(w)]
    assert not bad, f"per-fragment bar: {bad[:8]}\n" + "\n".join(lines)
    ends = [(s, w, r) for s, w, r in worst if s == "forward_host"]
    assert ends and all(r <= 2e-3 for _, _, r in ends), "\n".join(lines)
