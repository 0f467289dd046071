"""The tensor-core edge kernels on the tile lengths the planner picks below their compiled capacity.

plan_tiles (engine.cu) sets the tile length to 16 * rows-per-warp so that the tiles fill whole waves of CTAs, and runs it
in the smallest capacity ROWS of {32, 64, 96, 128} that holds it: 16 rows in edge_*_tc_kernel<32>, 48 in <64>, 80 in
<96>.  There the kernels' SIMT phases run fewer rows per warp than ROWS / 16, the gather warps of the warp-specialised
forward split fewer rows, and the second 64-row M half of <96> is only partly valid.  With 16-row tiles a target of
degree up to 32 spans three tiles, cut on both sides of the middle one.  And the plan is made once, from the
calibrated edge count plus a 3 % margin: when the edges of a later geometry outgrow it, the grid stays capped at the SM
count and CTAs loop over a second tile of the short length.

Every case here goes through the real planner on the card at hand: its geometry is built from a fixture's whole
fragments, taken until the edge count falls in the range of the wanted tile length, then single-atom fragments (one
atom, one self-loop edge each), which set the last tile's length and shift where tile boundaries cut the targets.  Each
case runs stage by stage against the fp64 hand adjoint (tools/stage_check.py) on the bars of
test_kernel_variants_gpu.py, and asserts what it ran: the resolved tile plan, the kernel instances, the last tile's
rows, whether the tiles outnumber the CTAs, the targets spanning three tiles.  The single atoms add two checks of their
own: their forces are exactly 0, and their energies agree to SINGLE_ULPS rounding steps.
test_every_case_reaches_its_tile_plan prints the plan of every case on 132 and on 114 SMs without a GPU.

On 132 SMs: t16-* run 16-row tiles in <32> with all 44 dense targets over three tiles (15 | 16 | 1, and 8 | 16 | 8 in
t16-span8), t48-* 48 rows in the warp-specialised <64>, t80-* 80 rows in <96>, t80-2wave 254 such tiles over 132 CTAs,
drift-48 / drift-16 135 tiles of 48 / 16 rows over 132 CTAs on a plan calibrated for 6,097 / 2,038 edges.
Worst per-fragment error of each case, measured on one H100 80GB HBM3 at 700 W (buffer, fragment):
    t16-span 4.9e-5 (g_vn_msg, 1)     t16-simt-te32 1.1e-5 (g_vn_msg, 1)   t16-simt-te64 1.1e-5 (g_vn_msg, 1)
    t16-span8 3.4e-5 (g_vn_msg, 8)    t48-r1 4.8e-5 (gvec_in3, 17)         t48-energy 5.2e-6 (va, 2)
    t48-r47 4.6e-5 (gvec_in3, 17)     drift-48 7.2e-5 (gvec_in2, 0)        t80-r1 7.5e-5 (gvec_in2, 11)
    t80-energy 1.2e-5 (va, 4)         t80-r79 7.5e-5 (gvec_in2, 11)        t80-2wave 5.4e-5 (gvec_out, 49)
    drift-16 3.4e-5 (gvec_in2, 0)
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLDEN = os.path.join(ROOT, "tests", "golden")

SINGLE_Z = 1          # the element of every single-atom fragment
# Identical single-atom fragments are not bit-identical: the embedding and SIMT node kernels start their K loops at a
# row that differs from CTA to CTA (spreading the weight reads over L2 slices), so each atom's sums run in an order set
# by its CTA.  Their energies agree to this many fp32 rounding steps (measured up to 6, on 79 single atoms); a row that
# read another row's data would miss by orders of magnitude more.
SINGLE_ULPS = 16


def plan_tiles(edges, sm):
    """engine.cu plan_tiles restated: (tile_rows, tc_rows, waves) for an edge count on a card of `sm` SMs."""
    padded = edges + edges * 3 // 100 + 1
    waves = max(1, -(-padded // (sm * 128)))
    rpw = -(-padded // (sm * waves * 16))
    if rpw >= 7:
        rpw = 8
    rows = 16 * min(8, max(1, rpw))
    return rows, 32 if rows <= 32 else 64 if rows <= 64 else 96 if rows <= 96 else 128, waves


def edge_range(rows, waves, sm):
    """[lo, hi] of the edge counts the planner runs in `waves` waves of `rows`-row tiles."""
    hit = [e for e in range(1, (waves + 1) * sm * 128) if plan_tiles(e, sm)[0::2] == (rows, waves)]
    return hit[0], hit[-1]


def _fixture(name):
    if name == "dense44":
        r = np.load(os.path.join(GOLDEN, "reference_outputs.npz"))
        return r["dense44_z"], r["dense44_pos"], r["dense44_batch"]
    g = np.load(os.path.join(GOLDEN, f"fragments_{name}.npz"))
    return g["z"], g["pos"], g["batch"]


def _frag_edges(name):
    """Edges of each fragment of a fixture (the radius graph stays inside a fragment)."""
    from oracle import visnet_ref as O
    z, pos, batch = _fixture(name)
    return np.bincount(batch, weights=O.radius_graph_canonical(pos, batch)[1]).astype(int)


def _assemble(lead, name, n_frags, trail):
    """`lead` single atoms, the first `n_frags` fragments of fixture `name`, `trail` single atoms: (z, pos, batch, the
    atoms that are single fragments).  The single atoms sit 8 A apart on a line away from the fragments."""
    z, pos, batch = _fixture(name)
    keep = batch < n_frags
    z, pos, batch = z[keep].astype(np.int64), pos[keep].astype(np.float32), batch[keep].astype(np.int64)

    def singles(n, x0):
        return (np.full(n, SINGLE_Z, np.int64),
                np.stack([x0 + 8.0 * np.arange(n), np.zeros(n), np.zeros(n)], 1).astype(np.float32))

    (zl, pl), (zt, pt) = singles(lead, -100.0 - 8.0 * lead), singles(trail, 100.0 + np.abs(pos).max())
    n_body = int(batch.max()) + 1
    b = np.concatenate([np.arange(lead), lead + batch, lead + n_body + np.arange(trail)])
    single = np.r_[np.ones(lead, bool), np.zeros(len(z), bool), np.ones(trail, bool)]
    return np.concatenate([zl, z, zt]), np.concatenate([pl, pos, pt]), b, single


def _fill(name, rows, waves, sm, last):
    """The largest prefix of whole fragments of `name` that stays in the edge range of (rows, waves) with room for up to
    rows - 1 single atoms, then the single atoms that leave `last` rows in the last tile (`last` None: none).  None when
    the fixture cannot reach the range on this card."""
    lo, hi = edge_range(rows, waves, sm)
    csum = np.cumsum(_frag_edges(name))
    room = 0 if last is None else rows - 1
    fits = np.flatnonzero(csum <= hi - room)
    if not len(fits) or csum[fits[-1]] < lo:
        return None
    e0 = int(csum[fits[-1]])
    trail = 0 if last is None else (last - e0) % rows
    return _assemble(0, name, int(fits[-1]) + 1, trail)


def contracted(pos, batch, rows, sm):
    """The atoms of every fragment contracted toward its centroid, by the mildest factor whose edges need more tiles of
    `rows` than `sm` CTAs: the plan calibrated on `pos` then runs several short tiles per CTA.  Milder than the "dense"
    decoy of stage_check (0.85 and 0.2 A noise), whose close contacts leave forces that even the fp32 SIMT edge kernels
    miss by more than the force bar on one Chignolin fragment."""
    from oracle import visnet_ref as O
    for factor in (0.97, 0.95, 0.93, 0.91, 0.89, 0.87, 0.85):
        out = pos.astype(np.float64)
        for g in np.unique(batch):
            m = batch == g
            c = out[m].mean(0)
            out[m] = c + factor * (out[m] - c)
        out = out.astype(np.float32)
        if -(-int(O.radius_graph_canonical(out, batch)[1].sum()) // rows) > sm:
            return out
    raise AssertionError(f"no contraction down to 0.85 outgrows {sm} tiles of {rows} rows")


# id -> (geometry (name, rows, waves, last) of _fill, or ("dense44", lead, trail)), options, derivative, drift,
#        plan (tile_rows, tc_rows), tiles outnumber the CTAs, fewest targets over three tiles)
CASES = {
    "t16-span": (("dense44", 1, 0), "", True, False, (16, 32), False, 40),
    "t16-simt-te32": (("dense44", 1, 0), "edge_tc=0,te_fwd=32,te_bwd=32", True, False, (16, 32), False, 40),
    "t16-simt-te64": (("dense44", 1, 0), "edge_tc=0,te_fwd=64,te_bwd=64", True, False, (16, 32), False, 40),
    "t16-span8": (("dense44", 8, 7), "", True, False, (16, 32), False, 40),
    "t48-r1": (("chig", 48, 1, 1), "", True, False, (48, 64), False, 0),
    "t48-energy": (("chig", 48, 1, 1), "", False, False, (48, 64), False, 0),
    "t48-r47": (("chig", 48, 1, 47), "", True, False, (48, 64), False, 0),
    "drift-48": (("chig", 48, 1, 1), "", True, True, (48, 64), True, 0),
    "t80-r1": (("trpcage", 80, 1, 1), "", True, False, (80, 96), False, 0),
    "t80-energy": (("trpcage", 80, 1, 1), "", False, False, (80, 96), False, 0),
    "t80-r79": (("trpcage", 80, 1, 79), "", True, False, (80, 96), False, 0),
    "t80-2wave": (("ww", 80, 2, None), "", True, False, (80, 96), True, 0),
    "drift-16": (("chig", 16, 1, None), "", True, True, (16, 32), True, 0),
}
# the kernels a case must run: the tensor-core pair of its capacity, or the SIMT pair of its tile length
SIMT = {"t16-simt-te32": ["edge_fwd_kernel<32,8>", "edge_bwd_kernel<32,8>"],
        "t16-simt-te64": ["edge_fwd_kernel<64,8>", "edge_bwd_kernel<64,8>"]}


def build_case(case, sm):
    """(z, pos, batch, single-atom mask, positions the plan is calibrated on) of a case on a card of `sm` SMs, or None
    when the fixture cannot reach the case's range there."""
    geo, _, _, drift, _, _, _ = CASES[case]
    if geo[0] == "dense44":
        z, pos, batch, single = _assemble(geo[1], "dense44", 1, geo[2])
    else:
        built = _fill(*geo[:3], sm, geo[3])
        if built is None:
            return None
        z, pos, batch, single = built
    if drift:
        return z, contracted(pos, batch, geo[1], sm), batch, single, pos
    return z, pos, batch, single, pos


def tile_facts(deg, rows):
    """(edges, tiles, rows of the last tile, targets whose edges span three or more tiles) of a degree list."""
    rp = np.concatenate([[0], np.cumsum(deg)])
    E = int(rp[-1])
    tiles = -(-E // rows)
    has = deg > 0
    spans = int(((rp[1:][has] - 1) // rows - rp[:-1][has] // rows >= 2).sum())
    return E, tiles, E - (tiles - 1) * rows, spans


def expected_plan(case, sm):
    """Restated plan, tiles, last-tile rows, three-tile spans and edge counts of a case, from the oracle's neighbour
    lists, or None when the case cannot be built on this card."""
    from oracle import visnet_ref as O
    built = build_case(case, sm)
    if built is None:
        return None
    z, pos, batch, single, cal = built
    e_cal = int(O.radius_graph_canonical(cal, batch)[1].sum())
    rows, cap, waves = plan_tiles(e_cal, sm)
    deg = O.radius_graph_canonical(pos, batch)[1]
    E, tiles, last, spans = tile_facts(deg, rows)
    return dict(rows=rows, cap=cap, waves=waves, e_cal=e_cal, E=E, tiles=tiles, last=last, spans=spans,
                multi=tiles > sm)


# ---- on the host: the cases reach their paths on a 132- and a 114-SM card --------------------------------------
@pytest.mark.parametrize("sm", [132, 114])
def test_every_case_reaches_its_tile_plan(sm):
    """The geometry builder on two SM counts, with the restated planner: each case lands on its tile length, capacity,
    last-tile rows, one tile per CTA or several, and three-tile spans.  (The GPU test asserts the same on the card
    and against the engine's own plan.)"""
    print(f"\n{sm} SMs: case            edges  tile_rows tc_rows  tiles  waves  multi  last  spans")
    for case, (geo, _, _, drift, plan, multi, spans) in CASES.items():
        x = expected_plan(case, sm)
        if x is None:
            assert case == "t80-2wave", f"{case} cannot be built on {sm} SMs"
            continue
        print(f"  {case:16s} {x['E']:6d} {x['rows']:9d} {x['cap']:7d} {x['tiles']:6d} {x['waves']:6d} "
              f"{x['multi']!s:6s} {x['last']:5d} {x['spans']:6d}")
        assert (x["rows"], x["cap"]) == plan, case
        assert x["multi"] == multi, case
        assert x["spans"] >= spans, case
        if geo[0] == "dense44":
            assert x["last"] == (1 if geo[1] == 1 else 15), case
        elif geo[3] is not None and not drift:
            assert x["last"] == geo[3], case
        if drift:
            assert x["E"] > x["e_cal"] * 1.03, case


# ---- on the GPU ---------------------------------------------------------------------------------------------------
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
def test_uncalibrated_plan_matches_the_restated_planner(real_weights):
    """Before any evaluation the plan comes from 17 edges per atom: N single-atom fragments for N = 1 .. 2000."""
    from ai2bmd_b200.engine import Engine
    sm = _sm_count()
    eng = Engine(real_weights, 0)
    bad = []
    for n in range(1, 2001):
        eng.set_topology(np.full(n, SINGLE_Z), np.arange(n))
        got = (eng.get_option("tile_rows"), eng.get_option("tc_rows"))
        if got != plan_tiles(17 * n, sm)[:2]:
            bad.append((n, got, plan_tiles(17 * n, sm)[:2]))
    assert not bad, f"{len(bad)} atom counts planned otherwise, first {bad[:8]}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_short_tiles_against_the_fp64_adjoint_oracle(case):
    from stage_check import stage_report
    from test_kernel_variants_gpu import _kernel_set, frag_bar
    sm = _sm_count()
    geo, opts, derivative, drift, plan, multi, min_spans = CASES[case]
    x = expected_plan(case, sm)
    if x is None:
        pytest.skip(f"{case}: the {geo[0]} fixture has too few edges to reach {geo[1]}-row tiles in {geo[2]} waves "
                    f"on {sm} SMs")
    z, pos, batch, single, cal = build_case(case, sm)
    detail = {}
    lines, worst = stage_report((z, pos, batch), "real", opts=opts, calibrate=True, detail=detail,
                                derivative=derivative, calibrate_pos=cal if drift else None)
    opt = detail["options"]
    grid = dict((s, g) for s, _, g in detail["kernels"])["edge_fwd0"]
    frag = max(detail["fragments"], key=lambda t: t[2])
    print(f"\n{case}: tile_rows {opt['tile_rows']} in <{opt['tc_rows']}>, {x['tiles']} tiles over {grid} CTAs, "
          f"last tile {x['last']} rows, {x['spans']} targets over three tiles, edges {x['E']} (plan {x['e_cal']}), "
          f"worst per-fragment {frag[2]:.2e} ({frag[1]}, fragment {frag[3]})")
    # what the case ran
    assert detail["n_edges"] == x["E"]
    assert (opt["tile_rows"], opt["tc_rows"]) == (x["rows"], x["cap"]) == plan, f"{case}: plan {opt}"
    assert (opt["tile_rows_after"], opt["tc_rows_after"]) == plan, f"{case}: the plan moved to {opt}"
    ran = _kernel_set(detail["kernels"])
    want = set(SIMT.get(case, [f"edge_fwd_tc_kernel<{plan[1]}>", f"edge_bwd_tc_kernel<{plan[1]}>"]))
    if not derivative:
        want = {k for k in want if "_bwd" not in k}
    assert want <= ran, f"{case} does not run {sorted(want - ran)}; it runs {sorted(ran)}"
    if case not in SIMT:
        assert (x["tiles"] > grid) == multi, f"{case}: {x['tiles']} edge tiles over {grid} CTAs"
    assert x["spans"] >= min_spans
    # the bars of the kernel-variant matrix
    bad = [(s, w, r) for s, w, r in worst if not r <= 2e-3]
    assert not bad, "buffer bar:\n" + "\n".join(lines)
    bad = [(s, w, r, g) for s, w, r, g in detail["fragments"] if not r <= frag_bar(w)]
    assert not bad, f"per-fragment bar: {bad[:8]}\n" + "\n".join(lines)
    # the single atoms: no force, and one energy to a few rounding steps (SINGLE_ULPS)
    e, f = detail["host"]
    g_single = np.unique(batch[single])
    if len(g_single):
        spread = np.ptp(e[g_single]) / np.spacing(np.abs(e[g_single]).max())
        assert spread <= SINGLE_ULPS, f"single-atom energies {np.unique(e[g_single])} ({spread:.0f} ulps apart)"
        if f is not None:
            assert np.all(f[single] == 0), f"single-atom forces up to {np.abs(f[single]).max():.3e}"
