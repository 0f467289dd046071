#!/usr/bin/env python
"""Stage-by-stage parity of the CUDA engine against the hand-adjoint oracle (GPU box diagnostic).

    python tools/stage_check.py [--weights real|random] [--frags chig] [--calibrate] [--decoy dense|nan] [--energy]
                                [--out stage_check.txt]

Runs the evaluation one launch at a time (``vb_debug_run``), reads the engine's internal buffers after
each stage and compares them with the tensors of ``oracle/adjoint_ref.py`` (fp64).  The first stage whose
relative error jumps is where a kernel bug lives.  Every comparison is reported twice: relative to the largest
reference entry of the whole buffer, and per fragment (the worst fragment is named), so that a fault confined to
one tile, one fragment or a few rows is not diluted by whichever fragment holds the largest entry.
Test infrastructure; not part of the product path.
"""
import argparse
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

from oracle import visnet_ref as O                      # noqa: E402
from oracle.adjoint_ref import AdjointViSNet            # noqa: E402
from ai2bmd_b200.engine import Engine                   # noqa: E402

D, L = 128, 6


def fragment_rel(got, ref, frag, n_frags):
    """Per-fragment relative error of got vs ref (rows grouped by ``frag``): the largest error over a fragment's rows
    divided by the larger of max|ref| over those rows and 1e-3 max|ref| of the whole buffer (a floor, so that near-zero
    fragments do not blow up).  Returns (worst relative error, its fragment)."""
    err = np.abs(got - ref).reshape(len(ref), -1).max(1)
    mag = np.abs(ref).reshape(len(ref), -1).max(1)
    e_g, m_g = np.zeros(n_frags), np.zeros(n_frags)
    np.maximum.at(e_g, frag, err)
    np.maximum.at(m_g, frag, mag)
    rel = e_g / np.maximum(m_g, 1e-3 * mag.max())
    g = int(np.argmax(rel))
    return float(rel[g]), g


def decoy_positions(pos, batch, kind, seed=0):
    """Positions of another geometry on the same z / batch topology, to run just before the geometry under test, so
    that whatever a stage reads before this evaluation writes it holds some other evaluation's data (float32 [N,3]).

    "dense": every fragment contracted toward its centroid by 0.85, then a seeded 0.2 A Gaussian displacement.  The
    neighbour lists, degrees, row pointers and the edge count all change, and the edge count grows by more than one
    128-row tile, so every edge row of the target and the rows past its last edge hold some other edge's finite data.
    "nan": the dense decoy with the second atom of every fragment of >= 2 atoms placed exactly on the first one.  The
    coordinates stay finite and the pair stays neighbours, so r = 0 for j != i gives d = 0/0 in edge_geom: NaN spreads
    through every vector feature and every later buffer of that fragment (and the shared memory the kernels leave
    behind).  No kernel turns a feature value into an index (the only float-to-int reinterpretation is the atomic number
    edge_geom copies into the geometry rows, and the VecLayerNorm max / min paths compare keys whose index bits are the
    channel, whatever the value), so the poison stays in values."""
    pos = np.asarray(pos, dtype=np.float64)
    batch = np.asarray(batch)
    if kind not in ("dense", "nan"):
        raise ValueError(f"decoy kind {kind!r}: 'dense' or 'nan'")
    out = pos.copy()
    for g in np.unique(batch):
        m = batch == g
        c = out[m].mean(0)
        out[m] = c + 0.85 * (out[m] - c)
    out = (out + 0.2 * np.random.default_rng(seed).standard_normal(out.shape)).astype(np.float32)
    if kind == "nan":
        first = np.flatnonzero(np.r_[True, batch[1:] != batch[:-1]])
        for a in first:
            if a + 1 < len(batch) and batch[a + 1] == batch[a]:
                out[a + 1] = out[a]
    return out


# Forward-only workspace (derivative = 0): layer l of a per-layer buffer lives in slot l % 2, and layer 0 of V / V123 /
# TU in a zeroed slot of its own (DESIGN section 3).  vb_debug_read refuses a layer that a later layer shares its slot
# with; the checks read each layer right after the stage that writes it, before that slot is written again, so they ask
# for the same slot under the last layer that maps to it.  No forward check of the full plan has to be skipped: each one
# reads only buffers its own stage writes (node stage k: X / V / VN / QKV / V123 / VDOT / TU of layer k and O of layer
# k - 1; tensor-core "norm k": VDOT of layer k - 1; edge stage l: F of layer l + 1), and no stage writes two layers that
# share a slot.  The adjoint's checks (gx_out / gvec_out at the head, every backward stage) have no buffers here.
PER_LAYER = ("X", "V", "F", "VN", "QKV", "V123", "VDOT", "TU", "O")
OWN_ZERO_LAYER = ("V", "V123", "TU")


def energy_slot_layer(name, layer):
    if layer == 0 and name in OWN_ZERO_LAYER:
        return 0
    n = L + 1 if name in ("X", "V") else L
    return max(range(layer, n, 2))


_oracle_cache = {}


def _geometry_key(z, pos, batch):
    """Cache key of a geometry given as arrays: a hash of its atomic numbers, positions and fragment indices."""
    h = hashlib.sha256()
    for a in (z, pos, batch):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _pins_key(pins):
    """Cache key of VecLayerNorm pins {site: (amx, amn)} (None: the natural branch)."""
    if pins is None:
        return None
    h = hashlib.sha256()
    for site in sorted(pins):
        h.update(str(site).encode())
        for a in pins[site]:
            h.update(np.ascontiguousarray(np.asarray(a, dtype=np.int64)).tobytes())
    return h.hexdigest()


def _oracle(key, sd, z, pos, batch, ei, pins=None):
    """fp64 hand-adjoint tensors of one geometry (on the VecLayerNorm branch ``pins``, AdjointViSNet); the last one is
    kept, so that runs of cases on one geometry (one case under several decoys, options or launch plans) build it
    once."""
    if key is not None and key in _oracle_cache:
        return _oracle_cache[key]
    adj = AdjointViSNet(O.OracleViSNet(sd, torch.float64))
    Eo, Fo, S, B = adj.energy_and_forces(z, pos, batch, ei, pins=pins)
    out = ({k: v.numpy() for k, v in S.items()}, {k: v.numpy() for k, v in B.items()})
    _oracle_cache.clear()
    if key is not None:
        _oracle_cache[key] = out
    return out


def stage_report(frags="chig", weights="real", max_frags=0, opts="", calibrate=False, detail=None, decoy=None,
                 derivative=True, calibrate_pos=None, pins=None):
    """Run the evaluation one launch at a time and compare every buffer a stage produces with the fp64 hand-adjoint
    oracle.  Returns (lines, worst) where worst = [(stage, what, rel)] of the comparisons, rel relative to the largest
    reference entry of the buffer.

    frags: a fixture name (tests/golden/fragments_<name>.npz) or a (z, pos, batch) tuple.  opts: "key=value,..." for
    vb_set_option.  calibrate: evaluate once, then re-plan the edge tiles from the real edge count (the plan the host
    entry points run).  calibrate_pos: positions [N, 3] of another geometry on the same topology (before the max_frags
    selection, as the positions of frags); the edge tiles are then calibrated on that geometry instead, as a plan
    calibrated earlier in a trajectory meets the geometry under test (implies calibrate).  detail: an optional dict,
    filled with "fragments" = [(stage, what, rel, fragment)] (the per-fragment metric of every comparison, see
    fragment_rel), "kernels" = Engine.stage_kernels(), "options" (resolved tile_rows, tc_rows, gxa_parts, node_tc,
    node_nb, edge_tc, npw, and use_pdl / tile_rows / tc_rows again after the last evaluation, as "<key>_after"),
    "n_edges", "n_atoms", "max_degree", and "host" = (energies, forces or None) of the last evaluation through the host
    entry point, and "vectors" = V[0..L] the engine's last evaluation left (oracle/vecln_branch.py reads its VecLayerNorm
    branch from them).  pins: the VecLayerNorm branch of the oracle ({site: (amx, amn)} over the selected atoms, see
    AdjointViSNet); None is the natural one."""
    if isinstance(frags, str):
        g = np.load(os.path.join(ROOT, "tests", "golden", f"fragments_{frags}.npz"))
        z, pos, batch = g["z"], g["pos"], g["batch"]
    else:
        z, pos, batch = (np.asarray(a) for a in frags)
        z, pos, batch = z.astype(np.int64), pos.astype(np.float32), batch.astype(np.int64)
    if calibrate_pos is not None:
        calibrate_pos = np.asarray(calibrate_pos, dtype=np.float32)
        assert calibrate_pos.shape == pos.shape, "calibrate_pos must be a geometry of the same atoms"
        calibrate = True
    if max_frags:
        keep = batch < max_frags
        z, pos, batch = z[keep], pos[keep], batch[keep]
        if calibrate_pos is not None:
            calibrate_pos = calibrate_pos[keep]
    sd = O.load_state_dict(os.path.join(ROOT, "tests", "golden", "weights_2ef43f29.npz")) if weights == "real" \
        else O.random_state_dict(int(weights) if str(weights).isdigit() else 0)
    slots, deg = O.radius_graph_canonical(pos, batch)
    ei = torch.from_numpy(O.slots_to_edge_index(slots, deg))
    E, N = ei.shape[1], len(z)
    key = frags if isinstance(frags, str) else _geometry_key(z, pos, batch)
    S, B = _oracle((key, max_frags, str(weights), _pins_key(pins)), sd, z, pos, batch, ei, pins)

    eng = Engine({k: v.numpy() for k, v in sd.items()}, 0, derivative=derivative)
    G = int(batch.max()) + 1
    eng.set_topology(z, batch, n_graphs=G)
    for kv in filter(None, opts.split(",")):
        k, v = kv.split("=")
        eng.set_option(k, int(v))
    host_eval = eng.forward_host if derivative else eng.energy_host
    if calibrate:
        host_eval(pos if calibrate_pos is None else calibrate_pos)
        eng.set_option("calibrate", 1)
    names = eng.stage_names()
    dpos = torch.from_numpy(pos).cuda()
    ddecoy = torch.from_numpy(decoy_positions(pos, batch, decoy)).cuda() if decoy else None
    lines, worst = [], []
    assert E != N, "node and edge rows must be told apart by their count"
    row_frag = {N: batch, E: batch[ei[1].numpy()], G: np.arange(G)}
    per_frag = []
    if detail is not None:
        detail["fragments"] = per_frag
        detail["kernels"] = eng.stage_kernels()
        detail["options"] = {k: eng.get_option(k) for k in ("tile_rows", "tc_rows", "gxa_parts", "node_tc", "node_nb",
                                                             "edge_tc", "npw", "use_pdl")}
        detail["n_edges"], detail["n_atoms"], detail["max_degree"] = E, N, int(deg.max())

    def report(stage, what, got, ref):
        ref = np.asarray(ref, dtype=np.float64)
        got = np.asarray(got, dtype=np.float64).reshape(ref.shape)
        err = np.abs(got - ref).max() if ref.size else 0.0
        mag = np.abs(ref).max() if ref.size else 0.0
        rel = err / mag if mag > 0 else err
        frel, fg = fragment_rel(got, ref, row_frag[len(ref)], G) if mag > 0 else (float(err), 0)
        flag = "  <<<<<<" if (not np.isfinite(err)) or rel > 2e-3 else ""
        lines.append(f"{stage:16s} {what:14s} maxabs {err:10.3e}  ref {mag:10.3e}  rel {rel:9.2e}  "
                     f"frag {frel:9.2e} @{fg:<4d}{flag}")
        worst.append((stage, what, float(rel) if np.isfinite(err) else float("inf")))
        per_frag.append((stage, what, frel if np.isfinite(frel) else float("inf"), fg))

    def flagline(stage, text, ok):
        lines.append(f"{stage:16s} {text}: {bool(ok)}")
        worst.append((stage, text, 0.0 if ok else float("inf")))
        per_frag.append((stage, text, 0.0 if ok else float("inf"), 0))

    def rd(name, layer, shape):
        if not derivative and name in PER_LAYER:
            layer = energy_slot_layer(name, layer)
        return eng.debug_read(name, layer, shape)

    def cat(*xs):
        return np.concatenate(xs, axis=-1)

    def node_fwd_checks(st, k):
        if k >= 1:
            report(st, f"x_in{k}", rd("X", k, (N, D)), S[f"x_in{k}"] if k < L else S["x_out"])
            report(st, f"vec_in{k}", rd("V", k, (N, 3, D)), S[f"vec_in{k}"] if k < L else S["vec_out"])
            report(st, f"o{k-1}", rd("O", k - 1, (N, 3 * D)), S[f"o{k-1}"])
        if k < L:
            report(st, "vn", rd("VN", k, (N, 3, D)), S[f"vn{k}"])
            report(st, "qkv", rd("QKV", k, (N, 3 * D)), cat(S[f"q{k}"], S[f"k{k}"], S[f"v{k}"]))
            report(st, "v123", rd("V123", k, (N, 3, 3 * D)), cat(S[f"v1{k}"], S[f"v2{k}"], S[f"v3{k}"]))
            report(st, "vdot", rd("VDOT", k, (N, D)), S[f"vdot{k}"])
            if k < L - 1:
                report(st, "tu", rd("TU", k, (N, 3, 2 * D)), cat(S[f"t{k}"], S[f"u{k}"]))

    def node_bwd_checks(st, k):
        if k <= L - 1:
            report(st, f"gx_in{k}", rd("GX", 0, (N, D)), B[f"gx_in{k}"])
            report(st, f"gvec_in{k}", rd("GVEC", 0, (N, 3, D)), B[f"gvec_in{k}"])
        if k >= 1:
            report(st, f"g_xa{k-1}", rd("GXA", 0, (N, D)), B[f"g_xa{k-1}"])

    def edge_bwd_checks(st, l):
        report(st, f"gf_in{l}", rd("GF", 0, (N * 32, D))[:E], B[f"gf_in{l}"])
        report(st, "g_qkv", rd("GQKV", 0, (N, 3 * D)), cat(B[f"g_q{l}"], B[f"g_k{l}"], B[f"g_v{l}"]))
        report(st, "g_vn_msg", rd("GVNMSG", 0, (N, 3, D)), B[f"g_vn_msg{l}"])
        if l < L - 1:
            report(st, "g_tu", rd("GTU", 0, (N, 3, 2 * D)), cat(B[f"g_t{l}"], B[f"g_u{l}"]))

    for si, st in enumerate(names):
        if ddecoy is not None:
            eng.debug_run(ddecoy.data_ptr(), -1)
        eng.debug_run(dpos.data_ptr(), si + 1)
        if st == "nbr_build":
            s2, d2 = eng.get_edges()
            flagline(st, "neighbour list identical", (s2 == slots).all() and (d2 == deg).all())
        elif st == "rowptr_scan":
            rp = rd("rowptr", 0, (N + 1,)).view(np.int32)
            flagline(st, "rowptr ok", (rp == np.concatenate([[0], np.cumsum(deg)])).all())
        elif st == "edge_geom":
            ge = rd("geom", 0, (N * 32, 8))[:E]
            report(st, "r", ge[:, 0], S["r"]); report(st, "C", ge[:, 1], S["C"]); report(st, "d", ge[:, 2:5], S["d"])
            report(st, "rbf", rd("rbf", 0, (N * 32, 32))[:E], S["rbf"])
            es, ed = rd("esrc", 0, (N * 32,)).view(np.int32)[:E], rd("edst", 0, (N * 32,)).view(np.int32)[:E]
            flagline(st, "edge_index ok", (es == ei[0].numpy()).all() and (ed == ei[1].numpy()).all())
        elif st == "embed_node":
            report(st, "x_emb", rd("X", 0, (N, D)), S["x_emb"])
        elif st == "embed_edge":
            report(st, "f0", rd("F", 0, (N * 32, D))[:E], S["f_in0"])
        elif st.startswith("node_fwd"):
            node_fwd_checks(st, int(st[8:]))
        elif st.startswith("oproj"):            # tensor-core node stage: O of the previous layer
            k = int(st[5:])
            report(st, f"o{k-1}", rd("O", k - 1, (N, 3 * D)), S[f"o{k-1}"])
        elif st.startswith("norm"):
            k = int(st[4:])
            if k >= 1:
                report(st, f"x_in{k}", rd("X", k, (N, D)), S[f"x_in{k}"] if k < L else S["x_out"])
                report(st, f"vec_in{k}", rd("V", k, (N, 3, D)), S[f"vec_in{k}"] if k < L else S["vec_out"])
                report(st, f"vdot{k-1}", rd("VDOT", k - 1, (N, D)), S[f"vdot{k-1}"])
            if k < L:
                report(st, "vn", rd("VN", k, (N, 3, D)), S[f"vn{k}"])
        elif st.startswith("proj"):
            k = int(st[4:])
            report(st, "qkv", rd("QKV", k, (N, 3 * D)), cat(S[f"q{k}"], S[f"k{k}"], S[f"v{k}"]))
            report(st, "v123", rd("V123", k, (N, 3, 3 * D)), cat(S[f"v1{k}"], S[f"v2{k}"], S[f"v3{k}"]))
            if k < L - 1:
                report(st, "tu", rd("TU", k, (N, 3, 2 * D)), cat(S[f"t{k}"], S[f"u{k}"]))
        elif st.startswith("bnorm"):
            k = int(st[5:])
            if k <= L - 1:
                report(st, f"gx_in{k}", rd("GX", 0, (N, D)), B[f"gx_in{k}"])
                report(st, f"gvec_in{k}", rd("GVEC", 0, (N, 3, D)), B[f"gvec_in{k}"])
        elif st.startswith("bwdB"):
            k = int(st[4:])
            report(st, f"g_xa{k-1}", rd("GXA3", 0, (3, N, D)).sum(0), B[f"g_xa{k-1}"])
        elif st.startswith("bwdA"):
            pass                                 # K-chunk partials only; their sums are checked at bnorm
        elif st.startswith("edge_fwd"):
            l = int(st[8:])
            report(st, "xa", rd("XA", 0, (N, D)), S[f"xa{l}"])
            report(st, "va", rd("VA", 0, (N, 3, D)), S[f"va{l}"])
            if l < L - 1:
                report(st, f"f_in{l+1}", rd("F", l + 1, (N * 32, D))[:E], S[f"f_in{l+1}"])
        elif st == "head":
            report(st, "e_atom", rd("eatom", 0, (N,)), S["e_atom"][:, 0])
            if derivative:                       # the energy plan's head stops at the per-atom energies
                report(st, "gx_out", rd("GX", 0, (N, D)), B["gx_out"])
                report(st, "gvec_out", rd("GVEC", 0, (N, 3, D)), B["gvec_out"])
        elif st in ("energy_reduce", "finalize"):
            report(st, "E", rd("energy", 0, (eng.n_graphs,)), S["E"][:, 0])
        elif st.startswith("node_bwd"):
            node_bwd_checks(st, int(st[8:]))
        elif st.startswith("edge_bwd"):
            edge_bwd_checks(st, int(st[8:]))
        elif st == "embed_edge_bwd":
            report(st, "gx_emb", rd("GX", 0, (N, D)), B["gx_emb"])
        elif st == "embed_node_bwd":
            ea = rd("eacc", 0, (N * 32, 4))[:E]
            report(st, "g_d", ea[:, 1:4] * S["mask"][:, None], B["g_d"] * S["mask"][:, None])
            report(st, "forces", rd("forces", 0, (N, 3)), B["forces"])
    # full evaluation through the public host entry
    if ddecoy is not None:
        eng.debug_run(ddecoy.data_ptr(), -1)
    if derivative:
        e, f = eng.forward_host(pos)
        report("forward_host", "E", e, S["E"][:, 0])
        report("forward_host", "forces", f, B["forces"])
    else:
        e, f = eng.energy_host(pos), None
        report("energy_host", "E", e, S["E"][:, 0])
    if detail is not None:
        for k in ("use_pdl", "tile_rows", "tc_rows"):
            detail["options"][f"{k}_after"] = eng.get_option(k)
        detail["host"] = (e, f)
        if derivative:
            detail["vectors"] = np.stack([eng.debug_read("V", k, (N, 3, D)) for k in range(L + 1)])
    return lines, worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--weights", default="real")
    ap.add_argument("--frags", default="chig")
    ap.add_argument("--max-frags", type=int, default=0)
    ap.add_argument("--out", default="")
    ap.add_argument("--opts", default="", help="comma list key=value for vb_set_option")
    ap.add_argument("--calibrate", action="store_true", help="plan the edge tiles from the real edge count first")
    ap.add_argument("--decoy", default=None, choices=["dense", "nan"], help="evaluate a decoy geometry before each prefix")
    ap.add_argument("--energy", action="store_true", help="check the energy plan on a derivative = 0 handle")
    args = ap.parse_args()
    lines, _ = stage_report(args.frags, args.weights, args.max_frags, args.opts, args.calibrate, decoy=args.decoy,
                            derivative=not args.energy)
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
