"""Which VecLayerNorm(max_min) branch the engine took, and the fp64 oracle on that branch.  TEST INFRASTRUCTURE ONLY.

VecLayerNorm(max_min) routes the energy gradient through each atom's argmax and argmin channel norm.  Where two channel
norms agree to fp32 rounding, the engine's fp32 norms and the fp64 oracle's norms can name different channels, and the
force jumps between the two branches by up to ~1e-2 eV/A (DESIGN section 2).  On one fixed branch the model is smooth,
so the engine's forces must match the fp64 oracle evaluated on the engine's own branch at the normal bar.

Sites: site l < L is layer l's ``vec_layernorm`` on V[l] (V[0] = 0), site L is the head's ``vec_out_norm`` on V[L].
The engine's backward (``vecln_backward``, ai2bmd_b200/csrc/k_node.cuh) reads exactly these V[0..L] from the workspace,
so the channel norms of the V an evaluation left behind decide its branch.  They are recomputed here in fp64 from that
fp32 data.  The engine's own ``sqrtf`` of an fp32 sum of squares, fused or not, sits up to 1.45 fp32 ulps from them
(measured over V[0..6] of the 160- and 512-fragment synthetic batches on one H100 80GB HBM3 at 700 W), so two channels
more than 2 x 1.45 ulps apart keep their order in the engine, and every channel within ULPS = 3 ulps of the max (min)
is a candidate for the engine's argmax (argmin).  2 ulps would not cover two roundings of 1.45 ulps each.  Widening the
window costs nothing there: those batches have no channel pair within 8 ulps of an extreme.
"""
from __future__ import annotations

import itertools

import numpy as np
import torch

from .adjoint_ref import AdjointViSNet
from .visnet_ref import HP, OracleViSNet, radius_graph_canonical, slots_to_edge_index

L = HP["L"]
SITES = L + 1
ULPS = 3
EPS = 1e-12                     # the clamp of the channel norms (VLN_EPS)
MAX_BRANCHES = 16


def engine_vectors(eng, n=None):
    """V[0..L] of the engine's last evaluation, fp32 [SITES, N, 3, D] -- what the adjoint's VecLayerNorms read."""
    n = eng.n_atoms if n is None else n
    return np.stack([eng.debug_read("V", k, (n, 3, HP["D"])) for k in range(SITES)])


class Candidates:
    """Per site and node, the channels the engine's argmax / argmin can be, from fp32 vectors ``vs`` [S, N, 3, D].

    ``rep_mx`` / ``rep_mn`` [S, N, D] (bool): the distinct choices to enumerate.  ``eq_mx`` / ``eq_mn``: every channel
    whose choice gives the same gradient as one of them (membership test for another evaluation's branch).  Collapsed,
    because the choice cannot matter there: max == min (delta == 0 zeroes g_mx and g_mn; every node at site 0, isolated
    atoms) keeps channel 0 only, and min candidates whose norm is below the clamp (their gradient is masked by
    n >= eps) keep the lowest of them."""

    def __init__(self, vs, ulps=ULPS):
        v = np.asarray(vs, dtype=np.float64)
        n = np.sqrt((v * v).sum(-2))                              # [S, N, D]
        nc = np.maximum(n, EPS)
        mx, mn = nc.max(-1, keepdims=True), nc.min(-1, keepdims=True)
        wmx = ulps * np.spacing(mx.astype(np.float32)).astype(np.float64)
        wmn = ulps * np.spacing(mn.astype(np.float32)).astype(np.float64)
        self.norms = nc
        self.eq_mx = nc >= mx - wmx
        self.eq_mn = nc <= mn + wmn
        self.rep_mx, self.rep_mn = self.eq_mx.copy(), self.eq_mn.copy()
        flat = (mx == mn)[..., 0]                                 # [S, N]
        first = np.zeros_like(self.rep_mx)
        first[..., 0] = True
        self.rep_mx[flat], self.rep_mn[flat] = first[flat], first[flat]
        self.eq_mx[flat], self.eq_mn[flat] = True, True
        clamped = self.rep_mn & (n < EPS)
        lowest = clamped & (np.cumsum(clamped, -1) == 1)
        self.rep_mn = (self.rep_mn & ~clamped) | lowest
        self.eq_mn |= n < EPS

    def ambiguous(self):
        """(site, node) pairs with more than one distinct choice."""
        return np.argwhere((self.rep_mx.sum(-1) > 1) | (self.rep_mn.sum(-1) > 1))

    def contains(self, natural, lo, hi):
        """True when the branch ``natural`` = {site: (amx, amn)} over nodes lo..hi-1 is one of the engine's."""
        ar = np.arange(lo, hi)
        for s, (amx, amn) in natural.items():
            amx, amn = np.asarray(amx), np.asarray(amn)
            if not (self.eq_mx[s, ar, amx].all() and self.eq_mn[s, ar, amn].all()):
                return False
        return True

    def branches(self, lo, hi, limit=MAX_BRANCHES):
        """Every branch the engine may have taken on nodes lo..hi-1: a list of pins {site: (amx, amn)} (int64 arrays
        over those nodes, every site pinned).  The product of the ambiguous sites' choices; more than ``limit``
        raises."""
        base = {s: (self.rep_mx[s, lo:hi].argmax(-1), self.rep_mn[s, lo:hi].argmax(-1)) for s in range(len(self.rep_mx))}
        amb = [(s, a) for s, a in self.ambiguous() if lo <= a < hi]
        opts = [[(s, a, i, j) for i in np.flatnonzero(self.rep_mx[s, a]) for j in np.flatnonzero(self.rep_mn[s, a])]
                for s, a in amb]
        count = int(np.prod([len(o) for o in opts])) if opts else 1
        if count > limit:
            raise RuntimeError(f"nodes {lo}..{hi - 1}: {count} VecLayerNorm branches (> {limit}) at {amb}")
        out = []
        for combo in itertools.product(*opts):
            pins = {s: (mx.copy(), mn.copy()) for s, (mx, mn) in base.items()}
            for s, a, i, j in combo:
                pins[s][0][a - lo], pins[s][1][a - lo] = i, j
            out.append(pins)
        return out


def natural_branch(vec_in):
    """The fp64 argmax / argmin {site: (amx, amn)} of the vectors ``vec_in`` = [V[0], .., V[L]] (torch or numpy)."""
    out = {}
    for s, v in enumerate(vec_in):
        v = torch.as_tensor(v)
        nc = torch.sqrt((v * v).sum(1)).clamp(min=EPS)
        out[s] = (nc.max(-1).indices.cpu().numpy(), nc.min(-1).indices.cpu().numpy())
    return out


def pinned_energy_and_forces(sd, z, pos, branches, batch=None):
    """fp64 hand-adjoint energy [G] and forces [N, 3] of one geometry on each branch of ``branches`` (CPU).  sd: state
    dict (numpy or torch); batch defaults to one graph."""
    z = np.asarray(z, dtype=np.int64)
    pos = np.asarray(pos, dtype=np.float32)
    batch = np.zeros(len(z), dtype=np.int64) if batch is None else np.asarray(batch, dtype=np.int64)
    slots, deg = radius_graph_canonical(pos, batch)
    ei = torch.from_numpy(slots_to_edge_index(slots, deg))
    adj = AdjointViSNet(OracleViSNet({k: torch.as_tensor(np.asarray(v)) for k, v in sd.items()}, torch.float64))
    out = []
    for pins in branches:
        E, F, _, _ = adj.energy_and_forces(z, pos, batch, ei, pins=pins)
        out.append((E.numpy()[:, 0], F.numpy()))
    return out


def best_branch(sd, cand, z, pos, lo, hi, f):
    """Of every branch ``cand`` allows on nodes lo..hi-1 -- one whole graph, z / pos / f indexed like them -- the fp64
    evaluation closest to the engine's forces f: (E, F [hi - lo, 3], branches tried)."""
    runs = pinned_energy_and_forces(sd, z[lo:hi], pos[lo:hi], cand.branches(lo, hi))
    er, fr = min(runs, key=lambda r: np.abs(np.asarray(f[lo:hi], np.float64) - r[1]).max())
    return float(er[0]), fr, len(runs)
