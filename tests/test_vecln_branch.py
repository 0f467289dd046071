"""The branch-pinned fp64 oracle and the helper that names the VecLayerNorm(max_min) branch the engine took
(oracle/vecln_branch.py), without a GPU.

a. Pinned to its own natural argmax / argmin, the hand adjoint is bit for bit the unpinned one.
b. Pinned to a non-maximal (non-minimal) channel, it is the exact gradient of the pinned forward: torch.autograd in fp64
   and central finite differences.
c. The pin matters: in whole Chignolin (one graph) the two branches of the layer-4 tie at atom 130 give forces further
   apart than the force bar, so a check on the wrong branch fails.
d. Engine.vecln_near_ties scans the head's vec_out_norm site too.
e. The candidate sets on constructed channel norms: ulp window, collapse at delta == 0 and below the clamp, the cap.
"""
import os
import types

import numpy as np
import pytest
import torch

from ai2bmd_b200.engine import Engine
from oracle import visnet_ref as O
from oracle.adjoint_ref import AdjointViSNet
from oracle.vecln_branch import MAX_BRANCHES, SITES, Candidates, natural_branch, pinned_energy_and_forces

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
D = 128


def _weights(real_weights, which):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in real_weights.items()} if which == "real" \
        else O.random_state_dict(3)


def _sub(chig):
    fd, _ = chig
    sub = fd[0:4]
    s, d = O.radius_graph_canonical(sub.pos, sub.batch)
    return sub, torch.from_numpy(O.slots_to_edge_index(s, d))


def _site_vectors(S):
    return [S[f"vec_in{l}"] for l in range(SITES - 1)] + [S["vec_out"]]


def _norms(v):
    return torch.sqrt((v * v).sum(1)).clamp(min=1e-12)


# ---- a. natural pins are the unpinned oracle -------------------------------------------------------------------------
@pytest.mark.parametrize("weights", ["real", "random"])
def test_natural_pins_are_bit_identical(real_weights, chig, weights):
    sub, ei = _sub(chig)
    adj = AdjointViSNet(O.OracleViSNet(_weights(real_weights, weights), torch.float64))
    E, F, S, B = adj.energy_and_forces(sub.z, sub.pos, sub.batch, ei)
    pins = natural_branch(_site_vectors(S))
    E2, F2, S2, B2 = adj.energy_and_forces(sub.z, sub.pos, sub.batch, ei, pins=pins)
    assert torch.equal(E, E2) and torch.equal(F, F2)
    assert all(torch.equal(B[k], B2[k]) for k in B) and all(torch.equal(S[k], S2[k]) for k in S)


# ---- b. a pinned branch is differentiated exactly --------------------------------------------------------------------
def _second(nc, node, largest):
    order = torch.argsort(nc[node], descending=largest)
    return int(order[1])


@pytest.mark.parametrize("weights", ["real", "random"])
def test_pinned_adjoint_is_the_gradient_of_the_pinned_forward(real_weights, chig, weights, monkeypatch):
    sub, ei = _sub(chig)
    adj = AdjointViSNet(O.OracleViSNet(_weights(real_weights, weights), torch.float64))
    z, batch = torch.as_tensor(sub.z, dtype=torch.long), torch.as_tensor(sub.batch, dtype=torch.long)
    pos0 = torch.as_tensor(sub.pos, dtype=torch.float64)
    with torch.no_grad():
        S = adj.forward(z, pos0, batch, ei)
    nat = natural_branch(_site_vectors(S))
    pins = {s: (torch.from_numpy(a.copy()), torch.from_numpy(b.copy())) for s, (a, b) in nat.items()}
    vs = _site_vectors(S)
    moved = []                                       # (site, node): argmax -> second largest, or argmin -> second smallest
    for s, node, largest in [(1, 3, True), (2, 20, True), (4, 11, False), (5, 40, True), (6, 7, True), (6, 30, False)]:
        alt = _second(_norms(vs[s]), node, largest)
        pins[s][0 if largest else 1][node] = alt
        moved.append((s, node))
    _, F, _, _ = adj.energy_and_forces(z, pos0, batch, ei, pins=pins)
    _, F_nat, _, _ = adj.energy_and_forces(z, pos0, batch, ei)
    assert (F - F_nat).abs().max() > 1e-4                                  # the pins change the forces

    calls = []

    def pinned_vecln(vec, weight):                   # visnet_ref.vec_layer_norm_max_min, max / min gathered at the pins
        site = len(calls)
        calls.append(site)
        dist = torch.norm(vec, dim=1, keepdim=True)
        if (dist == 0).all():
            return torch.zeros_like(vec) * weight.view(1, 1, -1)
        dist = dist.clamp(min=1e-12)
        ar = torch.arange(vec.shape[0])
        max_val, min_val = dist[ar, 0, pins[site][0]], dist[ar, 0, pins[site][1]]
        delta = max_val - min_val
        delta = torch.where(delta == 0, torch.ones_like(delta), delta)
        y = (dist - min_val.view(-1, 1, 1)) / delta.view(-1, 1, 1)
        return torch.relu(y) * (vec / dist) * weight.view(1, 1, -1)

    monkeypatch.setattr(O, "vec_layer_norm_max_min", pinned_vecln)
    _, g = adj.o.energy_and_forces(z, pos0, batch, edge_index=ei)           # torch.autograd of the pinned forward
    assert calls == list(range(SITES))
    assert (F - g).abs().max().item() <= 1e-11 * g.abs().max().item()

    def energy(p):
        with torch.no_grad():
            return adj.forward(z, p, batch, ei, pins=pins)["E"].sum().item()

    h, tol = 1e-5, lambda f: 2e-6 + 1e-5 * abs(f)                         # noqa: E731
    atoms = sorted({node for _, node in moved})
    for a in atoms:
        for c in range(3):
            dp = torch.zeros_like(pos0)
            dp[a, c] = h
            fd_force = -(energy(pos0 + dp) - energy(pos0 - dp)) / (2 * h)
            assert abs(fd_force - F[a, c].item()) <= tol(F[a, c].item()), (a, c, fd_force, F[a, c])
    assert (F - F_nat)[atoms].abs().max() > 100 * tol(F[atoms].abs().max().item())   # the pins move these forces


# ---- c. the pin changes the answer -----------------------------------------------------------------------------------
def test_the_chignolin_tie_branches_differ_by_more_than_the_bar(real_weights):
    g = np.load(os.path.join(ROOT, "tests", "golden", "reference_visnet_mode.npz"))
    z, pos = g["chig_z"], g["chig_pos"]
    batch = np.zeros(len(z), dtype=np.int64)
    s, d = O.radius_graph_canonical(pos, batch)
    ei = torch.from_numpy(O.slots_to_edge_index(s, d))
    adj = AdjointViSNet(O.OracleViSNet(_weights(real_weights, "real"), torch.float64))
    _, F, S, _ = adj.energy_and_forces(z, pos, batch, ei)
    nc = _norms(S["vec_in4"])[130]
    top = torch.topk(nc, 2)
    assert (top.values[0] - top.values[1]) / top.values[0] < 1e-5           # the tie
    nat = natural_branch(_site_vectors(S))
    assert nat[4][0][130] == int(top.indices[0])
    alt = {k: (a.copy(), b.copy()) for k, (a, b) in nat.items()}
    alt[4][0][130] = int(top.indices[1])
    (e_nat, f_nat), (e_alt, f_alt) = pinned_energy_and_forces(real_weights, z, pos, [nat, alt])
    assert np.array_equal(f_nat, F.numpy())
    f_bar = 5e-5 + 2e-5 * np.abs(f_nat).max()
    jump = np.abs(f_alt - f_nat).max()
    print(f"whole Chignolin, atom 130 layer 4: branch jump {jump:.3e} eV/A, bar {f_bar:.3e}")
    assert jump > 10 * f_bar
    assert abs(e_alt[0] - e_nat[0]) <= 1e-6 * abs(e_nat[0])                # the same energy, to the tie's gap


# ---- d. the tie scan covers the output norm --------------------------------------------------------------------------
def _spread_vectors(rng, n):
    """[n, 3, D] vectors whose channel norms are 1 + c / D in a random order per node: no two within 1e-5."""
    dirs = rng.standard_normal((n, 3, D))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    norms = np.stack([1.0 + rng.permutation(D) / D for _ in range(n)])
    return (dirs * norms[:, None, :]).astype(np.float32)


def test_near_ties_scan_the_output_norm():
    rng = np.random.default_rng(0)
    n = 6
    V = [np.zeros((n, 3, D), np.float32)] + [_spread_vectors(rng, n) for _ in range(SITES - 1)]
    nc = np.linalg.norm(V[6][3].astype(np.float64), axis=0)
    top, second = np.argsort(nc)[-1], np.argsort(nc)[-2]
    V[6][3, :, second] *= np.float32(nc[top] * (1 - 1e-7) / nc[second])   # a tie planted only at vec_out_norm
    stub = types.SimpleNamespace(n_atoms=n, debug_read=lambda name, k, shape: V[k].reshape(shape))
    assert list(Engine.vecln_near_ties(stub)) == [3]
    V[6][3, :, second] *= np.float32(0.9)
    assert list(Engine.vecln_near_ties(stub)) == []


# ---- e. candidate sets -----------------------------------------------------------------------------------------------
def _vectors_from_norms(norms):
    """fp32 [SITES, N, 3, D] vectors along y with the given fp32 channel norms [N, D] at every site."""
    v = np.zeros((SITES,) + norms.shape[:1] + (3, D), np.float32)
    v[:, :, 1, :] = norms
    return v


def test_candidate_sets_on_constructed_norms():
    f = np.float32(1.5)
    below = lambda k: np.float32(f - k * np.spacing(f))                      # noqa: E731
    norms = np.tile(np.linspace(0.5, 1.25, D, dtype=np.float32), (6, 1))     # node 0: a clear max and min
    norms[1, 10], norms[1, 20] = f, below(1)                                 # node 1: two max channels 1 ulp apart
    norms[2, 10], norms[2, 30] = f, below(8)                                 # node 2: the second 8 ulps down
    norms[3] = 0.0                                                           # node 3: all zero -> delta == 0
    norms[4, [5, 9, 70]] = 0.0                                               # node 4: three channels below the clamp
    norms[5] = 0.75                                                          # node 5: equal positive norms
    c = Candidates(_vectors_from_norms(norms))
    rmx, rmn = c.rep_mx[3], c.rep_mn[3]
    assert list(np.flatnonzero(rmx[0])) == [D - 1] and list(np.flatnonzero(rmn[0])) == [0]
    assert list(np.flatnonzero(rmx[1])) == [10, 20]
    assert list(np.flatnonzero(rmx[2])) == [10]
    assert list(np.flatnonzero(rmx[3])) == [0] and list(np.flatnonzero(rmn[3])) == [0] and c.eq_mx[3, 3].all()
    assert list(np.flatnonzero(rmn[4])) == [5] and list(np.flatnonzero(c.eq_mn[3, 4])) == [5, 9, 70]
    assert list(np.flatnonzero(rmx[5])) == [0] and list(np.flatnonzero(rmn[5])) == [0]
    assert {(int(s), int(a)) for s, a in c.ambiguous()} == {(s, 1) for s in range(SITES)}
    assert len(c.branches(0, 1)) == 1 and len(c.branches(2, 6)) == 1
    with pytest.raises(RuntimeError, match="branches"):
        c.branches(0, 6)                                                     # 2 ** 7 > MAX_BRANCHES
    c1 = Candidates(_vectors_from_norms(norms)[:1])                         # site 0 only: one ambiguous pair
    b = c1.branches(1, 2)
    assert len(b) == 2 and sorted(int(p[0][0][0]) for p in b) == [10, 20] and MAX_BRANCHES >= 2
    nat = {0: (np.array([20]), np.array([0]))}
    assert c1.contains(nat, 1, 2) and not c1.contains({0: (np.array([30]), np.array([0]))}, 1, 2)
    assert c1.contains({0: (np.array([7]), np.array([9]))}, 3, 4)           # delta == 0: any choice
    assert c1.contains({0: (np.array([D - 1]), np.array([70]))}, 4, 5)      # below the clamp: any of them
