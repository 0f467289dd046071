"""Hand-derived adjoint (analytic -dE/dr) of the ViSNet hot path in plain PyTorch ops, NO autograd.
TEST INFRASTRUCTURE ONLY.

Purpose: the CUDA engine does not use autograd (the reference does: ``visnet.py:152-165``); its force
pass is a hand-written reverse sweep.  This file is the executable specification of that sweep, stage
by stage in the same decomposition as the kernels (node stage A/B, edge stage, embedding, head,
geometry), and is validated against ``torch.autograd`` on the oracle in fp64 (tests/test_adjoint.py).
``tools/stage_check.py`` compares the engine's per-stage buffers with the tensors saved here.

Conventions: edge e has source j = edge_index[0], target i = edge_index[1]; r, d = |pos_j-pos_i| and
its unit vector (0 on self-loops); W matrices are ``nn.Linear`` weights [out, in].
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from .visnet_ref import HP, OracleViSNet, cosine_cutoff


def silu(x):
    return x * torch.sigmoid(x)


def dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def ln_fwd(x, w, b, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    return (x - mu) * rstd * w + b


def ln_bwd(x, w, gy, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = (x - mu) * rstd
    gh = gy * w
    return rstd * (gh - gh.mean(-1, keepdim=True) - xh * (gh * xh).mean(-1, keepdim=True))


def _extremes(nc, pin):
    """(mx, amx, mn, amn) of the clamped channel norms nc [N,D]: the natural max / min, or with ``pin`` = (amx, amn)
    (long [N]) the norms of the pinned channels.  A pinned evaluation is one smooth branch of the model: the gather
    below is what the max / min are away from a tie, and its gradient goes to the pinned channels."""
    if pin is None:
        mx, amx = nc.max(-1)
        mn, amn = nc.min(-1)
        return mx, amx, mn, amn
    amx, amn = (torch.as_tensor(a, dtype=torch.long, device=nc.device) for a in pin)
    ar = torch.arange(nc.shape[0], device=nc.device)
    return nc[ar, amx], amx, nc[ar, amn], amn


def vecln_fwd(vec, w, eps=1e-12, pin=None):
    """utils.py:200-228.  The global ``(dist==0).all()`` early-out is value- and gradient-neutral
    (all-zero rows give 0 either way), so it is not restated.  pin: optional (amx, amn) per node (see _extremes)."""
    n = torch.sqrt((vec * vec).sum(1))                      # [N,D]
    nc = n.clamp(min=eps)
    mx, _, mn, _ = _extremes(nc, pin)
    delta = mx - mn
    delta = torch.where(delta == 0, torch.ones_like(delta), delta)
    y = (nc - mn[:, None]) / delta[:, None]
    return torch.relu(y)[:, None, :] * (vec / nc[:, None, :]) * w


def vecln_bwd(vec, w, gout, eps=1e-12, pin=None):
    n = torch.sqrt((vec * vec).sum(1))
    nc = n.clamp(min=eps)
    mx, amx, mn, amn = _extremes(nc, pin)
    delta_raw = mx - mn
    zero = delta_raw == 0
    delta = torch.where(zero, torch.ones_like(delta_raw), delta_raw)
    y = (nc - mn[:, None]) / delta[:, None]
    ry = torch.relu(y)
    dirv = vec / nc[:, None, :]
    gw = gout * w
    g_dir = gw * ry[:, None, :]
    g_y = (gw * dirv).sum(1) * (y > 0).to(vec.dtype)
    g_nc = g_y / delta[:, None]
    g_mn = -(g_y / delta[:, None]).sum(-1)
    g_delta = -(g_y * y).sum(-1) / delta
    g_delta = torch.where(zero, torch.zeros_like(g_delta), g_delta)
    g_mx = g_delta
    g_mn = g_mn - g_delta
    g_nc = g_nc.clone()
    ar = torch.arange(vec.shape[0], device=vec.device)
    g_nc[ar, amx] += g_mx
    g_nc[ar, amn] += g_mn
    g_vec = g_dir / nc[:, None, :]
    g_nc = g_nc - (g_dir * vec).sum(1) / (nc * nc)
    g_n = torch.where(n >= eps, g_nc, torch.zeros_like(g_nc))
    inv_n = torch.where(n > 0, 1.0 / torch.where(n > 0, n, torch.ones_like(n)), torch.zeros_like(n))
    return g_vec + (g_n * inv_n)[:, None, :] * vec


class AdjointViSNet:
    """Explicit forward (saving what the reverse sweep needs) + explicit reverse sweep.

    ``pins`` (forward, backward, energy_and_forces): optional {site: (amx [N], amn [N])} fixing the channels the
    VecLayerNorm(max_min) max / min take at a site; site l < L is layer l's ``vec_layernorm``, site L is
    ``vec_out_norm``.  Sites without a pin take the natural argmax / argmin.  Where two channel norms tie to fp32
    rounding the engine's branch is not the fp64 argmax (DESIGN section 2); pinned to the engine's channels the
    oracle is the smooth function whose gradient the engine computes (oracle/vecln_branch.py)."""

    def __init__(self, oracle: OracleViSNet):
        self.o = oracle
        self.sd = oracle.sd
        self.dtype = oracle.dtype
        self.D, self.L, self.H = HP["D"], HP["L"], HP["H"]

    # ---------------------------------------------------------------------------------- forward
    def forward(self, z, pos, batch, edge_index, pins=None) -> Dict[str, torch.Tensor]:
        sd, D, H, L = self.sd, self.D, self.H, self.L
        pins = pins or {}
        rm = "representation_model."
        S: Dict[str, torch.Tensor] = {}
        src, dst = edge_index[0], edge_index[1]
        n = z.shape[0]
        pos = pos.to(self.dtype)
        ev = pos[src] - pos[dst]
        mask = (src != dst)
        fm = mask.to(self.dtype)
        r = torch.sqrt((ev * ev).sum(-1)) * fm
        inv_r = torch.where(mask, 1.0 / torch.where(mask, r, torch.ones_like(r)), torch.zeros_like(r))
        d = ev * inv_r[:, None]
        C = cosine_cutoff(r, self.o.cutoff)
        rbf = self.o.rbf(r)
        S.update(r=r, d=d, C=C, rbf=rbf, mask=fm, inv_r=inv_r)

        p = rm + "neighbor_embedding."
        nb = sd[p + "embedding.weight"][z]
        dp = rbf @ sd[p + "distance_proj.weight"].T + sd[p + "distance_proj.bias"]
        agg = torch.zeros(n, D, dtype=self.dtype).index_add_(0, dst, dp * (C * fm)[:, None] * nb[src])
        x0 = sd[rm + "embedding.weight"][z]
        x = torch.cat([x0, agg], 1) @ sd[p + "combine.weight"].T + sd[p + "combine.bias"]
        ep = rbf @ sd[rm + "edge_embedding.edge_proj.weight"].T + sd[rm + "edge_embedding.edge_proj.bias"]
        f = (x[dst] + x[src]) * ep
        vec = torch.zeros(n, 3, D, dtype=self.dtype)
        S.update(x_emb=x, nb=nb, dp=dp, ep=ep)

        hsel = torch.arange(D) // (D // H)                    # channel -> head
        for l in range(L):
            last = l == L - 1
            p = rm + f"vis_mp_layers.{l}."
            S[f"x_in{l}"], S[f"vec_in{l}"], S[f"f_in{l}"] = x, vec, f
            # node stage A
            xn = ln_fwd(x, sd[p + "layernorm.weight"], sd[p + "layernorm.bias"])
            vn = vecln_fwd(vec, sd[p + "vec_layernorm.weight"], pin=pins.get(l))
            q = xn @ sd[p + "q_proj.weight"].T + sd[p + "q_proj.bias"]
            k = xn @ sd[p + "k_proj.weight"].T + sd[p + "k_proj.bias"]
            v = xn @ sd[p + "v_proj.weight"].T + sd[p + "v_proj.bias"]
            vp = vn @ sd[p + "vec_proj.weight"].T
            v1, v2, v3 = vp[..., :D], vp[..., D:2 * D], vp[..., 2 * D:]
            vdot = (v1 * v2).sum(1)
            S.update({f"xn{l}": xn, f"vn{l}": vn, f"q{l}": q, f"k{l}": k, f"v{l}": v, f"v1{l}": v1, f"v2{l}": v2,
                      f"v3{l}": v3, f"vdot{l}": vdot})
            if not last:
                t = vn @ sd[p + "w_trg_proj.weight"].T
                u = vn @ sd[p + "w_src_proj.weight"].T
                S[f"t{l}"], S[f"u{l}"] = t, u
            # edge stage
            dk = silu(f @ sd[p + "dk_proj.weight"].T + sd[p + "dk_proj.bias"])
            dv = silu(f @ sd[p + "dv_proj.weight"].T + sd[p + "dv_proj.bias"])
            a = (q[dst] * k[src] * dk).view(-1, H, D // H).sum(-1)
            A = silu(a) * C[:, None]
            m = v[src] * dv * A[:, hsel]
            s = silu(m @ sd[p + "s_proj.weight"].T + sd[p + "s_proj.bias"])
            s1, s2 = s[:, :D], s[:, D:]
            M = vn[src] * s1[:, None, :] + s2[:, None, :] * d[:, :, None]
            xa = torch.zeros(n, D, dtype=self.dtype).index_add_(0, dst, m)
            va = torch.zeros(n, 3, D, dtype=self.dtype).index_add_(0, dst, M)
            S[f"xa{l}"], S[f"va{l}"] = xa, va
            if not last:
                ti, uj = t[dst], u[src]
                a1 = (ti * d[:, :, None]).sum(1)
                a2 = (uj * d[:, :, None]).sum(1)
                w1 = ti - a1[:, None, :] * d[:, :, None]
                w2 = uj - a2[:, None, :] * d[:, :, None]
                wdot = (w1 * w2).sum(1)
                df = silu(f @ sd[p + "f_proj.weight"].T + sd[p + "f_proj.bias"]) * wdot
            # node stage B
            o = xa @ sd[p + "o_proj.weight"].T + sd[p + "o_proj.bias"]
            S[f"o{l}"] = o
            o1, o2, o3 = o[:, :D], o[:, D:2 * D], o[:, 2 * D:]
            x = x + vdot * o2 + o3
            vec = vec + v3 * o1[:, None, :] + va
            if not last:
                f = f + df
        S["x_out"], S["vec_out"] = x, vec

        # head (per atom)
        X = ln_fwd(x, sd[rm + "out_norm.weight"], sd[rm + "out_norm.bias"])
        V = vecln_fwd(vec, sd[rm + "vec_out_norm.weight"], pin=pins.get(L))
        o0, o1_ = "output_model.output_network.0.", "output_model.output_network.1."
        p1 = V @ sd[o0 + "vec1_proj.weight"].T
        n1 = torch.sqrt((p1 * p1).sum(1))
        p2 = V @ sd[o0 + "vec2_proj.weight"].T
        pre = torch.cat([X, n1], -1) @ sd[o0 + "update_net.0.weight"].T + sd[o0 + "update_net.0.bias"]
        y = silu(pre) @ sd[o0 + "update_net.2.weight"].T + sd[o0 + "update_net.2.bias"]
        xs, g = silu(y[:, :64]), y[:, 64:]
        Vp = g[:, None, :] * p2
        p1b = Vp @ sd[o1_ + "vec1_proj.weight"].T
        n1b = torch.sqrt((p1b * p1b).sum(1))
        preb = torch.cat([xs, n1b], -1) @ sd[o1_ + "update_net.0.weight"].T + sd[o1_ + "update_net.0.bias"]
        yb = silu(preb) @ sd[o1_ + "update_net.2.weight"].T + sd[o1_ + "update_net.2.bias"]
        e_atom = yb[:, :1] * sd["std"] + sd["prior_model.atomref.weight"][z]
        S.update(X=X, V=V, p1=p1, n1=n1, p2=p2, pre=pre, y=y, xs=xs, g=g, Vp=Vp, p1b=p1b, n1b=n1b, preb=preb,
                 e_atom=e_atom)
        G = int(batch.max().item()) + 1
        S["E"] = torch.zeros(G, 1, dtype=self.dtype).index_add_(0, batch, e_atom) + sd["mean"]
        return S

    # --------------------------------------------------------------------------------- backward
    def backward(self, z, pos, batch, edge_index, S, pins=None) -> Dict[str, torch.Tensor]:
        """Reverse sweep for dE_total/dpos; returns forces and every stage's adjoint (for stage checks).  ``pins``: as
        given to the forward that made S."""
        sd, D, H, L = self.sd, self.D, self.H, self.L
        pins = pins or {}
        rm = "representation_model."
        B: Dict[str, torch.Tensor] = {}
        src, dst = edge_index[0], edge_index[1]
        n, E = z.shape[0], src.shape[0]
        r, d, C, rbf, fm, inv_r = S["r"], S["d"], S["C"], S["rbf"], S["mask"], S["inv_r"]
        hsel = torch.arange(D) // (D // H)
        zN = lambda *sh: torch.zeros(*sh, dtype=self.dtype)

        def safe_div(a, b):
            return torch.where(b > 0, a / torch.where(b > 0, b, torch.ones_like(b)), torch.zeros_like(a))

        # ---- head ----
        o0, o1_ = "output_model.output_network.0.", "output_model.output_network.1."
        g_e = torch.ones(n, 1, dtype=self.dtype) * sd["std"]
        g_hb = g_e * sd[o1_ + "update_net.2.weight"][0:1, :]
        g_preb = g_hb * dsilu(S["preb"])
        g_catb = g_preb @ sd[o1_ + "update_net.0.weight"]
        g_xs, g_n1b = g_catb[:, :64], g_catb[:, 64:]
        g_p1b = safe_div(g_n1b, S["n1b"])[:, None, :] * S["p1b"]
        g_Vp = g_p1b @ sd[o1_ + "vec1_proj.weight"]
        g_g = (g_Vp * S["p2"]).sum(1)
        g_p2 = g_Vp * S["g"][:, None, :]
        g_y = torch.cat([g_xs * dsilu(S["y"][:, :64]), g_g], -1)
        g_h = g_y @ sd[o0 + "update_net.2.weight"]
        g_pre = g_h * dsilu(S["pre"])
        g_cat = g_pre @ sd[o0 + "update_net.0.weight"]
        g_X, g_n1 = g_cat[:, :D], g_cat[:, D:]
        g_p1 = safe_div(g_n1, S["n1"])[:, None, :] * S["p1"]
        g_V = g_p1 @ sd[o0 + "vec1_proj.weight"] + g_p2 @ sd[o0 + "vec2_proj.weight"]
        gvec = vecln_bwd(S["vec_out"], sd[rm + "vec_out_norm.weight"], g_V, pin=pins.get(L))
        gx = ln_bwd(S["x_out"], sd[rm + "out_norm.weight"], g_X)
        B["gx_out"], B["gvec_out"] = gx, gvec

        g_C = zN(E)          # accumulates dE/dC(r_e) over layers + neighbour embedding
        g_d = zN(E, 3)       # accumulates dE/dd_e
        gf = zN(E, D)        # dE/df_{l+1}
        for l in reversed(range(L)):
            last = l == L - 1
            p = rm + f"vis_mp_layers.{l}."
            x_in, vec_in, f = S[f"x_in{l}"], S[f"vec_in{l}"], S[f"f_in{l}"]
            vn, q, k, v = S[f"vn{l}"], S[f"q{l}"], S[f"k{l}"], S[f"v{l}"]
            v1, v2, v3, vdot, o = S[f"v1{l}"], S[f"v2{l}"], S[f"v3{l}"], S[f"vdot{l}"], S[f"o{l}"]
            o1, o2 = o[:, :D], o[:, D:2 * D]
            # ---- node stage B adjoint (o-projection) ----
            g_o = torch.cat([(gvec * v3).sum(1), gx * vdot, gx], -1)
            g_vdot = gx * o2
            g_v3 = gvec * o1[:, None, :]
            g_xa = g_o @ sd[p + "o_proj.weight"]
            g_va = gvec
            B[f"g_xa{l}"] = g_xa
            # ---- edge stage adjoint (recompute forward pieces) ----
            Pdk = f @ sd[p + "dk_proj.weight"].T + sd[p + "dk_proj.bias"]
            Pdv = f @ sd[p + "dv_proj.weight"].T + sd[p + "dv_proj.bias"]
            dk, dv = silu(Pdk), silu(Pdv)
            qi, kj, vj, vnj = q[dst], k[src], v[src], vn[src]
            a = (qi * kj * dk).view(-1, H, D // H).sum(-1)
            sa = silu(a)
            A = sa * C[:, None]
            m = vj * dv * A[:, hsel]
            Spre = m @ sd[p + "s_proj.weight"].T + sd[p + "s_proj.bias"]
            s = silu(Spre)
            s1, s2 = s[:, :D], s[:, D:]
            gM = g_va[dst]                                           # [E,3,D]
            g_s = torch.cat([(gM * vnj).sum(1), (gM * d[:, :, None]).sum(1)], -1)
            g_vn = zN(n, 3, D).index_add_(0, src, gM * s1[:, None, :])
            g_d = g_d + (gM * s2[:, None, :]).sum(-1)
            g_Spre = g_s * dsilu(Spre)
            g_m = g_xa[dst] + g_Spre @ sd[p + "s_proj.weight"]
            g_v = zN(n, D).index_add_(0, src, g_m * dv * A[:, hsel])
            g_dv = g_m * vj * A[:, hsel]
            g_A = (g_m * vj * dv).view(-1, H, D // H).sum(-1)
            g_a = g_A * C[:, None] * dsilu(a)
            g_C = g_C + (g_A * sa).sum(-1)
            g_q = zN(n, D).index_add_(0, dst, g_a[:, hsel] * kj * dk)
            g_k = zN(n, D).index_add_(0, src, g_a[:, hsel] * qi * dk)
            g_dk = g_a[:, hsel] * qi * kj
            g_P = [g_dk * dsilu(Pdk), g_dv * dsilu(Pdv)]
            Wcat = [sd[p + "dk_proj.weight"], sd[p + "dv_proj.weight"]]
            if not last:
                t, u = S[f"t{l}"], S[f"u{l}"]
                Pf = f @ sd[p + "f_proj.weight"].T + sd[p + "f_proj.bias"]
                fp = silu(Pf)
                ti, uj = t[dst], u[src]
                dd = d[:, :, None]
                a1 = (ti * dd).sum(1)
                a2 = (uj * dd).sum(1)
                w1 = ti - a1[:, None, :] * dd
                w2 = uj - a2[:, None, :] * dd
                wdot = (w1 * w2).sum(1)
                g_fp = gf * wdot
                g_wdot = gf * fp
                g_w1 = g_wdot[:, None, :] * w2
                g_w2 = g_wdot[:, None, :] * w1
                c1 = (g_w1 * dd).sum(1)                               # [E,D]
                c2 = (g_w2 * dd).sum(1)
                g_ti = g_w1 - c1[:, None, :] * dd
                g_uj = g_w2 - c2[:, None, :] * dd
                g_d = g_d - (ti * c1[:, None, :]).sum(-1) - (a1[:, None, :] * g_w1).sum(-1) \
                    - (uj * c2[:, None, :]).sum(-1) - (a2[:, None, :] * g_w2).sum(-1)
                g_t = zN(n, 3, D).index_add_(0, dst, g_ti)
                g_u = zN(n, 3, D).index_add_(0, src, g_uj)
                g_P.append(g_fp * dsilu(Pf))
                Wcat.append(sd[p + "f_proj.weight"])
            gf = gf + torch.cat(g_P, -1) @ torch.cat(Wcat, 0)
            B[f"gf_in{l}"] = gf
            B[f"g_q{l}"], B[f"g_k{l}"], B[f"g_v{l}"], B[f"g_vn_msg{l}"] = g_q, g_k, g_v, g_vn
            # ---- node stage A adjoint ----
            g_xn = torch.cat([g_q, g_k, g_v], -1) @ torch.cat(
                [sd[p + "q_proj.weight"], sd[p + "k_proj.weight"], sd[p + "v_proj.weight"]], 0)
            g_vp = torch.cat([g_vdot[:, None, :] * v2, g_vdot[:, None, :] * v1, g_v3], -1)
            g_vn = g_vn + g_vp @ sd[p + "vec_proj.weight"]
            if not last:
                B[f"g_t{l}"], B[f"g_u{l}"] = g_t, g_u
                g_vn = g_vn + g_t @ sd[p + "w_trg_proj.weight"] + g_u @ sd[p + "w_src_proj.weight"]
            B[f"g_vn{l}"], B[f"g_xn{l}"] = g_vn, g_xn
            gvec = gvec + vecln_bwd(vec_in, sd[p + "vec_layernorm.weight"], g_vn, pin=pins.get(l))
            gx = gx + ln_bwd(x_in, sd[p + "layernorm.weight"], g_xn)
            B[f"gx_in{l}"], B[f"gvec_in{l}"] = gx, gvec

        # ---- embedding adjoint ----
        x, ep, dp, nb = S["x_emb"], S["ep"], S["dp"], S["nb"]
        gfe = gf * ep
        gx = gx + zN(n, D).index_add_(0, dst, gfe) + zN(n, D).index_add_(0, src, gfe)
        g_ep = gf * (x[dst] + x[src])
        g_rbf = g_ep @ sd[rm + "edge_embedding.edge_proj.weight"]
        p = rm + "neighbor_embedding."
        g_agg = (gx @ sd[p + "combine.weight"])[:, D:]
        g_We = g_agg[dst] * nb[src] * fm[:, None]
        g_C = g_C + (g_We * dp).sum(-1)
        g_rbf = g_rbf + (g_We * C[:, None]) @ sd[p + "distance_proj.weight"]
        B["gx_emb"], B["g_rbf"], B["g_C"], B["g_d"] = gx, g_rbf, g_C, g_d
        # ---- geometry adjoint ----
        pp = rm + "distance_expansion."
        means, betas = sd[pp + "means"], sd[pp + "betas"]
        alpha = 5.0 / self.o.cutoff
        cut = self.o.cutoff
        dC = -0.5 * math.pi / cut * torch.sin(r * math.pi / cut) * (r < cut).to(self.dtype)
        ex = torch.exp(-alpha * r)[:, None]
        gk = torch.exp(-betas * (ex - means) ** 2)
        drbf = dC[:, None] * gk + C[:, None] * gk * (2 * betas * alpha) * (ex - means) * ex
        g_r = g_C * dC + (g_rbf * drbf).sum(-1)
        g_ev = (g_r[:, None] * d + (g_d - (g_d * d).sum(-1, keepdim=True) * d) * inv_r[:, None]) * fm[:, None]
        dpos = zN(n, 3).index_add_(0, src, g_ev).index_add_(0, dst, -g_ev)
        B["g_r"], B["g_ev"] = g_r, g_ev
        B["forces"] = -dpos
        return B

    def energy_and_forces(self, z, pos, batch, edge_index, pins=None):
        z = torch.as_tensor(z, dtype=torch.long)
        batch = torch.as_tensor(batch, dtype=torch.long)
        pos = torch.as_tensor(pos).to(self.dtype)
        with torch.no_grad():
            S = self.forward(z, pos, batch, edge_index, pins)
            B = self.backward(z, pos, batch, edge_index, S, pins)
        return S["E"], B["forces"], S, B
