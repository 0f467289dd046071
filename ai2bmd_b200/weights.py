"""Checkpoint -> flat fp32 weight blob in the order of ``vb_weight_manifest()``.

The checkpoint keys are the reference's (``/root/reference/src/ViSNet/model/visnet.py:73-93`` strips the
leading ``model.``; tensor inventory in SURVEY.md App. B).  "T" entries are the transposed ``nn.Linear``
weights ([in][out]) read by the forward GEMMs, "N" entries the native [out][in] layout read by the adjoint
GEMMs; fused matrices ([q|k|v], [dk|dv|f], [w_trg|w_src]) are concatenated along the output dimension.
"""
from __future__ import annotations

import re
from typing import Dict, Optional, Tuple

import numpy as np

D, L = 128, 6


def load_state_dict(path: str) -> Dict[str, np.ndarray]:
    """``.ckpt`` (Lightning checkpoint as shipped by the reference) or ``.npz`` (extracted state_dict)."""
    return load_checkpoint(path)[0]


def resolve_derivative(checkpoint_derivative: bool, derivative: Optional[bool] = None) -> bool:
    """The reference's rule (``load_model(path, derivative=...)``, ``visnet.py:73-81``): the checkpoint's hyper-parameter,
    overridden by an explicit keyword."""
    return bool(checkpoint_derivative) if derivative is None else bool(derivative)


def load_checkpoint(path: str) -> Tuple[Dict[str, np.ndarray], bool]:
    """(state_dict, the checkpoint's ``derivative`` hyper-parameter).  An ``.npz`` carries no hyper-parameters and counts
    as ``derivative=True``, as does a checkpoint that does not set it.  Every other hyper-parameter must be the one the
    kernels are specialised for."""
    if path.endswith(".npz"):
        z = np.load(path)
        return {k: np.asarray(z[k], dtype=np.float32) for k in z.files}, True
    import torch
    try:
        ck = torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:      # Lightning checkpoints may pickle non-tensor objects in hyper_parameters
        raise RuntimeError(f"{path}: torch.load(weights_only=True) refused the file ({e}); the reference loads it with full "
                           "unpickling -- for a TRUSTED file, re-save its state_dict (or an .npz of it) and load that") from e
    hp = ck.get("hyper_parameters", {})
    if hp:
        want = dict(embedding_dimension=128, num_layers=6, num_heads=8, num_rbf=32, lmax=1, max_num_neighbors=32,
                    vecnorm_type="max_min", rbf_type="expnorm", activation="silu", attn_activation="silu", cutoff=5.0,
                    max_z=100, prior_model="Atomref", reduce_op="add")
        for k, v in want.items():
            if k in hp and hp[k] != v:
                raise ValueError(f"checkpoint hyper-parameter {k}={hp.get(k)!r} is not the supported {v!r}")
        if "derivative" in hp and hp["derivative"] not in (True, False):
            raise ValueError(f"checkpoint hyper-parameter derivative={hp['derivative']!r} is not a bool")
    sd = {re.sub(r"^model\.", "", k): v.float().numpy() for k, v in ck["state_dict"].items()}
    return sd, bool(hp.get("derivative", True)) if hp else True


def _named_arrays(sd: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    f = lambda k: np.asarray(sd[k], dtype=np.float32)
    rm = "representation_model."
    o0, o1 = "output_model.output_network.0.", "output_model.output_network.1."
    out: Dict[str, np.ndarray] = {}
    out["emb"] = f(rm + "embedding.weight")
    out["nb_emb"] = f(rm + "neighbor_embedding.embedding.weight")
    out["rbf_means"] = f(rm + "distance_expansion.means")
    out["rbf_betas"] = f(rm + "distance_expansion.betas")
    out["WdN"] = f(rm + "neighbor_embedding.distance_proj.weight")
    out["WdT"] = out["WdN"].T
    out["bd"] = f(rm + "neighbor_embedding.distance_proj.bias")
    wc = f(rm + "neighbor_embedding.combine.weight")
    out["WcT"], out["bc"], out["WcN"] = wc.T, f(rm + "neighbor_embedding.combine.bias"), wc
    out["WeN"] = f(rm + "edge_embedding.edge_proj.weight")
    out["WeT"] = out["WeN"].T
    out["be"] = f(rm + "edge_embedding.edge_proj.bias")
    out["on_w"], out["on_b"] = f(rm + "out_norm.weight"), f(rm + "out_norm.bias")
    out["von_w"] = f(rm + "vec_out_norm.weight")
    for tag, pre in (("h0", o0), ("h1", o1)):
        w1 = f(pre + "vec1_proj.weight")
        out[f"{tag}_W1T"], out[f"{tag}_W1N"] = w1.T, w1
        u0 = f(pre + "update_net.0.weight")
        out[f"{tag}_U0T"], out[f"{tag}_b0"], out[f"{tag}_U0N"] = u0.T, f(pre + "update_net.0.bias"), u0
    w2 = f(o0 + "vec2_proj.weight")
    out["h0_W2T"], out["h0_W2N"] = w2.T, w2
    u2 = f(o0 + "update_net.2.weight")
    out["h0_U2T"], out["h0_b2"], out["h0_U2N"] = u2.T, f(o0 + "update_net.2.bias"), u2
    out["h1_u2"] = f(o1 + "update_net.2.weight")[0]
    out["h1_b2"] = np.array([f(o1 + "update_net.2.bias")[0], 0, 0, 0], dtype=np.float32)
    # absent prior / standardisation tensors mean "no prior", std 1, mean 0 (visnet.py:141-149)
    out["atomref"] = (f("prior_model.atomref.weight").reshape(-1) if "prior_model.atomref.weight" in sd
                      else np.zeros(100, dtype=np.float32))
    out["scalars"] = np.array([float(sd.get("std", 1.0)), float(sd.get("mean", 0.0)), 0, 0], dtype=np.float32)
    for l in range(L):
        p = rm + f"vis_mp_layers.{l}."
        last = l == L - 1
        z = np.zeros((D, D), dtype=np.float32)
        zb = np.zeros((D,), dtype=np.float32)
        k = f"layer{l}."
        out[k + "ln_w"], out[k + "ln_b"] = f(p + "layernorm.weight"), f(p + "layernorm.bias")
        out[k + "vln_w"] = f(p + "vec_layernorm.weight")
        wqkv = np.concatenate([f(p + "q_proj.weight"), f(p + "k_proj.weight"), f(p + "v_proj.weight")], 0)
        out[k + "WqkvT"], out[k + "WqkvN"] = wqkv.T, wqkv
        out[k + "bqkv"] = np.concatenate([f(p + "q_proj.bias"), f(p + "k_proj.bias"), f(p + "v_proj.bias")])
        wv = f(p + "vec_proj.weight")
        out[k + "WvecT"], out[k + "WvecN"] = wv.T, wv
        wtu = np.concatenate([z if last else f(p + "w_trg_proj.weight"), z if last else f(p + "w_src_proj.weight")], 0)
        out[k + "WtuT"], out[k + "WtuN"] = wtu.T, wtu
        w1 = np.concatenate([f(p + "dk_proj.weight"), f(p + "dv_proj.weight"), z if last else f(p + "f_proj.weight")], 0)
        out[k + "W1T"], out[k + "W1N"] = w1.T, w1
        out[k + "b1"] = np.concatenate([f(p + "dk_proj.bias"), f(p + "dv_proj.bias"), zb if last else f(p + "f_proj.bias")])
        ws = f(p + "s_proj.weight")
        out[k + "WsT"], out[k + "bs"], out[k + "WsN"] = ws.T, f(p + "s_proj.bias"), ws
        wo = f(p + "o_proj.weight")
        out[k + "WoT"], out[k + "bo"], out[k + "WoN"] = wo.T, f(p + "o_proj.bias"), wo
        # tensor-core images: forward chunks use W[n_out][k_in]; adjoint chunks use (W[k_out-chunk][n_in])^T
        out[k + "tcW1"] = np.concatenate([tc_image(w1[c * D:(c + 1) * D]) for c in range(3)])
        out[k + "tcWs"] = np.concatenate([tc_image(ws[c * D:(c + 1) * D]) for c in range(2)])
        out[k + "tcWsN"] = np.concatenate([tc_image(ws[c * D:(c + 1) * D].T) for c in range(2)])
        out[k + "tcW1N"] = np.concatenate([tc_image(w1[c * D:(c + 1) * D].T) for c in range(3)])
        # node stage on tensor cores (k_node_tc.cuh)
        wvt = np.concatenate([wv, wtu], 0)                      # [v1 | v2 | v3 | t | u] : [640, 128]
        out[k + "tcWo"] = np.concatenate([tc_image(wo[c * D:(c + 1) * D]) for c in range(3)])
        out[k + "tcWqkv"] = np.concatenate([tc_image(wqkv[c * D:(c + 1) * D]) for c in range(3)])
        out[k + "tcWvt"] = np.concatenate([tc_image(wvt[c * D:(c + 1) * D]) for c in range(5)])
        out[k + "tcWoN"] = np.concatenate([tc_image(wo[c * D:(c + 1) * D].T) for c in range(3)])
        out[k + "tcWqkvN"] = np.concatenate([tc_image(wqkv[c * D:(c + 1) * D].T) for c in range(3)])
        out[k + "tcWvtN"] = np.concatenate([tc_image(wvt[c * D:(c + 1) * D].T) for c in range(5)])
    return out


def pack_weights(sd: Dict[str, np.ndarray], manifest: str) -> np.ndarray:
    """Flatten per the library's manifest string ``name:count;...``; sizes are cross-checked."""
    arrays = _named_arrays(sd)
    parts = []
    for item in manifest.strip(";").split(";"):
        name, count = item.split(":")
        a = np.ascontiguousarray(arrays[name], dtype=np.float32).reshape(-1)
        if a.size != int(count):
            raise ValueError(f"weight {name}: have {a.size} values, manifest wants {count}")
        parts.append(a)
    return np.concatenate(parts)


# ---- tensor-core weight images (wgmma path) -------------------------------------------------------------
def round_tf32(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest (ties away) to tf32: keep 10 explicit mantissa bits (PTX ``cvt.rna.tf32.f32``)."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def tc_image(w_nk: np.ndarray) -> np.ndarray:
    """Shared-memory image of a GEMM chunk for ``wgmma.mma_async`` (B operand, K-major, SWIZZLE_128B).

    ``w_nk`` is [128 output columns][K] (K multiple of 32): D[m][n] = sum_k A[m][k] * w_nk[n][k].
    Output: for every K-slab of 32 a 16 KB "hi" plane then a 16 KB "lo" plane (3xTF32 split); inside a plane
    row n occupies bytes [n*128, n*128+128) and its 16-byte chunk c sits at chunk position c ^ (n & 7)."""
    w = np.ascontiguousarray(w_nk, dtype=np.float32)
    n, k = w.shape
    assert n == 128 and k % 32 == 0
    hi = round_tf32(w)
    lo = round_tf32(w - hi)
    rows = np.arange(128)
    out = np.empty((k // 32, 2, 128, 8, 4), dtype=np.float32)
    for s in range(k // 32):
        for p, plane in enumerate((hi, lo)):
            blk = plane[:, s * 32:(s + 1) * 32].reshape(128, 8, 4)
            for c in range(8):
                out[s, p, rows, c ^ (rows & 7), :] = blk[:, c, :]
    return out.reshape(-1)
