// Weight table and workspace layout of the ViSNet sm_90a engine (host + device views).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include "common.cuh"

namespace vb {

// ---- canonical weight manifest -----------------------------------------------------------------
// One flat fp32 blob, tensors in exactly this order.  "T" = stored [in][out] (transposed nn.Linear
// weight, forward GEMM reads rows by input index), "N" = stored [out][in] (nn.Linear layout, used by
// the adjoint GEMMs).  The Python packer (ai2bmd_b200/weights.py) follows vb_weight_manifest().
//   reference tensors: SURVEY.md App. B / checkpoint state_dict keys.
#define VB_GLOBAL_WEIGHTS(X)                                                                      \
    X(emb, 100 * D)        /* representation_model.embedding.weight                     */        \
    X(nb_emb, 100 * D)     /* neighbor_embedding.embedding.weight                        */        \
    X(rbf_means, NR) X(rbf_betas, NR)                                                              \
    X(WdN, D * NR) X(WdT, NR * D) X(bd, D) /* neighbor_embedding.distance_proj [128,32] (+ transposed) */     \
    X(WcT, 2 * D * D) X(bc, D) X(WcN, D * 2 * D) /* neighbor_embedding.combine [128,256] */        \
    X(WeN, D * NR) X(WeT, NR * D) X(be, D) /* edge_embedding.edge_proj [128,32] (+ transposed) */             \
    X(on_w, D) X(on_b, D) X(von_w, D)  /* out_norm, vec_out_norm                         */        \
    X(h0_W1T, D * D) X(h0_W1N, D * D)          /* head block 0 vec1_proj [128,128]       */        \
    X(h0_W2T, D * 64) X(h0_W2N, 64 * D)        /* head block 0 vec2_proj [64,128]        */        \
    X(h0_U0T, 2 * D * D) X(h0_b0, D) X(h0_U0N, D * 2 * D) /* update_net.0 [128,256]      */        \
    X(h0_U2T, D * D) X(h0_b2, D) X(h0_U2N, D * D)         /* update_net.2 [128,128]      */        \
    X(h1_W1T, 64 * 64) X(h1_W1N, 64 * 64)      /* head block 1 vec1_proj [64,64]         */        \
    X(h1_U0T, D * 64) X(h1_b0, 64) X(h1_U0N, 64 * D)      /* update_net.0 [64,128]       */        \
    X(h1_u2, 64) X(h1_b2, 4)                   /* update_net.2 row 0 [64], bias[0] (padded) */     \
    X(atomref, 100) X(scalars, 4)              /* atomref[100]; {std, mean, 0, 0}        */

#define VB_LAYER_WEIGHTS(X)                                                                       \
    X(ln_w, D) X(ln_b, D) X(vln_w, D)                                                              \
    X(WqkvT, D * 3 * D) X(bqkv, 3 * D) X(WqkvN, 3 * D * D)   /* [q|k|v]                 */        \
    X(WvecT, D * 3 * D) X(WvecN, 3 * D * D)                  /* vec_proj [384,128]      */        \
    X(WtuT, D * 2 * D) X(WtuN, 2 * D * D)                    /* [w_trg|w_src] (zeros in the last layer) */ \
    X(W1T, D * 3 * D) X(b1, 3 * D) X(W1N, 3 * D * D)         /* [dk|dv|f] (f zeros in the last layer)   */ \
    X(WsT, D * 2 * D) X(bs, 2 * D) X(WsN, 2 * D * D)         /* s_proj [256,128]        */        \
    X(WoT, D * 3 * D) X(bo, 3 * D) X(WoN, 3 * D * D)         /* o_proj [384,128]        */        \
    /* tensor-core weight images (weights.py::tc_image): 128x128 chunks, 4 K-slabs x (hi 16 KB + lo 16 KB) */ \
    X(tcW1, 3 * 4 * 8192)      /* forward  [dk | dv | f]   : 3 chunks                    */        \
    X(tcWs, 2 * 4 * 8192)      /* forward  [s1 | s2]       : 2 chunks                    */        \
    X(tcWsN, 2 * 4 * 8192)     /* adjoint  g_m = g_s Ws    : K-chunks s1-part, s2-part   */        \
    X(tcW1N, 3 * 4 * 8192)     /* adjoint  g_f += g_P W1   : K-chunks dk, dv, f parts    */        \
    /* node stage on tensor cores (k_node_tc.cuh): forward column chunks / adjoint K chunks */                 \
    X(tcWo, 3 * 4 * 8192)      /* forward  o = xa Wo^T     : chunks o1, o2, o3           */        \
    X(tcWqkv, 3 * 4 * 8192)    /* forward  [q | k | v]                                    */        \
    X(tcWvt, 5 * 4 * 8192)     /* forward  [v1 | v2 | v3 | t | u] (t, u zeros in the last layer) */ \
    X(tcWoN, 3 * 4 * 8192)     /* adjoint  g_xa = g_o Wo   : K-chunks                     */        \
    X(tcWqkvN, 3 * 4 * 8192)   /* adjoint  g_xn = g_qkv Wqkv                              */        \
    X(tcWvtN, 5 * 4 * 8192)    /* adjoint  g_vn = g_v123 Wvec + g_tu Wtu                  */

struct LayerW {
#define X(name, count) const float* name;
    VB_LAYER_WEIGHTS(X)
#undef X
};

struct ModelW {
#define X(name, count) const float* name;
    VB_GLOBAL_WEIGHTS(X)
#undef X
    LayerW layer[L];
    float cutoff;
};

// ---- per-run workspace ---------------------------------------------------------------------------
struct Workspace {
    int N, G, Ecap;
    // static topology
    const int* z;           // [N]
    const int* frag_of;     // [N]
    const int* frag_start;  // [G+1]
    // neighbour list (rebuilt every step)
    int* deg;               // [N]
    int* slots;             // [N][32]
    int* rowptr;            // [N+1]; rowptr[N] = E
    int* esrc;              // [Ecap] source j
    int* edst;              // [Ecap] target i
    float* geom;            // [Ecap][8]  r, C(r), dx, dy, dz, 1/r, 0, 0   (d = unit vector, 0 on self-loops)
    float* rbf;             // [Ecap][32]
    float* eacc;            // [Ecap][4]  adjoint accumulators: dE/dC, dE/dd[3]
    float* grbf;            // [Ecap][32] dE/drbf
    // residual stream at the input of layer l (index L = output of the last layer)
    float* X[L + 1];        // [N][128]
    float* V[L + 1];        // [N][3][128]
    float* F[L];            // [Ecap][128]
    // per-layer node tensors kept for the reverse sweep
    float* VN[L];           // [N][3][128]  VecLayerNorm(vec)
    float* QKV[L];          // [N][384]
    float* V123[L];         // [N][3][384]  vec_proj output [v1|v2|v3]
    float* VDOT[L];         // [N][128]
    float* TU[L];           // [N][3][256]  [w_trg vn | w_src vn]   (unused for the last layer)
    float* O[L];            // [N][384]     o_proj output
    // per-layer edge pre-activations written by the forward edge stage, read by its adjoint (no recompute)
    float* P1[L];           // [Ecap][384]  f W1^T + b1 = [Pdk | Pdv | Pf]
    float* SP[L];           // [Ecap][256]  m Ws^T + bs
    float* ATT[L];          // [Ecap][8]    attention pre-activation a_h
    // transient aggregates
    float* XA;              // [N][128]
    float* VA;              // [N][3][128]
    // adjoints
    float* GX;              // [N][128]
    float* GVEC;            // [N][3][128]
    float* GF;              // [Ecap][128]
    float* GXA;             // [gxa_parts][N][128]  dE/dxa; with the tensor-core node stage three K-chunk partials (summed by the edge adjoint)
    int gxa_parts;          // 1 or 3
    float* GQKV;            // [N][384]
    float* GVNMSG;          // [N][3][128]
    float* GTU;             // [N][3][256]
    float* eatom;           // [N]
    // tensor-core node stage (k_node_tc.cuh)
    float* XN;              // [N][128]      LayerNorm(x) of the current stage
    float* PX;              // [3][N][128]   partial products of g_qkv Wqkv (one per 128-deep K chunk)
    float* PV;              // [5][3N][128]  partial products of g_v123 Wvec (3) and g_tu Wtu (2)
    float* GO;              // [N][384]      [g_o1 | g_x vdot | g_x]
};

// dE/dxa of a node: the sum of its partials in a fixed order
__device__ __forceinline__ float4 load_gxa(const Workspace& ws, size_t node, int col) {
    float4 v = ld4(ws.GXA + node * D + col);
    if (ws.gxa_parts == 3) v = (v + ld4(ws.GXA + ((size_t)ws.N + node) * D + col)) + ld4(ws.GXA + (2 * (size_t)ws.N + node) * D + col);
    return v;
}

}  // namespace vb
