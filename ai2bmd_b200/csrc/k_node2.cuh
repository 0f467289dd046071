// Per-node stages of a ViS_MP layer (forward and adjoint), SIMT version: a CTA of 8 warps (16 in the 4-node variant used
// for small systems) owns NB consecutive nodes and spreads the (weight chunk x row block) GEMM units over its warps, so
// the critical path is 1-3 units instead of the 11 chunk-GEMMs of one warp per node; the 4-node variant also splits the
// o_proj K dimension over warps and sums the partials in a fixed order.
//   reference: visnet_block.py:237-250 (LayerNorm, VecLayerNorm, q/k/v, vec_proj, vec_dot),
//              :271-273 (o_proj, dx, dvec), :129-131,136-137 (residual updates),
//              utils.py:200-228 (VecLayerNorm max_min), :290-292 (w_trg/w_src applied per node here:
//              the reference applies them per edge after the gather; same per-row arithmetic).
// Bound at small sizes by streaming ~720 KB of weights per CTA from L2 (DESIGN.md section 5).
#pragma once
#include "k_node.cuh"

namespace vb {

// warps per CTA: 16 for the 4-node variant (small systems: more units in flight per node), 8 otherwise
template <int NB> struct N2Cfg {
    static constexpr int WARPS = (NB <= 4) ? 16 : 8; static constexpr int THREADS = WARPS * 32;
    static constexpr int KS = (NB <= 4) ? 2 : 1;       // K-split projection plan (see NodeFwd2Smem)
};
template <int NB> struct N2Rows { static constexpr int RB = (NB < 8) ? NB : 8; };   // rows per GEMM unit

// KS = 2 (4-node variant): every projection unit covers ALL rows of the CTA (one pass over each weight chunk instead of
// one per row block) and half of K; the second K-half leaves a partial row in shared memory.
template <int NB>
struct NodeFwd2Smem {
    static constexpr int KS = N2Cfg<NB>::KS;
    static constexpr int LDA = D + LDS_PAD;       // 132
    static constexpr int LDO = 3 * D + LDS_PAD;   // 388
    float xs[NB][LDA];                            // xa rows, later LayerNorm(x) rows
    float vs[3 * NB][LDA];                        // VecLayerNorm(vec) rows
    float os[NB][LDO];                            // o_proj output rows
    float osp[(NB <= 4) ? 3 : 1][NB][LDO];        // 4-node variant: K-quarter partials 1..3 of the o_proj rows
    float px[(KS == 2) ? NB : 1][3 * D];          // KS = 2: second-K-half partials of the q|k|v rows,
    float pv[(KS == 2) ? 3 * NB : 1][3 * D];      //         of the vec_proj rows
    float pt[(KS == 2) ? 3 * NB : 1][2 * D];      //         and of the w_trg|w_src rows
};

// ---------------------------------------------------------------------------------------------
// Forward node stage k (k = 0..L), CTA b owns nodes [b*NB, b*NB + NB):
//   if k >= 1: finish layer k-1:  o = xa Wo^T + bo ; x += vdot*o2 + o3 ; vec += v3*o1 + va
//   if k <  L: start layer k:     xn = LN(x) ; vn = VecLN(vec) ; q,k,v ; [v1|v2|v3] = vn Wvec^T ; vdot ;
//                                 [t|u] = vn [Wtrg|Wsrc]^T (k < L-1)
//   zeroes XA / VA for the edge stage that follows.
// ---------------------------------------------------------------------------------------------
template <int NB>
__global__ void __launch_bounds__(N2Cfg<NB>::THREADS) node_fwd2_kernel(NodeArgs a) {
    pdl_entry();
    extern __shared__ __align__(16) float dyn_smem[];
    const ModelW& mw = a.mw;
    const Workspace& ws = a.ws;
    const int k = a.layer, n0 = (int)blockIdx.x * NB;
    unsigned long long* const tl = a.tl;
    const int krot = a.krot ? (int)blockIdx.x * 16 : 0;
#define N2_TL(i) do { if (tl != nullptr && n0 == 0 && (threadIdx.x & 31) == 0) tl[(i) * 16 + (threadIdx.x >> 5)] = (unsigned long long)clock64(); } while (0)
    N2_TL(0);
    constexpr int N2_WARPS = N2Cfg<NB>::WARPS, N2_THREADS = N2Cfg<NB>::THREADS, KS = N2Cfg<NB>::KS;
    using S = NodeFwd2Smem<NB>;
    constexpr int LDA = S::LDA;
    constexpr int N2_RB = N2Rows<NB>::RB;
    S& sm = *reinterpret_cast<S*>(dyn_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, col = lane * 4;
    const int nn = min(NB, ws.N - n0);            // valid nodes in this CTA

    if (k >= 1) {
        const LayerW& lw = mw.layer[k - 1];
        for (int idx = threadIdx.x; idx < NB * 32; idx += N2_THREADS) {
            const int nd = idx >> 5, c4 = (idx & 31) * 4;
            st4(&sm.xs[nd][c4], nd < nn ? ld4(ws.XA + (size_t)(n0 + nd) * D + c4) : f4s(0.f));
        }
        [[maybe_unused]] WarpGemmPre<D / 4, 4> go;               // KS = 2: weight rows of this warp's o_proj unit, issued before the barrier
        if constexpr (KS == 2) {
            if (warp < 12) go.prefetch(lw.WoT + (size_t)(warp / 3) * (D / 4) * 3 * D + (warp % 3) * D, 3 * D, lane, krot);
        }
        __syncthreads();
        N2_TL(1);
        // o = xa Wo^T + bo : units = 3 chunks x NB/8 row blocks (x 4 K-quarters in the 16-warp variant)
        if constexpr (KS == 2) {
            if (warp < 12) {
                const int ch = warp % 3, kq = warp / 3;
                float acc[N2_RB][4];
                if (kq == 0) acc_set_bias<N2_RB>(acc, lw.bo + ch * D, lane);
                else acc_zero<N2_RB>(acc);
                go.template run<N2_RB, LDA>(acc, &sm.xs[0][kq * (D / 4)]);
#pragma unroll
                for (int r = 0; r < N2_RB; r++) {
                    if (kq == 0) st4(&sm.os[r][ch * D + col], arr4(acc[r]));
                    else st4(&sm.osp[kq - 1][r][ch * D + col], arr4(acc[r]));
                }
            }
            N2_TL(2);
            __syncthreads();
            N2_TL(3);
            for (int idx = threadIdx.x; idx < NB * 96; idx += N2_THREADS) {      // fixed-order sum of the K-quarters
                const int r = idx / 96, c4 = (idx % 96) * 4;
                st4(&sm.os[r][c4], (ld4(&sm.os[r][c4]) + ld4(&sm.osp[0][r][c4])) + (ld4(&sm.osp[1][r][c4]) + ld4(&sm.osp[2][r][c4])));
            }
        } else if constexpr (NB <= 4) {
            for (int u = warp; u < 12; u += N2_WARPS) {
                const int ch = u % 3, kq = u / 3;
                float acc[N2_RB][4];
                if (kq == 0) acc_set_bias<N2_RB>(acc, lw.bo + ch * D, lane);
                else acc_zero<N2_RB>(acc);
                warp_gemm<N2_RB, D / 4, LDA, 4>(acc, &sm.xs[0][kq * (D / 4)], lw.WoT + (size_t)kq * (D / 4) * 3 * D + ch * D, 3 * D, lane, krot);
#pragma unroll
                for (int r = 0; r < N2_RB; r++) {
                    if (kq == 0) st4(&sm.os[r][ch * D + col], arr4(acc[r]));
                    else st4(&sm.osp[kq - 1][r][ch * D + col], arr4(acc[r]));
                }
            }
            N2_TL(2);
            __syncthreads();
            N2_TL(3);
            for (int idx = threadIdx.x; idx < NB * 96; idx += N2_THREADS) {      // fixed-order sum of the K-quarters
                const int r = idx / 96, c4 = (idx % 96) * 4;
                st4(&sm.os[r][c4], (ld4(&sm.os[r][c4]) + ld4(&sm.osp[0][r][c4])) + (ld4(&sm.osp[1][r][c4]) + ld4(&sm.osp[2][r][c4])));
            }
        } else {
            for (int u = warp; u < 3 * (NB / N2_RB); u += N2_WARPS) {
                const int ch = u % 3, rb = u / 3;
                float acc[N2_RB][4];
                acc_set_bias<N2_RB>(acc, lw.bo + ch * D, lane);
                warp_gemm<N2_RB, D, LDA, (NB <= 8 ? 4 : 2)>(acc, &sm.xs[rb * N2_RB][0], lw.WoT + ch * D, 3 * D, lane);
#pragma unroll
                for (int r = 0; r < N2_RB; r++) st4(&sm.os[rb * N2_RB + r][ch * D + col], arr4(acc[r]));
            }
        }
        __syncthreads();
        N2_TL(4);
    }
    // per-node phase: residual update, LayerNorm, VecLayerNorm (warp per node)
    for (int nd = warp; nd < NB; nd += N2_WARPS) {
        const int node = n0 + nd;
        const bool ok = nd < nn;
        float4 x = f4s(0.f), vec[3] = {f4s(0.f), f4s(0.f), f4s(0.f)};
        if (k >= 1) {
            if (ok) {
                const float4 o1 = ld4(&sm.os[nd][col]), o2 = ld4(&sm.os[nd][D + col]), o3 = ld4(&sm.os[nd][2 * D + col]);
                float* orow = ws.O[k - 1] + (size_t)node * 3 * D;
                st4(orow + col, o1); st4(orow + D + col, o2); st4(orow + 2 * D + col, o3);
                x = ld4(ws.X[k - 1] + (size_t)node * D + col) + ld4(ws.VDOT[k - 1] + (size_t)node * D + col) * o2 + o3;
                st4(ws.X[k] + (size_t)node * D + col, x);
#pragma unroll
                for (int s = 0; s < 3; s++) {
                    const size_t r3 = (size_t)node * 3 + s;
                    vec[s] = ld4(ws.V[k - 1] + r3 * D + col) + ld4(ws.V123[k - 1] + r3 * 3 * D + 2 * D + col) * o1 +
                             ld4(ws.VA + r3 * D + col);
                    st4(ws.V[k] + r3 * D + col, vec[s]);
                }
            }
        } else if (ok) {
            x = ld4(ws.X[0] + (size_t)node * D + col);
        }
        if (ok) {
            st4(ws.XA + (size_t)node * D + col, f4s(0.f));
#pragma unroll
            for (int s = 0; s < 3; s++) st4(ws.VA + ((size_t)node * 3 + s) * D + col, f4s(0.f));
        }
        if (k < L) {
            const LayerW& lw = mw.layer[k];
            st4(&sm.xs[nd][col], ln_forward(x, lw.ln_w, lw.ln_b, lane));
            float4 vn[3];
            vecln_forward(vec, vn, lw.vln_w, lane);
#pragma unroll
            for (int s = 0; s < 3; s++) {
                st4(&sm.vs[nd * 3 + s][col], vn[s]);
                if (ok) st4(ws.VN[k] + ((size_t)node * 3 + s) * D + col, vn[s]);
            }
        }
    }
    N2_TL(5);
    if (k >= L) return;
    const LayerW& lw = mw.layer[k];
    // KS = 2 plan (16 units, one per warp): (q|k|v chunk, K half) x3x2 on the NB scalar rows, (vec_proj chunk, K half) x3x2
    // and (w_trg|w_src chunk, K half) x2x2 on all 3*NB vector rows.  Every weight element is read once per CTA (the
    // row-block plan below reads the vector weights once per 4 rows); half 1 parks its partial rows in shared memory,
    // half 0 adds them (fixed order) and writes the result.  The first weight rows are requested before the barrier.
    constexpr int RV = 3 * NB, KH = D / 2;
    [[maybe_unused]] WarpGemmPre<KH, 2> gm;
    [[maybe_unused]] const int nunits2 = (k < L - 1) ? 16 : 12;
    [[maybe_unused]] const int kind = warp < 6 ? 0 : (warp < 12 ? 1 : 2);
    [[maybe_unused]] const int uv = kind == 0 ? warp : (kind == 1 ? warp - 6 : warp - 12);
    [[maybe_unused]] const int ch2 = kind == 2 ? (uv & 1) : uv % 3, half = kind == 2 ? (uv >> 1) : uv / 3;
    [[maybe_unused]] const bool active = warp < nunits2;
    if constexpr (KS == 2) {
        if (active) {
            const float* W = kind == 0 ? lw.WqkvT : (kind == 1 ? lw.WvecT : lw.WtuT);
            const int ldw = kind == 2 ? 2 * D : 3 * D;
            gm.prefetch(W + (size_t)half * KH * ldw + ch2 * D, ldw, lane, krot);
        }
    }
    __syncthreads();
    N2_TL(6);
    if constexpr (KS == 2) {
        const int ch = ch2;
        float acc[RV][4];
        float (&accx)[NB][4] = *reinterpret_cast<float (*)[NB][4]>(&acc[0][0]);
        if (active) {
            if (kind == 0) {
                if (half == 0) acc_set_bias<NB>(accx, lw.bqkv + ch * D, lane);
                else acc_zero<NB>(accx);
                gm.template run<NB, LDA>(accx, &sm.xs[0][half * KH]);
                if (half == 1) {
#pragma unroll
                    for (int r = 0; r < NB; r++) st4(&sm.px[r][ch * D + col], arr4(accx[r]));
                }
            } else {
                acc_zero<RV>(acc);
                gm.template run<RV, LDA>(acc, &sm.vs[0][half * KH]);
                if (half == 1) {
#pragma unroll
                    for (int r = 0; r < RV; r++) {
                        if (kind == 1) st4(&sm.pv[r][ch * D + col], arr4(acc[r]));
                        else           st4(&sm.pt[r][ch * D + col], arr4(acc[r]));
                    }
                }
            }
        }
        N2_TL(7);
        __syncthreads();
        N2_TL(8);
        if (active && half == 0) {
            if (kind == 0) {
#pragma unroll
                for (int r = 0; r < NB; r++)
                    if (r < nn) st4(ws.QKV[k] + (size_t)(n0 + r) * 3 * D + ch * D + col, arr4(accx[r]) + ld4(&sm.px[r][ch * D + col]));
            } else if (kind == 1) {
#pragma unroll
                for (int r = 0; r < RV; r++)
                    if (r / 3 < nn) st4(ws.V123[k] + ((size_t)n0 * 3 + r) * 3 * D + ch * D + col, arr4(acc[r]) + ld4(&sm.pv[r][ch * D + col]));
            } else {
#pragma unroll
                for (int r = 0; r < RV; r++)
                    if (r / 3 < nn) st4(ws.TU[k] + ((size_t)n0 * 3 + r) * 2 * D + ch * D + col, arr4(acc[r]) + ld4(&sm.pt[r][ch * D + col]));
            }
        }
    } else {
        // GEMM units: [0, UQ): qkv ; [UQ, UQ+UV): vec_proj ; then w_trg|w_src
        constexpr int UQ = 3 * (NB / N2_RB), UV = 3 * (3 * NB / N2_RB), UT = 2 * (3 * NB / N2_RB);
        const int nunits = UQ + UV + ((k < L - 1) ? UT : 0);
        for (int u = warp; u < nunits; u += N2_WARPS) {
            float acc[N2_RB][4];
            if (u < UQ) {
                const int ch = u % 3, rb = u / 3;
                acc_set_bias<N2_RB>(acc, lw.bqkv + ch * D, lane);
                warp_gemm<N2_RB, D, LDA, (NB <= 8 ? 4 : 2)>(acc, &sm.xs[rb * N2_RB][0], lw.WqkvT + ch * D, 3 * D, lane);
    #pragma unroll
                for (int r = 0; r < N2_RB; r++) {
                    const int nd = rb * N2_RB + r;
                    if (nd < nn) st4(ws.QKV[k] + (size_t)(n0 + nd) * 3 * D + ch * D + col, arr4(acc[r]));
                }
            } else if (u < UQ + UV) {
                const int v = u - UQ, ch = v % 3, rb = v / 3;
                acc_zero<N2_RB>(acc);
                warp_gemm<N2_RB, D, LDA, (NB <= 8 ? 4 : 2)>(acc, &sm.vs[rb * N2_RB][0], lw.WvecT + ch * D, 3 * D, lane);
    #pragma unroll
                for (int r = 0; r < N2_RB; r++) {
                    const int row = rb * N2_RB + r;                  // = nd*3 + s
                    if (row / 3 < nn) st4(ws.V123[k] + ((size_t)n0 * 3 + row) * 3 * D + ch * D + col, arr4(acc[r]));
                }
            } else {
                const int v = u - UQ - UV, ch = v % 2, rb = v / 2;
                acc_zero<N2_RB>(acc);
                warp_gemm<N2_RB, D, LDA, (NB <= 8 ? 4 : 2)>(acc, &sm.vs[rb * N2_RB][0], lw.WtuT + ch * D, 2 * D, lane);
    #pragma unroll
                for (int r = 0; r < N2_RB; r++) {
                    const int row = rb * N2_RB + r;
                    if (row / 3 < nn) st4(ws.TU[k] + ((size_t)n0 * 3 + row) * 2 * D + ch * D + col, arr4(acc[r]));
                }
            }
        }
    }
    N2_TL(9);
    __syncthreads();     // V123 rows of this CTA are visible block-wide
    N2_TL(10);
    for (int nd = warp; nd < nn; nd += N2_WARPS) {
        const size_t r3 = (size_t)(n0 + nd) * 3;
        float4 vd = f4s(0.f);
#pragma unroll
        for (int s = 0; s < 3; s++) vd = vd + ld4(ws.V123[k] + (r3 + s) * 3 * D + col) * ld4(ws.V123[k] + (r3 + s) * 3 * D + D + col);
        st4(ws.VDOT[k] + (size_t)(n0 + nd) * D + col, vd);
    }
    N2_TL(11);
}

// KS = 2 (4-node variant): units of (all rows of the CTA) x (half a 128-deep K chunk): each weight element is read once
// per CTA, 16 (12 in the last layer) units = one per warp; the o_proj adjoint is cut into 12 units of K = 32.
template <int NB>
struct NodeBwd2Smem {
    static constexpr int KS = N2Cfg<NB>::KS;
    static constexpr int LD3 = 3 * D + LDS_PAD;   // 388
    static constexpr int LD2 = 2 * D + LDS_PAD;   // 260
    static constexpr int NVB = 3 * NB / N2Rows<NB>::RB;    // vector row blocks
    static constexpr int NXB = NB / N2Rows<NB>::RB;        // scalar row blocks
    float gq[NB][LD3];                            // g_qkv rows -> later g_o rows
    float gvp[3 * NB][LD3];                       // [g_vdot*v2 | g_vdot*v1 | gvec*o1] rows
    float gtu[3 * NB][LD2];                       // [g_t | g_u] rows
    float part_x[3 * KS][NB][D];                  // partial products of the scalar rows (3 K-chunks x KS)
    float part_v[5 * KS][3 * NB][D];              // partial products of the vector rows ((3 + 2) K-chunks x KS); KS = 2: later
                                                  // also the 12 K = 32 partials of the o_proj adjoint ([12][NB][D])
};

// ---------------------------------------------------------------------------------------------
// Backward node stage k (k = L..0), CTA b owns nodes [b*NB, b*NB + NB):
//   if k <= L-1: adjoint of the first half of layer k (needs the edge adjoint of layer k):
//        g_xn = [gq|gk|gv] Wqkv ; g_vn = g_vn_msg + [g_vdot*v2 | g_vdot*v1 | gvec*o1] Wvec + [gt|gu] Wtu
//        gvec += VecLN'(vec_in, g_vn) ; gx += LN'(x_in, g_xn)
//   if k >= 1:   adjoint of the second half of layer k-1:
//        g_xa = [sum_s gvec*v3 | gx*vdot | gx] Wo          (feeds the edge adjoint of layer k-1)
//   GQKV / GVNMSG / GTU are the accumulators the edge adjoint of layer k added into; they are consumed and re-zeroed
//   here (atomic targets of the next edge adjoint).
// K-split units: every (row block, 128-wide K chunk) is one unit writing a partial [8][128] product into its own shared
// slot; slots are summed in a fixed order afterwards (deterministic).
// ---------------------------------------------------------------------------------------------
template <int NB>
__global__ void __launch_bounds__(N2Cfg<NB>::THREADS) node_bwd2_kernel(NodeArgs a) {
    pdl_entry();
    extern __shared__ __align__(16) float dyn_smem[];
    const ModelW& mw = a.mw;
    const Workspace& ws = a.ws;
    const int k = a.layer, n0 = (int)blockIdx.x * NB;
    unsigned long long* const tl = a.tl;
    const int krot = a.krot ? (int)blockIdx.x * 16 : 0;
    // the accumulators alias nothing else this kernel accesses: __restrict__ lets their loads move ahead of other stores
    float* __restrict__ const GQKV = ws.GQKV;
    float* __restrict__ const GVNMSG = ws.GVNMSG;
    float* __restrict__ const GTU = ws.GTU;
    constexpr int N2_WARPS = N2Cfg<NB>::WARPS, KS = N2Cfg<NB>::KS;
    N2_TL(0);
    using S = NodeBwd2Smem<NB>;
    constexpr int LD3 = S::LD3, LD2 = S::LD2;
    constexpr int N2_RB = N2Rows<NB>::RB;
    S& sm = *reinterpret_cast<S*>(dyn_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, col = lane * 4;
    const int nn = min(NB, ws.N - n0);
    const bool has_a = (k <= L - 1), has_b = (k >= 1);
    const bool has_tu = (k < L - 1);
    const float4 z4 = f4s(0.f);

    if (has_a) {
        const LayerW& lw = mw.layer[k];
        // stage the A-operand rows (warp per node)
        for (int nd = warp; nd < NB; nd += N2_WARPS) {
            const int node = n0 + nd;
            const bool ok = nd < nn;
            const float4 gx = ok ? ld4(ws.GX + (size_t)node * D + col) : z4;
            const float* orow = ws.O[k] + (size_t)node * 3 * D;
            const float4 o1 = ok ? ld4(orow + col) : z4, o2 = ok ? ld4(orow + D + col) : z4;
            const float4 g_vdot = gx * o2;
            const float* gq = GQKV + (size_t)node * 3 * D;
            st4(&sm.gq[nd][col], ok ? ld4(gq + col) : z4);
            st4(&sm.gq[nd][D + col], ok ? ld4(gq + D + col) : z4);
            st4(&sm.gq[nd][2 * D + col], ok ? ld4(gq + 2 * D + col) : z4);
#pragma unroll
            for (int s = 0; s < 3; s++) {
                const size_t r3 = (size_t)node * 3 + s;
                const float* vrow = ws.V123[k] + r3 * 3 * D;
                const float4 gv = ok ? ld4(ws.GVEC + r3 * D + col) : z4;
                st4(&sm.gvp[nd * 3 + s][col], g_vdot * (ok ? ld4(vrow + D + col) : z4));
                st4(&sm.gvp[nd * 3 + s][D + col], g_vdot * (ok ? ld4(vrow + col) : z4));
                st4(&sm.gvp[nd * 3 + s][2 * D + col], gv * o1);
                if (has_tu) {
                    const float* gt = GTU + r3 * 2 * D;
                    st4(&sm.gtu[nd * 3 + s][col], ok ? ld4(gt + col) : z4);
                    st4(&sm.gtu[nd * 3 + s][D + col], ok ? ld4(gt + D + col) : z4);
                }
            }
        }
        // KS = 2: one unit per warp, (K chunk, K half) on all scalar rows (6 units) / on all vector rows (10, or 6 without
        // w_trg|w_src); the first weight rows are requested before the barrier (13 of the 16 warps have nothing to stage)
        constexpr int RV = 3 * NB, KH = D / 2;
        [[maybe_unused]] WarpGemmPre<KH, 2> gm;
        [[maybe_unused]] const int kv2 = has_tu ? 5 : 3;
        if constexpr (KS == 2) {
            const int u = warp;
            if (u < 6) gm.prefetch(lw.WqkvN + ((size_t)(u >> 1) * D + (u & 1) * KH) * D, D, lane, krot);
            else if (u < 6 + 2 * kv2) {
                const int v = u - 6, kc = v >> 1, hf = v & 1;
                gm.prefetch((kc < 3 ? lw.WvecN + (size_t)kc * D * D : lw.WtuN + (size_t)(kc - 3) * D * D) + (size_t)hf * KH * D, D, lane, krot);
            }
        }
        N2_TL(1);
        __syncthreads();
        N2_TL(2);
        if constexpr (KS == 2) {
            const int u = warp;
            if (u < 6) {
                const int kc = u >> 1, half = u & 1;
                float acc[NB][4];
                acc_zero<NB>(acc);
                gm.template run<NB, LD3>(acc, &sm.gq[0][kc * D + half * KH]);
#pragma unroll
                for (int r = 0; r < NB; r++) st4(&sm.part_x[u][r][col], arr4(acc[r]));
            } else if (u < 6 + 2 * kv2) {
                const int v = u - 6, kc = v >> 1, half = v & 1;
                float acc[RV][4];
                acc_zero<RV>(acc);
                if (kc < 3) gm.template run<RV, LD3>(acc, &sm.gvp[0][kc * D + half * KH]);
                else        gm.template run<RV, LD2>(acc, &sm.gtu[0][(kc - 3) * D + half * KH]);
#pragma unroll
                for (int r = 0; r < RV; r++) st4(&sm.part_v[v][r][col], arr4(acc[r]));
            }
        } else {
            // units: scalar rows x 3 K-chunks (Wqkv) ; vector rows x (3 K-chunks Wvec + 2 K-chunks Wtu)
            constexpr int UX = 3 * S::NXB;
            const int kv = has_tu ? 5 : 3;
            const int nunits = UX + kv * S::NVB;
            for (int u = warp; u < nunits; u += N2_WARPS) {
                float acc[N2_RB][4];
                acc_zero<N2_RB>(acc);
                if (u < UX) {
                    const int kc = u % 3, rb = u / 3;
                    warp_gemm<N2_RB, D, LD3, 4>(acc, &sm.gq[rb * N2_RB][kc * D], lw.WqkvN + (size_t)kc * D * D, D, lane);
    #pragma unroll
                    for (int r = 0; r < N2_RB; r++) st4(&sm.part_x[kc][rb * N2_RB + r][col], arr4(acc[r]));
                } else {
                    const int v = u - UX, kc = v % kv, rb = v / kv;
                    if (kc < 3) warp_gemm<N2_RB, D, LD3, 4>(acc, &sm.gvp[rb * N2_RB][kc * D], lw.WvecN + (size_t)kc * D * D, D, lane);
                    else        warp_gemm<N2_RB, D, LD2, 4>(acc, &sm.gtu[rb * N2_RB][(kc - 3) * D], lw.WtuN + (size_t)(kc - 3) * D * D, D, lane);
    #pragma unroll
                    for (int r = 0; r < N2_RB; r++) st4(&sm.part_v[kc][rb * N2_RB + r][col], arr4(acc[r]));
                }
            }
        }
        N2_TL(3);
        __syncthreads();
        N2_TL(4);
    }
    // per-node phase
    for (int nd = warp; nd < NB; nd += N2_WARPS) {
        const int node = n0 + nd;
        const bool ok = nd < nn;
        float4 gx = ok ? ld4(ws.GX + (size_t)node * D + col) : z4, gvec[3];
#pragma unroll
        for (int s = 0; s < 3; s++) gvec[s] = ok ? ld4(ws.GVEC + ((size_t)node * 3 + s) * D + col) : z4;
        float4 v3p[3] = {z4, z4, z4}, vdp = z4;             // layer k-1 rows of the g_o products: requested now, used last
        if (has_b && ok) {
#pragma unroll
            for (int s = 0; s < 3; s++) v3p[s] = ld4(ws.V123[k - 1] + ((size_t)node * 3 + s) * 3 * D + 2 * D + col);
            vdp = ld4(ws.VDOT[k - 1] + (size_t)node * D + col);
        }
        if (has_a && ok) {
            const LayerW& lw = mw.layer[k];
            const auto px = [&](int kc) {              // K chunk kc of the scalar rows (KS = 2: its two halves, fixed order)
                if constexpr (KS == 2) return ld4(&sm.part_x[2 * kc][nd][col]) + ld4(&sm.part_x[2 * kc + 1][nd][col]);
                else return ld4(&sm.part_x[kc][nd][col]);
            };
            const float4 gxn = (px(0) + px(1)) + px(2);
            float4 vin[3], gout[3], gv[3];
#pragma unroll
            for (int s = 0; s < 3; s++) {
                const int row = nd * 3 + s;
                const auto pv = [&](int kc) {
                    if constexpr (KS == 2) return ld4(&sm.part_v[2 * kc][row][col]) + ld4(&sm.part_v[2 * kc + 1][row][col]);
                    else return ld4(&sm.part_v[kc][row][col]);
                };
                float4 g = ld4(GVNMSG + ((size_t)node * 3 + s) * D + col);
                g = g + ((pv(0) + pv(1)) + pv(2));
                if (has_tu) g = g + (pv(3) + pv(4));
                gout[s] = g;
                vin[s] = ld4(ws.V[k] + ((size_t)node * 3 + s) * D + col);
            }
            vecln_backward(vin, gout, gv, lw.vln_w, lane);
#pragma unroll
            for (int s = 0; s < 3; s++) gvec[s] = gvec[s] + gv[s];
            gx = gx + ln_backward(ld4(ws.X[k] + (size_t)node * D + col), gxn, lw.ln_w, lane);
        }
        if (ok) {
            float* gq = GQKV + (size_t)node * 3 * D;
            st4(gq + col, z4); st4(gq + D + col, z4); st4(gq + 2 * D + col, z4);
#pragma unroll
            for (int s = 0; s < 3; s++) {
                const size_t r3 = (size_t)node * 3 + s;
                st4(GVNMSG + r3 * D + col, z4);
                st4(GTU + r3 * 2 * D + col, z4);
                st4(GTU + r3 * 2 * D + D + col, z4);
                st4(ws.GVEC + r3 * D + col, gvec[s]);
            }
            st4(ws.GX + (size_t)node * D + col, gx);
        }
        if (has_b) {
            float4 go1 = z4;
#pragma unroll
            for (int s = 0; s < 3; s++) go1 = go1 + gvec[s] * v3p[s];
            __syncwarp();
            st4(&sm.gq[nd][col], go1);
            st4(&sm.gq[nd][D + col], gx * vdp);
            st4(&sm.gq[nd][2 * D + col], gx);
        }
    }
    N2_TL(5);
    if (!has_b) return;
    const LayerW& lwo = mw.layer[k - 1];
    [[maybe_unused]] WarpGemmPre<D / 4, 4> go;
    if constexpr (KS == 2) {
        if (warp < 12) go.prefetch(lwo.WoN + ((size_t)(warp >> 2) * D + (warp & 3) * (D / 4)) * D, D, lane, krot);
    }
    __syncthreads();
    N2_TL(6);
    if constexpr (KS == 2) {
        // g_xa = g_o Wo: 12 units of K = 32 (3 chunks x 4 quarters), one per warp; partial rows in the (now free) part_v area
        float (*po)[NB][D] = reinterpret_cast<float (*)[NB][D]>(&sm.part_v[0][0][0]);
        if (warp < 12) {
            const int kc = warp >> 2, q = warp & 3;
            float acc[NB][4];
            acc_zero<NB>(acc);
            go.template run<NB, LD3>(acc, &sm.gq[0][kc * D + q * (D / 4)]);
#pragma unroll
            for (int r = 0; r < NB; r++) st4(&po[warp][r][col], arr4(acc[r]));
        }
        N2_TL(7);
        __syncthreads();
        N2_TL(8);
        for (int nd = warp; nd < nn; nd += N2_WARPS) {
            float4 t[3];
#pragma unroll
            for (int kc = 0; kc < 3; kc++)
                t[kc] = (ld4(&po[4 * kc][nd][col]) + ld4(&po[4 * kc + 1][nd][col])) + (ld4(&po[4 * kc + 2][nd][col]) + ld4(&po[4 * kc + 3][nd][col]));
            st4(ws.GXA + (size_t)(n0 + nd) * D + col, (t[0] + t[1]) + t[2]);
        }
        N2_TL(9);
    } else {
        for (int u = warp; u < 3 * S::NXB; u += N2_WARPS) {
            const int kc = u % 3, rb = u / 3;
            float acc[N2_RB][4];
            acc_zero<N2_RB>(acc);
            warp_gemm<N2_RB, D, LD3, 4>(acc, &sm.gq[rb * N2_RB][kc * D], lwo.WoN + (size_t)kc * D * D, D, lane);
#pragma unroll
            for (int r = 0; r < N2_RB; r++) st4(&sm.part_x[kc][rb * N2_RB + r][col], arr4(acc[r]));
        }
        __syncthreads();
        for (int nd = warp; nd < nn; nd += N2_WARPS)
            st4(ws.GXA + (size_t)(n0 + nd) * D + col,
                (ld4(&sm.part_x[0][nd][col]) + ld4(&sm.part_x[1][nd][col])) + ld4(&sm.part_x[2][nd][col]));
    }
}
#undef N2_TL

}  // namespace vb
