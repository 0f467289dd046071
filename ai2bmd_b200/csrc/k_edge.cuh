// Per-edge stage of a ViS_MP layer: edge MLPs, attention, gather of source/target node rows, message,
// segmented scatter-add onto the targets, edge-feature update -- forward and hand-derived adjoint.
//   reference: visnet_block.py:244-245 (dk, dv), :276-288 (message), :297-307 (aggregate),
//              :206-209,290-295 (vector rejection, edge_update), :131 (f += df)
// A CTA processes a tile of TE consecutive edges (edges are target-major, so a target's edges are
// contiguous); warp w owns rows w*R..w*R+R-1 of the tile through all GEMM phases (rows are warp-private,
// only the final aggregation phase is CTA-wide).  Lane owns channels lane*4..+3 -> every gather/scatter
// of a node row is one coalesced 512 B request per warp.
#pragma once
#include "model.h"

namespace vb {

struct EdgeArgs {
    int layer;
    ModelW mw;
    Workspace ws;
};

constexpr int LE1 = D + LDS_PAD;       // 132
constexpr int LE2 = 2 * D + LDS_PAD;   // 260
constexpr int LE3 = 3 * D + LDS_PAD;   // 388

template <int TE>
struct EdgeMeta {
    int src[TE];
    int dst[TE];
    float C[TE];
    float4 d[TE];   // unit vector (x,y,z,0)
};

template <int TE, int NT>
__device__ __forceinline__ void load_edge_meta(EdgeMeta<TE>& m, const Workspace& ws, int e0, int nvalid) {
    for (int idx = threadIdx.x; idx < TE; idx += NT) {
        if (idx < nvalid) {
            const int e = e0 + idx;
            m.src[idx] = ws.esrc[e];
            m.dst[idx] = ws.edst[e];
            const float4 g0 = ld4(ws.geom + (size_t)e * 8);
            const float4 g1 = ld4(ws.geom + (size_t)e * 8 + 4);
            m.C[idx] = g0.y;
            m.d[idx] = f4(g0.z, g0.w, g1.x, 0.f);
        } else {   // padding rows: harmless indices, zero weight
            m.src[idx] = 0;
            m.dst[idx] = 0;
            m.C[idx] = 0.f;
            m.d[idx] = f4s(0.f);
        }
    }
}

template <int TE, int NT>
__device__ __forceinline__ void load_f_tile(float* Fs, const float* __restrict__ Fin, int e0, int nvalid) {
    for (int idx = threadIdx.x; idx < TE * 32; idx += NT) {
        const int row = idx >> 5, c4 = (idx & 31) * 4;
        st4(Fs + row * LE1 + c4, row < nvalid ? ldg4(Fin + (size_t)(e0 + row) * D + c4) : f4s(0.f));
    }
}

template <int TE>
constexpr size_t edge_fwd_smem_bytes() {
    return (size_t)TE * (LE1 + LE2) * sizeof(float) + sizeof(EdgeMeta<TE>);
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
template <int TE, int NW>
__global__ void __launch_bounds__(NW * 32) edge_fwd_kernel(EdgeArgs a) {
    pdl_entry();
    constexpr int R = TE / NW, NT = NW * 32;
    static_assert(TE % NW == 0 && NT % D == 0, "tile shape");
    extern __shared__ __align__(16) float dyn_smem[];
    float* Fs = dyn_smem;                       // [TE][132]  f tile, later the message m
    float* Ss = Fs + TE * LE1;                  // [TE][260]  silu(s_proj(m))
    EdgeMeta<TE>& meta = *reinterpret_cast<EdgeMeta<TE>*>(Ss + TE * LE2);
    const Workspace& ws = a.ws;
    const int l = a.layer;
    const LayerW& lw = a.mw.layer[l];
    const bool upd = (l < L - 1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, col = lane * 4;
    const int E = ws.rowptr[ws.N];
    const float* __restrict__ Fin = ws.F[l];
    float* __restrict__ Fout = upd ? ws.F[l + 1] : nullptr;
    const float* __restrict__ QKV = ws.QKV[l];
    const float* __restrict__ VN = ws.VN[l];
    const float* __restrict__ TU = ws.TU[l];
    float* __restrict__ P1 = ws.P1[l];
    float* __restrict__ SP = ws.SP[l];
    float* __restrict__ ATT = ws.ATT[l];
    const int r0 = warp * R;

    for (int e0 = blockIdx.x * TE; e0 < E; e0 += gridDim.x * TE) {
        const int nvalid = min(TE, E - e0);
        load_f_tile<TE, NT>(Fs, Fin, e0, nvalid);
        load_edge_meta<TE, NT>(meta, ws, e0, nvalid);
        __syncthreads();
        float acc[R][4];
        // ---- edge update: f_next = f + silu(f Wf^T + bf) * <rej(t_i, d), rej(u_j, -d)> ----
        if (upd) {
            acc_set_bias<R>(acc, lw.b1 + 2 * D, lane);
            warp_gemm<R, D, LE1>(acc, Fs + r0 * LE1, lw.W1T + 2 * D, 3 * D, lane);
#pragma unroll
            for (int r = 0; r < R; r++) {
                const int row = r0 + r;
                const int i = meta.dst[row], j = meta.src[row];
                const float4 dd = meta.d[row];
                const float4 fp = silu4(arr4(acc[r]));
                float4 ti[3], uj[3];
#pragma unroll
                for (int s = 0; s < 3; s++) {
                    ti[s] = ldg4(TU + ((size_t)i * 3 + s) * 2 * D + col);
                    uj[s] = ldg4(TU + ((size_t)j * 3 + s) * 2 * D + D + col);
                }
                const float4 a1 = ti[0] * dd.x + ti[1] * dd.y + ti[2] * dd.z;
                const float4 a2 = uj[0] * dd.x + uj[1] * dd.y + uj[2] * dd.z;
                const float4 wdot = (ti[0] - a1 * dd.x) * (uj[0] - a2 * dd.x) + (ti[1] - a1 * dd.y) * (uj[1] - a2 * dd.y) +
                                    (ti[2] - a1 * dd.z) * (uj[2] - a2 * dd.z);
                if (row < nvalid) {
                    st4(Fout + (size_t)(e0 + row) * D + col, ld4(Fs + row * LE1 + col) + fp * wdot);
                    st4(P1 + (size_t)(e0 + row) * 3 * D + 2 * D + col, arr4(acc[r]));
                }
            }
        }
        // ---- attention weight A_h = silu(sum_{c in h} q_i k_j dk) * C(r) ----
        float Areg[R];
        acc_set_bias<R>(acc, lw.b1, lane);
        warp_gemm<R, D, LE1>(acc, Fs + r0 * LE1, lw.W1T, 3 * D, lane);
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int row = r0 + r;
            const float4 qi = ldg4(QKV + (size_t)meta.dst[row] * 3 * D + col);
            const float4 kj = ldg4(QKV + (size_t)meta.src[row] * 3 * D + D + col);
            const float av = quad_sum(hsum4(qi * kj * silu4(arr4(acc[r]))));
            Areg[r] = silu_(av) * meta.C[row];
            if (row < nvalid) {
                st4(P1 + (size_t)(e0 + row) * 3 * D + col, arr4(acc[r]));
                if ((lane & 3) == 0) ATT[(size_t)(e0 + row) * H + (lane >> 2)] = av;
            }
        }
        // ---- message m = v_j * dv * A  (overwrites this warp's rows of the f tile) ----
        acc_set_bias<R>(acc, lw.b1 + D, lane);
        warp_gemm<R, D, LE1>(acc, Fs + r0 * LE1, lw.W1T + D, 3 * D, lane);
        __syncwarp();
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int row = r0 + r;
            const float4 vj = ldg4(QKV + (size_t)meta.src[row] * 3 * D + 2 * D + col);
            st4(Fs + row * LE1 + col, vj * silu4(arr4(acc[r])) * Areg[r]);
            if (row < nvalid) st4(P1 + (size_t)(e0 + row) * 3 * D + D + col, arr4(acc[r]));
        }
        __syncwarp();
        // ---- [s1|s2] = silu(m Ws^T + bs) ----
#pragma unroll 1
        for (int ch = 0; ch < 2; ch++) {
            acc_set_bias<R>(acc, lw.bs + ch * D, lane);
            warp_gemm<R, D, LE1>(acc, Fs + r0 * LE1, lw.WsT + ch * D, 2 * D, lane);
#pragma unroll
            for (int r = 0; r < R; r++) {
                st4(Ss + (r0 + r) * LE2 + ch * D + col, silu4(arr4(acc[r])));
                if (r0 + r < nvalid) st4(SP + (size_t)(e0 + r0 + r) * 2 * D + ch * D + col, arr4(acc[r]));
            }
        }
        __syncthreads();
        // ---- segmented reduction onto the targets present in this tile ----
        {
            const int c = threadIdx.x & (D - 1), grp = threadIdx.x >> 7;
            const int i_first = meta.dst[0], i_last = meta.dst[nvalid - 1];
            for (int i = i_first + grp; i <= i_last; i += NT / D) {
                const int lo = max(ws.rowptr[i], e0) - e0;
                const int hi = min(ws.rowptr[i + 1], e0 + nvalid) - e0;
                float xa = 0.f, va0 = 0.f, va1 = 0.f, va2 = 0.f;
                int e = lo;
                for (; e + 4 <= hi; e += 4) {                  // 12 independent gathers in flight
                    float g[4][3];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const size_t j3 = (size_t)meta.src[e + u] * 3;
                        g[u][0] = __ldg(VN + (j3 + 0) * D + c); g[u][1] = __ldg(VN + (j3 + 1) * D + c); g[u][2] = __ldg(VN + (j3 + 2) * D + c);
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const float4 dd = meta.d[e + u];
                        const float s1 = Ss[(e + u) * LE2 + c], s2 = Ss[(e + u) * LE2 + D + c];
                        xa += Fs[(e + u) * LE1 + c];
                        va0 += g[u][0] * s1 + s2 * dd.x;
                        va1 += g[u][1] * s1 + s2 * dd.y;
                        va2 += g[u][2] * s1 + s2 * dd.z;
                    }
                }
                for (; e < hi; e++) {
                    const size_t j3 = (size_t)meta.src[e] * 3;
                    const float4 dd = meta.d[e];
                    const float s1 = Ss[e * LE2 + c], s2 = Ss[e * LE2 + D + c];
                    xa += Fs[e * LE1 + c];
                    va0 += __ldg(VN + (j3 + 0) * D + c) * s1 + s2 * dd.x;
                    va1 += __ldg(VN + (j3 + 1) * D + c) * s1 + s2 * dd.y;
                    va2 += __ldg(VN + (j3 + 2) * D + c) * s1 + s2 * dd.z;
                }
                atomicAdd(ws.XA + (size_t)i * D + c, xa);
                atomicAdd(ws.VA + ((size_t)i * 3 + 0) * D + c, va0);
                atomicAdd(ws.VA + ((size_t)i * 3 + 1) * D + c, va1);
                atomicAdd(ws.VA + ((size_t)i * 3 + 2) * D + c, va2);
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------
// adjoint.  The forward stage left the pre-activations P1 = [Pdk|Pdv|Pf], SP = s_proj pre-activation and the
// attention pre-activation ATT in HBM/L2, so the reverse sweep only runs the two adjoint contractions
//   g_m = g_xa_i + g_Spre Ws            (K = 256)
//   g_f = g_f_next + [g_Pdk|g_Pdv|g_Pf] W1   (K = 384, 256 in the last layer)
// (the stage is contraction bound, not HBM bound, so 2.5 KB/edge of stored state is cheaper than recomputing
// five 128x128 contractions per edge tile).
// ---------------------------------------------------------------------------------------------
constexpr int LEQ = 2 * D + 2 * LDS_PAD;   // 264: g_Spre row (256) / later the two per-edge tiles g_q (0..127) and g_wdot (132..259)

template <int TE>
constexpr size_t edge_bwd_smem_bytes() {
    return (size_t)TE * (LEQ + LE3) * sizeof(float) + sizeof(EdgeMeta<TE>);
}

template <int TE, int NW>
__global__ void __launch_bounds__(NW * 32) edge_bwd_kernel(EdgeArgs a) {
    pdl_entry();
    constexpr int R = TE / NW, NT = NW * 32;
    static_assert(TE % NW == 0 && NT % D == 0, "tile shape");
    extern __shared__ __align__(16) float dyn_smem[];
    float* Ss = dyn_smem;                 // [TE][264]  g_Spre (A operand of g_m), later g_q | g_wdot per-edge tiles
    float* Ps = Ss + TE * LEQ;            // [TE][388]  g_P (A operand of g_f)
    EdgeMeta<TE>& meta = *reinterpret_cast<EdgeMeta<TE>*>(Ps + TE * LE3);
    const Workspace& ws = a.ws;
    const int l = a.layer;
    const LayerW& lw = a.mw.layer[l];
    const bool upd = (l < L - 1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, col = lane * 4, hd = lane >> 2;
    const int E = ws.rowptr[ws.N];
    const float* __restrict__ QKV = ws.QKV[l];
    const float* __restrict__ VN = ws.VN[l];
    const float* __restrict__ TU = ws.TU[l];
    const float* __restrict__ P1 = ws.P1[l];
    const float* __restrict__ SP = ws.SP[l];
    const float* __restrict__ ATT = ws.ATT[l];
    const int r0 = warp * R;
    constexpr int QOFF = 0, WOFF = D + LDS_PAD;   // column offsets of the two per-edge tiles inside an Ss row

    for (int e0 = blockIdx.x * TE; e0 < E; e0 += gridDim.x * TE) {
        const int nvalid = min(TE, E - e0);
        load_edge_meta<TE, NT>(meta, ws, e0, nvalid);
        __syncthreads();
        float acc[R][4];
        float gdx[R], gdy[R], gdz[R], gC[R];
        // ---- adjoint of M = vn_j*s1 + s2*d and of silu(s_proj) ----
        // (all loads of a batch are issued before the first atomic: atomics are compiler barriers for load hoisting)
        constexpr int RBB = (R < 2) ? R : 2;
#pragma unroll
        for (int rb = 0; rb < R; rb += RBB) {
            float4 sp1r[RBB], sp2r[RBB], gMr[RBB][3], vnr[RBB][3];
#pragma unroll
            for (int u = 0; u < RBB; u++) {
                const int row = r0 + rb + u;
                const size_t e = (size_t)(e0 + (row < nvalid ? row : 0));
                const size_t i3 = (size_t)meta.dst[row] * 3, j3 = (size_t)meta.src[row] * 3;
                sp1r[u] = ldg4(SP + e * 2 * D + col);
                sp2r[u] = ldg4(SP + e * 2 * D + D + col);
#pragma unroll
                for (int s = 0; s < 3; s++) { gMr[u][s] = ldg4(ws.GVEC + (i3 + s) * D + col); vnr[u][s] = ldg4(VN + (j3 + s) * D + col); }
            }
#pragma unroll
            for (int u = 0; u < RBB; u++) {
                const int r = rb + u, row = r0 + r;
                const bool ok = row < nvalid;
                const size_t j3 = (size_t)meta.src[row] * 3;
                const float4 dd = meta.d[row];
                const float4 s1 = silu4(sp1r[u]), s2 = silu4(sp2r[u]);
                const float4 gs1 = gMr[u][0] * vnr[u][0] + gMr[u][1] * vnr[u][1] + gMr[u][2] * vnr[u][2];
                const float4 gs2 = gMr[u][0] * dd.x + gMr[u][1] * dd.y + gMr[u][2] * dd.z;
                gdx[r] = warp_sum(hsum4(gMr[u][0] * s2));
                gdy[r] = warp_sum(hsum4(gMr[u][1] * s2));
                gdz[r] = warp_sum(hsum4(gMr[u][2] * s2));
                st4(Ss + row * LEQ + col, ok ? gs1 * dsilu4(sp1r[u]) : f4s(0.f));
                st4(Ss + row * LEQ + D + col, ok ? gs2 * dsilu4(sp2r[u]) : f4s(0.f));
                if (ok) {
                    red4(ws.GVNMSG + (j3 + 0) * D + col, gMr[u][0] * s1);
                    red4(ws.GVNMSG + (j3 + 1) * D + col, gMr[u][1] * s1);
                    red4(ws.GVNMSG + (j3 + 2) * D + col, gMr[u][2] * s1);
                }
            }
        }
        __syncwarp();
        // ---- g_m = g_xa_i + g_Spre Ws ----
#pragma unroll
        for (int r = 0; r < R; r++) {
            const float4 t = load_gxa(ws, (size_t)meta.dst[r0 + r], col);
            acc[r][0] = t.x; acc[r][1] = t.y; acc[r][2] = t.z; acc[r][3] = t.w;
        }
        warp_gemm<R, 2 * D, LEQ>(acc, Ss + r0 * LEQ, lw.WsN, D, lane);
        __syncwarp();
#pragma unroll
        for (int rb = 0; rb < R; rb += RBB) {
            float4 vjr[RBB], pdvr[RBB], pdkr[RBB], qir[RBB], kjr[RBB];
            float avr[RBB];
#pragma unroll
            for (int u = 0; u < RBB; u++) {
                const int row = r0 + rb + u;
                const size_t e = (size_t)(e0 + (row < nvalid ? row : 0));
                const size_t i = meta.dst[row], j = meta.src[row];
                vjr[u] = ldg4(QKV + j * 3 * D + 2 * D + col);
                pdvr[u] = ldg4(P1 + e * 3 * D + D + col);
                pdkr[u] = ldg4(P1 + e * 3 * D + col);
                qir[u] = ldg4(QKV + i * 3 * D + col);
                kjr[u] = ldg4(QKV + j * 3 * D + D + col);
                avr[u] = row < nvalid ? __ldg(ATT + e * H + hd) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < RBB; u++) {
                const int r = rb + u, row = r0 + r;
                const bool ok = row < nvalid;
                const size_t j = meta.src[row];
                const float4 gm = arr4(acc[r]);
                const float Ce = meta.C[row];
                const float av = avr[u], sa = silu_(av), A = sa * Ce;
                const float4 dv = silu4(pdvr[u]), dk = silu4(pdkr[u]);
                st4(Ps + row * LE3 + D + col, ok ? gm * vjr[u] * A * dsilu4(pdvr[u]) : f4s(0.f));
                const float gA = quad_sum(hsum4(gm * vjr[u] * dv));
                const float ga = gA * Ce * dsilu_(av);
                gC[r] = warp_sum((lane & 3) == 0 ? gA * sa : 0.f);
                st4(Ss + row * LEQ + QOFF + col, kjr[u] * dk * ga);                        // per-edge g_q contribution
                st4(Ps + row * LE3 + col, ok ? qir[u] * kjr[u] * ga * dsilu4(pdkr[u]) : f4s(0.f));
                if (ok) {
                    red4(ws.GQKV + j * 3 * D + 2 * D + col, gm * dv * A);
                    red4(ws.GQKV + j * 3 * D + D + col, qir[u] * dk * ga);                  // g_k (source side)
                }
            }
        }
        // ---- adjoint of the edge update ----
        if (upd) {
#pragma unroll
            for (int rb = 0; rb < R; rb += RBB) {
                float4 gfr[RBB], pfr[RBB], tir[RBB][3], ujr[RBB][3];
#pragma unroll
                for (int u = 0; u < RBB; u++) {
                    const int row = r0 + rb + u;
                    const bool ok = row < nvalid;
                    const size_t e = (size_t)(e0 + (ok ? row : 0));
                    const size_t i3 = (size_t)meta.dst[row] * 3, j3 = (size_t)meta.src[row] * 3;
                    gfr[u] = ok ? ld4(ws.GF + e * D + col) : f4s(0.f);
                    pfr[u] = ldg4(P1 + e * 3 * D + 2 * D + col);
#pragma unroll
                    for (int s = 0; s < 3; s++) {
                        tir[u][s] = ldg4(TU + (i3 + s) * 2 * D + col);
                        ujr[u][s] = ldg4(TU + (j3 + s) * 2 * D + D + col);
                    }
                }
#pragma unroll
                for (int u = 0; u < RBB; u++) {
                    const int r = rb + u, row = r0 + r;
                    const bool ok = row < nvalid;
                    const size_t j3 = (size_t)meta.src[row] * 3;
                    const float4 dd = meta.d[row];
                    const float4 gfn = gfr[u], pf = pfr[u];
                    const float4 fp = silu4(pf);
                    const float dv3[3] = {dd.x, dd.y, dd.z};
                    const float4 a1 = tir[u][0] * dd.x + tir[u][1] * dd.y + tir[u][2] * dd.z;
                    const float4 a2 = ujr[u][0] * dd.x + ujr[u][1] * dd.y + ujr[u][2] * dd.z;
                    float4 w1[3], w2[3];
#pragma unroll
                    for (int s = 0; s < 3; s++) { w1[s] = tir[u][s] - a1 * dv3[s]; w2[s] = ujr[u][s] - a2 * dv3[s]; }
                    const float4 wdot = w1[0] * w2[0] + w1[1] * w2[1] + w1[2] * w2[2];
                    const float4 gwd = gfn * fp;
                    st4(Ss + row * LEQ + WOFF + col, gwd);
                    st4(Ps + row * LE3 + 2 * D + col, gfn * wdot * dsilu4(pf));
                    const float4 c1 = gwd * (w2[0] * dd.x + w2[1] * dd.y + w2[2] * dd.z);
                    const float4 c2 = gwd * (w1[0] * dd.x + w1[1] * dd.y + w1[2] * dd.z);
                    float gdl[3];
                    float4 gu[3];
#pragma unroll
                    for (int s = 0; s < 3; s++) {
                        const float4 gw1 = gwd * w2[s], gw2 = gwd * w1[s];
                        gu[s] = gw2 - c2 * dv3[s];
                        gdl[s] = warp_sum(hsum4(tir[u][s] * c1 + a1 * gw1 + ujr[u][s] * c2 + a2 * gw2));
                    }
                    gdx[r] -= gdl[0]; gdy[r] -= gdl[1]; gdz[r] -= gdl[2];
                    acc[r][0] = gfn.x; acc[r][1] = gfn.y; acc[r][2] = gfn.z; acc[r][3] = gfn.w;
                    if (ok) {
                        red4(ws.GTU + (j3 + 0) * 2 * D + D + col, gu[0]);   // g_u (source side)
                        red4(ws.GTU + (j3 + 1) * 2 * D + D + col, gu[1]);
                        red4(ws.GTU + (j3 + 2) * 2 * D + D + col, gu[2]);
                    }
                }
            }
        } else {
            acc_zero<R>(acc);
        }
        __syncwarp();
        // ---- g_f = g_f_next + [g_Pdk|g_Pdv|g_Pf] [Wdk;Wdv;Wf] ----
        if (upd) warp_gemm<R, 3 * D, LE3>(acc, Ps + r0 * LE3, lw.W1N, D, lane);
        else     warp_gemm<R, 2 * D, LE3>(acc, Ps + r0 * LE3, lw.W1N, D, lane);
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int row = r0 + r;
            if (row < nvalid) {
                st4(ws.GF + (size_t)(e0 + row) * D + col, arr4(acc[r]));
                if (lane == 0) {
                    float* ea = ws.eacc + (size_t)(e0 + row) * 4;
                    st4(ea, ld4(ea) + f4(gC[r], gdx[r], gdy[r], gdz[r]));
                }
            }
        }
        __syncthreads();
        // ---- segmented reduction of the target-side adjoints: g_q and g_t ----
        {
            const int c = threadIdx.x & (D - 1), grp = threadIdx.x >> 7;
            const int i_first = meta.dst[0], i_last = meta.dst[nvalid - 1];
            for (int i = i_first + grp; i <= i_last; i += NT / D) {
                const int lo = max(ws.rowptr[i], e0) - e0;
                const int hi = min(ws.rowptr[i + 1], e0 + nvalid) - e0;
                float gq = 0.f, gt0 = 0.f, gt1 = 0.f, gt2 = 0.f;
                for (int e = lo; e < hi; e++) {
                    gq += Ss[e * LEQ + QOFF + c];
                    if (upd) {
                        const size_t j3 = (size_t)meta.src[e] * 3;
                        const float4 dd = meta.d[e];
                        const float gw = Ss[e * LEQ + WOFF + c];
                        const float u0 = __ldg(TU + (j3 + 0) * 2 * D + D + c), u1 = __ldg(TU + (j3 + 1) * 2 * D + D + c),
                                    u2 = __ldg(TU + (j3 + 2) * 2 * D + D + c);
                        const float a2 = u0 * dd.x + u1 * dd.y + u2 * dd.z;
                        const float w20 = u0 - a2 * dd.x, w21 = u1 - a2 * dd.y, w22 = u2 - a2 * dd.z;
                        const float wd = w20 * dd.x + w21 * dd.y + w22 * dd.z;
                        gt0 += gw * (w20 - wd * dd.x);
                        gt1 += gw * (w21 - wd * dd.y);
                        gt2 += gw * (w22 - wd * dd.z);
                    }
                }
                atomicAdd(ws.GQKV + (size_t)i * 3 * D + c, gq);
                if (upd) {
                    atomicAdd(ws.GTU + ((size_t)i * 3 + 0) * 2 * D + c, gt0);
                    atomicAdd(ws.GTU + ((size_t)i * 3 + 1) * 2 * D + c, gt1);
                    atomicAdd(ws.GTU + ((size_t)i * 3 + 2) * 2 * D + c, gt2);
                }
            }
        }
        __syncthreads();
    }
}

}  // namespace vb
