// Output stage: out_norm / vec_out_norm, the two gated equivariant blocks, atomref prior -- forward and
// adjoint fused in one per-node kernel (the head is node-local, so dE/dx6, dE/dvec6 follow immediately).
//   reference: visnet_block.py:139-140, output_modules.py:52-62,136-140, priors.py:86-87, visnet.py:141-149
#pragma once
#include "k_node.cuh"

namespace vb {

template <int NPW>
struct HeadSmem {
    static constexpr int L128 = D + LDS_PAD;       // 132
    static constexpr int L256 = 2 * D + LDS_PAD;   // 260
    static constexpr int L64 = 64 + LDS_PAD;       // 68
    static constexpr int OFF_VS = 0;                              // [3NPW][132]  V rows  -> later g_p1 rows
    static constexpr int OFF_CAT = OFF_VS + 3 * NPW * L128;       // [NPW][260]   [X | n1]
    static constexpr int OFF_HS = OFF_CAT + NPW * L256;           // [NPW][132]   h       -> later g_y
    static constexpr int OFF_YS = OFF_HS + NPW * L128;            // [NPW][132]   y
    static constexpr int OFF_VP = OFF_YS + NPW * L128;            // [3NPW][68]   V'      -> g_p1b -> g_p2
    static constexpr int OFF_CB = OFF_VP + 3 * NPW * L64;         // [NPW][132]   [xs|n1b] -> g_catb
    static constexpr int OFF_GPB = OFF_CB + NPW * L128;           // [NPW][68]    g_preb
    static constexpr int OFF_GPRE = OFF_GPB + NPW * L64;          // [NPW][132]   g_pre
    static constexpr int PER_WARP = OFF_GPRE + NPW * L128;
    static constexpr size_t BYTES = (size_t)NODE_WARPS * PER_WARP * sizeof(float);
};

template <int NPW>
__global__ void __launch_bounds__(NODE_WARPS * 32) head_kernel(ModelW mw, Workspace ws) {
    pdl_entry();
    using S = HeadSmem<NPW>;
    constexpr int L128 = S::L128, L256 = S::L256, L64 = S::L64;
    extern __shared__ __align__(16) float dyn_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* sm = dyn_smem + (size_t)warp * S::PER_WARP;
    float* Vs = sm + S::OFF_VS;
    float* cat = sm + S::OFF_CAT;
    float* hs = sm + S::OFF_HS;
    float* ys = sm + S::OFF_YS;
    float* Vp = sm + S::OFF_VP;
    float* cb = sm + S::OFF_CB;
    float* gpb = sm + S::OFF_GPB;
    float* gpre = sm + S::OFF_GPRE;
    const int n0 = (blockIdx.x * NODE_WARPS + warp) * NPW;
    if (n0 >= ws.N) return;
    const int col = lane * 4, c2 = lane * 2;
    const float stdv = __ldg(mw.scalars);

    float4 x6[NPW], v6[NPW][3];
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
        const int node = n0 + nd;
        const bool ok = node < ws.N;
        x6[nd] = ok ? ld4(ws.X[L] + (size_t)node * D + col) : f4s(0.f);
#pragma unroll
        for (int s = 0; s < 3; s++) v6[nd][s] = ok ? ld4(ws.V[L] + ((size_t)node * 3 + s) * D + col) : f4s(0.f);
        st4(cat + nd * L256 + col, ln_forward(x6[nd], mw.on_w, mw.on_b, lane));
        float4 vn[3];
        vecln_forward(v6[nd], vn, mw.von_w, lane);
#pragma unroll
        for (int s = 0; s < 3; s++) st4(Vs + (nd * 3 + s) * L128 + col, vn[s]);
    }
    __syncwarp();
    // ---- block 0 ----
    float p1[3 * NPW][4], p2[3 * NPW][2];
    acc_zero<3 * NPW>(p1);
    warp_gemm<3 * NPW, D, L128>(p1, Vs, mw.h0_W1T, D, lane);
#pragma unroll
    for (int r = 0; r < 3 * NPW; r++) p2[r][0] = p2[r][1] = 0.f;
    warp_gemm2<3 * NPW, D, L128>(p2, Vs, mw.h0_W2T, 64, lane);
    float4 n1[NPW];
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
        const float4 a = arr4(p1[nd * 3]), b = arr4(p1[nd * 3 + 1]), c = arr4(p1[nd * 3 + 2]);
        const float4 q = a * a + b * b + c * c;
        n1[nd] = f4(sqrtf(q.x), sqrtf(q.y), sqrtf(q.z), sqrtf(q.w));
        st4(cat + nd * L256 + D + col, n1[nd]);
    }
    __syncwarp();
    float pre[NPW][4];
    acc_set_bias<NPW>(pre, mw.h0_b0, lane);
    warp_gemm<NPW, 2 * D, L256>(pre, cat, mw.h0_U0T, D, lane);
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) st4(hs + nd * L128 + col, silu4(arr4(pre[nd])));
    __syncwarp();
    {
        float y[NPW][4];
        acc_set_bias<NPW>(y, mw.h0_b2, lane);
        warp_gemm<NPW, D, L128>(y, hs, mw.h0_U2T, D, lane);
#pragma unroll
        for (int nd = 0; nd < NPW; nd++) st4(ys + nd * L128 + col, arr4(y[nd]));
    }
    __syncwarp();
    // xs = silu(y[:64]) ; g = y[64:] ; V' = g * p2   (2 columns per lane from here on)
    float gate[NPW][2];
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
        gate[nd][0] = ys[nd * L128 + 64 + c2];
        gate[nd][1] = ys[nd * L128 + 64 + c2 + 1];
        cb[nd * L128 + c2] = silu_(ys[nd * L128 + c2]);
        cb[nd * L128 + c2 + 1] = silu_(ys[nd * L128 + c2 + 1]);
#pragma unroll
        for (int s = 0; s < 3; s++) {
            Vp[(nd * 3 + s) * L64 + c2] = gate[nd][0] * p2[nd * 3 + s][0];
            Vp[(nd * 3 + s) * L64 + c2 + 1] = gate[nd][1] * p2[nd * 3 + s][1];
        }
    }
    __syncwarp();
    // ---- block 1 ----
    float p1b[3 * NPW][2];
#pragma unroll
    for (int r = 0; r < 3 * NPW; r++) p1b[r][0] = p1b[r][1] = 0.f;
    warp_gemm2<3 * NPW, 64, L64>(p1b, Vp, mw.h1_W1T, 64, lane);
    float n1b[NPW][2];
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
#pragma unroll
        for (int q = 0; q < 2; q++) {
            n1b[nd][q] = sqrtf(p1b[nd * 3][q] * p1b[nd * 3][q] + p1b[nd * 3 + 1][q] * p1b[nd * 3 + 1][q] +
                               p1b[nd * 3 + 2][q] * p1b[nd * 3 + 2][q]);
            cb[nd * L128 + 64 + c2 + q] = n1b[nd][q];
        }
    }
    __syncwarp();
    float preb[NPW][2];
    {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(mw.h1_b0 + c2));
#pragma unroll
        for (int nd = 0; nd < NPW; nd++) { preb[nd][0] = bb.x; preb[nd][1] = bb.y; }
    }
    warp_gemm2<NPW, D, L128>(preb, cb, mw.h1_U0T, 64, lane);
    const float2 u2 = __ldg(reinterpret_cast<const float2*>(mw.h1_u2 + c2));
    const float b2 = __ldg(mw.h1_b2);
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
        const float e = warp_sum(silu_(preb[nd][0]) * u2.x + silu_(preb[nd][1]) * u2.y) + b2;
        const int node = n0 + nd;
        if (lane == 0 && node < ws.N) ws.eatom[node] = e * stdv + __ldg(mw.atomref + ws.z[node]);
    }
    if (ws.GX == nullptr) return;         // energy plan: no adjoint outputs in the workspace
    // ================= adjoint (dE_total/de_atom = 1) =================
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
        gpb[nd * L64 + c2] = stdv * u2.x * dsilu_(preb[nd][0]);
        gpb[nd * L64 + c2 + 1] = stdv * u2.y * dsilu_(preb[nd][1]);
    }
    __syncwarp();
    {
        float gcb[NPW][4];
        acc_zero<NPW>(gcb);
        warp_gemm<NPW, 64, L64>(gcb, gpb, mw.h1_U0N, D, lane);   // [g_xs | g_n1b]
        __syncwarp();
#pragma unroll
        for (int nd = 0; nd < NPW; nd++) st4(cb + nd * L128 + col, arr4(gcb[nd]));
    }
    __syncwarp();
    // g_p1b = g_n1b / n1b * p1b  -> rows in Vp ; g_Vp = g_p1b W1'
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
#pragma unroll
        for (int q = 0; q < 2; q++) {
            const float gn = cb[nd * L128 + 64 + c2 + q];
            const float sc = n1b[nd][q] > 0.f ? gn / n1b[nd][q] : 0.f;
#pragma unroll
            for (int s = 0; s < 3; s++) Vp[(nd * 3 + s) * L64 + c2 + q] = sc * p1b[nd * 3 + s][q];
        }
    }
    __syncwarp();
    float gVp[3 * NPW][2];
#pragma unroll
    for (int r = 0; r < 3 * NPW; r++) gVp[r][0] = gVp[r][1] = 0.f;
    warp_gemm2<3 * NPW, 64, L64>(gVp, Vp, mw.h1_W1N, 64, lane);
    __syncwarp();
    // g_g, g_p2 ; g_y = [g_xs * silu'(y[:64]) | g_g] -> hs ; g_p2 rows -> Vp
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
#pragma unroll
        for (int q = 0; q < 2; q++) {
            float gg = 0.f;
#pragma unroll
            for (int s = 0; s < 3; s++) {
                gg += gVp[nd * 3 + s][q] * p2[nd * 3 + s][q];
                Vp[(nd * 3 + s) * L64 + c2 + q] = gVp[nd * 3 + s][q] * gate[nd][q];
            }
            hs[nd * L128 + 64 + c2 + q] = gg;
            hs[nd * L128 + c2 + q] = cb[nd * L128 + c2 + q] * dsilu_(ys[nd * L128 + c2 + q]);
        }
    }
    __syncwarp();
    {
        float gh[NPW][4];
        acc_zero<NPW>(gh);
        warp_gemm<NPW, D, L128>(gh, hs, mw.h0_U2N, D, lane);
#pragma unroll
        for (int nd = 0; nd < NPW; nd++) st4(gpre + nd * L128 + col, arr4(gh[nd]) * dsilu4(arr4(pre[nd])));
    }
    __syncwarp();
    float gX[NPW][4], gn1[NPW][4];
    acc_zero<NPW>(gX);
    acc_zero<NPW>(gn1);
    warp_gemm<NPW, D, L128>(gX, gpre, mw.h0_U0N, 2 * D, lane);
    warp_gemm<NPW, D, L128>(gn1, gpre, mw.h0_U0N + D, 2 * D, lane);
    // g_p1 = g_n1 / n1 * p1 -> Vs rows
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
        const float4 g = arr4(gn1[nd]);
        const float4 sc = f4(n1[nd].x > 0.f ? g.x / n1[nd].x : 0.f, n1[nd].y > 0.f ? g.y / n1[nd].y : 0.f,
                             n1[nd].z > 0.f ? g.z / n1[nd].z : 0.f, n1[nd].w > 0.f ? g.w / n1[nd].w : 0.f);
#pragma unroll
        for (int s = 0; s < 3; s++) st4(Vs + (nd * 3 + s) * L128 + col, sc * arr4(p1[nd * 3 + s]));
    }
    __syncwarp();
    float gV[3 * NPW][4];
    acc_zero<3 * NPW>(gV);
    warp_gemm<3 * NPW, D, L128>(gV, Vs, mw.h0_W1N, D, lane);
    warp_gemm<3 * NPW, 64, L64>(gV, Vp, mw.h0_W2N, D, lane);
#pragma unroll
    for (int nd = 0; nd < NPW; nd++) {
        const int node = n0 + nd;
        if (node >= ws.N) continue;
        float4 gout[3], gv[3];
#pragma unroll
        for (int s = 0; s < 3; s++) gout[s] = arr4(gV[nd * 3 + s]);
        vecln_backward(v6[nd], gout, gv, mw.von_w, lane);
#pragma unroll
        for (int s = 0; s < 3; s++) st4(ws.GVEC + ((size_t)node * 3 + s) * D + col, gv[s]);
        st4(ws.GX + (size_t)node * D + col, ln_backward(x6[nd], arr4(gX[nd]), mw.on_w, lane));
    }
}

}  // namespace vb

// =====================================================================================================
// K-split variant: one node per 4-warp CTA.  Every contraction of the head is split four ways along K
// (warp w multiplies K-quarter w), the partial rows are summed through shared memory in a fixed order and all
// warps continue with identical values.  Cuts the serial chain of 13 small GEMMs by ~4x for small systems,
// where the head is otherwise the longest single launch.
// =====================================================================================================
namespace vb {

struct Head2Smem {
    static constexpr int L128 = D + LDS_PAD, L256 = 2 * D + LDS_PAD, L64 = 64 + LDS_PAD;
    float Vs[3][L128];        // V rows -> g_p1 rows
    float cat[L256];          // [X | n1]
    float hs[L128];           // h -> g_y
    float ys[L128];           // y
    float Vp[3][L64];         // V' -> g_p1b -> g_p2
    float cb[L128];           // [xs | n1b] -> g_catb
    float gpb[L64];           // g_preb
    float gpre[L128];         // g_pre
    float red[4][3][D];       // K-split partial rows
};

template <int R, int K, int LDA>
__device__ __forceinline__ void ksplit_gemm(float (&acc)[R][4], const float* As, const float* __restrict__ W, int ldw,
                                            int lane, int warp, float (&red)[4][3][D]) {
    float part[R][4];
    acc_zero<R>(part);
    warp_gemm<R, K / 4, LDA, 4>(part, As + warp * (K / 4), W + (size_t)warp * (K / 4) * ldw, ldw, lane);
#pragma unroll
    for (int r = 0; r < R; r++) st4(&red[warp][r][lane * 4], arr4(part[r]));
    __syncthreads();
#pragma unroll
    for (int r = 0; r < R; r++) {
        const float4 s = (ld4(&red[0][r][lane * 4]) + ld4(&red[1][r][lane * 4])) + (ld4(&red[2][r][lane * 4]) + ld4(&red[3][r][lane * 4]));
        acc[r][0] += s.x; acc[r][1] += s.y; acc[r][2] += s.z; acc[r][3] += s.w;
    }
    __syncthreads();
}
template <int R, int K, int LDA>
__device__ __forceinline__ void ksplit_gemm2(float (&acc)[R][2], const float* As, const float* __restrict__ W, int ldw,
                                             int lane, int warp, float (&red)[4][3][D]) {
    float part[R][2];
#pragma unroll
    for (int r = 0; r < R; r++) part[r][0] = part[r][1] = 0.f;
    warp_gemm2<R, K / 4, LDA>(part, As + warp * (K / 4), W + (size_t)warp * (K / 4) * ldw, ldw, lane);
#pragma unroll
    for (int r = 0; r < R; r++) { red[warp][r][lane * 2] = part[r][0]; red[warp][r][lane * 2 + 1] = part[r][1]; }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < R; r++) {
        acc[r][0] += (red[0][r][lane * 2] + red[1][r][lane * 2]) + (red[2][r][lane * 2] + red[3][r][lane * 2]);
        acc[r][1] += (red[0][r][lane * 2 + 1] + red[1][r][lane * 2 + 1]) + (red[2][r][lane * 2 + 1] + red[3][r][lane * 2 + 1]);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(128) head2_kernel(ModelW mw, Workspace ws) {
    pdl_entry();
    constexpr int L128 = Head2Smem::L128, L256 = Head2Smem::L256, L64 = Head2Smem::L64;
    __shared__ __align__(16) Head2Smem sm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int node = blockIdx.x;
    if (node >= ws.N) return;
    const int col = lane * 4, c2 = lane * 2;
    const bool w0 = (warp == 0);
    const float stdv = __ldg(mw.scalars);

    float4 x6 = ld4(ws.X[L] + (size_t)node * D + col), v6[3];
#pragma unroll
    for (int s = 0; s < 3; s++) v6[s] = ld4(ws.V[L] + ((size_t)node * 3 + s) * D + col);
    {
        const float4 xn = ln_forward(x6, mw.on_w, mw.on_b, lane);
        float4 vn[3];
        vecln_forward(v6, vn, mw.von_w, lane);
        if (w0) {
            st4(&sm.cat[col], xn);
#pragma unroll
            for (int s = 0; s < 3; s++) st4(&sm.Vs[s][col], vn[s]);
        }
    }
    __syncthreads();
    // ---- block 0 ----
    float p1[3][4], p2[3][2];
    acc_zero<3>(p1);
    ksplit_gemm<3, D, L128>(p1, &sm.Vs[0][0], mw.h0_W1T, D, lane, warp, sm.red);
#pragma unroll
    for (int r = 0; r < 3; r++) p2[r][0] = p2[r][1] = 0.f;
    ksplit_gemm2<3, D, L128>(p2, &sm.Vs[0][0], mw.h0_W2T, 64, lane, warp, sm.red);
    float4 n1;
    {
        const float4 a = arr4(p1[0]), b = arr4(p1[1]), c = arr4(p1[2]);
        const float4 q = a * a + b * b + c * c;
        n1 = f4(sqrtf(q.x), sqrtf(q.y), sqrtf(q.z), sqrtf(q.w));
        if (w0) st4(&sm.cat[D + col], n1);
    }
    __syncthreads();
    float pre[1][4];
    acc_set_bias<1>(pre, mw.h0_b0, lane);
    ksplit_gemm<1, 2 * D, L256>(pre, &sm.cat[0], mw.h0_U0T, D, lane, warp, sm.red);
    if (w0) st4(&sm.hs[col], silu4(arr4(pre[0])));
    __syncthreads();
    {
        float y[1][4];
        acc_set_bias<1>(y, mw.h0_b2, lane);
        ksplit_gemm<1, D, L128>(y, &sm.hs[0], mw.h0_U2T, D, lane, warp, sm.red);
        if (w0) st4(&sm.ys[col], arr4(y[0]));
    }
    __syncthreads();
    float gate[2];
    gate[0] = sm.ys[64 + c2];
    gate[1] = sm.ys[64 + c2 + 1];
    if (w0) {
        sm.cb[c2] = silu_(sm.ys[c2]);
        sm.cb[c2 + 1] = silu_(sm.ys[c2 + 1]);
#pragma unroll
        for (int s = 0; s < 3; s++) {
            sm.Vp[s][c2] = gate[0] * p2[s][0];
            sm.Vp[s][c2 + 1] = gate[1] * p2[s][1];
        }
    }
    __syncthreads();
    // ---- block 1 ----
    float p1b[3][2];
#pragma unroll
    for (int r = 0; r < 3; r++) p1b[r][0] = p1b[r][1] = 0.f;
    ksplit_gemm2<3, 64, L64>(p1b, &sm.Vp[0][0], mw.h1_W1T, 64, lane, warp, sm.red);
    float n1b[2];
#pragma unroll
    for (int q = 0; q < 2; q++) {
        n1b[q] = sqrtf(p1b[0][q] * p1b[0][q] + p1b[1][q] * p1b[1][q] + p1b[2][q] * p1b[2][q]);
        if (w0) sm.cb[64 + c2 + q] = n1b[q];
    }
    __syncthreads();
    float preb[1][2];
    {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(mw.h1_b0 + c2));
        preb[0][0] = bb.x; preb[0][1] = bb.y;
    }
    ksplit_gemm2<1, D, L128>(preb, &sm.cb[0], mw.h1_U0T, 64, lane, warp, sm.red);
    const float2 u2 = __ldg(reinterpret_cast<const float2*>(mw.h1_u2 + c2));
    {
        const float e = warp_sum(silu_(preb[0][0]) * u2.x + silu_(preb[0][1]) * u2.y) + __ldg(mw.h1_b2);
        if (threadIdx.x == 0) ws.eatom[node] = e * stdv + __ldg(mw.atomref + ws.z[node]);
    }
    if (ws.GX == nullptr) return;         // energy plan: no adjoint outputs in the workspace
    // ================= adjoint =================
    if (w0) {
        sm.gpb[c2] = stdv * u2.x * dsilu_(preb[0][0]);
        sm.gpb[c2 + 1] = stdv * u2.y * dsilu_(preb[0][1]);
    }
    __syncthreads();
    {
        float gcb[1][4];
        acc_zero<1>(gcb);
        ksplit_gemm<1, 64, L64>(gcb, &sm.gpb[0], mw.h1_U0N, D, lane, warp, sm.red);   // [g_xs | g_n1b]
        if (w0) st4(&sm.cb[col], arr4(gcb[0]));
    }
    __syncthreads();
    if (w0) {
#pragma unroll
        for (int q = 0; q < 2; q++) {
            const float gn = sm.cb[64 + c2 + q];
            const float sc = n1b[q] > 0.f ? gn / n1b[q] : 0.f;
#pragma unroll
            for (int s = 0; s < 3; s++) sm.Vp[s][c2 + q] = sc * p1b[s][q];
        }
    }
    __syncthreads();
    float gVp[3][2];
#pragma unroll
    for (int r = 0; r < 3; r++) gVp[r][0] = gVp[r][1] = 0.f;
    ksplit_gemm2<3, 64, L64>(gVp, &sm.Vp[0][0], mw.h1_W1N, 64, lane, warp, sm.red);
    if (w0) {
#pragma unroll
        for (int q = 0; q < 2; q++) {
            float gg = 0.f;
#pragma unroll
            for (int s = 0; s < 3; s++) {
                gg += gVp[s][q] * p2[s][q];
                sm.Vp[s][c2 + q] = gVp[s][q] * gate[q];
            }
            sm.hs[64 + c2 + q] = gg;
            sm.hs[c2 + q] = sm.cb[c2 + q] * dsilu_(sm.ys[c2 + q]);
        }
    }
    __syncthreads();
    {
        float gh[1][4];
        acc_zero<1>(gh);
        ksplit_gemm<1, D, L128>(gh, &sm.hs[0], mw.h0_U2N, D, lane, warp, sm.red);
        if (w0) st4(&sm.gpre[col], arr4(gh[0]) * dsilu4(arr4(pre[0])));
    }
    __syncthreads();
    float gX[1][4], gn1[1][4];
    acc_zero<1>(gX);
    acc_zero<1>(gn1);
    ksplit_gemm<1, D, L128>(gX, &sm.gpre[0], mw.h0_U0N, 2 * D, lane, warp, sm.red);
    ksplit_gemm<1, D, L128>(gn1, &sm.gpre[0], mw.h0_U0N + D, 2 * D, lane, warp, sm.red);
    if (w0) {
        const float4 g = arr4(gn1[0]);
        const float4 sc = f4(n1.x > 0.f ? g.x / n1.x : 0.f, n1.y > 0.f ? g.y / n1.y : 0.f, n1.z > 0.f ? g.z / n1.z : 0.f,
                             n1.w > 0.f ? g.w / n1.w : 0.f);
#pragma unroll
        for (int s = 0; s < 3; s++) st4(&sm.Vs[s][col], sc * arr4(p1[s]));
    }
    __syncthreads();
    float gV[3][4];
    acc_zero<3>(gV);
    ksplit_gemm<3, D, L128>(gV, &sm.Vs[0][0], mw.h0_W1N, D, lane, warp, sm.red);
    ksplit_gemm<3, 64, L64>(gV, &sm.Vp[0][0], mw.h0_W2N, D, lane, warp, sm.red);
    if (w0) {
        float4 gout[3], gv[3];
#pragma unroll
        for (int s = 0; s < 3; s++) gout[s] = arr4(gV[s]);
        vecln_backward(v6, gout, gv, mw.von_w, lane);
#pragma unroll
        for (int s = 0; s < 3; s++) st4(ws.GVEC + ((size_t)node * 3 + s) * D + col, gv[s]);
        st4(ws.GX + (size_t)node * D + col, ln_backward(x6, arr4(gX[0]), mw.on_w, lane));
    }
}

}  // namespace vb
