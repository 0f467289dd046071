// Helpers shared by the node stages (k_node2.cuh, k_node_tc.cuh) and the head (k_head.cuh): the launch arguments of a
// node stage and the per-node LayerNorm / VecLayerNorm (max_min) forward and adjoint, one warp per node with lane owning
// channels lane*4..lane*4+3.
//   reference: visnet_block.py:238-239 (LayerNorm, VecLayerNorm), utils.py:200-228 (VecLayerNorm max_min).
#pragma once
#include "model.h"

namespace vb {

constexpr int NODE_WARPS = 4;
constexpr float LN_EPS = 1e-5f;
constexpr float VLN_EPS = 1e-12f;

struct NodeArgs {
    int layer;      // forward: stage k in 0..L ; backward: stage k in L..0
    ModelW mw;
    Workspace ws;
    unsigned long long* tl = nullptr;   // optional timeline (SM clock stamps of every warp of CTA 0 at the phase boundaries of
                                        // the CTA-cooperative kernels, k_node2.cuh: slot = stamp * 16 + warp); nullptr = off
    int krot = 0;                       // 1: every CTA starts the K loops of its GEMM units at a different row (common.cuh)
};
constexpr int N2_TL_SLOTS = 256;

// ---- small per-lane helpers ----------------------------------------------------------------------
__device__ __forceinline__ float4 ln_forward(float4 x, const float* __restrict__ w, const float* __restrict__ b,
                                             int lane) {
    const float mean = warp_sum(hsum4(x)) * (1.0f / D);
    const float4 dlt = x - f4s(mean);
    const float var = warp_sum(hsum4(dlt * dlt)) * (1.0f / D);
    const float rstd = 1.0f / sqrtf(var + LN_EPS);
    return dlt * rstd * ldg4(w + lane * 4) + ldg4(b + lane * 4);
}

// gx += LN'(x)^T gy
__device__ __forceinline__ float4 ln_backward(float4 x, float4 gy, const float* __restrict__ w, int lane) {
    const float mean = warp_sum(hsum4(x)) * (1.0f / D);
    const float4 dlt = x - f4s(mean);
    const float var = warp_sum(hsum4(dlt * dlt)) * (1.0f / D);
    const float rstd = 1.0f / sqrtf(var + LN_EPS);
    const float4 xh = dlt * rstd;
    const float4 gh = gy * ldg4(w + lane * 4);
    const float m1 = warp_sum(hsum4(gh)) * (1.0f / D);
    const float m2 = warp_sum(hsum4(gh * xh)) * (1.0f / D);
    return (gh - f4s(m1) - xh * m2) * rstd;
}

__device__ __forceinline__ float max4(float4 a) { return fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)); }
__device__ __forceinline__ float min4(float4 a) { return fminf(fminf(a.x, a.y), fminf(a.z, a.w)); }

// VecLayerNorm(max_min) forward for one node; v[s] = lane's 4 channels of component s.
__device__ __forceinline__ void vecln_forward(const float4 (&v)[3], float4 (&out)[3],
                                              const float* __restrict__ w, int lane) {
    float4 n;
    n.x = sqrtf(v[0].x * v[0].x + v[1].x * v[1].x + v[2].x * v[2].x);
    n.y = sqrtf(v[0].y * v[0].y + v[1].y * v[1].y + v[2].y * v[2].y);
    n.z = sqrtf(v[0].z * v[0].z + v[1].z * v[1].z + v[2].z * v[2].z);
    n.w = sqrtf(v[0].w * v[0].w + v[1].w * v[1].w + v[2].w * v[2].w);
    const float4 nc = f4(fmaxf(n.x, VLN_EPS), fmaxf(n.y, VLN_EPS), fmaxf(n.z, VLN_EPS), fmaxf(n.w, VLN_EPS));
    const float mx = warp_max(max4(nc));
    const float mn = warp_min(min4(nc));
    float delta = mx - mn;
    if (delta == 0.f) delta = 1.f;
    const float4 ww = ldg4(w + lane * 4);
    float4 y = f4((nc.x - mn) / delta, (nc.y - mn) / delta, (nc.z - mn) / delta, (nc.w - mn) / delta);
    y = f4(fmaxf(y.x, 0.f), fmaxf(y.y, 0.f), fmaxf(y.z, 0.f), fmaxf(y.w, 0.f));
#pragma unroll
    for (int s = 0; s < 3; s++)
        out[s] = f4(y.x * (v[s].x / nc.x) * ww.x, y.y * (v[s].y / nc.y) * ww.y, y.z * (v[s].z / nc.z) * ww.z,
                    y.w * (v[s].w / nc.w) * ww.w);
}

// VecLayerNorm(max_min) adjoint (oracle/adjoint_ref.py: vecln_bwd).  Returns dE/dvec in gv.
__device__ __forceinline__ void vecln_backward(const float4 (&v)[3], const float4 (&gout)[3], float4 (&gv)[3],
                                               const float* __restrict__ w, int lane) {
    float nn[4], ncv[4];
    const float* vp[3] = {&v[0].x, &v[1].x, &v[2].x};
    const float* gp[3] = {&gout[0].x, &gout[1].x, &gout[2].x};
    float ww[4];
    {
        const float4 t = ldg4(w + lane * 4);
        ww[0] = t.x; ww[1] = t.y; ww[2] = t.z; ww[3] = t.w;
    }
    unsigned long long kmax = 0ull, kmin = ~0ull;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        nn[q] = sqrtf(vp[0][q] * vp[0][q] + vp[1][q] * vp[1][q] + vp[2][q] * vp[2][q]);
        ncv[q] = fmaxf(nn[q], VLN_EPS);
        const unsigned idx = (unsigned)(lane * 4 + q);
        const unsigned long long bits = (unsigned long long)__float_as_uint(ncv[q]) << 32;
        const unsigned long long ka = bits | (unsigned long long)(0xFFFFFFFFu - idx);  // max: ties -> lowest index
        const unsigned long long ki = bits | (unsigned long long)idx;                  // min: ties -> lowest index
        kmax = ka > kmax ? ka : kmax;
        kmin = ki < kmin ? ki : kmin;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long a = __shfl_xor_sync(0xffffffffu, kmax, o);
        const unsigned long long b = __shfl_xor_sync(0xffffffffu, kmin, o);
        kmax = a > kmax ? a : kmax;
        kmin = b < kmin ? b : kmin;
    }
    const float mx = __uint_as_float((unsigned)(kmax >> 32));
    const float mn = __uint_as_float((unsigned)(kmin >> 32));
    const int amx = (int)(0xFFFFFFFFu - (unsigned)(kmax & 0xFFFFFFFFull));
    const int amn = (int)(unsigned)(kmin & 0xFFFFFFFFull);
    const float draw = mx - mn;
    const bool zero = (draw == 0.f);
    const float delta = zero ? 1.f : draw;
    float y[4], gdir[3][4], gy[4];
    float s_gy = 0.f, s_gyy = 0.f;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        y[q] = (ncv[q] - mn) / delta;
        const float ry = fmaxf(y[q], 0.f);
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < 3; s++) {
            const float gw = gp[s][q] * ww[q];
            gdir[s][q] = gw * ry;
            acc += gw * (vp[s][q] / ncv[q]);
        }
        gy[q] = (y[q] > 0.f) ? acc : 0.f;
        s_gy += gy[q] / delta;
        s_gyy += gy[q] * y[q];
    }
    s_gy = warp_sum(s_gy);
    s_gyy = warp_sum(s_gyy);
    float g_mn = -s_gy;
    const float g_delta = zero ? 0.f : -s_gyy / delta;
    const float g_mx = g_delta;
    g_mn -= g_delta;
    float outv[3][4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int idx = lane * 4 + q;
        float g_nc = gy[q] / delta;
        if (idx == amx) g_nc += g_mx;
        if (idx == amn) g_nc += g_mn;
        float dotv = 0.f;
#pragma unroll
        for (int s = 0; s < 3; s++) dotv += gdir[s][q] * vp[s][q];
        g_nc -= dotv / (ncv[q] * ncv[q]);
        const float g_n = (nn[q] >= VLN_EPS) ? g_nc : 0.f;
        const float inv_n = (nn[q] > 0.f) ? 1.0f / nn[q] : 0.f;
#pragma unroll
        for (int s = 0; s < 3; s++) outv[s][q] = gdir[s][q] / ncv[q] + g_n * inv_n * vp[s][q];
    }
#pragma unroll
    for (int s = 0; s < 3; s++) gv[s] = f4(outv[s][0], outv[s][1], outv[s][2], outv[s][3]);
}

}  // namespace vb
