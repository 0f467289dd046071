// Shared device helpers for the ViSNet sm_90a engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vb {

constexpr int D = 128;        // channels
constexpr int H = 8;          // heads (head_dim 16)
constexpr int NR = 32;        // radial basis functions
constexpr int L = 6;          // interaction layers
constexpr int KNB = 32;       // neighbour slots per atom (incl. self)
constexpr int LDS_PAD = 4;    // smem row padding (floats) keeps rows 16 B aligned

// Activations use the hardware exp2 / reciprocal (MUFU.EX2, MUFU.RCP): ~1e-6 relative error, far inside the stated
// force tolerance, and cheaper than the IEEE expf + division in the latency-bound edge stages.
__device__ __forceinline__ float sigmoidf_(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float silu_(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// d/dx [x*sigmoid(x)] = s*(1 + x*(1-s))
__device__ __forceinline__ float dsilu_(float x) {
    float s = sigmoidf_(x);
    return s * (1.0f + x * (1.0f - s));
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void red4(float* p, float4 v) { atomicAdd(reinterpret_cast<float4*>(p), v); }

__device__ __forceinline__ float4 f4(float a, float b, float c, float d) { return make_float4(a, b, c, d); }
__device__ __forceinline__ float4 f4s(float a) { return make_float4(a, a, a, a); }
__device__ __forceinline__ float4 operator+(float4 a, float4 b) { return f4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 operator-(float4 a, float4 b) { return f4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
__device__ __forceinline__ float4 operator*(float4 a, float4 b) { return f4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 operator*(float4 a, float b) { return f4(a.x * b, a.y * b, a.z * b, a.w * b); }
__device__ __forceinline__ float4 operator*(float b, float4 a) { return f4(a.x * b, a.y * b, a.z * b, a.w * b); }
__device__ __forceinline__ float hsum4(float4 a) { return (a.x + a.y) + (a.z + a.w); }
__device__ __forceinline__ float4 silu4(float4 a) { return f4(silu_(a.x), silu_(a.y), silu_(a.z), silu_(a.w)); }
__device__ __forceinline__ float4 dsilu4(float4 a) { return f4(dsilu_(a.x), dsilu_(a.y), dsilu_(a.z), dsilu_(a.w)); }
__device__ __forceinline__ float4 arr4(const float (&a)[4]) { return f4(a[0], a[1], a[2], a[3]); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// sum over the 4 lanes that share one attention head (lanes 4h..4h+3)
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    return v;
}

// ---------------------------------------------------------------------------------------------
// Warp-level fp32 GEMM micro-kernel.
//   acc[r][0..3] += sum_k A[r][k] * W[k][lane*4 + 0..3]      r < R, k < K
// A: shared memory, row-major, row stride LDA floats (16 B aligned rows), rows private to the warp
//    (every lane reads the same address -> broadcast, no bank conflicts).
// W: global memory, row-major [K][ldw]; the caller pre-offsets W to the first of the 128 columns this
//    call produces.  Lanes read consecutive float4 -> one coalesced 512 B request per k.
// ---------------------------------------------------------------------------------------------
template <int R>
__device__ __forceinline__ void warp_gemm_group(float (&acc)[R][4], const float* __restrict__ As, int lda, int k,
                                                const float4 (&w)[4]) {
#pragma unroll
    for (int r = 0; r < R; r++) {
        const float4 a = ld4(As + r * lda + k);
        acc[r][0] = fmaf(a.x, w[0].x, acc[r][0]); acc[r][1] = fmaf(a.x, w[0].y, acc[r][1]);
        acc[r][2] = fmaf(a.x, w[0].z, acc[r][2]); acc[r][3] = fmaf(a.x, w[0].w, acc[r][3]);
        acc[r][0] = fmaf(a.y, w[1].x, acc[r][0]); acc[r][1] = fmaf(a.y, w[1].y, acc[r][1]);
        acc[r][2] = fmaf(a.y, w[1].z, acc[r][2]); acc[r][3] = fmaf(a.y, w[1].w, acc[r][3]);
        acc[r][0] = fmaf(a.z, w[2].x, acc[r][0]); acc[r][1] = fmaf(a.z, w[2].y, acc[r][1]);
        acc[r][2] = fmaf(a.z, w[2].z, acc[r][2]); acc[r][3] = fmaf(a.z, w[2].w, acc[r][3]);
        acc[r][0] = fmaf(a.w, w[3].x, acc[r][0]); acc[r][1] = fmaf(a.w, w[3].y, acc[r][1]);
        acc[r][2] = fmaf(a.w, w[3].z, acc[r][2]); acc[r][3] = fmaf(a.w, w[3].w, acc[r][3]);
    }
}
__device__ __forceinline__ void warp_gemm_loadw(float4 (&w)[4], const float* __restrict__ Wp, int ldw, int k) {
    w[0] = ldg4(Wp + (size_t)(k + 0) * ldw);
    w[1] = ldg4(Wp + (size_t)(k + 1) * ldw);
    w[2] = ldg4(Wp + (size_t)(k + 2) * ldw);
    w[3] = ldg4(Wp + (size_t)(k + 3) * ldw);
}

// Software-pipelined: the weight rows of the next k-groups are in flight while the current group is
// multiplied (register ring of NBUF groups; NBUF = 4 for small R where the math does not cover L2 latency).
// krot (a multiple of 4, taken modulo K; K a power of two when it is non-zero): the k loop starts at row krot of this
// call's K range and wraps, so that CTAs walking the same weight chunk at the same time do not all ask the same L2 slices
// for the same rows (the caller derives it from its block index; the summation order then depends on the block).
template <int R, int K, int LDA, int NBUF = (R <= 4 ? 4 : 2)>
__device__ __forceinline__ void warp_gemm(float (&acc)[R][4], const float* __restrict__ As,
                                          const float* __restrict__ W, int ldw, int lane, int krot = 0) {
    static_assert(K % 16 == 0, "K must be a multiple of 16");
    const float* Wp = W + lane * 4;
    const auto kk = [&](int k) { return (k + krot) & (K - 1 | -(int)((K & (K - 1)) != 0)); };   // non-power-of-two K: krot must be 0
    if constexpr (NBUF == 4) {
        float4 w0[4], w1[4], w2[4], w3[4];
        warp_gemm_loadw(w0, Wp, ldw, kk(0));
        warp_gemm_loadw(w1, Wp, ldw, kk(4));
        warp_gemm_loadw(w2, Wp, ldw, kk(8));
#pragma unroll 1
        for (int k = 0; k < K; k += 16) {
            warp_gemm_loadw(w3, Wp, ldw, kk(k + 12));
            warp_gemm_group<R>(acc, As, LDA, kk(k), w0);
            if (k + 16 < K) warp_gemm_loadw(w0, Wp, ldw, kk(k + 16));
            warp_gemm_group<R>(acc, As, LDA, kk(k + 4), w1);
            if (k + 16 < K) warp_gemm_loadw(w1, Wp, ldw, kk(k + 20));
            warp_gemm_group<R>(acc, As, LDA, kk(k + 8), w2);
            if (k + 16 < K) warp_gemm_loadw(w2, Wp, ldw, kk(k + 24));
            warp_gemm_group<R>(acc, As, LDA, kk(k + 12), w3);
        }
    } else {
        float4 w0[4], w1[4];
        warp_gemm_loadw(w0, Wp, ldw, kk(0));
#pragma unroll 1
        for (int k = 0; k < K; k += 8) {
            warp_gemm_loadw(w1, Wp, ldw, kk(k + 4));
            warp_gemm_group<R>(acc, As, LDA, kk(k), w0);
            if (k + 8 < K) warp_gemm_loadw(w0, Wp, ldw, kk(k + 8));
            warp_gemm_group<R>(acc, As, LDA, kk(k + 4), w1);
        }
    }
}

// Two-phase variant for the CTA-cooperative node kernels: prefetch() issues the first NPRE groups of weight rows -- they
// do not depend on the A rows, so a warp that is idle while others finish the previous phase calls it BEFORE the barrier
// that publishes A and the ~0.9 us L2 round trip overlaps that phase; run() consumes group g and refills its registers with
// group g + NPRE.  K a power of two, K / 4 a multiple of NPRE; krot as in warp_gemm.
template <int K, int NPRE>
struct WarpGemmPre {
    static_assert((K & (K - 1)) == 0 && K % (4 * NPRE) == 0, "K: power of two and a multiple of the ring");
    float4 w[NPRE][4];
    const float* Wp;
    int ldw, krot;
    __device__ __forceinline__ int kk(int k) const { return (k + krot) & (K - 1); }
    __device__ __forceinline__ void prefetch(const float* __restrict__ W, int ldw_, int lane, int krot_) {
        Wp = W + lane * 4; ldw = ldw_; krot = krot_;
#pragma unroll
        for (int g = 0; g < NPRE; g++) warp_gemm_loadw(w[g], Wp, ldw, kk(4 * g));
    }
    template <int R, int LDA>
    __device__ __forceinline__ void run(float (&acc)[R][4], const float* __restrict__ As) {
#pragma unroll 1
        for (int k = 0; k < K; k += 4 * NPRE) {
#pragma unroll
            for (int g = 0; g < NPRE; g++) {
                warp_gemm_group<R>(acc, As, LDA, kk(k + 4 * g), w[g]);
                if (k + 4 * (g + NPRE) < K) warp_gemm_loadw(w[g], Wp, ldw, kk(k + 4 * (g + NPRE)));
            }
        }
    }
};

// Narrow variant: 64 output columns, 2 per lane (head blocks).  W row-major [K][ldw].
template <int R, int K, int LDA>
__device__ __forceinline__ void warp_gemm2(float (&acc)[R][2], const float* __restrict__ As,
                                           const float* __restrict__ W, int ldw, int lane) {
    const float* Wp = W + lane * 2;
#pragma unroll 4
    for (int k = 0; k < K; k += 4) {
        const float2 w0 = __ldg(reinterpret_cast<const float2*>(Wp + (size_t)(k + 0) * ldw));
        const float2 w1 = __ldg(reinterpret_cast<const float2*>(Wp + (size_t)(k + 1) * ldw));
        const float2 w2 = __ldg(reinterpret_cast<const float2*>(Wp + (size_t)(k + 2) * ldw));
        const float2 w3 = __ldg(reinterpret_cast<const float2*>(Wp + (size_t)(k + 3) * ldw));
#pragma unroll
        for (int r = 0; r < R; r++) {
            const float4 a = ld4(As + r * LDA + k);
            acc[r][0] = fmaf(a.x, w0.x, acc[r][0]); acc[r][1] = fmaf(a.x, w0.y, acc[r][1]);
            acc[r][0] = fmaf(a.y, w1.x, acc[r][0]); acc[r][1] = fmaf(a.y, w1.y, acc[r][1]);
            acc[r][0] = fmaf(a.z, w2.x, acc[r][0]); acc[r][1] = fmaf(a.z, w2.y, acc[r][1]);
            acc[r][0] = fmaf(a.w, w3.x, acc[r][0]); acc[r][1] = fmaf(a.w, w3.y, acc[r][1]);
        }
    }
}

template <int R>
__device__ __forceinline__ void acc_set_bias(float (&acc)[R][4], const float* __restrict__ b, int lane) {
    const float4 bb = ldg4(b + lane * 4);
#pragma unroll
    for (int r = 0; r < R; r++) { acc[r][0] = bb.x; acc[r][1] = bb.y; acc[r][2] = bb.z; acc[r][3] = bb.w; }
}
template <int R>
__device__ __forceinline__ void acc_zero(float (&acc)[R][4]) {
#pragma unroll
    for (int r = 0; r < R; r++) { acc[r][0] = 0.f; acc[r][1] = 0.f; acc[r][2] = 0.f; acc[r][3] = 0.f; }
}

// Programmatic dependent launch (engine.cu Launcher::launch, option "use_pdl"): wait until the previous kernel of the
// stream has completed and its writes are visible.  No kernel triggers its dependents early (an entry-time
// griddepcontrol.launch_dependents parked the next kernels' CTAs on the SMs and cost more than it hid), so with the
// attribute the next grid starts launching when the last CTA of this one exits, overlapping only the completion
// latency.  Nothing before this call may touch data produced by another kernel.  A no-op without the attribute.
__device__ __forceinline__ void pdl_entry() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

// cosine cutoff and its derivative (utils.py:16-19), cutoff passed in
__device__ __forceinline__ float cutoff_fn(float r, float rc) {
    return (r < rc) ? 0.5f * (cosf(r * (3.14159265358979323846f / rc)) + 1.0f) : 0.0f;
}
__device__ __forceinline__ float cutoff_dfn(float r, float rc) {
    const float w = 3.14159265358979323846f / rc;
    return (r < rc) ? -0.5f * w * sinf(r * w) : 0.0f;
}

}  // namespace vb
