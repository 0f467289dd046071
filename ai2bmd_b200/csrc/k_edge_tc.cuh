// Tensor-core (wgmma / TMA) version of the per-edge stage.
//
// Weight images: for every 128-column GEMM chunk and every K-slab of 32: a 16 KB "hi" plane then a 16 KB "lo"
// plane, each already in the K-major SWIZZLE_128B shared-memory layout (see tc_common.cuh), so one
// contiguous 32 KB bulk copy fills a ring stage.  Built by ai2bmd_b200/weights.py::tc_image().
#pragma once
#include "k_edge.cuh"
#include "tc_common.cuh"

namespace vb {

constexpr int TC_TE = 128;           // rows per tile (two wgmma M = 64 halves)
constexpr int TC_STAGES = 2;         // 32 KB stages in `ring`: with the fp32 A operand in shared memory, two fit
constexpr int TC_MAX_STAGES = 3;     // + one in the unused upper half of `abuf` when the tile capacity is <= 64 rows
constexpr int TC_SLABS = D / tc::SLAB_K;   // K-slabs (ring stages) per product
static_assert((TC_SLABS & (TC_SLABS - 1)) == 0, "tc_slab rotates the slab order with a mask: TC_SLABS must be a power of two");
constexpr int TC_MAXJOBS = 12;
constexpr int TC_LT = D + LDS_PAD;   // padded row length of the staging tile and of the A operand (132 floats)
typedef float TcRow[TC_LT];           // one padded row: a [rows][TC_LT] shared buffer is addressed through TcRow*

struct TcJob {
    const float* img;   // weight image of this 128x128 chunk (4 slabs x 32 KB)
    int accumulate;     // 0: the product overwrites the accumulator, 1: adds to it
};

struct TcShared {
    alignas(1024) uint8_t ring[TC_STAGES][tc::STAGE_BYTES];
    alignas(16) float tile[TC_TE][TC_LT];
    alignas(16) float abuf[TC_TE][TC_LT];   // A operand of the products in flight (fp32; split into tf32 hi / lo as it is loaded)
    EdgeMeta<TC_TE> meta;
    alignas(8) uint64_t b_full[TC_MAX_STAGES];
    uint64_t b_tile;                    // per-edge feature rows landed in `tile` (one arrival + byte count per compute warp)
    uint32_t released[TC_MAX_STAGES];   // warps done with the stage's current slab (counts on, mod TC2_CWARPS, never reset)
    const TcJob* jobs;                  // the ring's slab sequence: `ntiles` passes over `njobs` jobs of TC_SLABS slabs
    int njobs, nslabs;
    alignas(16) float eacc[TC_TE][4];   // per-edge adjoint scalars of the current tile: dE/dC, dE/dd[3]
    float gattn[TC_TE][H];              // adjoint kernel: dE/da_h per edge
};

// the ring must start on a 1024 B boundary of the shared window (swizzle atom): align the dynamic block by hand
__device__ __forceinline__ TcShared* tc_shared_base(uint8_t* raw) {
    const uint32_t s = tc::smem_u32(raw);
    return reinterpret_cast<TcShared*>(raw + (((s + 1023u) & ~1023u) - s));
}
constexpr size_t TC_SMEM_BYTES = sizeof(TcShared) + 1024;
static_assert(TC_SMEM_BYTES <= 227 * 1024, "tensor-core kernels must fit the 227 KB of shared memory of an H100 block");

// ring stages for a tile capacity of `rows`.  A capacity of <= 64 rows never touches rows 64.. of `tile` and `abuf`, so a
// third stage lives in abuf[64..127] (33 KB, on a 1024 B boundary of the block).
__host__ __device__ constexpr int tc_nstages(int rows) { return rows <= 64 ? 3 : 2; }
constexpr size_t TC_STAGE2_OFF = offsetof(TcShared, abuf) + sizeof(float) * 64 * TC_LT;
static_assert(TC_STAGE2_OFF % 1024 == 0 && sizeof(float) * (TC_TE - 64) * TC_LT >= tc::STAGE_BYTES,
              "the third ring stage must fit the upper half of abuf on a swizzle-atom boundary");
__device__ __forceinline__ uint8_t* tc_stage_ptr(TcShared& sh, int stage) {
    return stage < TC_STAGES ? sh.ring[stage] : reinterpret_cast<uint8_t*>(&sh.abuf[64][0]);
}

// K-slab of a product that the CTA streams in position s (0 .. TC_SLABS-1): every CTA starts at a different slab, so
// the CTAs of a wave do not all ask the same L2 lines for the same 32 KB at once
__device__ __forceinline__ int tc_slab(int s) { return (s + (int)blockIdx.x) & (TC_SLABS - 1); }

// refill: slab k of the sequence -> ring stage k % NS (one thread; the stage's previous slab is released)
template <int NS>
__device__ __forceinline__ void tc_issue(TcShared& sh, int k) {
    if (k >= sh.nslabs) return;
    const int stage = k % NS, job = (k / TC_SLABS) % sh.njobs, s = tc_slab(k % TC_SLABS);
    const char* src = reinterpret_cast<const char*>(sh.jobs[job].img) + (size_t)s * tc::STAGE_BYTES;
    tc::mbar_arrive_expect_tx(&sh.b_full[stage], tc::STAGE_BYTES);
    tc::tma_load_1d(tc_stage_ptr(sh, stage), src, tc::STAGE_BYTES, &sh.b_full[stage]);
}

}  // namespace vb


// =====================================================================================================
// Tensor-core edge stage, hybrid layout.
//   * 16 compute warps keep the coalesced "lane owns 4 channels" layout of k_edge.cuh for every global
//     gather / scatter / elementwise step (one 512 B request per node row per warp);
//   * the five 128x128x128 contractions per tile run on wgmma: every warpgroup multiplies one part of the product (A
//     fragments split into 3xTF32 hi / lo in registers from a padded shared buffer, B = the weight ring): each
//     warpgroup computes a 64 x 64 quarter (rows x columns halves), and a warpgroup whose 64 product rows are all past
//     the tile's edges skips its MMAs;
//   * buffers: a tile of 96 / 128 rows has two, the staging tile and the A operand (`tc2_tile_to_a` copies an operand
//     that a phase wrote into the tile); a tile of <= 64 rows has three, `tile`, `abuf` and `tc_aux` (rows 64.. of
//     `tile`), so every operand is read where it was written, a phase that produces two row sets writes both at once,
//     and nothing is copied or gathered twice;
//   * the forward of a tile of <= 64 rows is warp-specialised: warpgroups 0 and 2 run the products, 1 and 3 the
//     gathers and SIMT phases (see tc2_is_mma_warp);
//   * there is no producer warp: the ring is refilled by whichever compute warp releases a stage last (tc2_release),
//     so the CTA is 512 threads with 128 registers each;
//   * a tile holds ROWS = 32 / 64 / 96 / 128 edges (template parameter): compute warp w owns rows
//     [w*ROWS/16, (w+1)*ROWS/16) in the coalesced phases.
// =====================================================================================================
namespace vb {

constexpr int TC2_CWARPS = 16;                      // compute warps
constexpr int TC2_CTHREADS = TC2_CWARPS * 32;       // 512
constexpr int TC2_THREADS = TC2_CTHREADS;           // the whole CTA computes (and refills the weight ring)
constexpr int TC2_NGRP = TC2_CTHREADS / D;          // channel groups in the per-target aggregation phases

struct EdgeTcArgs {
    int layer;
    ModelW mw;
    Workspace ws;
    TcJob jobs[TC_MAXJOBS];
    int njobs;
    int tile_rows;              // edges per tile, <= the kernel's ROWS
    unsigned long long* tl;     // optional timeline (SM clock stamps of CTA 0, first tile); nullptr = off
};
constexpr int TC_TL_SLOTS = 64;  // [0,32): compute thread 0 phase stamps, [32,64): thread 128 (a gather warp of a warp-specialised tile)
#define TC_TL(k) do { if (a.tl != nullptr && blockIdx.x == 0 && it == 0 && threadIdx.x == 0) a.tl[k] = (unsigned long long)clock64(); } while (0)

__device__ __forceinline__ void csync() { asm volatile("bar.sync 1, %0;" ::"n"(TC2_CTHREADS) : "memory"); }

// Warp-specialised tiles of <= 64 rows.  Such a tile has product rows for warpgroups 0 and 2 only (tc2_mma: rows
// 64 * (q & 1)), so those two warpgroups (the MMA warps) run the tile's products back to back and the other two (the
// gather warps, 256 threads) run the SIMT phases: each phase issues its loads and computes what needs no product
// result before it waits for the product.  A hand-off between the roles is a named barrier of all 512 threads: the
// producing role arrives (bar.arrive, no wait), the consuming role waits (bar.sync).  Every id is used once per tile,
// and the tile ends with a CTA barrier, so an arrival can never complete a later phase of the same id.
constexpr int TC2_WS_THREADS = TC2_CTHREADS / 2;    // threads per role
__device__ __forceinline__ bool tc2_is_mma_warp(int warp) { return ((warp >> 2) & 1) == 0; }
// named barrier ids: 0 = __syncthreads, 1 = csync, 2 = the gather warps among themselves, 3..15 = a kernel's hand-offs
__device__ __forceinline__ void gather_sync() { asm volatile("bar.sync 2, %0;" ::"n"(TC2_WS_THREADS) : "memory"); }
__device__ __forceinline__ void handoff_arrive(int id) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "n"(TC2_CTHREADS) : "memory"); }
__device__ __forceinline__ void handoff_wait(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(TC2_CTHREADS) : "memory"); }

// position of a thread in the ring's slab sequence (every thread walks the same sequence), for a tile capacity of ROWS
template <int ROWS>
struct TcRing {
    static constexpr int NS = tc_nstages(ROWS);     // ring stages
    int next = 0;                                   // sequence index of the next slab to consume
};

// barriers, the ring's slab sequence (`ntiles` passes over `njobs` jobs) and its first NS slabs.  `jobs` may be shared
// memory written before this call (the barrier here publishes it).
template <int ROWS>
__device__ __forceinline__ void tc2_setup(TcShared& sh, const TcRing<ROWS>&, const TcJob* jobs, int njobs, int ntiles) {
    constexpr int NS = TcRing<ROWS>::NS;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NS; s++) { tc::mbar_init(&sh.b_full[s], 1); sh.released[s] = 0; }
        tc::mbar_init(&sh.b_tile, TC2_CWARPS);
        sh.jobs = jobs; sh.njobs = njobs; sh.nslabs = ntiles * njobs * TC_SLABS;
        tc::fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 0; k < NS; k++) tc_issue<NS>(sh, k);
}

// a warp is done with slab k (every MMA that read it has retired): the warp that releases it last refills the stage
// with slab k + NS.  No warp waits for a refill, so none can wait on one that only it would issue.  NW: the warps that
// walk the ring (all 16, or the 8 MMA warps of a warp-specialised tile)
template <int NS, int NW>
__device__ __forceinline__ void tc2_release(TcShared& sh, int k, int lane) {
    __syncwarp();
    if (lane == 0) {
        const uint32_t before = tc::atom_add_acq_rel(&sh.released[k % NS], 1u);
        if (before % NW == NW - 1) tc_issue<NS>(sh, k + NS);
    }
}

// staging tile -> A operand (rows below `rows`), after every compute warp is done with the previous A operand and
// has finished writing the tile
__device__ __forceinline__ void tc2_tile_to_a(TcShared& sh, int rows) {
    csync();
    for (int idx = threadIdx.x; idx < rows * (D / 4); idx += TC2_CTHREADS) {
        const int r = idx >> 5, c = (idx & 31) * 4;
        st4(&sh.abuf[r][c], ld4(&sh.tile[r][c]));
    }
}

// rows 64..127 of the staging tile, a third [64][TC_LT] buffer when the tile capacity is <= 64 rows (such a tile never
// touches them): products read their A operand and leave their results wherever the next phase wants them, so the
// small-tile kernels copy nothing between `tile` and `abuf`
__device__ __forceinline__ TcRow* tc_aux(TcShared& sh) { return sh.tile + 64; }

// acc (+)= A * W^T for the next job of the ring (all warps), A = a padded [rows][TC_LT] shared buffer: `abuf`, `tile`
// or, for a tile capacity of <= 64 rows, `tc_aux(sh)`.  Warpgroup q = warp / 4 computes rows 64 * (q & 1) .. +63
// and columns 64 * (q >> 1) .. +63 of the 128 x 128 product; each K-step is three tf32 MMAs, lo * hi + hi * lo + hi * hi
// (~ fp32 accuracy).  A warpgroup whose rows all lie at or past `nvalid` only releases the ring stages (so a tile
// capacity of <= 64 rows never reads rows 64.. of its A buffer: the third ring stage, or `tc_aux`).  Per K-slab the A
// fragments are split into tf32 hi / lo as they are loaded (before the slab's weights are waited for), one commit group
// of 12 MMAs runs, and the stage is released as soon as that group retires: a product streams 128 KB of weights through
// the ring, and an early release is worth more than MMAs kept in flight across slabs.  On return `acc` holds this
// thread's part of the product (layout: tc_common.cuh).  WS: a warp-specialised tile, where only the MMA warps call this
// (after a hand-off that publishes A) and they alone release the ring stages.
template <int ROWS, bool WS = false>
__device__ __forceinline__ void tc2_mma(TcShared& sh, TcRing<ROWS>& ring, const TcRow* A, float (&acc)[32], int accumulate,
                                        int warp, int lane, int nvalid) {
    constexpr int NS = TcRing<ROWS>::NS;
    static_assert(!WS || ROWS <= 64, "only tiles of <= 64 rows leave two warpgroups without product rows");
    if constexpr (!WS) csync();                                // the A operand is complete
    const int q = warp >> 2, m0 = (q & 1) * 64 + (warp & 3) * 16, g = lane >> 2, t = lane & 3;
    const bool active = WS || (q & 1) * 64 < nvalid;           // warpgroup-uniform
    if (!accumulate) {
#pragma unroll
        for (int i = 0; i < 32; i++) acc[i] = 0.f;
    }
#pragma unroll 1
    for (int s = 0; s < TC_SLABS; s++) {
        const int k = ring.next + s, stage = k % NS;
        if (active) {
            uint32_t ahi[4][4], alo[4][4];
            const int k0 = tc_slab(s) * tc::SLAB_K + t;
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                const int kc = k0 + kk * 8;
                tc::split_tf32(A[m0 + g][kc], ahi[kk][0], alo[kk][0]);
                tc::split_tf32(A[m0 + g + 8][kc], ahi[kk][1], alo[kk][1]);
                tc::split_tf32(A[m0 + g][kc + 4], ahi[kk][2], alo[kk][2]);
                tc::split_tf32(A[m0 + g + 8][kc + 4], ahi[kk][3], alo[kk][3]);
            }
            tc::mbar_wait(&sh.b_full[stage], (uint32_t)(k / NS) & 1u);
            const uint32_t bhi = tc::smem_u32(tc_stage_ptr(sh, stage)) + (uint32_t)(q >> 1) * (64 * 128);
            const uint32_t blo = bhi + tc::SLAB_BYTES;
            tc::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                const uint64_t dhi = tc::smem_desc_sw128(bhi + kk * 32);
                const uint64_t dlo = tc::smem_desc_sw128(blo + kk * 32);
                tc::mma_m64n64k8_tf32(acc, alo[kk], dhi);
                tc::mma_m64n64k8_tf32(acc, ahi[kk], dlo);
                tc::mma_m64n64k8_tf32(acc, ahi[kk], dhi);
            }
            tc::wgmma_commit();
            tc::wgmma_wait_all();
#pragma unroll
            for (int kk = 0; kk < 4; kk++)
#pragma unroll
                for (int i = 0; i < 4; i++) { tc::reg_fence(ahi[kk][i]); tc::reg_fence(alo[kk][i]); }
#pragma unroll
            for (int i = 0; i < 32; i++) tc::reg_fence(acc[i]);
        } else {
            tc::mbar_wait(&sh.b_full[stage], (uint32_t)(k / NS) & 1u);
        }
        tc2_release<NS, WS ? TC2_CWARPS / 2 : TC2_CWARPS>(sh, k, lane);
    }
    ring.next += TC_SLABS;
}

// accumulator -> a padded [rows][TC_LT] shared buffer (rows below `nvalid`)
__device__ __forceinline__ void tc2_acc_to(TcRow* dst, const float (&acc)[32], int warp, int lane, int nvalid) {
    const int q = warp >> 2, r = (q & 1) * 64 + (warp & 3) * 16 + (lane >> 2), c = (q >> 1) * 64 + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        if (r < nvalid) *reinterpret_cast<float2*>(&dst[r][c + 8 * i]) = make_float2(acc[4 * i], acc[4 * i + 1]);
        if (r + 8 < nvalid) *reinterpret_cast<float2*>(&dst[r + 8][c + 8 * i]) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
}

// ---------------------------------------------------------------------------------------------
// Self-test: Dout[ROWS][128] = A[ROWS][128] * W^T with W given as a tc image (validates descriptors,
// swizzle, fragment layouts, the ring and its barriers before the edge kernels use them).  ROWS <= 64 runs the
// three-stage ring of the small-tile edge kernels.
// ---------------------------------------------------------------------------------------------
template <int ROWS>
__global__ void __launch_bounds__(TC2_THREADS, 1) tc_selftest_kernel(const float* __restrict__ A, const float* __restrict__ img,
                                                                     float* __restrict__ Dout, int reps) {
    extern __shared__ __align__(1024) uint8_t dyn_raw[];
    TcShared& sh = *tc_shared_base(dyn_raw);
    __shared__ TcJob jobs[1];
    if (threadIdx.x == 0) jobs[0] = TcJob{img, 0};
    TcRing<ROWS> ring;
    tc2_setup(sh, ring, jobs, 1, reps);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc[32];
    for (int t = 0; t < reps; t++) {
        for (int idx = threadIdx.x; idx < ROWS * (D / 4); idx += TC2_CTHREADS) {
            const int r = idx >> 5, c = (idx & 31) * 4;
            st4(&sh.tile[r][c], ld4(A + (size_t)r * D + c));
        }
        tc2_tile_to_a(sh, ROWS);
        tc2_mma(sh, ring, sh.abuf, acc, 0, warp, lane, ROWS);
        csync();
        tc2_acc_to(sh.tile, acc, warp, lane, ROWS);
        csync();
        for (int idx = threadIdx.x; idx < ROWS * (D / 4); idx += TC2_CTHREADS) {
            const int r = idx >> 5, c = (idx & 31) * 4;
            st4(Dout + (size_t)r * D + c, ld4(&sh.tile[r][c]));
        }
        csync();
    }
}

// ---------------------------------------------------------------------------------------------
// forward (math and reference lines: see edge_fwd_kernel in k_edge.cuh)
// job order: dk, dv, [f], s1, s2
// ---------------------------------------------------------------------------------------------
// Per-target sums of the forward over a tile's targets.  Thread (channel c, group grp of ngrp) sums targets
// i_first + grp, + ngrp, ..; a target whose edges all lie in the tile is stored, a target cut by a tile boundary is added
// atomically.
// xa_i = sum_e m_e
__device__ __forceinline__ void tc_fwd_xa(const TcShared& sh, const Workspace& ws, const TcRow* mb, int e0, int nvalid,
                                          int c, int grp, int ngrp) {
    const int i_first = sh.meta.dst[0], i_last = sh.meta.dst[nvalid - 1];
    for (int i = i_first + grp; i <= i_last; i += ngrp) {
        const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
        const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
        float xa = 0.f;
        for (int r = lo; r < hi; r++) xa += mb[r][c];
        if (q0 >= e0 && q1 <= e0 + nvalid) ws.XA[(size_t)i * D + c] = xa;
        else atomicAdd(ws.XA + (size_t)i * D + c, xa);
    }
}
// s1 (D1): va_i = sum_e vn_j * silu(s1 + bs); the sums of cut targets (at most two per thread) stay in `bnd` for tc_fwd_s2
__device__ __forceinline__ void tc_fwd_s1(const TcShared& sh, const Workspace& ws, const LayerW& lw, const float* __restrict__ VN,
                                          float* __restrict__ SP, const TcRow* s1b, int e0, int nvalid, int c, int grp, int ngrp,
                                          float (&bnd)[2][3]) {
    const float b = __ldg(lw.bs + c);
    const int i_first = sh.meta.dst[0], i_last = sh.meta.dst[nvalid - 1];
    int nb = 0;
    for (int i = i_first + grp; i <= i_last; i += ngrp) {
        const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
        const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
        float v0 = 0.f, v1 = 0.f, v2 = 0.f;
        int r = lo;
        for (; r + 4 <= hi; r += 4) {              // 12 independent gathers in flight
            float g[4][3], s1[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const size_t j3 = (size_t)sh.meta.src[r + u] * 3;
                g[u][0] = __ldg(VN + (j3 + 0) * D + c); g[u][1] = __ldg(VN + (j3 + 1) * D + c); g[u][2] = __ldg(VN + (j3 + 2) * D + c);
                const float sp = s1b[r + u][c] + b;
                SP[(size_t)(e0 + r + u) * 2 * D + c] = sp;
                s1[u] = silu_(sp);
            }
#pragma unroll
            for (int u = 0; u < 4; u++) { v0 += g[u][0] * s1[u]; v1 += g[u][1] * s1[u]; v2 += g[u][2] * s1[u]; }
        }
        for (; r < hi; r++) {
            const size_t j3 = (size_t)sh.meta.src[r] * 3;
            const float sp = s1b[r][c] + b;
            SP[(size_t)(e0 + r) * 2 * D + c] = sp;
            const float s1 = silu_(sp);
            v0 += __ldg(VN + (j3 + 0) * D + c) * s1;
            v1 += __ldg(VN + (j3 + 1) * D + c) * s1;
            v2 += __ldg(VN + (j3 + 2) * D + c) * s1;
        }
        if (q0 >= e0 && q1 <= e0 + nvalid) {
            ws.VA[((size_t)i * 3 + 0) * D + c] = v0;
            ws.VA[((size_t)i * 3 + 1) * D + c] = v1;
            ws.VA[((size_t)i * 3 + 2) * D + c] = v2;
        } else if (nb < 2) {
            bnd[nb][0] = v0; bnd[nb][1] = v1; bnd[nb][2] = v2;
            nb++;
        }
    }
}
// s2 (D0): va_i += sum_e silu(s2 + bs) * d (the same threads and targets as tc_fwd_s1)
__device__ __forceinline__ void tc_fwd_s2(const TcShared& sh, const Workspace& ws, const LayerW& lw, float* __restrict__ SP,
                                          const TcRow* s2b, int e0, int nvalid, int c, int grp, int ngrp, const float (&bnd)[2][3]) {
    const float b = __ldg(lw.bs + D + c);
    const int i_first = sh.meta.dst[0], i_last = sh.meta.dst[nvalid - 1];
    int nb = 0;
    for (int i = i_first + grp; i <= i_last; i += ngrp) {
        const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
        const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
        float v0 = 0.f, v1 = 0.f, v2 = 0.f;
        for (int r = lo; r < hi; r++) {
            const float4 de = sh.meta.d[r];
            const float sp = s2b[r][c] + b;
            SP[(size_t)(e0 + r) * 2 * D + D + c] = sp;
            const float s2 = silu_(sp);
            v0 += s2 * de.x; v1 += s2 * de.y; v2 += s2 * de.z;
        }
        if (q0 >= e0 && q1 <= e0 + nvalid) {
            ws.VA[((size_t)i * 3 + 0) * D + c] += v0;
            ws.VA[((size_t)i * 3 + 1) * D + c] += v1;
            ws.VA[((size_t)i * 3 + 2) * D + c] += v2;
        } else if (nb < 2) {
            atomicAdd(ws.VA + ((size_t)i * 3 + 0) * D + c, bnd[nb][0] + v0);
            atomicAdd(ws.VA + ((size_t)i * 3 + 1) * D + c, bnd[nb][1] + v1);
            atomicAdd(ws.VA + ((size_t)i * 3 + 2) * D + c, bnd[nb][2] + v2);
            nb++;
        }
    }
}

// gather-warp stamps of the timeline (thread 128 = lane 0 of warp 4, the first gather warp): slots [32, 64)
#define TC_TLG(k) do { if (a.tl != nullptr && blockIdx.x == 0 && it == 0 && threadIdx.x == 128) a.tl[32 + (k)] = (unsigned long long)clock64(); } while (0)

template <int ROWS>
__global__ void __launch_bounds__(TC2_THREADS, 1) edge_fwd_tc_kernel(const __grid_constant__ EdgeTcArgs a) {
    pdl_entry();
    extern __shared__ __align__(1024) uint8_t dyn_raw[];
    TcShared& sh = *tc_shared_base(dyn_raw);
    const Workspace& ws = a.ws;
    const int l = a.layer;
    const LayerW& lw = a.mw.layer[l];
    const bool upd = (l < L - 1);
    const int J_DK = 0, J_DV = 1, J_F = 2, J_S1 = upd ? 3 : 2, J_S2 = upd ? 4 : 3;
    constexpr int RPW = ROWS / TC2_CWARPS;      // rows per compute warp in the coalesced phases
    constexpr bool SMALL = ROWS <= 64;          // warp-specialised schedule, three buffers: see below
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, col = lane * 4;
    const int E = ws.rowptr[ws.N];
    const int trows = min(ROWS, max(16, a.tile_rows));          // edges per tile (<= ROWS, chosen on the host so the tiles fill whole waves)
    const int ntiles_total = (E + trows - 1) / trows;
    const int my_tiles = ((int)blockIdx.x < ntiles_total) ? (ntiles_total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    if (a.tl != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.tl[0] = (unsigned long long)clock64();
    TcRing<ROWS> ring;
    tc2_setup(sh, ring, a.jobs, a.njobs, my_tiles);
    if (a.tl != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.tl[1] = (unsigned long long)clock64();

    float acc[32];
    const float* __restrict__ Fin = ws.F[l];
    float* __restrict__ Fout = upd ? ws.F[l + 1] : nullptr;
    const float* __restrict__ QKV = ws.QKV[l];
    const float* __restrict__ VN = ws.VN[l];
    const float* __restrict__ TU = ws.TU[l];
    float* __restrict__ P1 = ws.P1[l];
    float* __restrict__ SP = ws.SP[l];
    float* __restrict__ ATT = ws.ATT[l];
    for (int it = 0; it < my_tiles; it++) {
        const uint32_t tpar = (uint32_t)(it & 1);
        const int e0 = ((int)blockIdx.x + it * (int)gridDim.x) * trows;
        const int nvalid = min(trows, E - e0);
        // ---- per-edge feature rows -> the A operand buffer by TMA bulk copies (one 512 B row each, padded rows in
        //      shared memory), completion on an mbarrier: f is the A operand of the dk, dv and f products ----
        {
            constexpr int RW = ROWS / TC2_CWARPS;                 // rows a warp issues
            const int w0 = warp * RW, wn = max(0, min(RW, nvalid - w0));
            if (lane == 0) {
                if (wn > 0) tc::mbar_arrive_expect_tx(&sh.b_tile, (uint32_t)wn * D * 4);
                else tc::mbar_arrive(&sh.b_tile);
            }
            __syncwarp();
            if (lane < wn) tc::tma_load_1d(&sh.abuf[w0 + lane][0], Fin + (size_t)(e0 + w0 + lane) * D, D * 4, &sh.b_tile);
        }
        load_edge_meta<TC_TE, TC2_CTHREADS>(sh.meta, ws, e0, nvalid);
        if constexpr (SMALL) {
            // ---- warp-specialised tile.  Buffers: abuf = the f rows (A of dk, dv, f), then s1; tile = dk, then f, then
            //      s2; tc_aux = q_i * k_j, then dv, turned into m in place (A of s1 and s2).  The MMA warps run dk, dv
            //      and f back to back and s1, s2 as soon as m is complete; a result is stored once the phase that read
            //      the buffer before it is done.  The edge update reads f from global memory (the rows the TMA just
            //      brought into L2), so abuf is free for s1 once the f product has retired. ----
            enum : int { H_DK = 3, H_ATT, H_DV, H_F, H_M, H_EU };     // hand-offs (named barrier ids)
            TcRow* const xb = tc_aux(sh);
            csync();                                                  // meta
            if (tc2_is_mma_warp(warp)) {
                tc::mbar_wait(&sh.b_tile, tpar);
                TC_TL(2);
                tc2_mma<ROWS, true>(sh, ring, sh.abuf, acc, a.jobs[J_DK].accumulate, warp, lane, nvalid);
                tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
                handoff_arrive(H_DK);
                TC_TL(4);
                tc2_mma<ROWS, true>(sh, ring, sh.abuf, acc, a.jobs[J_DV].accumulate, warp, lane, nvalid);
                TC_TL(7);
                handoff_wait(H_ATT);                                  // the attention phase is done with dk and q_i * k_j
                tc2_acc_to(xb, acc, warp, lane, nvalid);
                handoff_arrive(H_DV);
                TC_TL(8);
                if (upd) {
                    tc2_mma<ROWS, true>(sh, ring, sh.abuf, acc, a.jobs[J_F].accumulate, warp, lane, nvalid);
                    tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
                    handoff_arrive(H_F);
                    TC_TL(11);
                }
                handoff_wait(H_M);                                    // m complete (and every MMA warp is past the f rows)
                TC_TL(3);
                tc2_mma<ROWS, true>(sh, ring, xb, acc, a.jobs[J_S1].accumulate, warp, lane, nvalid);
                tc2_acc_to(sh.abuf, acc, warp, lane, nvalid);
                TC_TL(13);
                if (threadIdx.x == 0 && it + 1 < my_tiles) {         // next tile's feature rows -> L2 (bulk prefetch), shortly before use
                    const int en = ((int)blockIdx.x + (it + 1) * (int)gridDim.x) * trows;
                    tc::tma_prefetch_l2(Fin + (size_t)en * D, (uint32_t)min(trows, E - en) * D * 4);
                }
                tc2_mma<ROWS, true>(sh, ring, xb, acc, a.jobs[J_S2].accumulate, warp, lane, nvalid);
                TC_TL(16);
                if (upd) handoff_wait(H_EU);                          // the edge update is done with the tile
                tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
                TC_TL(17);
            } else {
                // gather warps: gw = 0..7 owns rows [gw * grpw, (gw + 1) * grpw), grpw = ceil(nvalid / 8)
                constexpr int GRPW = ROWS / (TC2_CWARPS / 2);
                const int gw = (warp >> 3) * 4 + (warp & 3), gt = gw * 32 + lane;
                const int grpw = (nvalid + 7) / 8, g0 = gw * grpw;
                const int gch = gt & (D - 1), ggrp = gt >> 7;          // per-target sums: channel, target parity
                // ---- attention weights: q_i * k_j (-> tc_aux) before dk lands ----
#pragma unroll 4
                for (int r = 0; r < GRPW; r++) {
                    if (r >= grpw) break;
                    const int row = g0 + r;
                    st4(&xb[row][col], ldg4(QKV + (size_t)sh.meta.dst[row] * 3 * D + col) * ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + D + col));
                }
                TC_TLG(0);
                float Areg[GRPW];
                {
                    const float4 bb = ldg4(lw.b1 + col);
                    handoff_wait(H_DK);
                    TC_TLG(1);
#pragma unroll
                    for (int r = 0; r < GRPW; r++) {
                        if (r >= grpw) break;
                        const int row = g0 + r;
                        const float4 P = ld4(&sh.tile[row][col]) + bb;
                        const float av = quad_sum(hsum4(ld4(&xb[row][col]) * silu4(P)));
                        Areg[r] = silu_(av) * sh.meta.C[row];
                        if (row < nvalid) {
                            st4(P1 + (size_t)(e0 + row) * 3 * D + col, P);
                            if ((lane & 3) == 0) ATT[(size_t)(e0 + row) * H + (lane >> 2)] = av;
                        }
                    }
                    handoff_arrive(H_ATT);
                }
                TC_TLG(2);
                // ---- message m = v_j * silu(dv) * A (in place in tc_aux): v_j before dv lands ----
                {
                    float4 vj[GRPW];
#pragma unroll
                    for (int r = 0; r < GRPW; r++) {
                        if (r >= grpw) break;
                        vj[r] = ldg4(QKV + (size_t)sh.meta.src[g0 + r] * 3 * D + 2 * D + col);
                    }
                    const float4 bb = ldg4(lw.b1 + D + col);
                    handoff_wait(H_DV);
                    TC_TLG(3);
#pragma unroll
                    for (int r = 0; r < GRPW; r++) {
                        if (r >= grpw) break;
                        const int row = g0 + r;
                        const float4 P = ld4(&xb[row][col]) + bb;
                        st4(&xb[row][col], vj[r] * silu4(P) * Areg[r]);
                        if (row < nvalid) st4(P1 + (size_t)(e0 + row) * 3 * D + D + col, P);
                    }
                }
                gather_sync();
                handoff_arrive(H_M);
                TC_TLG(4);
                tc_fwd_xa(sh, ws, xb, e0, nvalid, gch, ggrp, 2);
                TC_TLG(5);
                // ---- edge update f' = f + silu(Pf) * wdot (f from global memory: abuf is s1's by now) ----
                if (upd) {
                    const float4 bb = ldg4(lw.b1 + 2 * D + col);
                    handoff_wait(H_F);
                    TC_TLG(6);
#pragma unroll 1
                    for (int rb = 0; rb < GRPW; rb += 2) {             // gathers of 2 rows in flight before the first global store
                        if (rb >= grpw) break;
                        float4 tir[2][3], ujr[2][3], fin[2];
#pragma unroll
                        for (int u = 0; u < 2; u++) {
                            const int row = g0 + rb + u;
                            const size_t i3 = (size_t)sh.meta.dst[row] * 3, j3 = (size_t)sh.meta.src[row] * 3;
                            fin[u] = (rb + u < grpw && row < nvalid) ? ldg4(Fin + (size_t)(e0 + row) * D + col) : f4s(0.f);
#pragma unroll
                            for (int s = 0; s < 3; s++) {
                                tir[u][s] = ldg4(TU + (i3 + s) * 2 * D + col);
                                ujr[u][s] = ldg4(TU + (j3 + s) * 2 * D + D + col);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < 2; u++) {
                            const int row = g0 + rb + u;
                            const float4 dd = sh.meta.d[row];
                            const float4 Pf = ld4(&sh.tile[row][col]) + bb;
                            const float4 fp = silu4(Pf);
                            const float4 a1 = tir[u][0] * dd.x + tir[u][1] * dd.y + tir[u][2] * dd.z;
                            const float4 a2 = ujr[u][0] * dd.x + ujr[u][1] * dd.y + ujr[u][2] * dd.z;
                            const float4 wdot = (tir[u][0] - a1 * dd.x) * (ujr[u][0] - a2 * dd.x) + (tir[u][1] - a1 * dd.y) * (ujr[u][1] - a2 * dd.y) +
                                                (tir[u][2] - a1 * dd.z) * (ujr[u][2] - a2 * dd.z);
                            if (rb + u < grpw && row < nvalid) {
                                st4(P1 + (size_t)(e0 + row) * 3 * D + 2 * D + col, Pf);
                                st4(Fout + (size_t)(e0 + row) * D + col, fin[u] + fp * wdot);
                            }
                        }
                    }
                    handoff_arrive(H_EU);
                }
                TC_TLG(7);
            }
            // ---- s1 (abuf), s2 (tile): va_i, by the whole CTA (the MMA warps have no product left) ----
            csync();
            TC_TL(18);
            const int cch = threadIdx.x & (D - 1), grp = threadIdx.x >> 7;
            float bnd[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
            tc_fwd_s1(sh, ws, lw, VN, SP, sh.abuf, e0, nvalid, cch, grp, TC2_NGRP, bnd);
            TC_TL(19);
            tc_fwd_s2(sh, ws, lw, SP, sh.tile, e0, nvalid, cch, grp, TC2_NGRP, bnd);
            TC_TL(20);
        } else {
            const int cch = threadIdx.x & (D - 1), grp = threadIdx.x >> 7;      // per-target sums: channel, target parity
            // rows are dealt to the compute warps in contiguous runs of rpw = ceil(nvalid / 16): a tile shorter than ROWS
            // keeps every warp busy (slot s of a warp is row warp * rpw + s, valid while s < rpw and the row exists)
            const int rpw = (nvalid + TC2_CWARPS - 1) / TC2_CWARPS, r0 = warp * rpw;
            tc::mbar_wait(&sh.b_tile, tpar);
            csync();
            TC_TL(2);
            // ---- dk -> attention weights ----
            float Areg[RPW];
            tc2_mma(sh, ring, sh.abuf, acc, a.jobs[J_DK].accumulate, warp, lane, nvalid);
            TC_TL(4);
            tc2_acc_to(sh.tile, acc, warp, lane, nvalid);         // (nothing reads the tile between the MMAs' barrier and here)
            csync();
            {
                TC_TL(5);
                const float4 bb = ldg4(lw.b1 + col);
#pragma unroll
                for (int r = 0; r < RPW; r++) {
                    if (r >= rpw) break;
                    const int row = r0 + r;
                    const float4 qi = ldg4(QKV + (size_t)sh.meta.dst[row] * 3 * D + col);
                    const float4 kj = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + D + col);
                    const float4 P = ld4(&sh.tile[row][col]) + bb;
                    const float av = quad_sum(hsum4(qi * kj * silu4(P)));
                    Areg[r] = silu_(av) * sh.meta.C[row];
                    if ((r < rpw && row < nvalid)) {
                        st4(P1 + (size_t)(e0 + row) * 3 * D + col, P);
                        if ((lane & 3) == 0) ATT[(size_t)(e0 + row) * H + (lane >> 2)] = av;
                    }
                }
            }
            TC_TL(6);
            // ---- dv -> message m (in place in the tile) ----
            tc2_mma(sh, ring, sh.abuf, acc, a.jobs[J_DV].accumulate, warp, lane, nvalid);
            TC_TL(7);
            csync();
            tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
            csync();
            {
                TC_TL(8);
                const float4 bb = ldg4(lw.b1 + D + col);
#pragma unroll
                for (int r = 0; r < RPW; r++) {
                    if (r >= rpw) break;
                    const int row = r0 + r;
                    const float4 vj = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + 2 * D + col);
                    const float4 P = ld4(&sh.tile[row][col]) + bb;
                    st4(&sh.tile[row][col], vj * silu4(P) * Areg[r]);
                    if ((r < rpw && row < nvalid)) st4(P1 + (size_t)(e0 + row) * 3 * D + D + col, P);
                }
            }
            csync();
            TC_TL(9);
            tc_fwd_xa(sh, ws, sh.tile, e0, nvalid, cch, grp, TC2_NGRP);
            TC_TL(10);
            // ---- f product; A = m for s1 and s2: m is copied into abuf ----
            if (upd) tc2_mma(sh, ring, sh.abuf, acc, a.jobs[J_F].accumulate, warp, lane, nvalid);
            tc2_tile_to_a(sh, nvalid);
            TC_TL(11);
            // ---- edge update from the f chunk (D0) ----
            if (upd) {
                csync();                                         // m tile fully consumed (xa + A copy)
                tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
                csync();
                const float4 bb = ldg4(lw.b1 + 2 * D + col);
#pragma unroll 1
                for (int rb = 0; rb < RPW; rb += 2) {       // gathers of 2 rows in flight before the first global store
                    if (rb >= rpw) break;
                    float4 tir[2][3], ujr[2][3], fin[2];
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const int row = r0 + rb + u;
                        const size_t i3 = (size_t)sh.meta.dst[row] * 3, j3 = (size_t)sh.meta.src[row] * 3;
                        if (rb + u < rpw && row < nvalid) fin[u] = ldg4(Fin + (size_t)(e0 + row) * D + col);
                        else fin[u] = f4s(0.f);
#pragma unroll
                        for (int s = 0; s < 3; s++) {
                            tir[u][s] = ldg4(TU + (i3 + s) * 2 * D + col);
                            ujr[u][s] = ldg4(TU + (j3 + s) * 2 * D + D + col);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const int row = r0 + rb + u;
                        const float4 dd = sh.meta.d[row];
                        const float4 Pf = ld4(&sh.tile[row][col]) + bb;
                        const float4 fp = silu4(Pf);
                        const float4 a1 = tir[u][0] * dd.x + tir[u][1] * dd.y + tir[u][2] * dd.z;
                        const float4 a2 = ujr[u][0] * dd.x + ujr[u][1] * dd.y + ujr[u][2] * dd.z;
                        const float4 wdot = (tir[u][0] - a1 * dd.x) * (ujr[u][0] - a2 * dd.x) + (tir[u][1] - a1 * dd.y) * (ujr[u][1] - a2 * dd.y) +
                                            (tir[u][2] - a1 * dd.z) * (ujr[u][2] - a2 * dd.z);
                        if ((rb + u < rpw && row < nvalid)) {
                            st4(P1 + (size_t)(e0 + row) * 3 * D + 2 * D + col, Pf);
                            st4(Fout + (size_t)(e0 + row) * D + col, fin[u] + fp * wdot);
                        }
                    }
                }
            }
            TC_TL(12);
            // ---- s1 (D1): va_i += sum_e vn_j * s1 ----
            float bnd[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
            tc2_mma(sh, ring, sh.abuf, acc, a.jobs[J_S1].accumulate, warp, lane, nvalid);
            TC_TL(13);
            csync();
            tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
            csync();
            TC_TL(14);
            tc_fwd_s1(sh, ws, lw, VN, SP, sh.tile, e0, nvalid, cch, grp, TC2_NGRP, bnd);
            TC_TL(15);
            if (threadIdx.x == 0 && it + 1 < my_tiles) {             // next tile's feature rows -> L2 (bulk prefetch), shortly before use
                const int en = ((int)blockIdx.x + (it + 1) * (int)gridDim.x) * trows;
                tc::tma_prefetch_l2(Fin + (size_t)en * D, (uint32_t)min(trows, E - en) * D * 4);
            }
            // ---- s2 (D0): va_i += sum_e s2 * d ----
            tc2_mma(sh, ring, sh.abuf, acc, a.jobs[J_S2].accumulate, warp, lane, nvalid);
            TC_TL(16);
            csync();
            tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
            csync();
            TC_TL(17);
            tc_fwd_s2(sh, ws, lw, SP, sh.tile, e0, nvalid, cch, grp, TC2_NGRP, bnd);
            TC_TL(18);
        }
        csync();                                              // tile / meta free for the next tile
    }
    if (a.tl != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.tl[31] = (unsigned long long)clock64();
}

}  // namespace vb

namespace vb {

// ---------------------------------------------------------------------------------------------
// adjoint on tensor cores (math and reference lines: see edge_bwd_kernel in k_edge.cuh).  Pre-activations come
// from the forward stage (P1, SP, ATT), so the tile runs only the two adjoint contractions:
// jobs (upd):  0 g3a   1 g3b (+)   2 g4dv   3 g4dk (+)   4 g4f (+)
// ---------------------------------------------------------------------------------------------
template <int ROWS>
__global__ void __launch_bounds__(TC2_THREADS, 1) edge_bwd_tc_kernel(const __grid_constant__ EdgeTcArgs a) {
    pdl_entry();
    extern __shared__ __align__(1024) uint8_t dyn_raw[];
    TcShared& sh = *tc_shared_base(dyn_raw);
    const Workspace& ws = a.ws;
    const int l = a.layer;
    const bool upd = (l < L - 1);
    const int J_G3A = 0, J_G3B = 1, J_G4DV = 2, J_G4DK = 3, J_G4F = 4;
    const int J_LAST = upd ? J_G4F : J_G4DK;
    constexpr int RPW = ROWS / TC2_CWARPS;
    constexpr int RB4 = (RPW % 4 == 0) ? 4 : 2;     // rows whose loads are issued together
    constexpr bool SMALL = ROWS <= 64;              // tile_to_a-free schedule: products read A where it was written, side
                                                    // results go to tc_aux, and no row set is gathered twice
    constexpr int RBM = SMALL ? 2 : RB4;            // g_m phase: its merged neighbours leave fewer registers (0 spills)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, col = lane * 4, hd = lane >> 2;
    const int E = ws.rowptr[ws.N];
    const int trows = min(ROWS, max(16, a.tile_rows));          // edges per tile (<= ROWS, chosen on the host so the tiles fill whole waves)
    const int ntiles_total = (E + trows - 1) / trows;
    const int my_tiles = ((int)blockIdx.x < ntiles_total) ? (ntiles_total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    if (a.tl != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.tl[0] = (unsigned long long)clock64();
    TcRing<ROWS> ring;
    tc2_setup(sh, ring, a.jobs, a.njobs, my_tiles);
    if (a.tl != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.tl[1] = (unsigned long long)clock64();

    float acc[32];
    const float* __restrict__ QKV = ws.QKV[l];
    const float* __restrict__ VN = ws.VN[l];
    const float* __restrict__ TU = ws.TU[l];
    const float* __restrict__ P1 = ws.P1[l];
    const float* __restrict__ SP = ws.SP[l];
    const float* __restrict__ ATT = ws.ATT[l];
    const int cch = threadIdx.x & (D - 1), grp = threadIdx.x >> 7;
    for (int it = 0; it < my_tiles; it++) {
        const int e0 = ((int)blockIdx.x + it * (int)gridDim.x) * trows;
        const int nvalid = min(trows, E - e0);
        // rows are dealt to the compute warps in contiguous runs of rpw = ceil(nvalid / 16): a tile shorter than ROWS
        // keeps every warp busy (slot s of a warp is row warp * rpw + s, valid while s < rpw and the row exists)
        const int rpw = (nvalid + TC2_CWARPS - 1) / TC2_CWARPS, r0 = warp * rpw;
        load_edge_meta<TC_TE, TC2_CTHREADS>(sh.meta, ws, e0, nvalid);
        csync();
        TC_TL(2);
        if constexpr (SMALL) {
            // ---- both halves in one pass (a target's GVEC rows are gathered once): g_Spre[:, 0:128] -> abuf (A of g3a),
            //      g_Spre[:, 128:256] -> tile (A of g3b), written in place (the previous tile's products are done) ;
            //      source-side g_vn, dE/dd ----
#pragma unroll 1
            for (int rb = 0; rb < RPW; rb += RB4) {
                if (rb >= rpw) break;
                float4 sp[RB4][2], gM[RB4][3], vn[RB4][3];
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = r0 + rb + u;
                    const size_t e = (size_t)(e0 + ((rb + u < rpw && row < nvalid) ? row : 0));
                    const size_t i3 = (size_t)sh.meta.dst[row] * 3, j3 = (size_t)sh.meta.src[row] * 3;
                    sp[u][0] = ldg4(SP + e * 2 * D + col);
                    sp[u][1] = ldg4(SP + e * 2 * D + D + col);
#pragma unroll
                    for (int s = 0; s < 3; s++) { gM[u][s] = ldg4(ws.GVEC + (i3 + s) * D + col); vn[u][s] = ldg4(VN + (j3 + s) * D + col); }
                }
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = r0 + rb + u;
                    const bool mine = rb + u < rpw, ok = (mine && row < nvalid);   // (a slot past the run is the next warp's row)
                    const size_t j3 = (size_t)sh.meta.src[row] * 3;
                    const float4 dd = sh.meta.d[row];
                    const float4 s1 = silu4(sp[u][0]), s2 = silu4(sp[u][1]);
                    const float4 gs1 = gM[u][0] * vn[u][0] + gM[u][1] * vn[u][1] + gM[u][2] * vn[u][2];
                    const float gx_ = warp_sum(hsum4(gM[u][0] * s2)), gy_ = warp_sum(hsum4(gM[u][1] * s2)), gz_ = warp_sum(hsum4(gM[u][2] * s2));
                    if (mine) {
                        st4(&sh.abuf[row][col], ok ? gs1 * dsilu4(sp[u][0]) : f4s(0.f));
                        st4(&sh.tile[row][col], ok ? (gM[u][0] * dd.x + gM[u][1] * dd.y + gM[u][2] * dd.z) * dsilu4(sp[u][1]) : f4s(0.f));
                        if (lane == 0) { sh.eacc[row][1] = gx_; sh.eacc[row][2] = gy_; sh.eacc[row][3] = gz_; }
                    }
                    if (ok) {
                        red4(ws.GVNMSG + (j3 + 0) * D + col, gM[u][0] * s1);
                        red4(ws.GVNMSG + (j3 + 1) * D + col, gM[u][1] * s1);
                        red4(ws.GVNMSG + (j3 + 2) * D + col, gM[u][2] * s1);
                    }
                }
            }
            TC_TL(3);
        } else {
            // ---- s1 half: g_Spre[:, 0:128] -> A (written in place: the previous tile's products are done) ; source-side g_vn ----
            // (loads of 4 rows are issued together: the atomics below are compiler barriers for load hoisting)
#pragma unroll 1
            for (int rb = 0; rb < RPW; rb += RB4) {
                if (rb >= rpw) break;
                float4 sp[RB4], gM[RB4][3], vn[RB4][3];
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = r0 + rb + u;
                    const size_t e = (size_t)(e0 + ((rb + u < rpw && row < nvalid) ? row : 0));
                    const size_t i3 = (size_t)sh.meta.dst[row] * 3, j3 = (size_t)sh.meta.src[row] * 3;
                    sp[u] = ldg4(SP + e * 2 * D + col);
#pragma unroll
                    for (int s = 0; s < 3; s++) { gM[u][s] = ldg4(ws.GVEC + (i3 + s) * D + col); vn[u][s] = ldg4(VN + (j3 + s) * D + col); }
                }
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = r0 + rb + u;
                    const bool ok = (rb + u < rpw && row < nvalid);
                    const size_t j3 = (size_t)sh.meta.src[row] * 3;
                    const float4 s1 = silu4(sp[u]);
                    const float4 gs1 = gM[u][0] * vn[u][0] + gM[u][1] * vn[u][1] + gM[u][2] * vn[u][2];
                    if (rb + u < rpw) st4(&sh.abuf[row][col], ok ? gs1 * dsilu4(sp[u]) : f4s(0.f));   // (a slot past the run is the next warp's row)
                    if (ok) {
                        red4(ws.GVNMSG + (j3 + 0) * D + col, gM[u][0] * s1);
                        red4(ws.GVNMSG + (j3 + 1) * D + col, gM[u][1] * s1);
                        red4(ws.GVNMSG + (j3 + 2) * D + col, gM[u][2] * s1);
                    }
                }
            }
            TC_TL(3);
            // ---- s2 half (into the tile; the g3a product's barrier publishes the A rows above) ----
#pragma unroll 4
            for (int r = 0; r < RPW; r++) {
                if (r >= rpw) break;
                const int row = r0 + r;
                const bool ok = (r < rpw && row < nvalid);
                const size_t e = (size_t)(e0 + (ok ? row : 0));
                const size_t i3 = (size_t)sh.meta.dst[row] * 3;
                const float4 dd = sh.meta.d[row];
                const float4 sp = ldg4(SP + e * 2 * D + D + col);
                const float4 s2 = silu4(sp);
                const float4 gM0 = ldg4(ws.GVEC + (i3 + 0) * D + col), gM1 = ldg4(ws.GVEC + (i3 + 1) * D + col),
                             gM2 = ldg4(ws.GVEC + (i3 + 2) * D + col);
                const float gx_ = warp_sum(hsum4(gM0 * s2)), gy_ = warp_sum(hsum4(gM1 * s2)), gz_ = warp_sum(hsum4(gM2 * s2));
                if (lane == 0) { sh.eacc[row][1] = gx_; sh.eacc[row][2] = gy_; sh.eacc[row][3] = gz_; }
                st4(&sh.tile[row][col], ok ? (gM0 * dd.x + gM1 * dd.y + gM2 * dd.z) * dsilu4(sp) : f4s(0.f));
            }
            TC_TL(5);
        }
        csync();
        tc2_mma(sh, ring, sh.abuf, acc, a.jobs[J_G3A].accumulate, warp, lane, nvalid);
        TC_TL(6);
        if constexpr (!SMALL) {
            tc2_tile_to_a(sh, nvalid);
            TC_TL(7);
        }
        // ---- g_m = g_xa_i + g_Spre Ws ; adjoint of m = v_j dv A ----
        tc2_mma(sh, ring, SMALL ? sh.tile : sh.abuf, acc, a.jobs[J_G3B].accumulate, warp, lane, nvalid);
        TC_TL(8);
        csync();                                 // (a tile of <= 64 rows: every warp is done with the tile as g3b's A)
        tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
        csync();
        TC_TL(9);
#pragma unroll 1
        for (int rb = 0; rb < RPW; rb += RBM) {
            if (rb >= rpw) break;
            float4 gxa[RBM], vjr[RBM], pdvr[RBM];
            float avr[RBM];
#pragma unroll
            for (int u = 0; u < RBM; u++) {
                const int row = r0 + rb + u;
                const size_t e = (size_t)(e0 + ((rb + u < rpw && row < nvalid) ? row : 0));
                gxa[u] = load_gxa(ws, (size_t)sh.meta.dst[row], col);
                vjr[u] = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + 2 * D + col);
                pdvr[u] = ldg4(P1 + e * 3 * D + D + col);
                avr[u] = (rb + u < rpw && row < nvalid) ? __ldg(ATT + e * H + hd) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < RBM; u++) {
                const int row = r0 + rb + u;
                const bool ok = (rb + u < rpw && row < nvalid);
                const size_t j = sh.meta.src[row];
                const float Ce = sh.meta.C[row];
                const float av = avr[u], sa = silu_(av), A = sa * Ce;
                const bool mine = rb + u < rpw;                 // a slot past the run is the next warp's row: no shared accesses
                const float4 gm = mine ? ld4(&sh.tile[row][col]) + gxa[u] : f4s(0.f);   // (its owner rewrites it in this phase)
                const float4 dv = silu4(pdvr[u]);
                if (mine) st4(&sh.abuf[row][col], ok ? gm * vjr[u] * A * dsilu4(pdvr[u]) : f4s(0.f));      // g_Pdv -> A (g3a, g3b done)
                const float gA = quad_sum(hsum4(gm * vjr[u] * dv));
                if (mine && (lane & 3) == 0) sh.gattn[row][hd] = gA * Ce * dsilu_(av);
                const float gc = warp_sum((lane & 3) == 0 ? gA * sa : 0.f);
                if (mine && lane == 0) sh.eacc[row][0] = gc;
                if (ok) red4(ws.GQKV + j * 3 * D + 2 * D + col, gm * dv * A);
            }
        }
        TC_TL(10);
        csync();                                 // gattn / A = g_Pdv complete
        // ---- adjoint of a_h = sum q_i k_j dk : g_Pdk (next A operand) ; in a tile of <= 64 rows also the per-edge g_q
        //      rows (-> tc_aux), a longer tile gathers them again below once g_Pdk is copied into abuf ----
#pragma unroll 1
        for (int rb = 0; rb < RPW; rb += RB4) {
            if (rb >= rpw) break;
            float4 pdkr[RB4], qir[RB4], kjr[RB4];
#pragma unroll
            for (int u = 0; u < RB4; u++) {
                const int row = r0 + rb + u;
                const size_t e = (size_t)(e0 + ((rb + u < rpw && row < nvalid) ? row : 0));
                pdkr[u] = ldg4(P1 + e * 3 * D + col);
                qir[u] = ldg4(QKV + (size_t)sh.meta.dst[row] * 3 * D + col);
                kjr[u] = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + D + col);
            }
#pragma unroll
            for (int u = 0; u < RB4; u++) {
                const int row = r0 + rb + u;
                const bool ok = (rb + u < rpw && row < nvalid);
                const size_t j = sh.meta.src[row];
                const float4 dk = silu4(pdkr[u]);
                const float gav = sh.gattn[row][hd];
                if (rb + u < rpw) st4(&sh.tile[row][col], ok ? qir[u] * kjr[u] * gav * dsilu4(pdkr[u]) : f4s(0.f));   // g_Pdk
                if (SMALL && rb + u < rpw) st4(&tc_aux(sh)[row][col], kjr[u] * dk * gav);                            // g_q
                if (ok) red4(ws.GQKV + j * 3 * D + D + col, qir[u] * dk * gav);
            }
        }
        TC_TL(12);
        csync();
        tc2_mma(sh, ring, sh.abuf, acc, a.jobs[J_G4DV].accumulate, warp, lane, nvalid);
        TC_TL(13);
        if constexpr (!SMALL) {
            tc2_tile_to_a(sh, nvalid);           // A = g_Pdk
            TC_TL(14);
            csync();
#pragma unroll 4
            for (int r = 0; r < RPW; r++) {
                if (r >= rpw) break;
                const int row = r0 + r;
                const size_t e = (size_t)(e0 + ((r < rpw && row < nvalid) ? row : 0));
                const float4 dk = silu4(ldg4(P1 + e * 3 * D + col));
                const float4 kj = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + D + col);
                st4(&sh.tile[row][col], kj * dk * sh.gattn[row][hd]);                // per-edge g_q contribution
            }
            csync();
        }
        {
            const TcRow* const gqb = SMALL ? tc_aux(sh) : sh.tile;
            const int i_first = sh.meta.dst[0], i_last = sh.meta.dst[nvalid - 1];
            for (int i = i_first + grp; i <= i_last; i += TC2_NGRP) {
                const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
                const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
                float gq = 0.f;
                for (int r = lo; r < hi; r++) gq += gqb[r][cch];
                if (q0 >= e0 && q1 <= e0 + nvalid) ws.GQKV[(size_t)i * 3 * D + cch] = gq;
                else atomicAdd(ws.GQKV + (size_t)i * 3 * D + cch, gq);
            }
        }
        TC_TL(15);
        // ---- adjoint of the edge update: g_Pf (A operand: abuf in a tile of <= 64 rows, free once g4dv has retired,
        //      while `tile` still holds g_Pdk for g4dk) ; in a tile of <= 64 rows also the g_wdot rows (-> tc_aux, free once
        //      the g_q sums are done), a longer tile gathers them again below once g_Pf is copied into abuf ----
        if (upd) {
            TcRow* const gpfb = SMALL ? sh.abuf : sh.tile;
            csync();
#pragma unroll 1
            for (int rb = 0; rb < RPW; rb += 2) {
                if (rb >= rpw) break;
                float4 gfr[2], pfr[2], tir[2][3], ujr[2][3];
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const int row = r0 + rb + u;
                    const bool ok = (rb + u < rpw && row < nvalid);
                    const size_t e = (size_t)(e0 + (ok ? row : 0));
                    const size_t i3 = (size_t)sh.meta.dst[row] * 3, j3 = (size_t)sh.meta.src[row] * 3;
                    gfr[u] = ok ? ld4(ws.GF + e * D + col) : f4s(0.f);
                    pfr[u] = ldg4(P1 + e * 3 * D + 2 * D + col);
#pragma unroll
                    for (int s = 0; s < 3; s++) {
                        tir[u][s] = ldg4(TU + (i3 + s) * 2 * D + col);
                        ujr[u][s] = ldg4(TU + (j3 + s) * 2 * D + D + col);
                    }
                }
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const int row = r0 + rb + u;
                    const bool ok = (rb + u < rpw && row < nvalid);
                    const size_t e = (size_t)(e0 + (ok ? row : 0));
                    const size_t j3 = (size_t)sh.meta.src[row] * 3;
                    const float4 dd = sh.meta.d[row];
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
                    if (rb + u < rpw) {
                        st4(&gpfb[row][col], gfn * wdot * dsilu4(pf));                                     // g_Pf
                        if (SMALL) st4(&tc_aux(sh)[row][col], gwd);                                        // g_wdot
                    }
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
                    if (lane == 0 && rb + u < rpw) { sh.eacc[row][1] -= gdl[0]; sh.eacc[row][2] -= gdl[1]; sh.eacc[row][3] -= gdl[2]; }
                    if (ok) {
                        red4(ws.GTU + (j3 + 0) * 2 * D + D + col, gu[0]);
                        red4(ws.GTU + (j3 + 1) * 2 * D + D + col, gu[1]);
                        red4(ws.GTU + (j3 + 2) * 2 * D + D + col, gu[2]);
                    }
                    (void)e;
                }
            }
            TC_TL(16);
            csync();
            tc2_mma(sh, ring, SMALL ? sh.tile : sh.abuf, acc, a.jobs[J_G4DK].accumulate, warp, lane, nvalid);
            TC_TL(17);
            if constexpr (!SMALL) {
                tc2_tile_to_a(sh, nvalid);       // A = g_Pf
                TC_TL(18);
                csync();
#pragma unroll 4
                for (int r = 0; r < RPW; r++) {
                    if (r >= rpw) break;
                    const int row = r0 + r;
                    const bool ok = (r < rpw && row < nvalid);
                    const size_t e = (size_t)(e0 + (ok ? row : 0));
                    const float4 gfn = ok ? ld4(ws.GF + e * D + col) : f4s(0.f);
                    st4(&sh.tile[row][col], gfn * silu4(ldg4(P1 + e * 3 * D + 2 * D + col)));   // g_wdot
                }
                csync();
            }
            {
                const TcRow* const gwb = SMALL ? tc_aux(sh) : sh.tile;
                const int i_first = sh.meta.dst[0], i_last = sh.meta.dst[nvalid - 1];
                for (int i = i_first + grp; i <= i_last; i += TC2_NGRP) {
                    const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
                    const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
                    float gt0 = 0.f, gt1 = 0.f, gt2 = 0.f;
                    auto term = [&](int r, float u0, float u1, float u2) {
                        const float4 dd = sh.meta.d[r];
                        const float gw = gwb[r][cch];
                        const float a2 = u0 * dd.x + u1 * dd.y + u2 * dd.z;
                        const float w20 = u0 - a2 * dd.x, w21 = u1 - a2 * dd.y, w22 = u2 - a2 * dd.z;
                        const float wd = w20 * dd.x + w21 * dd.y + w22 * dd.z;
                        gt0 += gw * (w20 - wd * dd.x);
                        gt1 += gw * (w21 - wd * dd.y);
                        gt2 += gw * (w22 - wd * dd.z);
                    };
                    int r = lo;
                    for (; r + 4 <= hi; r += 4) {              // 12 independent gathers in flight
                        float u[4][3];
#pragma unroll
                        for (int q = 0; q < 4; q++) {
                            const size_t j3 = (size_t)sh.meta.src[r + q] * 3;
                            u[q][0] = __ldg(TU + (j3 + 0) * 2 * D + D + cch);
                            u[q][1] = __ldg(TU + (j3 + 1) * 2 * D + D + cch);
                            u[q][2] = __ldg(TU + (j3 + 2) * 2 * D + D + cch);
                        }
#pragma unroll
                        for (int q = 0; q < 4; q++) term(r + q, u[q][0], u[q][1], u[q][2]);
                    }
                    for (; r < hi; r++) {
                        const size_t j3 = (size_t)sh.meta.src[r] * 3;
                        term(r, __ldg(TU + (j3 + 0) * 2 * D + D + cch), __ldg(TU + (j3 + 1) * 2 * D + D + cch),
                             __ldg(TU + (j3 + 2) * 2 * D + D + cch));
                    }
                    if (q0 >= e0 && q1 <= e0 + nvalid) {
                        ws.GTU[((size_t)i * 3 + 0) * 2 * D + cch] = gt0;
                        ws.GTU[((size_t)i * 3 + 1) * 2 * D + cch] = gt1;
                        ws.GTU[((size_t)i * 3 + 2) * 2 * D + cch] = gt2;
                    } else {
                        atomicAdd(ws.GTU + ((size_t)i * 3 + 0) * 2 * D + cch, gt0);
                        atomicAdd(ws.GTU + ((size_t)i * 3 + 1) * 2 * D + cch, gt1);
                        atomicAdd(ws.GTU + ((size_t)i * 3 + 2) * 2 * D + cch, gt2);
                    }
                }
            }
        }
        TC_TL(19);
        // next tile's stored pre-activations -> L2 (bulk prefetch, UBLKPF).  Issued late in the tile: a whole tile ahead
        // the rows were evicted again before their use (ncu: DRAM reads 1.0 -> 1.7 GB per launch on the 512-fragment batch)
        if (threadIdx.x < 3 && it + 1 < my_tiles) {
            const int en = ((int)blockIdx.x + (it + 1) * (int)gridDim.x) * trows;
            const uint32_t nn = (uint32_t)min(trows, E - en);
            if (threadIdx.x == 0) tc::tma_prefetch_l2(SP + (size_t)en * 2 * D, nn * 2 * D * 4);
            else if (threadIdx.x == 1) tc::tma_prefetch_l2(P1 + (size_t)en * 3 * D, nn * 3 * D * 4);
            else tc::tma_prefetch_l2(ATT + (size_t)en * H, nn * H * 4);
        }
        // ---- g_f = g_f_next + [g_Pdk|g_Pdv|g_Pf] W1 ----
        tc2_mma(sh, ring, (SMALL && !upd) ? sh.tile : sh.abuf, acc, a.jobs[J_LAST].accumulate, warp, lane, nvalid);
        TC_TL(20);
        if (!SMALL || !upd) csync();             // (the tile is free unless it was this product's A)
        tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
        csync();
        TC_TL(21);
#pragma unroll 4
        for (int r = 0; r < RPW; r++) {
            if (r >= rpw) break;
            const int row = r0 + r;
            if ((r < rpw && row < nvalid)) {
                float* g = ws.GF + (size_t)(e0 + row) * D + col;
                float4 v = ld4(&sh.tile[row][col]);
                if (upd) v = v + ld4(g);
                st4(g, v);
            }
        }
        if (threadIdx.x < nvalid) {
            float* ea = ws.eacc + (size_t)(e0 + threadIdx.x) * 4;
            st4(ea, ld4(ea) + ld4(&sh.eacc[threadIdx.x][0]));
        }
        TC_TL(22);
        csync();
    }
    if (a.tl != nullptr && blockIdx.x == 0 && threadIdx.x == 0) a.tl[31] = (unsigned long long)clock64();
}

}  // namespace vb
