// Fused per-layer kernels: ONE launch per ViS_MP layer and direction.
//
// A CTA owns a block of NB consecutive nodes.  Edges are target-major, so the edges whose TARGET is one of those nodes
// are one contiguous range [rowptr[n0], rowptr[n0 + NB)); the CTA walks that range in sub-tiles of <= 128 edges through
// the tensor-core edge stage of k_edge_tc.cuh (same phases, same weight ring and MMA helpers) and then runs the
// node stage for its own nodes without leaving the kernel:
//   forward  layer l : edge stage l  (messages, per-target sums, edge update)  ->  node stage l+1 of the block
//                      (o_proj + residual + LayerNorm + VecLayerNorm + q/k/v + vec_proj + w_trg/w_src, k_node2.cuh)
//   backward layer l : node adjoint l+1 of the block (produces dE/dvec, dE/dxa of its targets)  ->  edge adjoint l
// Every quantity the edge stage scatters onto its TARGET belongs to the CTA's own block, so the per-target sums are plain
// read-modify-writes by one CTA (no atomics, fixed order) and need no grid-wide dependency before the node stage; what
// the edge stage gathers from SOURCE nodes (any node of the fragment) was written by the previous launch.  The adjoint's
// source-side sums (dE/dk, dE/dv, dE/dvn, dE/du of the sources) go to the accumulator set of parity l&1 while the node
// adjoint in the same launch consumes and re-zeroes the set of parity (l+1)&1, so the two never meet.
//   reference math: visnet_block.py:237-295 (ViS_MP.forward / message / aggregate / edge_update), utils.py:200-249.
#pragma once
#include "k_edge_tc.cuh"
#include "k_node2.cuh"

namespace vb {

struct FusedArgs {
    int layer;                  // edge layer l (the node stage is l + 1)
    ModelW mw;
    Workspace ws;
    TcJob jobs[8];
    int njobs;
    // adjoint only: accumulators written by this launch's edge adjoint / consumed by its node adjoint
    float *acc_qkv, *acc_vn, *acc_tu;
    float *con_qkv, *con_vn, *con_tu;
};

constexpr int FU_NB = 4;                 // nodes per block: a 4-node block has <= 128 edges, i.e. one sub-tile
static_assert(sizeof(NodeFwd2Smem<FU_NB>) <= sizeof(float) * (TC_TE * TC_LT + TC_TILE_EXT), "node stage rows must fit the staging tile");
static_assert(sizeof(NodeBwd2Smem<FU_NB>) <= sizeof(float) * (TC_TE * TC_LT + TC_TILE_EXT), "node adjoint rows must fit the staging tile");
static_assert(N2Cfg<FU_NB>::WARPS == TC2_CWARPS, "the node stage runs on the compute warps");
constexpr int FU_RPW = TC_TE / TC2_CWARPS;   // up to 8 rows per compute warp

// Rows of a sub-tile are dealt to the compute warps in contiguous runs of rpw = ceil(nvalid / 16): consecutive rows mostly
// share their target node, so a warp's target-side gathers of one batch coalesce into one L2 request.  Row slot r of a
// warp is row warp * rpw + r (valid while r < rpw and the row is below nvalid).
struct FuRows {
    int rpw, base, nvalid;
    __device__ __forceinline__ FuRows(int nvalid_, int warp) : rpw((nvalid_ + TC2_CWARPS - 1) / TC2_CWARPS), base(warp * rpw), nvalid(nvalid_) {}
    __device__ __forceinline__ int row(int r) const { return base + r; }
    __device__ __forceinline__ bool ok(int r) const { return r < rpw && base + r < nvalid; }
};

// number of sub-tiles this CTA will run (sets the length of the weight ring's slab sequence)
__device__ __forceinline__ int fu_count_tiles(const Workspace& ws) {
    const int nblocks = (ws.N + FU_NB - 1) / FU_NB;
    int tiles = 0;
    for (int b = blockIdx.x; b < nblocks; b += gridDim.x) {
        const int n0 = b * FU_NB, n1 = min(n0 + FU_NB, ws.N);
        tiles += (ws.rowptr[n1] - ws.rowptr[n0] + TC_TE - 1) / TC_TE;
    }
    return tiles;
}

// =====================================================================================================
// forward: edge stage l of the block's edges, then node stage l + 1 of the block
// job order: dk, dv, [f], s1, s2        (as edge_fwd_tc_kernel)
// =====================================================================================================
__global__ void __launch_bounds__(TC2_THREADS, 1) fused_fwd_kernel(const __grid_constant__ FusedArgs a) {
    pdl_entry();
    extern __shared__ __align__(1024) uint8_t dyn_raw[];
    TcShared& sh = *tc_shared_base(dyn_raw);
    const Workspace& ws = a.ws;
    const int l = a.layer;
    const LayerW& lw = a.mw.layer[l];
    const bool upd = (l < L - 1);
    const int J_DK = 0, J_DV = 1, J_F = 2, J_S1 = upd ? 3 : 2, J_S2 = upd ? 4 : 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, col = lane * 4;
    const int my_tiles = fu_count_tiles(ws);
    TcRing<TC_TE> ring;
    tc2_setup(sh, ring, a.jobs, a.njobs, my_tiles);

    float acc[32];
    const float* __restrict__ Fin = ws.F[l];
    float* __restrict__ Fout = upd ? ws.F[l + 1] : nullptr;
    const float* __restrict__ QKV = ws.QKV[l];
    const float* __restrict__ VN = ws.VN[l];
    const float* __restrict__ TU = ws.TU[l];
    float* __restrict__ P1 = ws.P1[l];
    float* __restrict__ SP = ws.SP[l];
    float* __restrict__ ATT = ws.ATT[l];
    const int cch = threadIdx.x & (D - 1), grp = threadIdx.x >> 7;      // aggregation role: channel, target group
    const int nblocks = (ws.N + FU_NB - 1) / FU_NB;
    int t = 0;
    for (int b = blockIdx.x; b < nblocks; b += gridDim.x) {
        const int n0 = b * FU_NB, n1 = min(n0 + FU_NB, ws.N);
        const int eb = ws.rowptr[n0], ee = ws.rowptr[n1];
        for (int e0 = eb; e0 < ee; e0 += TC_TE, t++) {
            const int nvalid = min(TC_TE, ee - e0);
            const FuRows R(nvalid, warp);
            // ---- load f tile + meta (coalesced) ----
            for (int idx = threadIdx.x; idx < nvalid * 32; idx += TC2_CTHREADS) {
                const int row = idx >> 5, c4 = (idx & 31) * 4;
                st4(&sh.tile[row][c4], ldg4(Fin + (size_t)(e0 + row) * D + c4));
            }
            load_edge_meta<TC_TE, TC2_CTHREADS>(sh.meta, ws, e0, nvalid);
            csync();
            tc2_tile_to_a(sh, nvalid);
            // ---- dk -> attention weights ----
            float Areg[FU_RPW];
            tc2_mma(sh, ring, acc, a.jobs[J_DK].accumulate, warp, lane, nvalid);
            csync();                                              // everyone finished reading f from the tile
            tc2_acc_to_tile(sh, acc, warp, lane, nvalid);
            csync();
            {
                const float4 bb = ldg4(lw.b1 + col);
#pragma unroll
                for (int r = 0; r < FU_RPW; r++) {
                    const int row = R.row(r);
                    Areg[r] = 0.f;
                    if (R.ok(r)) {
                        const float4 qi = ldg4(QKV + (size_t)sh.meta.dst[row] * 3 * D + col);
                        const float4 kj = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + D + col);
                        const float4 P = ld4(&sh.tile[row][col]) + bb;
                        const float av = quad_sum(hsum4(qi * kj * silu4(P)));
                        Areg[r] = silu_(av) * sh.meta.C[row];
                        st4(P1 + (size_t)(e0 + row) * 3 * D + col, P);
                        if ((lane & 3) == 0) ATT[(size_t)(e0 + row) * H + (lane >> 2)] = av;
                    }
                }
            }
            // ---- dv -> message m (in place in the tile) ----
            tc2_mma(sh, ring, acc, a.jobs[J_DV].accumulate, warp, lane, nvalid);
            csync();
            tc2_acc_to_tile(sh, acc, warp, lane, nvalid);
            csync();
            {
                const float4 bb = ldg4(lw.b1 + D + col);
#pragma unroll
                for (int r = 0; r < FU_RPW; r++) {
                    const int row = R.row(r);
                    if (R.ok(r)) {
                        const float4 vj = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + 2 * D + col);
                        const float4 P = ld4(&sh.tile[row][col]) + bb;
                        st4(&sh.tile[row][col], vj * silu4(P) * Areg[r]);
                        st4(P1 + (size_t)(e0 + row) * 3 * D + D + col, P);
                    }
                }
            }
            csync();
            // ---- xa_i += sum_e m_e  (targets of this sub-tile all belong to this block: plain read-modify-write) ----
            const int i_first = sh.meta.dst[0], i_last = sh.meta.dst[nvalid - 1];
            for (int i = i_first + grp; i <= i_last; i += TC2_NGRP) {
                const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
                const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
                float xa = 0.f;
                for (int r = lo; r < hi; r++) xa += sh.tile[r][cch];
                ws.XA[(size_t)i * D + cch] += xa;
            }
            // ---- A = m, start s1 (-> D1) ----
            if (upd) tc2_mma(sh, ring, acc, a.jobs[J_F].accumulate, warp, lane, nvalid);
            tc2_tile_to_a(sh, nvalid);
            // ---- edge update from the f chunk (D0) ----
            if (upd) {
                csync();                                          // m tile fully consumed (xa + A copy)
                tc2_acc_to_tile(sh, acc, warp, lane, nvalid);
                csync();
                const float4 bb = ldg4(lw.b1 + 2 * D + col);
#pragma unroll 1
                for (int rb = 0; rb < FU_RPW; rb += 2) {       // gathers of 2 rows in flight before the first global store
                    if (!R.ok(rb)) break;
                    float4 tir[2][3], ujr[2][3], fin[2];
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const int row = R.row(rb + u);
                        const bool ok = R.ok(rb + u);
                        const size_t i3 = (size_t)sh.meta.dst[ok ? row : 0] * 3, j3 = (size_t)sh.meta.src[ok ? row : 0] * 3;
                        fin[u] = ok ? ldg4(Fin + (size_t)(e0 + row) * D + col) : f4s(0.f);
#pragma unroll
                        for (int s = 0; s < 3; s++) {
                            tir[u][s] = ldg4(TU + (i3 + s) * 2 * D + col);
                            ujr[u][s] = ldg4(TU + (j3 + s) * 2 * D + D + col);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const int row = R.row(rb + u);
                        if (R.ok(rb + u)) {
                            const float4 dd = sh.meta.d[row];
                            const float4 Pf = ld4(&sh.tile[row][col]) + bb;
                            const float4 fp = silu4(Pf);
                            const float4 a1 = tir[u][0] * dd.x + tir[u][1] * dd.y + tir[u][2] * dd.z;
                            const float4 a2 = ujr[u][0] * dd.x + ujr[u][1] * dd.y + ujr[u][2] * dd.z;
                            const float4 wdot = (tir[u][0] - a1 * dd.x) * (ujr[u][0] - a2 * dd.x) + (tir[u][1] - a1 * dd.y) * (ujr[u][1] - a2 * dd.y) +
                                                (tir[u][2] - a1 * dd.z) * (ujr[u][2] - a2 * dd.z);
                            st4(P1 + (size_t)(e0 + row) * 3 * D + 2 * D + col, Pf);
                            st4(Fout + (size_t)(e0 + row) * D + col, fin[u] + fp * wdot);
                        }
                    }
                }
            }
            // ---- s1 (D1): va_i += sum_e vn_j * s1 ----
            tc2_mma(sh, ring, acc, a.jobs[J_S1].accumulate, warp, lane, nvalid);
            csync();
            tc2_acc_to_tile(sh, acc, warp, lane, nvalid);
            csync();
            {
                const float bsv = __ldg(lw.bs + cch);
                for (int i = i_first + grp; i <= i_last; i += TC2_NGRP) {
                    const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
                    const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
                    float v0 = 0.f, v1 = 0.f, v2 = 0.f;
                    int r = lo;
                    for (; r + 4 <= hi; r += 4) {              // 12 independent gathers in flight
                        float g[4][3], s1[4];
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            const size_t j3 = (size_t)sh.meta.src[r + u] * 3;
                            g[u][0] = __ldg(VN + (j3 + 0) * D + cch); g[u][1] = __ldg(VN + (j3 + 1) * D + cch); g[u][2] = __ldg(VN + (j3 + 2) * D + cch);
                            const float sp = sh.tile[r + u][cch] + bsv;
                            SP[(size_t)(e0 + r + u) * 2 * D + cch] = sp;
                            s1[u] = silu_(sp);
                        }
#pragma unroll
                        for (int u = 0; u < 4; u++) { v0 += g[u][0] * s1[u]; v1 += g[u][1] * s1[u]; v2 += g[u][2] * s1[u]; }
                    }
                    for (; r < hi; r++) {
                        const size_t j3 = (size_t)sh.meta.src[r] * 3;
                        const float sp = sh.tile[r][cch] + bsv;
                        SP[(size_t)(e0 + r) * 2 * D + cch] = sp;
                        const float s1 = silu_(sp);
                        v0 += __ldg(VN + (j3 + 0) * D + cch) * s1;
                        v1 += __ldg(VN + (j3 + 1) * D + cch) * s1;
                        v2 += __ldg(VN + (j3 + 2) * D + cch) * s1;
                    }
                    ws.VA[((size_t)i * 3 + 0) * D + cch] += v0;
                    ws.VA[((size_t)i * 3 + 1) * D + cch] += v1;
                    ws.VA[((size_t)i * 3 + 2) * D + cch] += v2;
                }
            }
            // ---- s2 (D0): va_i += sum_e s2 * d ----
            tc2_mma(sh, ring, acc, a.jobs[J_S2].accumulate, warp, lane, nvalid);
            csync();
            tc2_acc_to_tile(sh, acc, warp, lane, nvalid);
            csync();
            {
                const float bsv = __ldg(lw.bs + D + cch);
                for (int i = i_first + grp; i <= i_last; i += TC2_NGRP) {
                    const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
                    const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
                    float v0 = 0.f, v1 = 0.f, v2 = 0.f;
                    for (int r = lo; r < hi; r++) {
                        const float4 de = sh.meta.d[r];
                        const float sp = sh.tile[r][cch] + bsv;
                        SP[(size_t)(e0 + r) * 2 * D + D + cch] = sp;
                        const float s2 = silu_(sp);
                        v0 += s2 * de.x; v1 += s2 * de.y; v2 += s2 * de.z;
                    }
                    ws.VA[((size_t)i * 3 + 0) * D + cch] += v0;
                    ws.VA[((size_t)i * 3 + 1) * D + cch] += v1;
                    ws.VA[((size_t)i * 3 + 2) * D + cch] += v2;
                }
            }
            csync();                                              // tile / meta free; XA / VA updates visible CTA-wide
        }
        // ---- node stage l + 1 of this block (its xa / va are complete) ----
        node_fwd2_body<FU_NB, 2>(a.mw, ws, l + 1, n0, reinterpret_cast<float*>(&sh.tile[0][0]), [] { csync(); });
        csync();                                                  // node-stage shared rows (aliasing the tile) are free
    }
}

// =====================================================================================================
// backward: node adjoint l + 1 of the block, then edge adjoint l of the block's edges
// jobs (upd):  0 g3a   1 g3b (+)   2 g4dv   3 g4dk (+)   4 g4f (+)     (as edge_bwd_tc_kernel)
// =====================================================================================================
__global__ void __launch_bounds__(TC2_THREADS, 1) fused_bwd_kernel(const __grid_constant__ FusedArgs a) {
    pdl_entry();
    extern __shared__ __align__(1024) uint8_t dyn_raw[];
    TcShared& sh = *tc_shared_base(dyn_raw);
    const Workspace& ws = a.ws;
    const int l = a.layer;
    const bool upd = (l < L - 1);
    const int J_G3A = 0, J_G3B = 1, J_G4DV = 2, J_G4DK = 3, J_G4F = 4;
    const int J_LAST = upd ? J_G4F : J_G4DK;
    constexpr int RB4 = 4;                          // rows whose loads are issued together
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, col = lane * 4, hd = lane >> 2;
    const int my_tiles = fu_count_tiles(ws);
    TcRing<TC_TE> ring;
    tc2_setup(sh, ring, a.jobs, a.njobs, my_tiles);

    float acc[32];
    const float* __restrict__ QKV = ws.QKV[l];
    const float* __restrict__ VN = ws.VN[l];
    const float* __restrict__ TU = ws.TU[l];
    const float* __restrict__ P1 = ws.P1[l];
    const float* __restrict__ SP = ws.SP[l];
    const float* __restrict__ ATT = ws.ATT[l];
    float* __restrict__ GQKV = a.acc_qkv;
    float* __restrict__ GVNMSG = a.acc_vn;
    float* __restrict__ GTU = a.acc_tu;
    const float* GVEC = ws.GVEC;            // written by this CTA's node adjoint below: coherent loads only (no ld.global.nc)
    const float* GXA = ws.GXA;
    const int cch = threadIdx.x & (D - 1), grp = threadIdx.x >> 7;
    const int nblocks = (ws.N + FU_NB - 1) / FU_NB;
    int t = 0;
    for (int b = blockIdx.x; b < nblocks; b += gridDim.x) {
        const int n0 = b * FU_NB, n1 = min(n0 + FU_NB, ws.N);
        // ---- node adjoint l + 1 of this block: consumes the accumulators of parity (l+1)&1, writes GX / GVEC / GXA ----
        node_bwd2_body<FU_NB, 2>(a.mw, ws, l + 1, n0, a.con_qkv, a.con_vn, a.con_tu, reinterpret_cast<float*>(&sh.tile[0][0]),
                              [] { csync(); });
        csync();                                                  // GVEC / GXA of the block visible; node rows (aliasing the tile) free
        const int eb = ws.rowptr[n0], ee = ws.rowptr[n1];
        for (int e0 = eb; e0 < ee; e0 += TC_TE, t++) {
            const int nvalid = min(TC_TE, ee - e0);
            const FuRows R(nvalid, warp);
            load_edge_meta<TC_TE, TC2_CTHREADS>(sh.meta, ws, e0, nvalid);
            csync();
            // ---- s1 half: g_Spre[:, 0:128] -> tile -> A ; source-side g_vn ----
#pragma unroll 1
            for (int rb = 0; rb < FU_RPW; rb += RB4) {
                if (!R.ok(rb)) break;
                float4 sp[RB4], gM[RB4][3], vn[RB4][3];
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = R.row(rb + u);
                    const int rr = R.ok(rb + u) ? row : 0;
                    const size_t e = (size_t)(e0 + rr);
                    const size_t i3 = (size_t)sh.meta.dst[rr] * 3, j3 = (size_t)sh.meta.src[rr] * 3;
                    sp[u] = ldg4(SP + e * 2 * D + col);
#pragma unroll
                    for (int s = 0; s < 3; s++) { gM[u][s] = ld4(GVEC + (i3 + s) * D + col); vn[u][s] = ldg4(VN + (j3 + s) * D + col); }
                }
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = R.row(rb + u);
                    if (R.ok(rb + u)) {
                        const size_t j3 = (size_t)sh.meta.src[row] * 3;
                        const float4 s1 = silu4(sp[u]);
                        const float4 gs1 = gM[u][0] * vn[u][0] + gM[u][1] * vn[u][1] + gM[u][2] * vn[u][2];
                        st4(&sh.tile[row][col], gs1 * dsilu4(sp[u]));
                        red4(GVNMSG + (j3 + 0) * D + col, gM[u][0] * s1);
                        red4(GVNMSG + (j3 + 1) * D + col, gM[u][1] * s1);
                        red4(GVNMSG + (j3 + 2) * D + col, gM[u][2] * s1);
                    }
                }
            }
            csync();
            tc2_tile_to_a(sh, nvalid);
            csync();
            // ---- s2 half ----
#pragma unroll 4
            for (int r = 0; r < FU_RPW; r++) {
                const int row = R.row(r);
                if (R.ok(r)) {
                    const size_t e = (size_t)(e0 + row);
                    const size_t i3 = (size_t)sh.meta.dst[row] * 3;
                    const float4 dd = sh.meta.d[row];
                    const float4 sp = ldg4(SP + e * 2 * D + D + col);
                    const float4 s2 = silu4(sp);
                    const float4 gM0 = ld4(GVEC + (i3 + 0) * D + col), gM1 = ld4(GVEC + (i3 + 1) * D + col),
                                 gM2 = ld4(GVEC + (i3 + 2) * D + col);
                    const float gx_ = warp_sum(hsum4(gM0 * s2)), gy_ = warp_sum(hsum4(gM1 * s2)), gz_ = warp_sum(hsum4(gM2 * s2));
                    if (lane == 0) { sh.eacc[row][1] = gx_; sh.eacc[row][2] = gy_; sh.eacc[row][3] = gz_; }
                    st4(&sh.tile[row][col], (gM0 * dd.x + gM1 * dd.y + gM2 * dd.z) * dsilu4(sp));
                }
            }
            csync();
            tc2_mma(sh, ring, acc, a.jobs[J_G3A].accumulate, warp, lane, nvalid);
            tc2_tile_to_a(sh, nvalid);
            // ---- g_m = g_xa_i + g_Spre Ws ; adjoint of m = v_j dv A ----
            tc2_mma(sh, ring, acc, a.jobs[J_G3B].accumulate, warp, lane, nvalid);
            csync();
            tc2_acc_to_tile(sh, acc, warp, lane, nvalid);
            csync();
#pragma unroll 1
            for (int rb = 0; rb < FU_RPW; rb += RB4) {
                if (!R.ok(rb)) break;
                float4 gxa[RB4], vjr[RB4], pdvr[RB4];
                float avr[RB4];
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = R.row(rb + u);
                    const int rr = R.ok(rb + u) ? row : 0;
                    const size_t e = (size_t)(e0 + rr);
                    gxa[u] = ld4(GXA + (size_t)sh.meta.dst[rr] * D + col);
                    vjr[u] = ldg4(QKV + (size_t)sh.meta.src[rr] * 3 * D + 2 * D + col);
                    pdvr[u] = ldg4(P1 + e * 3 * D + D + col);
                    avr[u] = __ldg(ATT + e * H + hd);
                }
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = R.row(rb + u);
                    if (R.ok(rb + u)) {                              // warp-uniform
                        const size_t j = sh.meta.src[row];
                        const float Ce = sh.meta.C[row];
                        const float av = avr[u], sa = silu_(av), A = sa * Ce;
                        const float4 gm = ld4(&sh.tile[row][col]) + gxa[u];
                        const float4 dv = silu4(pdvr[u]);
                        st4(&sh.tile[row][col], gm * vjr[u] * A * dsilu4(pdvr[u]));      // g_Pdv
                        const float gA = quad_sum(hsum4(gm * vjr[u] * dv));
                        if ((lane & 3) == 0) sh.gattn[row][hd] = gA * Ce * dsilu_(av);
                        const float gc = warp_sum((lane & 3) == 0 ? gA * sa : 0.f);
                        if (lane == 0) sh.eacc[row][0] = gc;
                        red4(GQKV + j * 3 * D + 2 * D + col, gm * dv * A);
                    }
                }
            }
            csync();
            tc2_tile_to_a(sh, nvalid);               // A = g_Pdv (A planes free: g3b done)
            csync();
            // ---- adjoint of a_h = sum q_i k_j dk : first g_Pdk (next A operand), then the g_q tile ----
#pragma unroll 1
            for (int rb = 0; rb < FU_RPW; rb += RB4) {
                if (!R.ok(rb)) break;
                float4 pdkr[RB4], qir[RB4], kjr[RB4];
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = R.row(rb + u);
                    const int rr = R.ok(rb + u) ? row : 0;
                    const size_t e = (size_t)(e0 + rr);
                    pdkr[u] = ldg4(P1 + e * 3 * D + col);
                    qir[u] = ldg4(QKV + (size_t)sh.meta.dst[rr] * 3 * D + col);
                    kjr[u] = ldg4(QKV + (size_t)sh.meta.src[rr] * 3 * D + D + col);
                }
#pragma unroll
                for (int u = 0; u < RB4; u++) {
                    const int row = R.row(rb + u);
                    if (R.ok(rb + u)) {
                        const size_t j = sh.meta.src[row];
                        const float4 dk = silu4(pdkr[u]);
                        const float gav = sh.gattn[row][hd];
                        st4(&sh.tile[row][col], qir[u] * kjr[u] * gav * dsilu4(pdkr[u]));   // g_Pdk
                        red4(GQKV + j * 3 * D + D + col, qir[u] * dk * gav);
                    }
                }
            }
            csync();
            tc2_mma(sh, ring, acc, a.jobs[J_G4DV].accumulate, warp, lane, nvalid);
            tc2_tile_to_a(sh, nvalid);               // A = g_Pdk
            csync();
#pragma unroll 4
            for (int r = 0; r < FU_RPW; r++) {
                const int row = R.row(r);
                if (R.ok(r)) {
                    const size_t e = (size_t)(e0 + row);
                    const float4 dk = silu4(ldg4(P1 + e * 3 * D + col));
                    const float4 kj = ldg4(QKV + (size_t)sh.meta.src[row] * 3 * D + D + col);
                    st4(&sh.tile[row][col], kj * dk * sh.gattn[row][hd]);                    // per-edge g_q contribution
                }
            }
            csync();
            const int i_first = sh.meta.dst[0], i_last = sh.meta.dst[nvalid - 1];
            for (int i = i_first + grp; i <= i_last; i += TC2_NGRP) {
                const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
                const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
                float gq = 0.f;
                for (int r = lo; r < hi; r++) gq += sh.tile[r][cch];
                GQKV[(size_t)i * 3 * D + cch] += gq;              // target side: this block's own rows
            }
            // ---- adjoint of the edge update: first g_Pf (A operand), then the g_wdot tile ----
            if (upd) {
                csync();
#pragma unroll 1
                for (int rb = 0; rb < FU_RPW; rb += 2) {
                    if (!R.ok(rb)) break;
                    float4 gfr[2], pfr[2], tir[2][3], ujr[2][3];
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const int row = R.row(rb + u);
                        const int rr = R.ok(rb + u) ? row : 0;
                        const size_t e = (size_t)(e0 + rr);
                        const size_t i3 = (size_t)sh.meta.dst[rr] * 3, j3 = (size_t)sh.meta.src[rr] * 3;
                        gfr[u] = ld4(ws.GF + e * D + col);
                        pfr[u] = ldg4(P1 + e * 3 * D + 2 * D + col);
#pragma unroll
                        for (int s = 0; s < 3; s++) {
                            tir[u][s] = ldg4(TU + (i3 + s) * 2 * D + col);
                            ujr[u][s] = ldg4(TU + (j3 + s) * 2 * D + D + col);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const int row = R.row(rb + u);
                        if (R.ok(rb + u)) {
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
                            st4(&sh.tile[row][col], gfn * wdot * dsilu4(pf));                    // g_Pf
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
                            if (lane == 0) { sh.eacc[row][1] -= gdl[0]; sh.eacc[row][2] -= gdl[1]; sh.eacc[row][3] -= gdl[2]; }
                            red4(GTU + (j3 + 0) * 2 * D + D + col, gu[0]);
                            red4(GTU + (j3 + 1) * 2 * D + D + col, gu[1]);
                            red4(GTU + (j3 + 2) * 2 * D + D + col, gu[2]);
                        }
                    }
                }
                csync();
                tc2_mma(sh, ring, acc, a.jobs[J_G4DK].accumulate, warp, lane, nvalid);
                tc2_tile_to_a(sh, nvalid);           // A = g_Pf
                csync();
#pragma unroll 4
                for (int r = 0; r < FU_RPW; r++) {
                    const int row = R.row(r);
                    if (R.ok(r)) {
                        const size_t e = (size_t)(e0 + row);
                        const float4 gfn = ld4(ws.GF + e * D + col);
                        st4(&sh.tile[row][col], gfn * silu4(ldg4(P1 + e * 3 * D + 2 * D + col)));   // g_wdot
                    }
                }
                csync();
                for (int i = i_first + grp; i <= i_last; i += TC2_NGRP) {
                    const int q0 = ws.rowptr[i], q1 = ws.rowptr[i + 1];
                    const int lo = max(q0, e0) - e0, hi = min(q1, e0 + nvalid) - e0;
                    float gt0 = 0.f, gt1 = 0.f, gt2 = 0.f;
                    auto term = [&](int r, float u0, float u1, float u2) {
                        const float4 dd = sh.meta.d[r];
                        const float gw = sh.tile[r][cch];
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
                    GTU[((size_t)i * 3 + 0) * 2 * D + cch] += gt0;    // target side: this block's own rows
                    GTU[((size_t)i * 3 + 1) * 2 * D + cch] += gt1;
                    GTU[((size_t)i * 3 + 2) * 2 * D + cch] += gt2;
                }
            }
            // ---- g_f = g_f_next + [g_Pdk|g_Pdv|g_Pf] W1 ----
            tc2_mma(sh, ring, acc, a.jobs[J_LAST].accumulate, warp, lane, nvalid);
            csync();
            tc2_acc_to_tile(sh, acc, warp, lane, nvalid);
            csync();
#pragma unroll 4
            for (int r = 0; r < FU_RPW; r++) {
                const int row = R.row(r);
                if (R.ok(r)) {
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
            csync();
        }
    }
}

}  // namespace vb
