// Neighbour build, edge geometry/RBF, neighbour + edge embedding (forward) and their adjoints.
//   reference: utils.py:259-276 (Distance), :53-57 (ExpNormalSmearing), :16-19 (CosineCutoff),
//              visnet_block.py:110-122, utils.py:296-317 (NeighborEmbedding), :331-337 (EdgeEmbedding)
#pragma once
#include "model.h"

namespace vb {

// ---------------------------------------------------------------------------------------------
// K1: canonical radius graph.  One thread per target atom scans the atoms of its own fragment in
// ascending index; d2 = fma(dz,dz, fma(dy,dy, dx*dx)) < rc^2 (strict), first 32 hits kept.
// Bit-exact contract with oracle/radius_graph.c.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) nbr_build_kernel(int N, const float* __restrict__ pos,
                                                        const int* __restrict__ frag_of,
                                                        const int* __restrict__ frag_start, float rc,
                                                        int* __restrict__ slots, int* __restrict__ deg,
                                                        float* __restrict__ forces) {
    pdl_entry();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    if (forces) { forces[3 * i] = 0.f; forces[3 * i + 1] = 0.f; forces[3 * i + 2] = 0.f; }   // accumulated by the last kernel of the sweep (none in the energy plan)
    const int g = frag_of[i];
    const int j0 = frag_start[g], j1 = frag_start[g + 1];
    const float xi = pos[3 * i], yi = pos[3 * i + 1], zi = pos[3 * i + 2];
    const float r2 = __fmul_rn(rc, rc);
    int cnt = 0;
    for (int j = j0; j < j1 && cnt < KNB; j++) {
        const float dx = __fsub_rn(__ldg(pos + 3 * j), xi);
        const float dy = __fsub_rn(__ldg(pos + 3 * j + 1), yi);
        const float dz = __fsub_rn(__ldg(pos + 3 * j + 2), zi);
        float d2 = __fmul_rn(dx, dx);
        d2 = __fmaf_rn(dy, dy, d2);
        d2 = __fmaf_rn(dz, dz, d2);
        if (d2 < r2) slots[i * KNB + cnt++] = j;
    }
    for (int k = cnt; k < KNB; k++) slots[i * KNB + k] = -1;
    deg[i] = cnt;
}

// K2: exclusive scan of deg -> rowptr (single block; N is small enough that this is latency only).
// A total above the workspace's edge capacity (a caller-trimmed max_edges that a step exceeded) raises flags[0]; the
// row pointers are clamped to the capacity, so nothing is written out of bounds and the host can report the overflow.
// `total` (a chunk's slot on a chunked handle, else null) receives the unclamped edge total: calibration and the
// overflow report of each chunk read it after later chunks have reused rowptr.
__global__ void __launch_bounds__(1024) rowptr_scan_kernel(int N, const int* __restrict__ deg,
                                                           int* __restrict__ rowptr, int ecap, int* __restrict__ flags,
                                                           int* __restrict__ total) {
    pdl_entry();
    __shared__ int wsum[32];
    __shared__ int carry_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < N; base += 1024) {
        const int i = base + tid;
        const int v = (i < N) ? deg[i] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += t;
            }
            wsum[lane] = w;  // inclusive over warps
        }
        __syncthreads();
        const int carry = carry_s;
        const int excl = carry + (warp ? wsum[warp - 1] : 0) + incl - v;
        if (i < N) rowptr[i] = min(excl, ecap);
        __syncthreads();
        if (tid == 1023) carry_s = carry + wsum[31];
        __syncthreads();
    }
    if (tid == 0) {
        rowptr[N] = min(carry_s, ecap);
        if (carry_s > ecap) flags[0] = 1;
        if (total) *total = carry_s;
    }
}

// K3: per-edge geometry + RBF.  One warp per target atom, lane k = neighbour slot k.
__global__ void __launch_bounds__(128) edge_geom_kernel(int N, const float* __restrict__ pos, ModelW mw,
                                                        Workspace ws) {
    pdl_entry();
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= N) return;
    const int dg = ws.deg[i];
    const int e0 = ws.rowptr[i];
    float r = 0.f, C = 0.f;
    if (lane < dg) {
        const int j = ws.slots[i * KNB + lane];
        const int e = e0 + lane;
        float dx = 0.f, dy = 0.f, dz = 0.f, inv_r = 0.f;
        if (j != i) {
            const float ex = __fsub_rn(pos[3 * j], pos[3 * i]);
            const float ey = __fsub_rn(pos[3 * j + 1], pos[3 * i + 1]);
            const float ez = __fsub_rn(pos[3 * j + 2], pos[3 * i + 2]);
            const float s2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez));
            r = __fsqrt_rn(s2);
            dx = __fdiv_rn(ex, r); dy = __fdiv_rn(ey, r); dz = __fdiv_rn(ez, r);
            inv_r = __fdiv_rn(1.0f, r);
        }
        C = cutoff_fn(r, mw.cutoff);
        if (e < ws.Ecap) {                // beyond a trimmed capacity: dropped (rowptr_scan raised the overflow flag)
            ws.esrc[e] = j;
            ws.edst[e] = i;
            st4(ws.geom + (size_t)e * 8, f4(r, C, dx, dy));
            st4(ws.geom + (size_t)e * 8 + 4, f4(dz, inv_r, __int_as_float(ws.z[j]), 0.f));   // [6]: z of the source atom (embed_node)
            if (ws.eacc) st4(ws.eacc + (size_t)e * 4, f4s(0.f));       // adjoint accumulators (absent in the energy plan)
        }
    }
    const float mu = __ldg(mw.rbf_means + lane), beta = __ldg(mw.rbf_betas + lane);
    const float alpha = 5.0f / mw.cutoff;
    for (int k = 0; k < dg; k++) {
        const float rk = __shfl_sync(0xffffffffu, r, k);
        const float Ck = __shfl_sync(0xffffffffu, C, k);
        const float t = expf(-alpha * rk) - mu;
        if (e0 + k < ws.Ecap) ws.rbf[(size_t)(e0 + k) * NR + lane] = Ck * expf(-beta * t * t);
    }
}

// ---------------------------------------------------------------------------------------------
// K4: neighbour embedding.  Block = 128 threads (thread = channel c), NB consecutive nodes per block.
//   agg_i[c] = sum_{e->i, j!=i} (rbf_e . Wd[c,:] + bd[c]) * C_e * nb_emb[z_j][c]
//   x_i = [emb[z_i] | agg_i] Wc^T + bc
// ---------------------------------------------------------------------------------------------
// NB consecutive nodes per 256-thread block (thread = channel x K-half): the per-edge loop and the final K = 256 product
// are serial latency chains, so both are split in two and the halves summed in a fixed order through shared memory.
// NB = 1 for small systems (one wave of per-node CTAs, shortest chain); NB = 8 for batches, where every CTA streaming the
// 128 KB combine weight for a single node made the kernel L2-bound (14k nodes: 1.8 GB of L2 -> SM traffic): a weight row is
// now loaded once per CTA and used for all NB nodes.
constexpr int EMB_THREADS = 2 * D;
template <int NB>
__global__ void __launch_bounds__(EMB_THREADS) embed_node_kernel(ModelW mw, Workspace ws) {
    pdl_entry();
    __shared__ float cat[NB][2 * D];
    __shared__ float part[NB][D];
    __shared__ int sj[KNB];
    __shared__ int sz[KNB];
    __shared__ float sC[KNB];
    const int c = threadIdx.x & (D - 1), half = threadIdx.x >> 7;
    const int n0 = blockIdx.x * NB;
    float wd[NR];
#pragma unroll
    for (int k = 0; k < NR; k += 4) {
        const float4 w = ldg4(mw.WdN + c * NR + k);
        wd[k] = w.x; wd[k + 1] = w.y; wd[k + 2] = w.z; wd[k + 3] = w.w;
    }
    const float bd = __ldg(mw.bd + c);
    for (int nb = 0; nb < NB; nb++) {
        const int i = n0 + nb;
        if (i >= ws.N) {                                 // (block-uniform)
            if (half == 0) { cat[nb][c] = 0.f; cat[nb][D + c] = 0.f; }
            continue;
        }
        const int e0 = ws.rowptr[i], dg = ws.rowptr[i + 1] - e0;
        if (threadIdx.x < dg) {                         // edge metadata first: breaks the esrc -> z -> embedding load chain
            const int j = ws.esrc[e0 + threadIdx.x];
            sj[threadIdx.x] = j;
            sz[threadIdx.x] = ws.z[j];
            sC[threadIdx.x] = ws.geom[(size_t)(e0 + threadIdx.x) * 8 + 1];
        }
        const float x0 = __ldg(mw.emb + ws.z[i] * D + c);
        __syncthreads();
        float acc = 0.f;
#pragma unroll 2
        for (int k2 = half; k2 < dg; k2 += 2) {         // even edges on one half, odd edges on the other
            if (sj[k2] == i) continue;
            const float nbv = __ldg(mw.nb_emb + sz[k2] * D + c);
            float dp = bd;
#pragma unroll
            for (int k = 0; k < NR; k += 4) {
                const float4 rb = ldg4(ws.rbf + (size_t)(e0 + k2) * NR + k);
                dp = fmaf(rb.x, wd[k], dp); dp = fmaf(rb.y, wd[k + 1], dp);
                dp = fmaf(rb.z, wd[k + 2], dp); dp = fmaf(rb.w, wd[k + 3], dp);
            }
            acc = fmaf(dp * sC[k2], nbv, acc);
        }
        if (half == 1) part[nb][c] = acc;
        __syncthreads();                                // (also: sj / sz / sC free for the next node)
        if (half == 0) { cat[nb][c] = x0; cat[nb][D + c] = acc + part[nb][c]; }
    }
    __syncthreads();
    // x_i = [emb | agg] Wc^T + bc : each half takes 128 of the 256 k's
    const int kb = half * D;
    if constexpr (NB == 1) {
        float o[8];
#pragma unroll
        for (int u = 0; u < 8; u++) o[u] = 0.f;
#pragma unroll 2
        for (int k = 0; k < D; k += 8) {
#pragma unroll
            for (int u = 0; u < 8; u++) o[u] = fmaf(cat[0][kb + k + u], __ldg(mw.WcT + (size_t)(kb + k + u) * D + c), o[u]);
        }
        const float sum = ((o[0] + o[1]) + (o[2] + o[3])) + ((o[4] + o[5]) + (o[6] + o[7]));
        if (half == 1) part[0][c] = sum;
        __syncthreads();
        if (half == 0 && n0 < ws.N) ws.X[0][(size_t)n0 * D + c] = (__ldg(mw.bc + c) + sum) + part[0][c];
    } else {
        float o[NB];
#pragma unroll
        for (int nb = 0; nb < NB; nb++) o[nb] = 0.f;
#pragma unroll 8
        for (int k = 0; k < D; k++) {
            const float w = __ldg(mw.WcT + (size_t)(kb + k) * D + c);
#pragma unroll
            for (int nb = 0; nb < NB; nb++) o[nb] = fmaf(cat[nb][kb + k], w, o[nb]);
        }
        if (half == 1) {
#pragma unroll
            for (int nb = 0; nb < NB; nb++) part[nb][c] = o[nb];
        }
        __syncthreads();
        if (half == 0) {
            const float bcv = __ldg(mw.bc + c);
#pragma unroll
            for (int nb = 0; nb < NB; nb++)
                if (n0 + nb < ws.N) ws.X[0][(size_t)(n0 + nb) * D + c] = (bcv + o[nb]) + part[nb][c];
        }
    }
}

// Small-system variant of K4: FOUR nodes per CTA of 512 threads = 128 channels x 4 slices.  Slice q aggregates node q (all of
// its <= 32 edges, rbf rows and edge metadata staged in shared memory by the whole CTA), then multiplies K-slice q of the
// combine weight for all four nodes, so a CTA reads the 128 KB weight once for four nodes.  With one node per CTA the ~400
// CTAs of a small protein all pulled the same 128 KB through L2 at the same time and that, not latency, bounded the kernel
// (cutting its dependent load rounds did not change its time); for the
// same reason every CTA starts its walk over the weight rows at a different row.
constexpr int EMS_THREADS = 4 * D, EMS_NB = 4;
__global__ void __launch_bounds__(EMS_THREADS) embed_node_small_kernel(ModelW mw, Workspace ws, unsigned long long* tl) {
#define EMS_TL(i) do { if (tl != nullptr && blockIdx.x == 0 && (threadIdx.x & 31) == 0) tl[(i) * 16 + (threadIdx.x >> 5)] = (unsigned long long)clock64(); } while (0)
    EMS_TL(0);
    pdl_entry();
    EMS_TL(1);
    __shared__ __align__(16) float rbf_s[EMS_NB][KNB][NR];
    __shared__ __align__(16) float cat[EMS_NB][2 * D];
    __shared__ float part[3][EMS_NB][D];
    __shared__ int sj[EMS_NB][KNB];
    __shared__ int sz[EMS_NB][KNB];
    __shared__ float sC[EMS_NB][KNB];
    __shared__ int sdg[EMS_NB];
    const int c = threadIdx.x & (D - 1), q = threadIdx.x >> 7;
    const int n0 = blockIdx.x * EMS_NB;
    float wd[NR];
#pragma unroll
    for (int k = 0; k < NR; k++) wd[k] = __ldg(mw.WdT + k * D + c);     // coalesced (the [c][k] image costs 32 sectors per request)
    const float bd = __ldg(mw.bd + c);
    // combine weight rows of this slice (k in [64 q, 64 q + 64), walked from a row that differs from CTA to CTA): the first
    // half is requested now, the second as soon as the registers of the neighbour rows are free -- neither waits for the
    // aggregation
    const int kb = q * (D / 2), rot = ((int)blockIdx.x * 16) & (D / 2 - 1);
    float wc[32];
#pragma unroll
    for (int u = 0; u < 32; u++) wc[u] = __ldg(mw.WcT + (size_t)(kb + ((rot + u) & (D / 2 - 1))) * D + c);
    const int i = n0 + q;                                    // this slice's node
    const bool ok = i < ws.N;
    const int e0 = ok ? ws.rowptr[i] : 0, dg = ok ? ws.rowptr[i + 1] - e0 : 0;
    const float x0 = ok ? __ldg(mw.emb + ws.z[i] * D + c) : 0.f;
    if (c < dg) {
        const float4 g0 = ld4(ws.geom + (size_t)(e0 + c) * 8);
        const float4 g1 = ld4(ws.geom + (size_t)(e0 + c) * 8 + 4);
        sj[q][c] = ws.esrc[e0 + c];
        sC[q][c] = g0.y;
        sz[q][c] = __float_as_int(g1.z);                  // z of the source atom, left there by edge_geom
    }
    for (int idx = c; idx < dg * NR; idx += D) (&rbf_s[q][0][0])[idx] = ws.rbf[(size_t)e0 * NR + idx];
    if (c == 0) sdg[q] = dg;
    EMS_TL(2);
    __syncthreads();
    // slice q takes the edges q, q + 4, ... of ALL four nodes (a slice per node would wait for the node with the most
    // neighbours); the eight 32-deep products of a node are independent chains (select instead of branch)
    float accn[EMS_NB] = {0.f, 0.f, 0.f, 0.f};
    {
        constexpr int EPQ = KNB / 4;
        float nbv[EMS_NB][EPQ];
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++)
#pragma unroll
            for (int t = 0; t < EPQ; t++) {
                const int k2 = q + 4 * t;
                nbv[nd][t] = (k2 < sdg[nd] && sj[nd][k2] != n0 + nd) ? __ldg(mw.nb_emb + sz[nd][k2] * D + c) : 0.f;
            }
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++) {
            if (q >= sdg[nd]) continue;                     // (uniform per slice: none of this slice's edges exist)
#pragma unroll
            for (int t = 0; t < EPQ; t++) {
                const int k2 = q + 4 * t;
                const bool on = k2 < sdg[nd] && sj[nd][k2] != n0 + nd;
                float dp = bd;
#pragma unroll
                for (int k = 0; k < NR; k += 4) {
                    const float4 rb = ld4(&rbf_s[nd][on ? k2 : 0][k]);
                    dp = fmaf(rb.x, wd[k], dp); dp = fmaf(rb.y, wd[k + 1], dp);
                    dp = fmaf(rb.z, wd[k + 2], dp); dp = fmaf(rb.w, wd[k + 3], dp);
                }
                accn[nd] += on ? dp * sC[nd][k2] * nbv[nd][t] : 0.f;
            }
        }
    }
    float wc2[32];
#pragma unroll
    for (int u = 0; u < 32; u++) wc2[u] = __ldg(mw.WcT + (size_t)(kb + ((rot + 32 + u) & (D / 2 - 1))) * D + c);
    cat[q][c] = x0;
    if (q > 0) {
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++) part[q - 1][nd][c] = accn[nd];
    }
    __syncthreads();
    if (q == 0) {
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++) cat[nd][D + c] = ((accn[nd] + part[0][nd][c]) + part[1][nd][c]) + part[2][nd][c];
    }
    EMS_TL(3);
    __syncthreads();
    // x = [emb | agg] Wc^T + bc : slice q multiplies its 64 k's for the four nodes
    float o[EMS_NB] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 32; u++) {
        const int k = kb + ((rot + u) & (D / 2 - 1));
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++) o[nd] = fmaf(cat[nd][k], wc[u], o[nd]);
    }
#pragma unroll
    for (int u = 0; u < 32; u++) {
        const int k = kb + ((rot + 32 + u) & (D / 2 - 1));
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++) o[nd] = fmaf(cat[nd][k], wc2[u], o[nd]);
    }
    if (q > 0) {
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++) part[q - 1][nd][c] = o[nd];
    }
    EMS_TL(4);
    __syncthreads();
    if (q == 0) {
        const float bcv = __ldg(mw.bc + c);
#pragma unroll
        for (int nd = 0; nd < EMS_NB; nd++)
            if (n0 + nd < ws.N) ws.X[0][(size_t)(n0 + nd) * D + c] = (bcv + ((o[nd] + part[0][nd][c]) + part[1][nd][c])) + part[2][nd][c];
    }
    EMS_TL(5);
#undef EMS_TL
}

// K5: edge embedding  f0_e[c] = (x_i[c] + x_j[c]) * (rbf_e . We[c,:] + be[c]).   thread = channel, four edges per pass.
// The four rbf rows reach the block as ONE coalesced load per thread (shared memory, read back as broadcasts): the former
// 32 same-address global loads per thread and edge kept the load queue full and every chain waiting (ncu: 52 % of the
// samples at the first fma).
__global__ void __launch_bounds__(128) embed_edge_kernel(ModelW mw, Workspace ws) {
    pdl_entry();
    constexpr int EU = 4;
    __shared__ __align__(16) float rbf_s[EU][NR];
    const int c = threadIdx.x;
    float we[NR];
#pragma unroll
    for (int k = 0; k < NR; k++) we[k] = __ldg(mw.WeT + k * D + c);     // coalesced
    const float be = __ldg(mw.be + c);
    const int E = ws.rowptr[ws.N];
    const float* __restrict__ X = ws.X[0];
    for (int e0 = blockIdx.x * EU; e0 < E; e0 += gridDim.x * EU) {
        {
            const int e = e0 + (c >> 5);
            rbf_s[c >> 5][c & 31] = (e < E) ? ws.rbf[(size_t)e * NR + (c & 31)] : 0.f;
        }
        int ii[EU], jj[EU];
#pragma unroll
        for (int u = 0; u < EU; u++) {
            const int e = min(e0 + u, E - 1);
            ii[u] = ws.edst[e]; jj[u] = ws.esrc[e];
        }
        float xs[EU], ep[EU];
#pragma unroll
        for (int u = 0; u < EU; u++) { xs[u] = X[(size_t)ii[u] * D + c] + X[(size_t)jj[u] * D + c]; ep[u] = be; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < NR; k += 4) {
#pragma unroll
            for (int u = 0; u < EU; u++) {
                const float4 rb = ld4(&rbf_s[u][k]);
                ep[u] = fmaf(rb.x, we[k], ep[u]); ep[u] = fmaf(rb.y, we[k + 1], ep[u]);
                ep[u] = fmaf(rb.z, we[k + 2], ep[u]); ep[u] = fmaf(rb.w, we[k + 3], ep[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < EU; u++)
            if (e0 + u < E) ws.F[0][(size_t)(e0 + u) * D + c] = xs[u] * ep[u];
        __syncthreads();                                    // rbf_s is rewritten by the next pass
    }
}

// ---------------------------------------------------------------------------------------------
// K14: adjoint of the edge embedding.  gf = dE/df0 (in ws.GF).  One warp per edge, no block barriers:
//   phase A (lane = 4 channels): ep = rbf.We^T + be ; gx_i += gf*ep, gx_j += gf*ep ; g_ep = gf*(x_i+x_j) -> smem
//   phase B (lane = rbf index k): g_rbf[e][k] = sum_c g_ep[c] * We[c][k]
// ---------------------------------------------------------------------------------------------
constexpr int EEB_WARPS = 8;
__global__ void __launch_bounds__(EEB_WARPS * 32) embed_edge_bwd_kernel(ModelW mw, Workspace ws) {
    pdl_entry();
    __shared__ __align__(16) float WeT_s[NR][D];          // [k][c]
    __shared__ float WeN_s[D][NR + 1];                    // [c][k] (+1: conflict-free column walks)
    __shared__ __align__(16) float gep_s[EEB_WARPS][2][D];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, col = lane * 4;
    for (int idx = threadIdx.x; idx < D * NR; idx += blockDim.x) {        // both images copied with consecutive addresses
        WeT_s[idx / D][idx % D] = __ldg(mw.WeT + idx);                    // (the former in-kernel transpose wrote 32-way bank conflicts)
        WeN_s[idx / NR][idx % NR] = __ldg(mw.WeN + idx);
    }
    __syncthreads();
    const float4 be = ldg4(mw.be + col);
    const int E = ws.rowptr[ws.N];
    const float* __restrict__ X = ws.X[0];
    // two edges per warp and pass: phase B reads every weight once for both and runs four independent fma chains
    for (int e0 = (blockIdx.x * EEB_WARPS + warp) * 2; e0 < E; e0 += gridDim.x * EEB_WARPS * 2) {
        const bool two = e0 + 1 < E;
        const int e1 = two ? e0 + 1 : e0;
        const int i0 = ws.edst[e0], j0 = ws.esrc[e0], i1 = ws.edst[e1], j1 = ws.esrc[e1];
        const float rk0 = __ldg(ws.rbf + (size_t)e0 * NR + lane), rk1 = __ldg(ws.rbf + (size_t)e1 * NR + lane);
        const float4 gf0 = ld4(ws.GF + (size_t)e0 * D + col), gf1 = ld4(ws.GF + (size_t)e1 * D + col);
        const float4 xs0 = ldg4(X + (size_t)i0 * D + col) + ldg4(X + (size_t)j0 * D + col);
        const float4 xs1 = ldg4(X + (size_t)i1 * D + col) + ldg4(X + (size_t)j1 * D + col);
        float4 ep0 = be, ep1 = be;
#pragma unroll
        for (int k = 0; k < NR; k++) {
            const float4 w = ld4(&WeT_s[k][col]);
            ep0 = ep0 + w * __shfl_sync(0xffffffffu, rk0, k);
            ep1 = ep1 + w * __shfl_sync(0xffffffffu, rk1, k);
        }
        const float4 gfe0 = gf0 * ep0, gfe1 = gf1 * ep1;
        red4(ws.GX + (size_t)i0 * D + col, gfe0);
        red4(ws.GX + (size_t)j0 * D + col, gfe0);
        if (two) {
            red4(ws.GX + (size_t)i1 * D + col, gfe1);
            red4(ws.GX + (size_t)j1 * D + col, gfe1);
        }
        __syncwarp();
        st4(&gep_s[warp][0][col], gf0 * xs0);
        st4(&gep_s[warp][1][col], gf1 * xs1);
        __syncwarp();
        float ga[2] = {0.f, 0.f}, gb[2] = {0.f, 0.f};
#pragma unroll 8
        for (int c = 0; c < D; c += 2) {
            const float w0 = WeN_s[c][lane], w1 = WeN_s[c + 1][lane];
            const float2 a = *reinterpret_cast<const float2*>(&gep_s[warp][0][c]);
            const float2 b = *reinterpret_cast<const float2*>(&gep_s[warp][1][c]);
            ga[0] = fmaf(a.x, w0, ga[0]); ga[1] = fmaf(a.y, w1, ga[1]);
            gb[0] = fmaf(b.x, w0, gb[0]); gb[1] = fmaf(b.y, w1, gb[1]);
        }
        ws.grbf[(size_t)e0 * NR + lane] = ga[0] + ga[1];
        if (two) ws.grbf[(size_t)e1 * NR + lane] = gb[0] + gb[1];
    }
}

// ---------------------------------------------------------------------------------------------
// K15: adjoint of the neighbour embedding + geometry adjoint + force accumulation.  One block (4 warps) per target
// node i (needs the complete gx); each warp takes every 4th edge of the node, no block barriers in the edge loop:
//   g_agg = (gx_i Wc)[128:256]
//   phase A (lane = 4 channels): dp = rbf.Wd^T + bd ; g_We = g_agg * nb[z_j] ; gC += sum_c g_We*dp ; g_We*C -> smem
//   phase B (lane = rbf index k): g_rbf[k] += sum_c g_We[c]*C*Wd[c][k] ; g_r = gC*C'(r) + sum_k g_rbf[k]*drbf_k/dr
//   g_ev = g_r d + (g_d - (g_d.d) d)/r ; dE/dpos_j += g_ev, dE/dpos_i -= g_ev ; forces = -dE/dpos
// ---------------------------------------------------------------------------------------------
constexpr int ENB_WARPS = 8;
__global__ void __launch_bounds__(ENB_WARPS * 32) embed_node_bwd_kernel(ModelW mw, Workspace ws,
                                                                        float* __restrict__ forces) {
    pdl_entry();
    __shared__ __align__(16) float WdT_s[NR][D];
    __shared__ float WdN_s[D][NR + 1];
    __shared__ __align__(16) float gx_s[D];
    __shared__ __align__(16) float gagg_s[ENB_WARPS][D];
    __shared__ __align__(16) float gwe_s[ENB_WARPS][D];
    __shared__ float fi_s[ENB_WARPS][3];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, col = lane * 4;
    for (int idx = threadIdx.x; idx < D * NR; idx += ENB_WARPS * 32) {      // once per CTA (a CTA walks several nodes of a batch)
        WdT_s[idx / D][idx % D] = __ldg(mw.WdT + idx);
        WdN_s[idx / NR][idx % NR] = __ldg(mw.WdN + idx);
    }
    const float alpha = 5.0f / mw.cutoff;
    const float mu = __ldg(mw.rbf_means + lane), beta = __ldg(mw.rbf_betas + lane);
    const float4 bd = ldg4(mw.bd + col);
    for (int i = blockIdx.x; i < ws.N; i += gridDim.x) {
    __syncthreads();                                    // previous node's shared rows are consumed; weights visible
    if (threadIdx.x < D) gx_s[threadIdx.x] = ws.GX[(size_t)i * D + threadIdx.x];
    __syncthreads();
    // g_agg = (gx_i Wc)[128:256]: K split over the warps (16 k's each, all loads in flight), fixed-order sum
    {
        constexpr int KW = D / ENB_WARPS;
        float4 part = f4s(0.f);
#pragma unroll
        for (int k = 0; k < KW; k++)
            part = part + ldg4(mw.WcN + (size_t)(warp * KW + k) * 2 * D + D + col) * gx_s[warp * KW + k];
        st4(&gagg_s[warp][col], part);
    }
    __syncthreads();
    float4 g_agg = f4s(0.f);
#pragma unroll
    for (int w = 0; w < ENB_WARPS; w++) g_agg = g_agg + ld4(&gagg_s[w][col]);
    float fix = 0.f, fiy = 0.f, fiz = 0.f;
    const int e1 = ws.rowptr[i + 1];
    // the (at most 4) edges of this warp: every row they need is requested before the first is used -- two L2 round trips
    // for the node instead of three per edge (edge data, then the neighbour-embedding rows by the z that edge_geom left in geom[6])
    constexpr int EPW = KNB / ENB_WARPS;
    float4 g0r[EPW], g1r[EPW], ear[EPW], nbr[EPW];
    float rkr[EPW], grr[EPW];
    int jr[EPW];
#pragma unroll
    for (int t = 0; t < EPW; t++) {
        const int e = ws.rowptr[i] + warp + t * ENB_WARPS;
        const bool on = e < e1;
        const int ec = on ? e : e1 - 1;                      // (e1 > rowptr[i]: every atom has its self loop)
        jr[t] = on ? ws.esrc[ec] : i;
        g0r[t] = ld4(ws.geom + (size_t)ec * 8);
        g1r[t] = ld4(ws.geom + (size_t)ec * 8 + 4);
        rkr[t] = __ldg(ws.rbf + (size_t)ec * NR + lane);
        ear[t] = ld4(ws.eacc + (size_t)ec * 4);
        grr[t] = ws.grbf[(size_t)ec * NR + lane];
    }
#pragma unroll
    for (int t = 0; t < EPW; t++) nbr[t] = ldg4(mw.nb_emb + __float_as_int(g1r[t].z) * D + col);
#pragma unroll
    for (int t = 0; t < EPW; t++) {
        const int j = jr[t];
        if (j == i) continue;     // self-loops carry no geometry and are masked out of the neighbour embedding (also: no edge)
        const float4 g0 = g0r[t], g1 = g1r[t];
        const float r = g0.x, Ce = g0.y, dx = g0.z, dy = g0.w, dz = g1.x, inv_r = g1.y;
        const float rk = rkr[t];
        const float4 nbj = nbr[t];
        const float4 ea = ear[t];
        const float grbf0 = grr[t];
        float4 dp = bd;
#pragma unroll
        for (int k = 0; k < NR; k++) dp = dp + ld4(&WdT_s[k][col]) * __shfl_sync(0xffffffffu, rk, k);
        const float4 gwe = g_agg * nbj;
        const float gc = warp_sum(hsum4(gwe * dp));
        __syncwarp();
        st4(&gwe_s[warp][col], gwe * Ce);
        __syncwarp();
        float g4[4] = {0.f, 0.f, 0.f, 0.f};               // four independent chains instead of one 128-deep one
#pragma unroll 4
        for (int cc = 0; cc < D; cc += 4) {
            const float4 gw = ld4(&gwe_s[warp][cc]);
            g4[0] = fmaf(gw.x, WdN_s[cc][lane], g4[0]); g4[1] = fmaf(gw.y, WdN_s[cc + 1][lane], g4[1]);
            g4[2] = fmaf(gw.z, WdN_s[cc + 2][lane], g4[2]); g4[3] = fmaf(gw.w, WdN_s[cc + 3][lane], g4[3]);
        }
        const float g = (g4[0] + g4[1]) + (g4[2] + g4[3]);
        const float gC = ea.x + gc;
        const float grbf = grbf0 + g;
        const float ex = __expf(-alpha * r);
        const float tt = ex - mu;
        const float gk = __expf(-beta * tt * tt);
        const float dC = cutoff_dfn(r, mw.cutoff);
        const float drbf = dC * gk + Ce * gk * (2.0f * beta * alpha) * tt * ex;
        const float g_r = gC * dC + warp_sum(grbf * drbf);
        if (lane == 0) {
            const float gdd = ea.y * dx + ea.z * dy + ea.w * dz;
            const float gx_ = g_r * dx + (ea.y - gdd * dx) * inv_r;
            const float gy_ = g_r * dy + (ea.z - gdd * dy) * inv_r;
            const float gz_ = g_r * dz + (ea.w - gdd * dz) * inv_r;
            // dE/dpos_j += g_ev  -> F_j -= g_ev ; dE/dpos_i -= g_ev -> F_i += g_ev
            atomicAdd(forces + 3 * j, -gx_);
            atomicAdd(forces + 3 * j + 1, -gy_);
            atomicAdd(forces + 3 * j + 2, -gz_);
            fix += gx_; fiy += gy_; fiz += gz_;
        }
    }
    if (lane == 0) { fi_s[warp][0] = fix; fi_s[warp][1] = fiy; fi_s[warp][2] = fiz; }
    __syncthreads();
    if (threadIdx.x < 3) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < ENB_WARPS; w++) t += fi_s[w][threadIdx.x];
        atomicAdd(forces + 3 * i + threadIdx.x, t);
    }
    }
}

}  // namespace vb
