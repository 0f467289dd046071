// Node stage on tensor cores (wgmma / TMA weight ring, 3xTF32): the dense node-feature x weight contractions of a
// ViS_MP layer -- q/k/v, vec_proj, w_trg/w_src, o_proj and their adjoints -- as 128-row GEMM tiles, one (row tile, column
// chunk) job per CTA for small systems (every CTA streams ONE 128 KB weight image instead of the layer's whole 720 KB, and
// the jobs of a stage spread over ~60-70 SMs), all chunks of a row tile in one CTA for large batches (A staged once).
//   reference math: visnet_block.py:237-250 (LayerNorm, VecLayerNorm, q/k/v, vec_proj), :271-273 (o_proj + updates),
//                   :291-292 (w_src / w_trg), utils.py:200-249 (VecLayerNorm max_min).
// A stage is three launches; the element-wise glue between the GEMMs is a warp-per-node SIMT kernel:
//   forward  k :  oproj   O   = xa Wo^T + bo                                   [N x 128] x 3 chunks   (k >= 1)
//                 norm    x, vec updates, LayerNorm, VecLayerNorm, vec_dot of the previous layer, xa / va re-zeroed
//                 proj    [q|k|v] = LN(x) Wqkv^T + b ;  [v1|v2|v3|t|u] = VecLN(vec) [Wvec|Wtu]^T     (k <  L)
//   backward k :  bwdA    partial products of the three K = 384 / 256 adjoint contractions, one 128-wide K chunk per CTA:
//                         g_qkv Wqkv, [g_vdot v2 | g_vdot v1 | g_vec o1] Wvec, g_tu Wtu                (k <= L-1)
//                 bnorm   fixed-order sum of the partials, VecLayerNorm / LayerNorm adjoints, accumulators re-zeroed,
//                         rows of the next product [g_o1 | g_x vdot | g_x]
//                 bwdB    dE/dxa = [g_o1 | g_x vdot | g_x] Wo as three K-chunk partials (summed by the edge adjoint) (k >= 1)
// Vector rows are the flat [3N][128] view of the [N][3][128] tensors (row = 3 * node + s): a 128-row tile is dense.
#pragma once
#include "k_edge_tc.cuh"
#include "k_node.cuh"

namespace vb {

enum { NT_OPROJ = 0, NT_PROJ = 1, NT_BWDA = 2, NT_BWDB = 3 };

struct NodeTcArgs {
    int layer;              // stage k
    ModelW mw;
    Workspace ws;
    int tx, tv;             // row tiles of the scalar rows (N) and of the vector rows (3N); tv = 0: no vector items
    int njx, njv;           // jobs (128-column chunks forward, 128-deep K chunks backward) per scalar / vector row tile
    int jx, jv;             // jobs one CTA runs (divides njx / njv)
    TcJob jobs_x[3];
    TcJob jobs_v[5];
    const float* acc_qkv;   // backward: accumulators the edge adjoint of layer k added into
    const float* acc_tu;
};

// ---------------------------------------------------------------------------------------------------------
// GEMM kernels: one row tile, `nj` jobs sharing one A operand (forward) or one job with its own A (backward)
// ---------------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(TC2_THREADS, 1) node_tc_kernel(const __grid_constant__ NodeTcArgs a) {
    pdl_entry();
    extern __shared__ __align__(1024) uint8_t dyn_raw[];
    TcShared& sh = *tc_shared_base(dyn_raw);
    __shared__ TcJob jl[5];
    const Workspace& ws = a.ws;
    const int k = a.layer;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, col = lane * 4;
    // ---- which item is this CTA? ----
    const int gx = a.njx / a.jx;                       // CTAs per scalar row tile
    const int nx_items = a.tx * gx;
    const bool is_x = (int)blockIdx.x < nx_items;
    int tile, j0, nj;
    if (is_x) { tile = (int)blockIdx.x / gx; j0 = ((int)blockIdx.x % gx) * a.jx; nj = a.jx; }
    else { const int b = (int)blockIdx.x - nx_items, gv = a.njv / a.jv; tile = b / gv; j0 = (b % gv) * a.jv; nj = a.jv; }
    const int total_rows = is_x ? ws.N : 3 * ws.N;
    const int row0 = tile * TC_TE;
    const int nvalid = min(TC_TE, total_rows - row0);
    constexpr bool KCHUNKS = (MODE == NT_BWDA || MODE == NT_BWDB);     // jobs = K chunks accumulated into one product
    if (threadIdx.x < nj) {
        TcJob j = is_x ? a.jobs_x[j0 + threadIdx.x] : a.jobs_v[j0 + threadIdx.x];
        j.accumulate = (KCHUNKS && threadIdx.x > 0) ? 1 : 0;
        jl[threadIdx.x] = j;
    }
    TcRing<TC_TE> ring;
    tc2_setup(sh, ring, jl, nj, 1);                    // (its __syncthreads publishes jl)

    float acc[32];
    // A operand rows of job jj -> staging tile (warp per row, lane owns 4 channels: coalesced 512 B rows)
    auto load_a = [&](int jj) {
        for (int r = warp; r < nvalid; r += TC2_CWARPS) {
            const size_t row = (size_t)(row0 + r);
            float4 v;
            if (MODE == NT_OPROJ) {
                v = ld4(ws.XA + row * D + col);
            } else if (MODE == NT_PROJ) {
                v = is_x ? ld4(ws.XN + row * D + col) : ld4(ws.VN[k] + row * D + col);
            } else if (MODE == NT_BWDA) {
                if (is_x) {
                    v = ld4(a.acc_qkv + row * 3 * D + jj * D + col);
                } else if (jj >= 3) {
                    v = ld4(a.acc_tu + row * 2 * D + (jj - 3) * D + col);
                } else {
                    const size_t node = row / 3;
                    const float* orow = ws.O[k] + node * 3 * D;
                    if (jj == 2) {
                        v = ld4(ws.GVEC + row * D + col) * ld4(orow + col);                         // g_vec * o1
                    } else {
                        const float4 g_vdot = ld4(ws.GX + node * D + col) * ld4(orow + D + col);    // g_x * o2
                        v = g_vdot * ld4(ws.V123[k] + row * 3 * D + (jj == 0 ? D : 0) + col);       // * v2 | * v1
                    }
                }
            } else {
                v = ld4(ws.GO + row * 3 * D + jj * D + col);
            }
            st4(&sh.tile[r][col], v);
        }
    };
    if (!KCHUNKS) {
        // ---- column chunks of one product: one A operand ----
        load_a(0);
        tc2_tile_to_a(sh, nvalid);
        for (int j = 0; j < nj; j++) {
            tc2_mma(sh, ring, sh.abuf, acc, jl[j].accumulate, warp, lane, nvalid);
            csync();                                          // the tile is free (A copied / previous chunk stored)
            tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
            csync();
            const int jj = j0 + j;
            for (int r = warp; r < nvalid; r += TC2_CWARPS) {
                const size_t row = (size_t)(row0 + r);
                const float4 v = ld4(&sh.tile[r][col]);
                if (MODE == NT_OPROJ) {
                    st4(ws.O[k - 1] + row * 3 * D + jj * D + col, v + ldg4(a.mw.layer[k - 1].bo + jj * D + col));
                } else {
                    if (is_x) st4(ws.QKV[k] + row * 3 * D + jj * D + col, v + ldg4(a.mw.layer[k].bqkv + jj * D + col));
                    else if (jj < 3) st4(ws.V123[k] + row * 3 * D + jj * D + col, v);
                    else st4(ws.TU[k] + row * 2 * D + (jj - 3) * D + col, v);
                }
            }
        }
    } else {
        // ---- K chunks of one product: every chunk has its own A operand, all accumulate into one product; with one
        //      chunk per CTA the result is the partial of chunk j0 (the glue kernel / the edge adjoint sums the partials) ----
        for (int j = 0; j < nj; j++) {
            load_a(j0 + j);                                   // (the previous chunk's MMAs began with a barrier: tile free)
            tc2_tile_to_a(sh, nvalid);
            tc2_mma(sh, ring, sh.abuf, acc, jl[j].accumulate, warp, lane, nvalid);
        }
        csync();
        tc2_acc_to(sh.tile, acc, warp, lane, nvalid);
        csync();
        for (int r = warp; r < nvalid; r += TC2_CWARPS) {
            const size_t row = (size_t)(row0 + r);
            const float4 v = ld4(&sh.tile[r][col]);
            if (MODE == NT_BWDA) {
                if (is_x) st4(ws.PX + ((size_t)j0 * ws.N + row) * D + col, v);
                else st4(ws.PV + ((size_t)j0 * 3 * ws.N + row) * D + col, v);
            } else {
                st4(ws.GXA + ((size_t)j0 * ws.N + row) * D + col, v);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// forward glue (warp per node): residual update, LayerNorm, VecLayerNorm   (the per-node phase of node_fwd2_kernel)
// ---------------------------------------------------------------------------------------------------------
constexpr int NN_WARPS = 8;
__global__ void __launch_bounds__(NN_WARPS * 32) node_norm_fwd_kernel(int k, ModelW mw, Workspace ws) {
    pdl_entry();
    const int lane = threadIdx.x & 31, col = lane * 4;
    const int node = blockIdx.x * NN_WARPS + (threadIdx.x >> 5);
    if (node >= ws.N) return;
    float4 x, vec[3];
    if (k >= 1) {
        const float* orow = ws.O[k - 1] + (size_t)node * 3 * D;
        const float4 o1 = ld4(orow + col), o2 = ld4(orow + D + col), o3 = ld4(orow + 2 * D + col);
        float4 vd = f4s(0.f), v3[3];
#pragma unroll
        for (int s = 0; s < 3; s++) {
            const float* vr = ws.V123[k - 1] + ((size_t)node * 3 + s) * 3 * D;
            vd = vd + ld4(vr + col) * ld4(vr + D + col);
            v3[s] = ld4(vr + 2 * D + col);
        }
        st4(ws.VDOT[k - 1] + (size_t)node * D + col, vd);
        x = ld4(ws.X[k - 1] + (size_t)node * D + col) + vd * o2 + o3;
        st4(ws.X[k] + (size_t)node * D + col, x);
#pragma unroll
        for (int s = 0; s < 3; s++) {
            const size_t r3 = (size_t)node * 3 + s;
            vec[s] = ld4(ws.V[k - 1] + r3 * D + col) + v3[s] * o1 + ld4(ws.VA + r3 * D + col);
            st4(ws.V[k] + r3 * D + col, vec[s]);
            st4(ws.VA + r3 * D + col, f4s(0.f));
        }
        st4(ws.XA + (size_t)node * D + col, f4s(0.f));
    } else {
        x = ld4(ws.X[0] + (size_t)node * D + col);
        vec[0] = vec[1] = vec[2] = f4s(0.f);
    }
    if (k < L) {
        const LayerW& lw = mw.layer[k];
        st4(ws.XN + (size_t)node * D + col, ln_forward(x, lw.ln_w, lw.ln_b, lane));
        float4 vn[3];
        vecln_forward(vec, vn, lw.vln_w, lane);
#pragma unroll
        for (int s = 0; s < 3; s++) st4(ws.VN[k] + ((size_t)node * 3 + s) * D + col, vn[s]);
    }
}

// ---------------------------------------------------------------------------------------------------------
// backward glue (warp per node): the per-node phase of node_bwd2_kernel around the partial products
// ---------------------------------------------------------------------------------------------------------
// `split`: the products arrive as one partial per K chunk (3 scalar, 3 + 2 vector) to be summed here; otherwise chunk 0
// holds the complete product (the GEMM CTA accumulated its chunks).
__global__ void __launch_bounds__(NN_WARPS * 32) node_norm_bwd_kernel(int k, ModelW mw, Workspace ws, float* __restrict__ GQKV,
                                                                      float* __restrict__ GVNMSG, float* __restrict__ GTU, int split) {
    pdl_entry();
    const int lane = threadIdx.x & 31, col = lane * 4;
    const int node = blockIdx.x * NN_WARPS + (threadIdx.x >> 5);
    if (node >= ws.N) return;
    const bool has_a = (k <= L - 1), has_b = (k >= 1), has_tu = (k < L - 1);
    const float4 z4 = f4s(0.f);
    const size_t N = ws.N;
    float4 gx = ld4(ws.GX + (size_t)node * D + col), gvec[3];
#pragma unroll
    for (int s = 0; s < 3; s++) gvec[s] = ld4(ws.GVEC + ((size_t)node * 3 + s) * D + col);
    if (has_a) {
        const LayerW& lw = mw.layer[k];
        float4 gxn = ld4(ws.PX + (0 * N + node) * D + col);
        if (split) gxn = (gxn + ld4(ws.PX + (1 * N + node) * D + col)) + ld4(ws.PX + (2 * N + node) * D + col);
        float4 vin[3], gout[3], gv[3];
#pragma unroll
        for (int s = 0; s < 3; s++) {
            const size_t r3 = (size_t)node * 3 + s;
            float4 g = ld4(GVNMSG + r3 * D + col);
            if (split) {
                g = g + ((ld4(ws.PV + (0 * 3 * N + r3) * D + col) + ld4(ws.PV + (1 * 3 * N + r3) * D + col)) + ld4(ws.PV + (2 * 3 * N + r3) * D + col));
                if (has_tu) g = g + (ld4(ws.PV + (3 * 3 * N + r3) * D + col) + ld4(ws.PV + (4 * 3 * N + r3) * D + col));
            } else {
                g = g + ld4(ws.PV + r3 * D + col);
            }
            gout[s] = g;
            vin[s] = ld4(ws.V[k] + r3 * D + col);
        }
        vecln_backward(vin, gout, gv, lw.vln_w, lane);
#pragma unroll
        for (int s = 0; s < 3; s++) gvec[s] = gvec[s] + gv[s];
        gx = gx + ln_backward(ld4(ws.X[k] + (size_t)node * D + col), gxn, lw.ln_w, lane);
    }
    {
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
        for (int s = 0; s < 3; s++) go1 = go1 + gvec[s] * ld4(ws.V123[k - 1] + ((size_t)node * 3 + s) * 3 * D + 2 * D + col);
        float* go = ws.GO + (size_t)node * 3 * D;
        st4(go + col, go1);
        st4(go + D + col, gx * ld4(ws.VDOT[k - 1] + (size_t)node * D + col));
        st4(go + 2 * D + col, gx);
    }
}

}  // namespace vb
