// Non-bonded MM term of the fragment calculator (SURVEY §8f rank 2): all ordered atom pairs (src j, dst i), i != j,
// not inside a common dipeptide, Lennard-Jones (Lorentz-Berthelot) + Coulomb, forces accumulated on dst, energy halved.
// Reference: MMNonBondedCalculator.__call__, src/Calculators/nonbonded.py:34-63; pair list Protein.initial_mm_adjmatrix,
// src/AIMD/protein.py:133-151; exclusions src/Fragmentation/distancefrag.py:355-363.  fp32 arithmetic in the
// reference's operation order per pair; per-atom sums are warp-ordered (the reference's scatter_add is atomic-ordered).
// The pair list is never materialised: a warp owns one destination atom and walks all sources; the excluded partners of
// that atom (a short sorted list) are binary-searched.
#pragma once
#include <cuda_runtime.h>

namespace vb {

struct NbParams {
    int n;                        // protein atoms
    int lo, hi;                   // destination atoms this rank owns
    const float* q;               // [n] charges (e)
    const float* sigma;           // [n] nm
    const float* eps;             // [n] kJ/mol
    const int* excl_rowptr;       // [n+1]
    const int* excl_col;          // sorted within a row
    float coulomb_k;              // 1/(4 pi eps0) in kJ/mol * Angstrom / e^2  (nonbonded.py:18)
    float kj_mol;                 // kJ/mol in eV
};

// FORCES = false is the energy-only instantiation: the same per-pair energy arithmetic and lane order, so e_atom is
// bit-identical to the full kernel's, without the force sums and the ef row stores (and ef is not read).
template <typename PosT, bool FORCES = true>
__global__ void __launch_bounds__(256) nonbonded_kernel(NbParams p, const PosT* __restrict__ pos, float* __restrict__ ef,
                                                        double* __restrict__ e_atom) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int i = p.lo + warp;
    if (i >= p.hi) return;
    const float xi = (float)pos[3 * i], yi = (float)pos[3 * i + 1], zi = (float)pos[3 * i + 2];
    const float qi = p.q[i], si = p.sigma[i], ei = p.eps[i];
    const int x0 = p.excl_rowptr[i], x1 = p.excl_rowptr[i + 1];
    float fx = 0.f, fy = 0.f, fz = 0.f;
    double e = 0.0;
    for (int j = lane; j < p.n; j += 32) {
        if (j == i) continue;
        int a = x0, b = x1;                       // binary search of j among the excluded partners of i
        while (a < b) {
            const int m = (a + b) >> 1;
            if (p.excl_col[m] < j) a = m + 1; else b = m;
        }
        if (a < x1 && p.excl_col[a] == j) continue;
        // vec = pos[dst] - pos[src]   (nonbonded.py:41-43)
        const float vx = xi - (float)pos[3 * j], vy = yi - (float)pos[3 * j + 1], vz = zi - (float)pos[3 * j + 2];
        // d2 and the LJ bracket are spelled out as the compiler contracts them in the force kernel, so that the energy-only
        // instantiation, where c12 has one use, cannot contract them otherwise (the force kernel's code is unchanged)
        const float d2 = fmaf(vz, vz, fmaf(vx, vx, vy * vy));
        const float d = sqrtf(d2);
        // LJ (nonbonded.py:46-51)
        const float sij = 0.5f * (p.sigma[j] + si) * 10.0f;
        const float eij = sqrtf(p.eps[j] * ei);
        const float t = sij * sij / d2;
        const float c6 = t * t * t, c12 = c6 * c6;
        const float e_lj = 4.0f * eij * __fsub_rn(c12, c6);
        const float f_lj = 24.0f * eij * (2.0f * c12 - c6) / d2;
        // Coulomb (nonbonded.py:54-55)
        const float e_c = p.coulomb_k * p.q[j] * qi / d;
        const float f_c = e_c / d2;
        if (FORCES) {
            const float f = f_lj + f_c;
            fx += f * vx; fy += f * vy; fz += f * vz;
        }
        e += (double)e_lj + (double)e_c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        if (FORCES) {
            fx += __shfl_xor_sync(0xffffffffu, fx, o); fy += __shfl_xor_sync(0xffffffffu, fy, o);
            fz += __shfl_xor_sync(0xffffffffu, fz, o);
        }
        e += __shfl_xor_sync(0xffffffffu, e, o);
    }
    if (lane == 0) {
        if (FORCES) { ef[3 * i] += fx * p.kj_mol; ef[3 * i + 1] += fy * p.kj_mol; ef[3 * i + 2] += fz * p.kj_mol; }
        e_atom[i] = e;
    }
}

// E += (sum_i e_atom[i]) * kJ/mol / 2 over the owned atoms, fixed order (nonbonded.py:58,61)
__global__ void __launch_bounds__(256) nonbonded_energy_kernel(NbParams p, const double* __restrict__ e_atom, float* __restrict__ ef) {
    __shared__ double red[8];
    double s = 0.0;
    for (int i = p.lo + threadIdx.x; i < p.hi; i += 256) s += e_atom[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; w++) t += red[w];
        ef[3 * p.n] += (float)(t * (double)p.kj_mol * 0.5);
    }
}

}  // namespace vb
