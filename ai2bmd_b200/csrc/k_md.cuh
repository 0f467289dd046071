// Device-resident MD step around the force evaluation (SURVEY §8f rank 3 and the first half of rank 1):
//   * Langevin / velocity-Verlet update of the whole-protein state -- the integrator the reference drives through
//     ASE (src/AIMD/simulator.py:96-137: Langevin, dt = 1 fs, 300 K, friction 0.001/fs; ASE 3.22 ase/md/langevin.py,
//     recalled, restated on the host in ai2bmd_b200/md.py which is this file's checker);
//   * placement of every packed fragment atom from the protein coordinates, cap hydrogens on the acceptor->removed ray
//     (src/Fragmentation/distancefrag.py:34-54; host restatement ai2bmd_b200/pdbfrag.py FragmentRecipe.positions).
//   * optional Hookean position / bond restraints on top of the calculator forces (see MdRestraints below).
// State (positions, velocities) is fp64 like ASE's numpy arrays; forces arrive as the fp32 whole-protein buffer
// [3*n_protein + 1] the signed fragment reduction writes.  Normals come from a counter-based Philox4x32-10 stream
// keyed by (seed; step, component), so every rank of a sharded run draws identical numbers without communication.
// An optional frame recorder (MdRecorder below) keeps every record step's state in a device ring and stops the
// integration itself when the temperature runs away, so an observed run needs no host round trip per frame.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vb {

struct MdParams {
    int n_protein;
    double dt, kT, fr;          // ASE units: Angstrom*sqrt(amu/eV), eV, 1/time
    unsigned long long seed;
    const double* pool;         // optional externally supplied normals [pool_steps][2][3*n_protein] (tests), else nullptr
    long long pool_steps;
};

// ---- Philox4x32-10 (Salmon et al. 2011), counter = (c0..c3), key = (k0, k1) -------------------------------
__host__ __device__ inline void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n1 = (uint32_t)p1;
        const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1, n3 = (uint32_t)p0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}

// two independent standard normals (xi, eta) for (step, component): Box-Muller on two 53-bit uniforms in (0, 1]
__device__ inline void md_normals(const MdParams& p, long long step, int comp, double& xi, double& eta) {
    if (p.pool != nullptr) {
        const size_t n3 = 3 * (size_t)p.n_protein;
        const double* row = p.pool + (size_t)(step % p.pool_steps) * 2 * n3;
        xi = row[comp]; eta = row[n3 + comp];
        return;
    }
    uint32_t c[4] = {(uint32_t)comp, (uint32_t)(unsigned long long)step, (uint32_t)((unsigned long long)step >> 32), 0u};
    philox4x32_10(c, (uint32_t)p.seed, (uint32_t)(p.seed >> 32));
    const double u1 = ((double)((((uint64_t)c[0] << 32) | c[1]) >> 11) + 1.0) * (1.0 / 9007199254740992.0);
    const double u2 = ((double)((((uint64_t)c[2] << 32) | c[3]) >> 11) + 1.0) * (1.0 / 9007199254740992.0);
    const double r = sqrt(-2.0 * log(u1));
    double s, co;
    sincospi(2.0 * u2, &s, &co);
    xi = r * co; eta = r * s;
}

// ---- frame recorder (vb_md_set_recorder / vb_md_read_frames) -------------------------------------------------------
// The reference observes its run every --record-per-steps steps (MDObserver, src/utils/utils.py:114-166): it prints
// Epot / Ekin / Etot, writes a trajectory frame and raises TemperatureRunawayError above 1.5 T0.  Here kick2 of a record
// step (a step after which the counter is a multiple of `every`) sums Ekin in a fixed order, decides the runaway, and
// writes the frame -- its scalars, and x and v copied by the threads that own those components -- into ring slot
// frame % capacity.  The copy lives in kick2 rather than in a launch of its own: kick2 already holds v, x is final since
// kick1, and a separate grid would add a launch to every step to move 8 KB (Chignolin) on a few of them.  Once the
// runaway guard fires, kick1 and kick2 leave the state and the ring alone, so the device stays at the halting step
// (whose frame is kept) however many steps are still enqueued behind it.  With the recorder off every pointer is null
// and the kernels do exactly what they do without it.
constexpr double MD_KB = 8.617330337217213e-05;     // eV / K, as ai2bmd_b200/md.py KB
enum { MD_REC_FRAMES = 0, MD_REC_HALT = 1, MD_REC_CTL = 2 };
struct MdRecorder {
    long long every = 0, capacity = 0;
    double runaway_factor = 0.0;   // > 0: halt when T > runaway_factor * T0, T0 = kT / k_B
    // ctl[MD_REC_FRAMES]  frames written so far (frame f lives in slot f % capacity)
    // ctl[MD_REC_HALT]    -1, or the step at which the guard fired
    long long* ctl = nullptr;
    long long* step = nullptr;     // per slot
    double* epot = nullptr;        // per slot: restrained potential energy, ef[3n] + rf[3n]
    double* ekin = nullptr;        // per slot: sum m v^2 / 2 after the centre-of-mass velocity removal
    int* halted = nullptr;         // per slot: 1 on the frame whose temperature fired the guard
    double* x = nullptr;           // [capacity][3 * n_protein]
    double* v = nullptr;           // [capacity][3 * n_protein]
};

__device__ inline bool md_halted(const long long* ctl) { return ctl != nullptr && ctl[MD_REC_HALT] >= 0; }

// Langevin coefficients of one atom (ase/md/langevin.py updatevars; md.py Langevin.__init__)
struct MdCoef { double c1, c2, c3, c4, c5; };
__device__ inline MdCoef md_coef(const MdParams& p, double mass) {
    const double dt = p.dt, fr = p.fr, sigma = sqrt(2.0 * p.kT * fr / mass);
    MdCoef c;
    c.c1 = dt / 2.0 - dt * dt * fr / 8.0;
    c.c2 = dt * fr / 2.0 - dt * dt * fr * fr / 8.0;
    c.c3 = sqrt(dt) * sigma / 2.0 - pow(dt, 1.5) * fr * sigma / 8.0;
    c.c5 = pow(dt, 1.5) * sigma / (2.0 * sqrt(3.0));
    c.c4 = fr / 2.0 * c.c5;
    return c;
}

// first half-kick + drift (ase/md/langevin.py step(): v += ..., x += dt v + c5 eta, v recomputed from the positions).
// With friction > 0 the integrator also keeps the centre of mass where it was (fix_com: old_com saved before the drift,
// atoms.set_center_of_mass(old_com) after it, THEN the velocity recomputation), so the kernel is one CTA: pass 1 drifts
// and sums m*x_old, m*x_new in a fixed order, pass 2 shifts every atom by old_com - new_com and recomputes v.
constexpr int MD_K1_THREADS = 1024;
__global__ void __launch_bounds__(MD_K1_THREADS) md_kick1_kernel(MdParams p, const long long* __restrict__ step_ctr,
                                                                 const double* __restrict__ mass, const float* __restrict__ ef,
                                                                 const double* __restrict__ rf,
                                                                 double* __restrict__ x, double* __restrict__ v,
                                                                 const long long* __restrict__ rec_ctl) {
    __shared__ double shift[3];
    if (md_halted(rec_ctl)) return;
    const int n3 = 3 * p.n_protein;
    const long long step = *step_ctr;
    const bool fixcm = p.fr > 0.0;
    double so[3] = {0.0, 0.0, 0.0}, sn[3] = {0.0, 0.0, 0.0}, sm = 0.0;
    // thread t handles components t, t + T, ...; T is a multiple of 3, so a thread stays on one Cartesian axis
    constexpr int T = (MD_K1_THREADS / 3) * 3;
    if (threadIdx.x < T) {
        for (int comp = threadIdx.x; comp < n3; comp += T) {
            const double m = mass[comp / 3];
            const MdCoef c = md_coef(p, m);
            double xi = 0.0, eta = 0.0;
            if (p.fr > 0.0) md_normals(p, step, comp, xi, eta);
            double f = (double)ef[comp];
            if (rf != nullptr) f += rf[comp];
            double vv = v[comp];
            vv = vv + (c.c1 * f / m - c.c2 * vv + c.c3 * xi - c.c4 * eta);
            const double x_old = x[comp];
            const double x_new = x_old + p.dt * vv + c.c5 * eta;
            x[comp] = x_new;
            if (fixcm) {
                v[comp] = x_old;                   // parked until pass 2
                so[0] += m * x_old; sn[0] += m * x_new;
                if (comp % 3 == 0) sm += m;
            } else {
                v[comp] = (x_new - x_old - c.c5 * eta) / p.dt;
            }
        }
    }
    if (!fixcm) return;
    // block reduction per axis (axis of thread t = t % 3), fixed order: warp shuffles cannot be used across axes, so
    // every thread publishes its partials and three threads sum them serially
    __shared__ double part_o[MD_K1_THREADS], part_n[MD_K1_THREADS], part_m[MD_K1_THREADS];
    part_o[threadIdx.x] = so[0]; part_n[threadIdx.x] = sn[0]; part_m[threadIdx.x] = sm;
    __syncthreads();
    if (threadIdx.x < 3) {
        double o = 0.0, n = 0.0, mt = 0.0;
        for (int t = threadIdx.x; t < T; t += 3) { o += part_o[t]; n += part_n[t]; }
        for (int t = 0; t < T; t += 3) mt += part_m[t];
        shift[threadIdx.x] = o / mt - n / mt;      // old_com - new_com
    }
    __syncthreads();
    if (threadIdx.x < T) {
        for (int comp = threadIdx.x; comp < n3; comp += T) {
            const double m = mass[comp / 3];
            const MdCoef c = md_coef(p, m);
            double xi = 0.0, eta = 0.0;
            md_normals(p, step, comp, xi, eta);
            const double x_old = v[comp];
            const double x_new = x[comp] + shift[comp % 3];
            x[comp] = x_new;
            v[comp] = (x_new - x_old - c.c5 * eta) / p.dt;
        }
    }
}

// ---- Hookean restraints (ASE 3.22 ase/constraints.py Hookean, recalled; host checker oracle/hookean_ref.py) -----------
// The reference's pre-equilibration tethers every protein atom to where it stood at the start of a stage
// (src/AIMD/simulator.py:139-166, ASE type 'point', rt = 0) and --constraints adds a spring between every hydrogen and its
// bonded partner (simulator.py:168-180, ASE type 'two atoms').  For one term, with d the vector from the atom to the
// anchor (tether) or to the partner (spring) and L = |d|: if L > rt, F += k (L - rt) d / L and E += k (L - rt)^2 / 2 (at
// L = 0 nothing is added).  ASE applies find_mic with the cell; here there is no minimum image: a tether moves far less
// than half a box length and a bond is about 1 A, so the minimum image is the displacement itself.
// Terms are a CSR over protein atoms built on the host: a spring appears once at each of its two atoms (the partner's
// entry sees -d, i.e. the opposite force), a tether once.  One thread sums an atom's terms in CSR order, no atomics; the
// energy of a spring is counted at its lower-indexed atom and reduced in a fixed order, so rf is bit-reproducible.
// The output rf[3*n_protein + 1] (forces, then the energy) is the engine's own fp64 buffer: the caller's ef stays the
// calculator output and the kicks add the two, as ASE's Atoms.get_forces() adds the constraint on top of the calculator.
struct MdRestraints {
    int n_protein;
    const int* rowptr;      // [n_protein + 1]
    const int* partner;     // per term: the other atom of a spring, or -1 for a tether
    const double* k;        // per term, eV/A^2
    const double* rt;       // per term, A
    const double* p0;       // [3 * terms]: the anchor of a tether (unused for springs)
    double* rf;             // [3 * n_protein + 1]
};

// evaluated by one CTA of blockDim.x threads (a multiple of 32, at most 1024)
__device__ inline void md_restraint_cta(const MdRestraints& r, const double* __restrict__ x) {
    __shared__ double red[32];
    double e = 0.0;
    for (int a = threadIdx.x; a < r.n_protein; a += blockDim.x) {
        const double xa = x[3 * a], ya = x[3 * a + 1], za = x[3 * a + 2];
        double fx = 0.0, fy = 0.0, fz = 0.0;
        for (int t = r.rowptr[a]; t < r.rowptr[a + 1]; t++) {
            const int j = r.partner[t];
            double dx, dy, dz;
            if (j < 0) { dx = r.p0[3 * t] - xa; dy = r.p0[3 * t + 1] - ya; dz = r.p0[3 * t + 2] - za; }
            else       { dx = x[3 * j] - xa;    dy = x[3 * j + 1] - ya;    dz = x[3 * j + 2] - za; }
            const double L = sqrt(dx * dx + dy * dy + dz * dz), rt = r.rt[t];
            if (L > rt) {
                const double mag = r.k[t] * (L - rt);
                fx += dx / L * mag; fy += dy / L * mag; fz += dz / L * mag;
                if (j < a) e += 0.5 * r.k[t] * ((L - rt) * (L - rt));    // tethers (j = -1) and each spring once
            }
        }
        r.rf[3 * a] = fx; r.rf[3 * a + 1] = fy; r.rf[3 * a + 2] = fz;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += red[w];
        r.rf[3 * r.n_protein] = t;
    }
}

// fragment atoms follow the protein: real atoms copy, cap hydrogens sit at P[acc] + unit(P[rem] - P[acc]) * blen.
// With restraints the launch has one CTA more than the placement needs, and that last CTA evaluates them into rf at the
// same protein coordinates: the restraints cost no launch of their own in the step (a grid of one CTA with n_atoms = 0
// evaluates only the restraints).
__global__ void md_place_kernel(int n_atoms, const int* __restrict__ real, const int* __restrict__ acc,
                                const int* __restrict__ rem, const float* __restrict__ blen,
                                const double* __restrict__ x, float* __restrict__ pos, MdRestraints rs) {
    if ((int)blockIdx.x == (n_atoms + (int)blockDim.x - 1) / (int)blockDim.x) { md_restraint_cta(rs, x); return; }
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    const int r = real[a];
    double px, py, pz;
    if (r >= 0) {
        px = x[3 * r]; py = x[3 * r + 1]; pz = x[3 * r + 2];
    } else {
        const int ia = acc[a], ir = rem[a];
        const double ax = x[3 * ia], ay = x[3 * ia + 1], az = x[3 * ia + 2];
        double dx = x[3 * ir] - ax, dy = x[3 * ir + 1] - ay, dz = x[3 * ir + 2] - az;
        const double n = sqrt(dx * dx + dy * dy + dz * dz);
        dx /= n; dy /= n; dz /= n;
        const double b = (double)blen[a];
        px = ax + dx * b; py = ay + dy * b; pz = az + dz * b;
    }
    pos[3 * a] = (float)px; pos[3 * a + 1] = (float)py; pos[3 * a + 2] = (float)pz;
}

// second half-kick (+ centre-of-mass velocity removal when friction > 0, as md.py does) and step counter advance; on
// record steps also the frame and the runaway guard.  One CTA: the momentum and kinetic-energy sums are
// reduced in a fixed order, so they are bit-reproducible for the same v.
constexpr int MD_K2_THREADS = 1024;
__global__ void __launch_bounds__(MD_K2_THREADS) md_kick2_kernel(MdParams p, long long* __restrict__ step_ctr,
                                                                 const double* __restrict__ mass, const float* __restrict__ ef,
                                                                 const double* __restrict__ rf,
                                                                 const double* __restrict__ x, double* __restrict__ v,
                                                                 double* __restrict__ epot_hist, long long hist_cap,
                                                                 MdRecorder rec) {
    __shared__ double red[3][MD_K2_THREADS / 32];
    __shared__ double com[3];
    if (md_halted(rec.ctl)) return;
    const long long step = *step_ctr;
    const int n3 = 3 * p.n_protein;
    for (int comp = threadIdx.x; comp < n3; comp += MD_K2_THREADS) {
        const double m = mass[comp / 3];
        const MdCoef c = md_coef(p, m);
        double xi = 0.0, eta = 0.0;
        if (p.fr > 0.0) md_normals(p, step, comp, xi, eta);
        double f = (double)ef[comp];
        if (rf != nullptr) f += rf[comp];
        double vv = v[comp];
        vv = vv + (c.c1 * f / m - c.c2 * vv + c.c3 * xi - c.c4 * eta);
        v[comp] = vv;
    }
    if (p.fr > 0.0) {
        __syncthreads();
        double s[3] = {0.0, 0.0, 0.0}, ms = 0.0;
        for (int a = threadIdx.x; a < p.n_protein; a += MD_K2_THREADS) {
            const double m = mass[a];
            s[0] += m * v[3 * a]; s[1] += m * v[3 * a + 1]; s[2] += m * v[3 * a + 2];
            ms += m;
        }
        // block reduction of (px, py, pz) and of the total mass (fixed order)
        __shared__ double redm[MD_K2_THREADS / 32];
        __shared__ double mtot;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s[0] += __shfl_xor_sync(0xffffffffu, s[0], o); s[1] += __shfl_xor_sync(0xffffffffu, s[1], o);
            s[2] += __shfl_xor_sync(0xffffffffu, s[2], o); ms += __shfl_xor_sync(0xffffffffu, ms, o);
        }
        if ((threadIdx.x & 31) == 0) {
            red[0][threadIdx.x >> 5] = s[0]; red[1][threadIdx.x >> 5] = s[1]; red[2][threadIdx.x >> 5] = s[2];
            redm[threadIdx.x >> 5] = ms;
        }
        __syncthreads();
        if (threadIdx.x < 4) {
            double t = 0.0;
            for (int w = 0; w < MD_K2_THREADS / 32; w++) t += (threadIdx.x < 3) ? red[threadIdx.x][w] : redm[w];
            if (threadIdx.x < 3) com[threadIdx.x] = t; else mtot = t;
        }
        __syncthreads();
        for (int comp = threadIdx.x; comp < n3; comp += MD_K2_THREADS) v[comp] -= com[comp % 3] / mtot;
    }
    // record step: the frame's x and v, and Ekin = sum m v^2 / 2 of the final velocities.  Each thread copies and sums
    // only the components it wrote itself; warp shuffles, then the warp partials summed serially (the momentum
    // reduction's pattern).  Every thread reads the frame count before the barrier, thread 0 advances it after.
    const bool record = rec.ctl != nullptr && (step + 1) % rec.every == 0;
    __shared__ double redk[MD_K2_THREADS / 32];
    long long frame = 0;
    if (record) {
        frame = rec.ctl[MD_REC_FRAMES];
        double* __restrict__ fx = rec.x + (frame % rec.capacity) * n3;
        double* __restrict__ fv = rec.v + (frame % rec.capacity) * n3;
        double e = 0.0;
        for (int comp = threadIdx.x; comp < n3; comp += MD_K2_THREADS) {
            const double vv = v[comp];
            fx[comp] = x[comp];
            fv[comp] = vv;
            e += mass[comp / 3] * (vv * vv);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
        if ((threadIdx.x & 31) == 0) redk[threadIdx.x >> 5] = e;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        // with restraints, the restrained potential energy (ASE get_potential_energy(apply_constraint=True))
        const double epot = (double)ef[n3] + (rf != nullptr ? rf[n3] : 0.0);
        if (epot_hist != nullptr && hist_cap > 0) epot_hist[step % hist_cap] = epot;
        if (record) {
            double s = 0.0;
            for (int w = 0; w < MD_K2_THREADS / 32; w++) s += redk[w];
            const double ekin = 0.5 * s;
            // md.py DeviceLangevin.temperature: T = 2 Ekin / (3 n k_B); the reference raises above 1.5 T0
            const double temp = 2.0 * ekin / (3.0 * p.n_protein) / MD_KB;
            const bool runaway = rec.runaway_factor > 0.0 && temp > rec.runaway_factor * p.kT / MD_KB;
            const long long slot = frame % rec.capacity;
            rec.step[slot] = step + 1;
            rec.epot[slot] = epot;
            rec.ekin[slot] = ekin;
            rec.halted[slot] = runaway ? 1 : 0;
            rec.ctl[MD_REC_FRAMES] = frame + 1;
            if (runaway) rec.ctl[MD_REC_HALT] = step + 1;
        }
        *step_ctr = step + 1;
    }
}

}  // namespace vb
