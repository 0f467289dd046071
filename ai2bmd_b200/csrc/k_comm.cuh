// One-shot all-reduce of the whole-protein force/energy buffer over NVLink peer memory (SURVEY section 8e).
//
// Replaces, per MD step, the reference's host-side concatenation of the per-device results and their re-upload
// (src/Calculators/bonded.py:74-89) ahead of the signed scatter (combiner.py:38-39).  The buffer is tiny ([3*N_prot + 1]
// floats: 2.1 KB for Chignolin, ~110 KB for the 512-fragment batch), so the cost of a collective is launch + latency, not
// bandwidth.  Every rank owns a window in its own HBM, mapped into every peer with CUDA IPC:
//     slots[parity][sender][max_floats]   and   flags[parity][sender]
// One kernel per rank and step, captured in the step's CUDA graph (no host call, no NCCL launch):
//   1. push   : every CTA stores its chunk of the local buffer into slot[parity][my_rank] of EVERY rank (peer stores
//               over NVLink / NVSwitch; the local copy takes the same path through the local pointer);
//   2. signal : the last CTA to finish pushing fences at system scope and writes the step's sequence number into
//               flags[parity][my_rank] of every rank;
//   3. wait   : every CTA spins until all `world` flags of this parity in its OWN memory carry the sequence number;
//   4. sum    : slots of this parity are added in rank order 0..world-1 -> every rank computes bit-identical sums
//               (replicated MD state stays in lock-step) and writes them over its local buffer.
// Two parities suffice: a rank can run at most one step ahead of the slowest one, because finishing step s+1 needs the
// slowest rank's push for s+1, which that rank issues only after it has summed step s.
// All CTAs of the kernel must be co-resident (they wait for each other): the grid is capped at COMM_MAX_CTAS.
// The wait has a deadline: a flag that does not arrive within COMM_WAIT_NS (a peer that died, a broken protocol) is
// counted in counters[3] and the kernel finishes with whatever the slots hold, so the stream never hangs.  Once the count
// is nonzero the ranks are out of step for good, and every later launch of the kernel (the rest of an md_run's replays)
// skips the wait, so one failure costs one deadline, not one per enqueued step.  The host reports the count
// (vb_get_option "comm_timeouts") and fails every later all-reduce and MD call of the handle but vb_md_get_state.
// The deadline bounds the skew between ranks, host side included: one rank stalled for more than 10 s between steps
// (I/O, a checkpoint) while its peers already wait in the next all-reduce also trips it.
// The sum starts at +0.0f, so an element that is -0.0 on every rank comes out as +0.0 (also with world = 1).
//
// With `gather` set the kernel is the join of an in-process group of handles (vb_group_*): one launch on the leader
// device, ordered after every member's evaluation by stream events, runs step 4 alone over slots[0 .. world), each the
// base of one member's complete [n] buffer (a peer pointer, a local one, or a row of a leader staging copy).  No push,
// no flags, no wait; the same rank-order sum from +0.0f, so a group's result is bit-identical to what the one-process-
// per-GPU path sums for the same partials.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vb {

constexpr int COMM_MAX_WORLD = 16;
constexpr int COMM_THREADS = 512;
constexpr int COMM_MAX_CTAS = 32;
constexpr unsigned long long COMM_WAIT_NS = 10ull * 1000 * 1000 * 1000;

struct CommParams {
    int rank, world;
    long long max_floats;                 // capacity of one slot
    float* slots[COMM_MAX_WORLD];         // slots[r]: base of rank r's slot array [2][world][max_floats] (peer-mapped)
    int* flags[COMM_MAX_WORLD];           // flags[r]: base of rank r's flag array [2][world]
    unsigned int* counters;               // local: [0] CTAs done pushing, [1] CTAs done summing, [2] sequence number,
                                          //        [3] flag waits that ran past COMM_WAIT_NS
    int gather;                           // 1: the group join -- buf[i] = sum over r of slots[r][i], nothing else
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ void st_release_sys(int* p, int v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float ld_relaxed_sys(const float* p) {
    float v;
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(COMM_THREADS) comm_allreduce_kernel(CommParams c, float* __restrict__ buf, long long n) {
    if (c.gather) {         // step 4 alone over complete member buffers (stream-ordered: plain loads)
        for (long long i = (long long)blockIdx.x * COMM_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * COMM_THREADS) {
            float s = 0.f;
            for (int r = 0; r < c.world; r++) s += c.slots[r][i];
            buf[i] = s;
        }
        return;
    }
    __shared__ unsigned int s_seq, s_broken;
    __shared__ int s_last;
    const int rank = c.rank, world = c.world;
    if (threadIdx.x == 0) {
        s_seq = *reinterpret_cast<volatile unsigned int*>(c.counters + 2);
        s_broken = *reinterpret_cast<volatile unsigned int*>(c.counters + 3);
    }
    __syncthreads();
    const unsigned int seq = s_seq + 1u;                    // this step's sequence number (starts at 1)
    const int par = (int)(seq & 1u);
    const size_t slot_off = ((size_t)par * world + rank) * (size_t)c.max_floats;
    // 1. push my chunk into my slot on every rank
    for (long long i = (long long)blockIdx.x * COMM_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * COMM_THREADS) {
        const float v = buf[i];
        for (int r = 0; r < world; r++) c.slots[r][slot_off + i] = v;
    }
    __threadfence_system();
    __syncthreads();
    // 2. the last CTA publishes the sequence number on every rank
    if (threadIdx.x == 0) s_last = (atomicAdd(c.counters + 0, 1u) == gridDim.x - 1) ? 1 : 0;
    __syncthreads();
    if (s_last) {
        __threadfence_system();
        if ((int)threadIdx.x < world) st_release_sys(c.flags[threadIdx.x] + par * world + rank, (int)seq);
    }
    // 3. wait for every rank's flag of this parity in my own memory
    if ((int)threadIdx.x < world && s_broken == 0u) {
        const int* f = c.flags[rank] + par * world + threadIdx.x;
        const unsigned long long t0 = globaltimer_ns();
        while (ld_acquire_sys(f) != (int)seq) {
            if (globaltimer_ns() - t0 > COMM_WAIT_NS) { atomicAdd(c.counters + 3, 1u); break; }
            __nanosleep(64);
        }
    }
    __syncthreads();
    // 4. fixed-order sum of the slots (same order on every rank)
    const float* mine = c.slots[rank] + (size_t)par * world * (size_t)c.max_floats;
    for (long long i = (long long)blockIdx.x * COMM_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * COMM_THREADS) {
        float s = 0.f;
        for (int r = 0; r < world; r++) s += ld_relaxed_sys(mine + (size_t)r * (size_t)c.max_floats + i);
        buf[i] = s;
    }
    __syncthreads();
    // bookkeeping: the last CTA to finish advances the sequence number and re-arms the counters
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(c.counters + 1, 1u) == gridDim.x - 1) {
            c.counters[0] = 0u;
            c.counters[1] = 0u;
            __threadfence();
            *reinterpret_cast<volatile unsigned int*>(c.counters + 2) = seq;
        }
    }
}

}  // namespace vb
