// Hopper (sm_90a) primitives used by the tensor-core kernels: mbarrier, 1-D TMA bulk copies, warpgroup MMA
// (wgmma.mma_async kind tf32, A from registers, B from shared memory).  Inline PTX only (no CUTLASS dependency).
// Layout facts used here:
//   * B operand from shared memory, K-major, 128-byte swizzle: one K-slab = 32 tf32 = 128 B per row;
//     row n at byte n*128, its 16-byte chunk c stored at chunk position c ^ (n & 7); 8-row groups are
//     1024 B apart (SBO = 1024).  One MMA consumes K = 8 (32 B): the descriptor start address advances by
//     32 B per K-step inside the slab; rows 64..127 of a plane (the second N = 64 half) start 8 KB in.
//   * A operand in registers (m64n64k8, per warp 16 rows): a0 = (g, t), a1 = (g + 8, t), a2 = (g, t + 4),
//     a3 = (g + 8, t + 4) with g = lane / 4, t = lane % 4 (row, k within the warp's 16 x 8 block).
//   * accumulator (m64n64, f32): d[4i + 0/1] = row g, columns 8i + 2t + 0/1; d[4i + 2/3] = row g + 8, same columns.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vb {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
// shared-memory counter add, acquire-release at CTA scope (orders a warp's retired reads of a ring stage before the refill
// that the last releasing warp issues); returns the old value
__device__ __forceinline__ uint32_t atom_add_acq_rel(uint32_t* p, uint32_t v) {
    uint32_t old;
    asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(smem_u32(p)), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// ---- TMA: 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP) ------------------
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// bulk prefetch global -> L2 (SASS: UBLKPF.L2): address and size multiples of 16 bytes
__device__ __forceinline__ void tma_prefetch_l2(const void* gmem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}

// ---- warpgroup MMA --------------------------------------------------------------------------------------
// shared-memory matrix descriptor (sm_90): K-major, SWIZZLE_128B, LBO unused (1), SBO = 1024 B
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps a register live and unmodified up to this point (the A fragments of MMAs still in flight)
__device__ __forceinline__ void reg_fence(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// d[64 x 64] += A[64 x 8] (registers) * B[64 x 8]^T (descriptor), tf32 inputs, f32 accumulation
__device__ __forceinline__ void mma_m64n64k8_tf32(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
    asm volatile(
        "{\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
        "{%32,%33,%34,%35}, %36, 1, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b)
        : "memory");
}

// round-to-nearest tf32 split: x ~= hi + lo, both exactly representable in tf32 (low 13 mantissa bits zero)
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
    const float rest = x - __uint_as_float(hi);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(rest));
}

constexpr int SLAB_K = 32;                         // tf32 elements per K-slab (= 128 B, one swizzle row)
constexpr int SLAB_BYTES = 128 * SLAB_K * 4;       // one plane (hi or lo) of a 128-column slab: 16 KB
constexpr int STAGE_BYTES = 2 * SLAB_BYTES;        // hi + lo

}  // namespace tc
}  // namespace vb
