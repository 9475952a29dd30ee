// Minimal hand-written Hopper tensor-core building blocks (sm_90a inline PTX) for the large-state sweep GEMM:
// wgmma shared-memory descriptors for the canonical K-major no-swizzle layout, wgmma.mma_async kind tf32 with
// register accumulators, mbarrier + TMA bulk copies.
//
// Canonical K-major, SWIZZLE_NONE operand layout (units of 16 bytes; cute/atom/mma_traits_sm90_gmma.hpp
// "LayoutType::INTERLEAVE : ((8,m),(T,2k)):((1T,SBO),(1,LBO))"): a core matrix is 8 rows x 16 bytes stored
// contiguously (128 B); core matrices adjacent along K are LBO bytes apart, adjacent 8-row groups
// SBO bytes apart.  For fp32/tf32 one 16-byte row piece holds 4 elements and one MMA consumes
// K = 8 (two core matrices along K).
//
// Accumulator fragment of wgmma m64nNk8 (f32): thread i of the warpgroup (warp w = i / 32, lane l) holds
// d[4j + 2h + e] = D(16 w + l / 4 + 8 h, 8 j + 2 (l % 4) + e),  j < N / 8, h, e in {0, 1}.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rxg {
namespace umma {

constexpr uint32_t LBO = 128;          // bytes between K-adjacent core matrices
__host__ __device__ constexpr uint32_t sbo_bytes(int K) { return (uint32_t)(K / 4) * 128u; }   // next 8-row group
// byte offset of element (row, k) of an operand with K columns in the canonical layout
__host__ __device__ constexpr uint32_t elem_off(int row, int k, int K) {
    return (uint32_t)(row / 8) * sbo_bytes(K) + (uint32_t)(k / 4) * LBO + (uint32_t)(row % 8) * 16u + (uint32_t)(k % 4) * 4u;
}

__device__ __forceinline__ uint64_t smem_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);            // start address       bits [0,14)
    d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;            // leading byte offset bits [16,30)
    d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;            // stride byte offset  bits [32,46)
    return d;                                              // base offset 0, layout type 0 = SWIZZLE_NONE
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]' (tf32 in, fp32 accumulate), A and B K-major in shared memory.
// accumulate = 0 ignores the previous contents of d.
template <int N>
__device__ __forceinline__ void mma_tf32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);

template <>
__device__ __forceinline__ void mma_tf32<16>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <>
__device__ __forceinline__ void mma_tf32<32>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// pin accumulator registers behind the wait: the compiler must not read them before wgmma_wait_all()
__device__ __forceinline__ void fence_reg(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t* mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(mbar)), "r"(count) : "memory");
}

// ---- TMA bulk copy (1-D, no tensor map): global -> shared, completion on an mbarrier (complete_tx)
__device__ __forceinline__ void mbar_expect_tx(uint64_t* mbar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(mbar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     (uint32_t)__cvta_generic_to_shared(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(mbar))
                 : "memory");
}
// bounded spin on an mbarrier phase: a mis-programmed pipeline traps instead of hanging the GPU
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* mbar, uint32_t parity) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(mbar);
    uint32_t done = 0;
    for (uint32_t spin = 0; spin < (1u << 27); ++spin) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n"
            : "=r"(done)
            : "r"(a), "r"(parity)
            : "memory");
        if (done) return;
    }
    __trap();
}

// split an fp32 value into a tf32-representable high part and the (tf32-rounded) remainder:
// x ~= hi + lo with ~21 bits, so A B ~= Ahi Bhi + Ahi Blo + Alo Bhi to fp32-level accuracy ("3xTF32")
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    uint32_t h;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
    hi = __uint_as_float(h);
    const float r = x - hi;
    uint32_t l;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(r));
    lo = __uint_as_float(l);
}

}  // namespace umma
}  // namespace rxg
