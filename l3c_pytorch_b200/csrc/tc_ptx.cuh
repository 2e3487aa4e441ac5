// tc_ptx.cuh -- thin PTX wrappers shared by the tensor-core convolution kernels (sm_90a): mbarriers, TMA
// (cp.async.bulk.tensor), wgmma shared-memory descriptors and warpgroup MMA issue, and the FP16 operand-image
// conversions.  The kernel skeleton built on them is in tc_conv.cuh.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace l3c {
namespace tcx {

constexpr int CONSUMER_WARPS = 8;              // two warpgroups
constexpr int THREADS = 32 * (CONSUMER_WARPS + 2);

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}

// K-major, 128B-swizzled operand tile as TMA writes it with CU_TENSOR_MAP_SWIZZLE_128B: rows of 128 B, 8-row
// groups `sbo` bytes apart (a multiple of 1024 B, so that every group has the start's phase in the 1024 B swizzle
// atom).  +32 B steps along K inside the swizzled row are +2 on the descriptor.  A start may also lie on any row
// inside the atom: the H100 applies the swizzle to the absolute shared-memory address bits, so the matrix base
// offset (bits 49-51) stays 0.  Setting it to the start's phase, (start >> 7) & 7, reads the rows in the wrong
// order (measured: every output of the 3x3 f16 kernel wrong).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t sbo = 1024) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFFu)      // start address
           | (1ull << 16)                              // leading byte offset (unused for SW128 K-major)
           | ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32)  // stride byte offset between 8-row groups
           | (1ull << 62);                             // SWIZZLE_128B
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// the accumulator registers become valid at wgmma_wait0(): keep the compiler from touching them earlier
__device__ __forceinline__ void acc_fence(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void acc_zero(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
}

#define L3C_WGMMA_D32                                                                                              \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "  \
    "%23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define L3C_WGMMA_ACC(d)                                                                                           \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),   \
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),     \
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),    \
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, FP16 operands, fp32 accumulate; issued by the whole warpgroup
__device__ __forceinline__ void wgmma_f16(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " L3C_WGMMA_D32 ", %32, %33, p, 1, 1, 0, 0;\n\t}"
        : L3C_WGMMA_ACC(d)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
// D[64 x 64] (+)= A[64 x 8] * B[64 x 8]^T, TF32 operands (both K-major), fp32 accumulate
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " L3C_WGMMA_D32 ", %32, %33, p, 1, 1;\n\t}"
        : L3C_WGMMA_ACC(d)
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

__device__ __forceinline__ float round_tf32(float x) {      // round-to-nearest TF32 image of x
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// named barrier of one consumer warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(wg + 1) : "memory"); }

// two floats -> packed fp16 pair, round-to-nearest-even, saturating to +-65504
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // d.hi = first source
    return r;
}
constexpr float LO_SCALE = 2048.0f, LO_INV = 1.0f / 2048.0f;   // precision mode f16x2: x = hi + lo / 2^11
// (hi, lo) pair images of two floats (precision mode f16x2)
__device__ __forceinline__ void split_h2(float a, float b, uint32_t &hi, uint32_t &lo) {
    hi = pack_h2(a, b);
    const float2 h = __half22float2(*reinterpret_cast<const __half2 *>(&hi));
    lo = pack_h2((a - h.x) * LO_SCALE, (b - h.y) * LO_SCALE);
}

// 4x4 transpose inside each quad of lanes: before, thread tq holds v[j] = element (column block j, pair tq);
// after, thread tq holds v[s] = element (column block tq, pair s) -> 8 consecutive channels = 16 bytes.
// Must be executed by all 32 lanes.
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int tq) {
    const bool hi2 = (tq & 2) != 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const uint32_t send = hi2 ? v[i] : v[i + 2];
        const uint32_t got = __shfl_xor_sync(0xFFFFFFFFu, send, 2);
        if (hi2) v[i] = got; else v[i + 2] = got;
    }
    const bool hi1 = (tq & 1) != 0;
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
        const uint32_t send = hi1 ? v[i] : v[i + 1];
        const uint32_t got = __shfl_xor_sync(0xFFFFFFFFu, send, 1);
        if (hi1) v[i] = got; else v[i + 1] = got;
    }
}

}  // namespace tcx
}  // namespace l3c
