// Thin inline-PTX wrappers for the sm_90a features the tensor-core ALS kernel and the batch top-k kernel use: mbarrier,
// cp.async (SASS LDGSTS), cp.async.bulk and warpgroup MMA (wgmma.mma_async, SASS HGMMA) with shared-memory matrix descriptors.  No CUTLASS: every string
// below is plain PTX ISA 8.x.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bfl {
namespace sm90 {

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(s32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// for waits that are expected to be long (an idle role): back off between polls so that the spinning warp does not take
// issue slots from the working warps of its scheduler
__device__ __forceinline__ void mbar_wait_idle(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(128);
}

// transaction-count completion: one arrival that also announces `bytes` of bulk-copy traffic for the current phase
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(bar)), "r"(bytes) : "memory");
}
// bulk asynchronous copy global -> shared (SASS UBLKCP): 16-byte aligned addresses, size a multiple of 16; its bytes
// complete on `bar`
__device__ __forceinline__ void cp_async_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     s32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(s32(bar))
                 : "memory");
}

// barrier `id` (1..15; 0 is __syncthreads) of the first `nthreads` threads that reach it, a multiple of 32
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// generic-proxy writes to shared memory -> visible to the async proxy (tensor-core operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- 16-byte cp.async (SASS LDGSTS), completion by commit / wait groups ---------------------------------
__device__ __forceinline__ void cp_async16_cg(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// waits until at most N of the executing thread's most recent commit groups are still pending
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- wgmma: operands from shared memory, fp32 accumulator in the registers of one warpgroup ----------------
// Shared-memory matrix descriptor (PTX ISA "matrix descriptor" of wgmma):
//   [0,14) start address >> 4 | [16,30) leading-dimension byte offset >> 4 | [32,46) stride-dimension byte offset >> 4
//   [62,64) swizzle mode (0 = none, "interleaved")
// K-major un-swizzled operand: core matrices of 8 rows (M/N) x 16 bytes (8 fp16 along K), stored as 128 contiguous
// bytes; SBO = distance between core matrices that are neighbours along M/N, LBO = distance between neighbours along K.
// One instruction covers K = 16 (two core matrices deep).
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr >> 4) & 0x3fffu) | ((uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// per-thread register budget of the executing warpgroup (all of its warps execute the same instruction)
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
// keeps the compiler from touching accumulator registers across a wgmma fence / wait
__device__ __forceinline__ void acc_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// D[64 x 128] (+)= (+/-A)[64 x 16] B[16 x 128]^T, fp16 operands (both K-major), fp32 accumulator.
// Fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4 n + 2 h + i] = D[16 w + l / 4 + 8 h][8 n + 2 (l % 4) + i].
#define BFL_WGMMA_ACC64(d)                                                                                              \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),         \
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),        \
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),       \
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),       \
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),       \
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),       \
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),       \
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define BFL_WGMMA_REGS64                                                                                                \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "   \
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, " \
    "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
template <bool NEG>
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    if (NEG) {
        asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " BFL_WGMMA_REGS64 ", %64, %65, 1, -1, 1, 0, 0;"
                     : BFL_WGMMA_ACC64(d)
                     : "l"(adesc), "l"(bdesc)
                     : "memory");
    } else {
        asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " BFL_WGMMA_REGS64 ", %64, %65, 1, 1, 1, 0, 0;"
                     : BFL_WGMMA_ACC64(d)
                     : "l"(adesc), "l"(bdesc)
                     : "memory");
    }
}
// D[64 x 64] (+)= (+/-A)[64 x 16] B[16 x 64]^T: the first 64 columns of the above, same fragment layout (n < 8)
#define BFL_WGMMA_ACC32(d)                                                                                              \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),         \
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),        \
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),       \
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define BFL_WGMMA_REGS32                                                                                                \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "   \
    "%24, %25, %26, %27, %28, %29, %30, %31}"
template <bool NEG>
__device__ __forceinline__ void wgmma_m64n64k16_f16(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
    if (NEG) {
        asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " BFL_WGMMA_REGS32 ", %32, %33, 1, -1, 1, 0, 0;"
                     : BFL_WGMMA_ACC32(d)
                     : "l"(adesc), "l"(bdesc)
                     : "memory");
    } else {
        asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " BFL_WGMMA_REGS32 ", %32, %33, 1, 1, 1, 0, 0;"
                     : BFL_WGMMA_ACC32(d)
                     : "l"(adesc), "l"(bdesc)
                     : "memory");
    }
}
#undef BFL_WGMMA_ACC64
#undef BFL_WGMMA_REGS64
#undef BFL_WGMMA_ACC32
#undef BFL_WGMMA_REGS32

// fp32 pairs (two FMULs / FFMAs: sm_90 has no packed fp32 arithmetic)
__device__ __forceinline__ float2 f2mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 f2fma(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
// Two-term fp16 split of a pair of fp32 values (k even -> low half, k odd -> high half of each 32-bit word):
// head = the value with its low 13 mantissa bits cleared (exactly an fp16 number while it is in the normal fp16 range),
// tail = value - head rounded to fp16; head + tail carries >= 21 significant bits.
__device__ __forceinline__ void split_f16x2(float2 s, uint32_t& head, uint32_t& tail) {
    float2 h;
    h.x = __uint_as_float(__float_as_uint(s.x) & 0xffffe000u);
    h.y = __uint_as_float(__float_as_uint(s.y) & 0xffffe000u);
    const float2 t = f2fma(h, make_float2(-1.f, -1.f), s);
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(head) : "f"(h.y), "f"(h.x));
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(tail) : "f"(t.y), "f"(t.x));
}

}  // namespace sm90
}  // namespace bfl
