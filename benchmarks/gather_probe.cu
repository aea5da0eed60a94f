// Micro-benchmark behind the producer design of the tensor-core ALS kernel (DESIGN.md 4.1): how fast can ONE SM's
// producer warps gather random 512-byte factor rows from HBM into a shared-memory ring?
//   mode 0: cp.async.bulk (TMA, SASS UBLKCP), one 512-byte copy per lane, mbarrier expect_tx completion
//   mode 1: cp.async 16 B per lane (SASS LDGSTS), one warp instruction = one coalesced 512-byte row,
//           completion by cp.async.mbarrier.arrive.noinc
//   mode 2: plain 128-bit loads into registers + st.shared (the synchronous baseline)
// P producer warps share the ring (stage s belongs to warp s % P); one consumer warp releases a stage as soon as it is
// full, so a configuration keeps up to `stages` tiles in flight per SM.  Persistent grid of one CTA per SM.  Prints
// GB/s per configuration.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gather_probe gather_probe.cu
//   ./gather_probe [rows of Y, default 1e7] [mode, default all]
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t par) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(s32(b)), "r"(par) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(dst)), "l"(src), "r"(bytes), "r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void cp16(void* dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s32(dst)), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_arrive_noinc(uint64_t* bar) { asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(s32(bar)) : "memory"); }

constexpr int ROWF = 128;          // floats per row
constexpr int TILE = 32;           // rows per stage
constexpr int RAWP = ROWF + 8;     // padded pitch
constexpr int MAXP = 8;

template <int MODE>
__global__ void __launch_bounds__(32 * (MAXP + 1), 1) probe(const float* __restrict__ Y, const int32_t* __restrict__ keys, int tiles_per_cta,
                                                        int P, int NS, float* sink) {
    extern __shared__ __align__(128) unsigned char smem_[];
    float* raw = reinterpret_cast<float*>(smem_);                       // [NS][TILE*RAWP]
    uint64_t* full = reinterpret_cast<uint64_t*>(raw + (size_t)NS * TILE * RAWP);
    uint64_t* empty = full + NS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(&full[i], MODE == 0 ? 1 : 32);
            mbar_init(&empty[i], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int32_t* mykeys = keys + (size_t)blockIdx.x * tiles_per_cta * TILE;
    if (warp < P) {
        int32_t knext = mykeys[(size_t)warp * TILE + lane];
        for (int t = warp; t < tiles_per_cta; t += P) {
            const int s = t % NS;
            const uint32_t ph = (uint32_t)((t / NS) & 1);
            const int32_t key = knext;
            if (t + P < tiles_per_cta) knext = mykeys[(size_t)(t + P) * TILE + lane];
            mbar_wait(&empty[s], ph ^ 1u);
            float* dst = raw + (size_t)s * TILE * RAWP;
            if (MODE == 0) {
                if (lane == 0) mbar_expect(&full[s], TILE * ROWF * 4);
                __syncwarp();
                bulk_g2s(dst + lane * RAWP, Y + (size_t)key * ROWF, ROWF * 4, &full[s]);
            } else if (MODE == 1) {
#pragma unroll 8
                for (int r = 0; r < TILE; ++r) {
                    const int32_t k = __shfl_sync(0xffffffffu, key, r);
                    cp16(dst + r * RAWP + lane * 4, Y + (size_t)k * ROWF + lane * 4);
                }
                cp_arrive_noinc(&full[s]);
            } else {
                float4 v[8];
#pragma unroll 1
                for (int r0 = 0; r0 < TILE; r0 += 8) {
#pragma unroll
                    for (int r = 0; r < 8; ++r) {
                        const int32_t k = __shfl_sync(0xffffffffu, key, r0 + r);
                        v[r] = __ldg(reinterpret_cast<const float4*>(Y + (size_t)k * ROWF + lane * 4));
                    }
#pragma unroll
                    for (int r = 0; r < 8; ++r) *reinterpret_cast<float4*>(dst + (r0 + r) * RAWP + lane * 4) = v[r];
                }
                mbar_arrive(&full[s]);
            }
        }
    } else if (warp == P) {
        float acc = 0.f;
        for (int t = 0; t < tiles_per_cta; ++t) {
            const int s = t % NS;
            const uint32_t ph = (uint32_t)((t / NS) & 1);
            mbar_wait(&full[s], ph);
            acc += raw[(size_t)s * TILE * RAWP + lane * RAWP + lane];
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        if (acc == 123.456f) sink[0] = acc;
    }
}

int main(int argc, char** argv) {
    const size_t rows = argc > 1 ? (size_t)atoll(argv[1]) : 10000000;
    const int only_mode = argc > 2 ? atoi(argv[2]) : -1;   // -1: every mode
    int grid = 0, clk_khz = 0;
    CK(cudaDeviceGetAttribute(&grid, cudaDevAttrMultiProcessorCount, 0));
    CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    const int tiles = 2000;
    float* Y;
    CK(cudaMalloc(&Y, rows * ROWF * 4));
    CK(cudaMemset(Y, 0, rows * ROWF * 4));
    std::vector<int32_t> hk((size_t)grid * tiles * TILE);
    uint64_t st = 88172645463325252ull;
    for (auto& k : hk) { st ^= st << 13; st ^= st >> 7; st ^= st << 17; k = (int32_t)(st % rows); }
    int32_t* dk;
    CK(cudaMalloc(&dk, hk.size() * 4));
    CK(cudaMemcpy(dk, hk.data(), hk.size() * 4, cudaMemcpyHostToDevice));
    float* sink;
    CK(cudaMalloc(&sink, 4));
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    const double bytes = (double)grid * tiles * TILE * ROWF * 4;
    for (int mode = 0; mode < 3; ++mode)
        for (int NS : {2, 4, 6, 8, 12})
            for (int P : {1, 2, 4, 8}) {
                if (P > NS || (only_mode >= 0 && mode != only_mode)) continue;
                const size_t smem = (size_t)NS * TILE * RAWP * 4 + 2 * NS * 8;
                auto launch = [&]() {
                    if (mode == 0) { CK(cudaFuncSetAttribute(probe<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); probe<0><<<grid, 32 * (MAXP + 1), smem>>>(Y, dk, tiles, P, NS, sink); }
                    if (mode == 1) { CK(cudaFuncSetAttribute(probe<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); probe<1><<<grid, 32 * (MAXP + 1), smem>>>(Y, dk, tiles, P, NS, sink); }
                    if (mode == 2) { CK(cudaFuncSetAttribute(probe<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); probe<2><<<grid, 32 * (MAXP + 1), smem>>>(Y, dk, tiles, P, NS, sink); }
                };
                launch();
                CK(cudaDeviceSynchronize());
                cudaEventRecord(e0);
                launch();
                cudaEventRecord(e1);
                CK(cudaDeviceSynchronize());
                float ms;
                cudaEventElapsedTime(&ms, e0, e1);
                printf("mode %d (%s) stages %2d producers %d: %8.1f GB/s  (%.0f clk per 32-row tile per SM at %.3f GHz)\n", mode,
                       mode == 0 ? "bulk 512B" : (mode == 1 ? "LDGSTS 16B/lane" : "LDG+STS"), NS, P, bytes / ms / 1e6,
                       ms * 1e-3 * clk_khz * 1e3 / tiles, clk_khz * 1e-6);
            }
    return 0;
}
