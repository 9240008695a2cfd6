// tma_ring_bench.cu -- microbenchmark of the persistent decode kernel's weight pipeline in isolation: one CTA per SM,
// one producer thread streaming a large buffer through a ring of `nstage` stages (each filled by `ncopy`
// cp.async.bulk copies), 16 consumer warps that only wait for a stage and release it (no arithmetic).
// Tells which ring geometry the HBM stream needs, independent of the MMA loop.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_ring_bench tma_ring_bench.cu && ./tma_ring_bench
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) { while (!mbar_try(bar, parity)) {} }
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar, uint64_t pol, int hint) {
    if (hint)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
    else
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

constexpr int CW = 16;
// work: every CTA streams `per_cta` bytes starting at base + cta * per_cta (mode 0: contiguous per CTA) or interleaved
// in stage-sized units across CTAs (mode 1), `touch` != 0: consumers also read the stage (one LDS.128 per lane per 512 B)
__global__ void __launch_bounds__(CW * 32 + 32, 1)
ring_kernel(const unsigned char *base, size_t per_cta, int stage_bytes, int nstage, int ncopy, int hint, int mode, int touch,
            unsigned *sink) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem);
    uint64_t *empty = full + 32;
    unsigned char *ring = smem + 1024;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < nstage; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CW); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    const size_t n_it = per_cta / stage_bytes;
    const int cb = stage_bytes / ncopy;
    if (warp == CW) {
        if (lane == 0) {
            uint64_t pol;
            asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
            int stage = 0; uint32_t phase = 0; bool wrapped = false;
            for (size_t it = 0; it < n_it; ++it) {
                const unsigned char *src = mode == 0 ? base + (size_t)blockIdx.x * per_cta + it * stage_bytes
                                                     : base + (it * gridDim.x + blockIdx.x) * (size_t)stage_bytes;
                if (wrapped) mbar_wait(&empty[stage], phase ^ 1u);
                mbar_expect_tx(&full[stage], (uint32_t)stage_bytes);
                for (int c = 0; c < ncopy; ++c)
                    bulk_g2s(ring + (size_t)stage * stage_bytes + (size_t)c * cb, src + (size_t)c * cb, (uint32_t)cb, &full[stage], pol, hint);
                if (++stage == nstage) { stage = 0; phase ^= 1u; wrapped = true; }
            }
        }
        return;
    }
    int stage = 0; uint32_t phase = 0; unsigned acc = 0;
    for (size_t it = 0; it < n_it; ++it) {
        mbar_wait(&full[stage], phase);
        if (touch) {
            const uint4 *p = reinterpret_cast<const uint4 *>(ring + (size_t)stage * stage_bytes);
            for (int i = warp * 32 + lane; i < stage_bytes / 16; i += CW * 32) { uint4 v = p[i]; acc += v.x ^ v.y ^ v.z ^ v.w; }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == nstage) { stage = 0; phase ^= 1u; }
    }
    if (acc == 0x12345678u) sink[0] = acc;
}

int main() {
    int dev = 0, sms = 0;
    cudaSetDevice(dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t total = (size_t)2 << 30;  // 2 GiB >> L2
    unsigned char *buf; unsigned *sink;
    cudaMalloc(&buf, total); cudaMalloc(&sink, 4);
    cudaMemset(buf, 1, total);
    cudaFuncSetAttribute(ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    printf("SMs %d\n%8s %6s %5s %4s %4s %5s | %8s\n", sms, "stageB", "nstage", "ncopy", "hint", "mode", "touch", "GB/s");
    const int stage_sizes[] = {9216, 18432, 36864};
    for (int touch = 0; touch <= 1; ++touch)
    for (int mode = 0; mode <= 1; ++mode)
    for (int hint = 0; hint <= 1; ++hint)
    for (int sb : stage_sizes)
    for (int ns : {3, 6, 12, 20})
    for (int nc : {1, 4, 8}) {
        if ((size_t)ns * sb + 1024 > 227 * 1024) continue;
        if (touch && (hint == 0 || nc == 8)) continue;   // keep the sweep short
        if (mode == 1 && (hint == 0 || nc == 8)) continue;
        size_t per_cta = total / sms / sb * sb;
        size_t smem = (size_t)ns * sb + 1024;
        float best = 1e9f;
        for (int rep = 0; rep < 3; ++rep) {
            cudaEventRecord(e0);
            ring_kernel<<<sms, CW * 32 + 32, smem>>>(buf, per_cta, sb, ns, nc, hint, mode, touch, sink);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            if (ms < best) best = ms;
        }
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
        printf("%8d %6d %5d %4d %4d %5d | %8.0f\n", sb, ns, nc, hint, mode, touch, (double)per_cta * sms / (best * 1e-3) / 1e9);
    }
    return 0;
}
