// mg_pair_bench.cu -- the M = 8 weight-loop body of decode_mega.cu (mg_pair<8,2,2>: 2 tiles x 2 blocks, 16 chained
// m16n8k16 + unpack + scale FMAs) timed in isolation: operands resident in shared memory, no TMA ring, no mbarriers,
// 1 CTA per SM.  Cycles per call and warp for 4/8/16 resident warps and with parts of the body removed -- which pipe (or
// which latency) sets the ~1300 cycles per ring stage that the kernel's weight loop was measured to take?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mg_pair_bench mg_pair_bench.cu
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

constexpr int SLOT = 16 * 576;  // one tile's 16 pairs
constexpr int MT = 8;

// MODE bits: 1 = no MMA (cc = float(a-bits) instead), 2 = weights not re-read from shared memory (first iteration's
// registers reused), 4 = fragments not re-read, 8 = no scale FMAs, 16 = chains interleaved in source order
// MODE bit 32: the ring holds random bytes, i.e. the A operands are f16 SUBNORMALS n * 2^-24 / n * 2^-20 as in the kernel
// (the default fill masks to 0x3C00 patterns, which the nibble masks turn into zeros)
template <int MODE>
__global__ void __launch_bounds__(544, 1) body_kernel(unsigned long long *out, int iters, float *sink, int maxreg_dummy) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char *ring = smem;                                   // [4 stages][2 tiles][SLOT]
    uint2 *bf = reinterpret_cast<uint2 *>(smem + 4 * 2 * SLOT);   // [16 pairs][2 blocks][16*MT]
    float2 *off2 = reinterpret_cast<float2 *>(bf + 16 * 2 * 16 * MT);  // [16 pairs][2][MT]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    for (int i = tid; i < (4 * 2 * SLOT + 16 * 2 * 16 * MT * 8 + 16 * 2 * MT * 8) / 4; i += blockDim.x)
        reinterpret_cast<uint32_t *>(smem)[i] = ((MODE & 32) && i < 4 * 2 * SLOT / 4) ? ((uint32_t)i * 2654435761u) ^ ((uint32_t)i >> 3) : ((uint32_t)i * 2654435761u & 0x3C003C00u);  // finite halves
    __syncthreads();
    float acc[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
    const uint32_t slot_q = (uint32_t)warp * 512u + (uint32_t)lane * 16u;
    const uint32_t slot_d = 16u * 512u + (uint32_t)warp * 64u + (uint32_t)g * 8u;
    uint4 wq[2];
    uint2 wd[2];
    uint4 fhk[2], fmk[2];
    float4 ok[2];
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
        const unsigned char *sb = ring + (size_t)(it & 3) * (2 * SLOT);
        const uint2 *bfp = bf + (size_t)(warp & 15) * (2 * 16 * MT);
        const float2 *ofp = off2 + (size_t)(warp & 15) * (2 * MT);
        if (!(MODE & 2) || it == 0) {
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                wq[u] = *reinterpret_cast<const uint4 *>(sb + (size_t)u * SLOT + slot_q);
                wd[u] = *reinterpret_cast<const uint2 *>(sb + (size_t)u * SLOT + slot_d);
            }
        }
#pragma unroll
        for (int bb = 0; bb < 2; ++bb) {
            if (!(MODE & 4) || it == 0) {
                const uint4 *bq = reinterpret_cast<const uint4 *>(bfp + (size_t)bb * (16 * MT));
                fhk[bb] = bq[lane];
                fmk[bb] = bq[32 + lane];
                ok[bb] = *reinterpret_cast<const float4 *>(ofp + bb * MT + 2 * t);
            }
            const uint4 fh = fhk[bb], fm = fmk[bb];
            const float4 o = ok[bb];
            uint32_t al[2][4], ah[2][4];
            float cc[2][4];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const uint32_t wg = bb ? wq[u].z : wq[u].x, wg8 = bb ? wq[u].w : wq[u].y;
                const uint32_t sg = wg >> 8, sg8 = wg8 >> 8;
                al[u][0] = wg & 0x000F000Fu; al[u][1] = wg8 & 0x000F000Fu; al[u][2] = sg & 0x000F000Fu; al[u][3] = sg8 & 0x000F000Fu;
                ah[u][0] = wg & 0x00F000F0u; ah[u][1] = wg8 & 0x00F000F0u; ah[u][2] = sg & 0x00F000F0u; ah[u][3] = sg8 & 0x00F000F0u;
                cc[u][0] = cc[u][1] = cc[u][2] = cc[u][3] = 0.f;
            }
            if (MODE & 1) {
#pragma unroll
                for (int u = 0; u < 2; ++u)
#pragma unroll
                    for (int q = 0; q < 4; ++q) cc[u][q] = __uint_as_float((al[u][q] ^ ah[u][q] ^ fh.x ^ fm.y) | 0x3F000000u);
            } else if (MODE & 16) {
#pragma unroll
                for (int u = 0; u < 2; ++u) mma16816(cc[u], al[u][0], al[u][1], al[u][2], al[u][3], fh.x, fh.y);
#pragma unroll
                for (int u = 0; u < 2; ++u) mma16816(cc[u], ah[u][0], ah[u][1], ah[u][2], ah[u][3], fh.z, fh.w);
#pragma unroll
                for (int u = 0; u < 2; ++u) mma16816(cc[u], al[u][0], al[u][1], al[u][2], al[u][3], fm.x, fm.y);
#pragma unroll
                for (int u = 0; u < 2; ++u) mma16816(cc[u], ah[u][0], ah[u][1], ah[u][2], ah[u][3], fm.z, fm.w);
            } else {
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    mma16816(cc[u], al[u][0], al[u][1], al[u][2], al[u][3], fh.x, fh.y);
                    mma16816(cc[u], ah[u][0], ah[u][1], ah[u][2], ah[u][3], fh.z, fh.w);
                    mma16816(cc[u], al[u][0], al[u][1], al[u][2], al[u][3], fm.x, fm.y);
                    mma16816(cc[u], ah[u][0], ah[u][1], ah[u][2], ah[u][3], fm.z, fm.w);
                }
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                if (MODE & 8) {
                    acc[u][0] += cc[u][0]; acc[u][1] += cc[u][1]; acc[u][2] += cc[u][2]; acc[u][3] += cc[u][3];
                } else {
                    const uint32_t dw = bb ? wd[u].y : wd[u].x;
                    const float2 d = __half22float2(*reinterpret_cast<const __half2 *>(&dw));
                    acc[u][0] = fmaf(d.x, fmaf(cc[u][0], o.y, o.x), acc[u][0]);
                    acc[u][1] = fmaf(d.x, fmaf(cc[u][1], o.w, o.z), acc[u][1]);
                    acc[u][2] = fmaf(d.y, fmaf(cc[u][2], o.y, o.x), acc[u][2]);
                    acc[u][3] = fmaf(d.y, fmaf(cc[u][3], o.w, o.z), acc[u][3]);
                }
            }
        }
    }
    const long long t1 = clock64();
    float s = 0.f;
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int q = 0; q < 4; ++q) s += acc[u][q];
    if (s == 123.456f) sink[0] = s;
    if (lane == 0) out[blockIdx.x * 32 + warp] = (unsigned long long)(t1 - t0);
}

template <int MODE>
void run(const char *name) {
    unsigned long long *d;
    float *sink;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&d, 8 * (size_t)sms * 32);
    cudaMalloc(&sink, 4);
    const int iters = 2000;
    const int smem = 4 * 2 * SLOT + 16 * 2 * 16 * MT * 8 + 16 * 2 * MT * 8;
    cudaFuncSetAttribute(body_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    printf("%-58s", name);
    for (int warps : {4, 8, 16}) {
        body_kernel<MODE><<<sms, warps * 32, smem>>>(d, iters, sink, 0);
        cudaDeviceSynchronize();
        unsigned long long h[32];
        cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
        unsigned long long mx = 0;
        for (int w = 0; w < warps; ++w) mx = h[w] > mx ? h[w] : mx;
        printf("  %2d warps: %7.1f cyc/call", warps, (double)mx / iters);
    }
    cudaError_t e = cudaGetLastError();
    printf("  [%s]\n", cudaGetErrorString(e));
    cudaFree(d);
    cudaFree(sink);
}

int main() {
    run<0>("full body (16 HMMA, unpack, scale FMAs, LDS)");
    run<32>("full body, subnormal A operands (random nibbles)");
    run<32 + 14>("MMA + unpack only, subnormal A operands");
    run<16>("full body, chains interleaved in source");
    run<1>("no MMA");
    run<2>("weights kept in registers (no LDS of qs/d)");
    run<4>("fragments kept in registers (no LDS of bf/off)");
    run<6>("no LDS at all");
    run<8>("no scale FMAs / conversions");
    run<14>("MMA + unpack only (no LDS, no scale FMAs)");
    run<15>("unpack only");
    return 0;
}
