// mma_rate_bench.cu -- issue rate of the LEGACY warp-level MMA instructions on sm_90a (they are what the decode matvec's
// arithmetic runs on): per SM sub-partition, cycles per instruction with 1..8 resident warps and 4 independent
// accumulator chains per warp.  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mma_rate_bench mma_rate_bench.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

template <int KIND>
__global__ void rate_kernel(unsigned long long *out, int iters, float *sink) {
    float c[4][4];
    int ci[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { c[i][j] = 0.f; ci[i][j] = 0; }
    uint32_t a0 = threadIdx.x * 3 + 1, a1 = a0 ^ 0x1234, a2 = a0 + 7, a3 = a1 + 9, b0 = a0 * 5, b1 = a1 * 3;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
            if (KIND == 0)
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+f"(c[ch][0]), "+f"(c[ch][1]), "+f"(c[ch][2]), "+f"(c[ch][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            else if (KIND == 1)
                asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+r"(ci[ch][0]), "+r"(ci[ch][1]), "+r"(ci[ch][2]), "+r"(ci[ch][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            else if (KIND == 2)
                asm volatile("mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+f"(c[ch][0]), "+f"(c[ch][1]), "+f"(c[ch][2]), "+f"(c[ch][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            else if (KIND == 3)
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+f"(c[ch][0]), "+f"(c[ch][1]), "+f"(c[ch][2]), "+f"(c[ch][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            else
                asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+f"(c[ch][0]), "+f"(c[ch][1]), "+f"(c[ch][2]), "+f"(c[ch][3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
        }
    }
    const long long t1 = clock64();
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s += c[i][j] + (float)ci[i][j];
    if (s == 123.456f) sink[0] = s;
    if (threadIdx.x == 0) out[blockIdx.x] = (unsigned long long)(t1 - t0);
}

template <int KIND>
void run(const char *name, int macs) {
    unsigned long long *d; float *sink;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&d, 8 * (size_t)sms); cudaMalloc(&sink, 4);
    const int iters = 4096;
    printf("%-28s", name);
    for (int warps : {4, 8, 16, 32}) {    // per CTA (1 CTA per SM): 1, 2, 4, 8 warps per sub-partition
        rate_kernel<KIND><<<sms, warps * 32>>>(d, iters, sink);
        cudaDeviceSynchronize();
        unsigned long long h0 = 0;   // CTA 0's cycle count
        cudaMemcpy(&h0, d, sizeof(h0), cudaMemcpyDeviceToHost);
        double cyc = (double)h0;
        const double per_smsp = (double)iters * 4 * (warps / 4);       // instructions issued per sub-partition
        printf("  %2d w/SMSP: %6.2f cyc/instr (%5.0f MAC/clk/SM)", warps / 4, cyc / per_smsp, macs * per_smsp * 4 / cyc);
    }
    printf("\n");
    cudaFree(d); cudaFree(sink);
}

int main() {
    run<0>("HMMA.16816 f16->f32", 16 * 8 * 16);
    run<3>("HMMA.16816 bf16->f32", 16 * 8 * 16);
    run<1>("IMMA.16832 u8.s8->s32", 16 * 8 * 32);
    run<2>("QMMA.16832 e4m3->f32", 16 * 8 * 32);
    run<4>("HMMA.1688 tf32->f32", 16 * 8 * 8);
    cudaError_t e = cudaGetLastError();
    printf("status: %s\n", cudaGetErrorString(e));
    return 0;
}
