// mma_denorm_test.cu -- micro-check for the tensor-core-assisted Q4 matvec idea:
//   (1) does mma.sync.m16n8k16 (f16 x f16 -> f32) treat f16 *subnormal* A inputs exactly?
//       A Q4 nibble n sitting in the low bits of a 16-bit lane is the f16 subnormal n * 2^-24
//       (and n << 4 is 16 n * 2^-24), i.e. nibbles can feed the MMA with one LOP3 per two weights.
//   (2) same with bf16 inputs built by the 0x4300|n magic (128 + n).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -o mma_denorm_test mma_denorm_test.cu
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>

__global__ void k_f16(const uint32_t *a, const uint32_t *b, float *c) {
    const int lane = threadIdx.x;
    uint32_t a0 = a[lane * 4 + 0], a1 = a[lane * 4 + 1], a2 = a[lane * 4 + 2], a3 = a[lane * 4 + 3];
    uint32_t b0 = b[lane * 2 + 0], b1 = b[lane * 2 + 1];
    float d0 = 0, d1 = 0, d2 = 0, d3 = 0;
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d0), "+f"(d1), "+f"(d2), "+f"(d3) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    c[lane * 4 + 0] = d0; c[lane * 4 + 1] = d1; c[lane * 4 + 2] = d2; c[lane * 4 + 3] = d3;
}
__global__ void k_bf16(const uint32_t *a, const uint32_t *b, float *c) {
    const int lane = threadIdx.x;
    uint32_t a0 = a[lane * 4 + 0], a1 = a[lane * 4 + 1], a2 = a[lane * 4 + 2], a3 = a[lane * 4 + 3];
    uint32_t b0 = b[lane * 2 + 0], b1 = b[lane * 2 + 1];
    float d0 = 0, d1 = 0, d2 = 0, d3 = 0;
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d0), "+f"(d1), "+f"(d2), "+f"(d3) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    c[lane * 4 + 0] = d0; c[lane * 4 + 1] = d1; c[lane * 4 + 2] = d2; c[lane * 4 + 3] = d3;
}

static float h2f(uint16_t h) { __half x; memcpy(&x, &h, 2); return __half2float(x); }
static uint16_t f2h(float f) { __half x = __float2half_rn(f); uint16_t h; memcpy(&h, &x, 2); return h; }
static float b2f(uint16_t h) { uint32_t u = (uint32_t)h << 16; float f; memcpy(&f, &u, 4); return f; }
static uint16_t f2b(float f) { __nv_bfloat16 x = __float2bfloat16_rn(f); uint16_t h; memcpy(&h, &x, 2); return h; }

int main() {
    // logical A[16][16], B[16][8]
    std::vector<uint16_t> A(256), B(128);
    std::vector<uint32_t> fa(128), fb(64);
    uint32_t *da, *db; float *dc;
    cudaMalloc(&da, 512); cudaMalloc(&db, 256); cudaMalloc(&dc, 512);
    std::vector<float> C(128);
    for (int mode = 0; mode < 3; ++mode) {
        srand(1 + mode);
        for (int i = 0; i < 256; ++i) {
            int n = rand() % 16;
            if (mode == 0) A[i] = (uint16_t)((i % 2) ? (n << 4) : n);     // f16 subnormals n*2^-24, 16n*2^-24
            else if (mode == 1) A[i] = (uint16_t)(0x4300 | n);            // bf16 128+n
            else A[i] = (uint16_t)(0x6400 | ((i % 2) ? (n << 4) : n));    // f16 1024+n, 1024+16n
        }
        for (int i = 0; i < 128; ++i) {
            float v = ((rand() % 2001) - 1000) / 37.0f;
            B[i] = (mode == 1) ? f2b(v) : f2h(v);
        }
        for (int lane = 0; lane < 32; ++lane) {
            int g = lane / 4, t = lane % 4;
            auto pk = [&](int r, int c) { return (uint32_t)A[r * 16 + c] | ((uint32_t)A[r * 16 + c + 1] << 16); };
            fa[lane * 4 + 0] = pk(g, 2 * t); fa[lane * 4 + 1] = pk(g + 8, 2 * t);
            fa[lane * 4 + 2] = pk(g, 2 * t + 8); fa[lane * 4 + 3] = pk(g + 8, 2 * t + 8);
            auto pb = [&](int k, int n) { return (uint32_t)B[k * 8 + n] | ((uint32_t)B[(k + 1) * 8 + n] << 16); };
            fb[lane * 2 + 0] = pb(2 * t, g); fb[lane * 2 + 1] = pb(2 * t + 8, g);
        }
        cudaMemcpy(da, fa.data(), 512, cudaMemcpyHostToDevice);
        cudaMemcpy(db, fb.data(), 256, cudaMemcpyHostToDevice);
        if (mode == 1) k_bf16<<<1, 32>>>(da, db, dc); else k_f16<<<1, 32>>>(da, db, dc);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { printf("mode %d: CUDA error %s\n", mode, cudaGetErrorString(e)); return 1; }
        cudaMemcpy(C.data(), dc, 512, cudaMemcpyDeviceToHost);
        double maxrel = 0, maxabs = 0;
        for (int lane = 0; lane < 32; ++lane) {
            int g = lane / 4, t = lane % 4;
            for (int j = 0; j < 4; ++j) {
                int r = g + (j >= 2 ? 8 : 0), c = 2 * t + (j & 1);
                double ref = 0;
                for (int k = 0; k < 16; ++k)
                    ref += (double)(mode == 1 ? b2f(A[r * 16 + k]) : h2f(A[r * 16 + k])) * (double)(mode == 1 ? b2f(B[k * 8 + c]) : h2f(B[k * 8 + c]));
                double err = fabs((double)C[lane * 4 + j] - ref);
                maxabs = fmax(maxabs, err);
                if (ref != 0) maxrel = fmax(maxrel, err / fabs(ref));
            }
        }
        const char *names[3] = {"f16 subnormal nibbles (n, 16n)*2^-24", "bf16 magic 128+n", "f16 magic 1024+n / 1024+16n"};
        printf("mode %d [%s]: max abs err %.3e, max rel err %.3e  (sample c=%.9g)\n", mode, names[mode], maxabs, maxrel, C[5]);
    }
    return 0;
}
