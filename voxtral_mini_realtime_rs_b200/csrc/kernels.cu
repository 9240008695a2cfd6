// kernels.cu -- sm_90a kernels for the Voxtral Q4_0 hot path (f32 arithmetic throughout, like the
// reference's WGSL/Burn path).  Reference semantics cited per kernel; none of this is derived from
// the reference's shaders beyond the arithmetic they define.
#include "kernels.h"

#include <atomic>
#include <cfloat>
#include <cmath>
#include <string>

#include "common.h"

namespace vox {

void smem_attr_check(cudaError_t e, const char *what) {
    if (e != cudaSuccess) fail(VOX_ECUDA, fmt("cudaFuncSetAttribute(%s, MaxDynamicSharedMemorySize): %s", what, cudaGetErrorString(e)));
}


static std::atomic<uint64_t> g_launches{0};
uint64_t kernel_launch_count() { return g_launches.load(); }
void add_graph_launches(int64_t n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

static inline void post_launch(const char *name) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) fail(VOX_ECUDA, fmt("%s launch failed: %s", name, cudaGetErrorString(e)));
}

void tc_count_launch(const char *name) { post_launch(name); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }

// =====================================================================================
// K2: Q4_0 fused dequant + matvec for M <= 8 activation rows (decode / batched decode).
//   y[m,n] = sum_k x[m,k] * (q[n,k]-8) * d[n,k/32]      (reference src/gguf/shader.wgsl:41-133)
// One warp owns two consecutive weight rows; lane l owns blocks l, l+32, ... of each row and reads
// them with one 128-bit load (the warp's request is 512 contiguous bytes).  x is staged in shared
// memory once per CTA (block stride padded to 36 floats => conflict-free 128-bit reads) together
// with the per-block sums used to fold the "-8" offset:  sum (q-8) x = sum q x - 8 sum x.
// =====================================================================================
constexpr int MV_THREADS = 256;
constexpr int MV_ROWS = 16;  // 8 warps x 2 rows
constexpr int XPAD = 36;

template <int M>
__device__ __forceinline__ void q4_block_dot(const uint4 q, const float dd, const float *__restrict__ xb,
                                             const int xs_stride, const float *__restrict__ xsum_b,
                                             const int xsum_stride, float (&acc)[M]) {
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
    float lo[16], hi[16];
#pragma unroll
    for (int wi = 0; wi < 4; ++wi) {
        const uint32_t l4 = w[wi] & 0x0F0F0F0Fu;
        const uint32_t h4 = (w[wi] >> 4) & 0x0F0F0F0Fu;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            lo[wi * 4 + t] = (float)((l4 >> (8 * t)) & 0xFFu);
            hi[wi * 4 + t] = (float)((h4 >> (8 * t)) & 0xFFu);
        }
    }
#pragma unroll
    for (int m = 0; m < M; ++m) {
        const float4 *x4 = reinterpret_cast<const float4 *>(xb + m * xs_stride);
        float s = 0.0f;
#pragma unroll
        for (int wi = 0; wi < 4; ++wi) {
            const float4 a = x4[wi];
            const float4 b = x4[4 + wi];
            s = fmaf(lo[wi * 4 + 0], a.x, s);
            s = fmaf(lo[wi * 4 + 1], a.y, s);
            s = fmaf(lo[wi * 4 + 2], a.z, s);
            s = fmaf(lo[wi * 4 + 3], a.w, s);
            s = fmaf(hi[wi * 4 + 0], b.x, s);
            s = fmaf(hi[wi * 4 + 1], b.y, s);
            s = fmaf(hi[wi * 4 + 2], b.z, s);
            s = fmaf(hi[wi * 4 + 3], b.w, s);
        }
        acc[m] = fmaf(dd, s - 8.0f * xsum_b[m * xsum_stride], acc[m]);
    }
}

template <int M, int EPI>
__global__ void __launch_bounds__(MV_THREADS)
q4_matvec_kernel(const uint4 *__restrict__ qs, const __half *__restrict__ ds, const int N, const int K,
                 const float *__restrict__ x, float *__restrict__ y, const int ldy,
                 const float *__restrict__ bias, const float *__restrict__ res, const int kcb,
                 const int n_chunks) {
    extern __shared__ __align__(16) float smem[];
    const int bpr = K >> 5;
    const int xs_stride = kcb * XPAD;
    float *xs = smem;                      // [M][kcb*36]
    float *xsum = smem + M * xs_stride;    // [M][kcb]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_rg = (N + MV_ROWS - 1) / MV_ROWS;

    auto stage = [&](int chunk) {
        const int b0 = chunk * kcb;
        const int nb = min(kcb, bpr - b0);
        for (int m = 0; m < M; ++m) {
            const float4 *src = reinterpret_cast<const float4 *>(x + (size_t)m * K + (size_t)b0 * 32);
            for (int i = threadIdx.x; i < nb * 8; i += MV_THREADS) {
                const float4 v = src[i];
                *reinterpret_cast<float4 *>(xs + m * xs_stride + (i >> 3) * XPAD + (i & 7) * 4) = v;
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < M * nb; i += MV_THREADS) {
            const int m = i / nb, bl = i - m * nb;
            const float *p = xs + m * xs_stride + bl * XPAD;
            float s = 0.0f;
#pragma unroll
            for (int j = 0; j < 32; ++j) s += p[j];
            xsum[m * kcb + bl] = s;
        }
        __syncthreads();
        return nb;
    };

    auto accumulate = [&](int rg, int chunk, int nb, float (&acc0)[M], float (&acc1)[M]) {
        const int r0 = rg * MV_ROWS + warp * 2;
        const int r1 = r0 + 1;
        const int b0 = chunk * kcb;
        const bool v0 = r0 < N, v1 = r1 < N;
        const uint4 *q0p = qs + (size_t)(v0 ? r0 : 0) * bpr + b0;
        const uint4 *q1p = qs + (size_t)(v1 ? r1 : 0) * bpr + b0;
        const __half *d0p = ds + (size_t)(v0 ? r0 : 0) * bpr + b0;
        const __half *d1p = ds + (size_t)(v1 ? r1 : 0) * bpr + b0;
#pragma unroll 2
        for (int bl = lane; bl < nb; bl += 32) {
            const uint4 q0 = __ldg(q0p + bl);
            const uint4 q1 = __ldg(q1p + bl);
            const float d0 = __half2float(__ldg(d0p + bl));
            const float d1 = __half2float(__ldg(d1p + bl));
            q4_block_dot<M>(q0, d0, xs + bl * XPAD, xs_stride, xsum + bl, kcb, acc0);
            q4_block_dot<M>(q1, d1, xs + bl * XPAD, xs_stride, xsum + bl, kcb, acc1);
        }
    };

    auto epilogue = [&](int rg, float (&acc0)[M], float (&acc1)[M]) {
        const int r0 = rg * MV_ROWS + warp * 2;
        const int r1 = r0 + 1;
#pragma unroll
        for (int m = 0; m < M; ++m) {
            const float a0 = warp_sum(acc0[m]);
            const float a1 = warp_sum(acc1[m]);
            if (lane == 0) {
                if (EPI == EPI_SILU_MUL) {
                    if (r1 < N) y[(size_t)m * ldy + (r0 >> 1)] = silu_f(a0) * a1;
                } else {
                    if (r0 < N) {
                        float v = a0 + (bias ? bias[r0] : 0.0f);
                        if (EPI == EPI_RESIDUAL) v += res[(size_t)m * ldy + r0];
                        if (EPI == EPI_GELU) v = gelu_erf(v);
                        y[(size_t)m * ldy + r0] = v;
                    }
                    if (r1 < N) {
                        float v = a1 + (bias ? bias[r1] : 0.0f);
                        if (EPI == EPI_RESIDUAL) v += res[(size_t)m * ldy + r1];
                        if (EPI == EPI_GELU) v = gelu_erf(v);
                        y[(size_t)m * ldy + r1] = v;
                    }
                }
            }
        }
    };

    if (n_chunks == 1) {
        const int nb = stage(0);
        for (int rg = blockIdx.x; rg < n_rg; rg += gridDim.x) {
            float acc0[M], acc1[M];
#pragma unroll
            for (int m = 0; m < M; ++m) acc0[m] = acc1[m] = 0.0f;
            accumulate(rg, 0, nb, acc0, acc1);
            epilogue(rg, acc0, acc1);
        }
    } else {
        const int rg = blockIdx.x;
        float acc0[M], acc1[M];
#pragma unroll
        for (int m = 0; m < M; ++m) acc0[m] = acc1[m] = 0.0f;
        for (int c = 0; c < n_chunks; ++c) {
            const int nb = stage(c);
            accumulate(rg, c, nb, acc0, acc1);
            __syncthreads();
        }
        epilogue(rg, acc0, acc1);
    }
}

template <int M, int EPI>
static void matvec_launch_t(const Q4Weight &w, const float *x, float *y, int ldy, const float *bias,
                            const float *res, cudaStream_t st) {
    const int bpr = w.K / 32;
    const size_t budget = 96 * 1024;
    int kcb = (int)(budget / ((size_t)M * (XPAD + 1) * sizeof(float)));
    if (kcb >= bpr) kcb = bpr;
    else kcb = (kcb / 32) * 32;
    const int n_chunks = (bpr + kcb - 1) / kcb;
    const size_t smem = (size_t)M * kcb * (XPAD + 1) * sizeof(float);
    static SmemAttr attr;
    smem_attr_check(ensure_dyn_smem(q4_matvec_kernel<M, EPI>, 100 * 1024, attr), "q4_matvec");
    const int n_rg = (w.N + MV_ROWS - 1) / MV_ROWS;
    int grid = n_rg;
    if (n_chunks == 1 && grid > VOX_NUM_SMS * 8) grid = VOX_NUM_SMS * 8;
    q4_matvec_kernel<M, EPI><<<grid, MV_THREADS, smem, st>>>(w.qs, w.d, w.N, w.K, x, y, ldy, bias, res, kcb, n_chunks);
    post_launch("q4_matvec");
}

template <int M>
static void matvec_launch_m(const Q4Weight &w, const float *x, float *y, int ldy, const float *bias,
                            const float *res, int epi, cudaStream_t st) {
    switch (epi) {
        case EPI_NONE: matvec_launch_t<M, EPI_NONE>(w, x, y, ldy, bias, res, st); break;
        case EPI_RESIDUAL: matvec_launch_t<M, EPI_RESIDUAL>(w, x, y, ldy, bias, res, st); break;
        case EPI_SILU_MUL: matvec_launch_t<M, EPI_SILU_MUL>(w, x, y, ldy, bias, res, st); break;
        case EPI_GELU: matvec_launch_t<M, EPI_GELU>(w, x, y, ldy, bias, res, st); break;
        default: fail(VOX_EINVAL, "bad epilogue");
    }
}

void launch_q4_matvec(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                      const float *res, int epi, cudaStream_t st) {
    VOX_CHECK(M >= 1 && M <= 8, VOX_EINVAL, "q4_matvec: M=%d out of range", M);
    VOX_CHECK(w.K % 32 == 0, VOX_EINVAL, "q4_matvec: K=%d not a multiple of 32", w.K);
    switch (M) {
        case 1: matvec_launch_m<1>(w, x, y, ldy, bias, res, epi, st); break;
        case 2: matvec_launch_m<2>(w, x, y, ldy, bias, res, epi, st); break;
        case 3: matvec_launch_m<3>(w, x, y, ldy, bias, res, epi, st); break;
        case 4: matvec_launch_m<4>(w, x, y, ldy, bias, res, epi, st); break;
        case 5: matvec_launch_m<5>(w, x, y, ldy, bias, res, epi, st); break;
        case 6: matvec_launch_m<6>(w, x, y, ldy, bias, res, epi, st); break;
        case 7: matvec_launch_m<7>(w, x, y, ldy, bias, res, epi, st); break;
        default: matvec_launch_m<8>(w, x, y, ldy, bias, res, epi, st); break;
    }
}

// =====================================================================================
// K3 (v1): tiled SIMT GEMM  C[M,N] = A[M,K] . W[N,K]^T  with the weight tile dequantised in
// shared memory (reference src/gguf/shader_naive.wgsl:31-98 computes the same sums without reuse).
// BMODE 0: W is Q4 (w = (q-8)*d in f32, exactly the reference's dequant), 1: W is f32 row-major.
// AMODE 0: A row-major [M][lda]; 1: implicit im2col of a time-major [B][T_in][C_in] tensor for a
// k=3, stride 2, pad 1 conv (reference src/models/layers/conv.rs:78-83), K = 3*C_in, k = tap*C_in+c.
// =====================================================================================
constexpr int GB_M = 64, GB_N = 64, GB_K = 32, GB_PAD = 4, GB_THREADS = 256;

struct GemmArgs {
    const float *a;
    int M, N, K, lda;
    const uint4 *qs;
    const __half *ds;
    const float *wf;
    float *y;
    int ldy;
    const float *bias;
    const float *res;
    int T_in, T_out, C_in;
    int t_off;  // implicit im2col: output row t of the launch is conv output t + t_off (streaming: only the new frames)
};

template <int BMODE, int AMODE, int EPI>
__global__ void __launch_bounds__(GB_THREADS) gemm_kernel(const GemmArgs p) {
    __shared__ __align__(16) float As[GB_K][GB_M + GB_PAD];
    __shared__ __align__(16) float Ws[GB_K][GB_N + GB_PAD];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * GB_M, n0 = blockIdx.x * GB_N;
    const int bpr = p.K >> 5;
    float c[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) c[i][j] = 0.0f;

    for (int k0 = 0; k0 < p.K; k0 += GB_K) {
        // ---- A tile -> As[k][m]
#pragma unroll
        for (int it = 0; it < 2; ++it) {
            const int idx = tid + it * GB_THREADS;
            const int row = idx >> 3, kq = idx & 7;
            const int gm = m0 + row;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gm < p.M) {
                if (AMODE == 0) {
                    v = *reinterpret_cast<const float4 *>(p.a + (size_t)gm * p.lda + k0 + kq * 4);
                } else {
                    const int b = gm / p.T_out, t = gm - b * p.T_out;
                    const int tap = k0 / p.C_in, c0 = k0 - tap * p.C_in;
                    const int tin = 2 * (t + p.t_off) - 1 + tap;
                    if (tin >= 0 && tin < p.T_in)
                        v = *reinterpret_cast<const float4 *>(p.a + ((size_t)b * p.T_in + tin) * p.C_in + c0 + kq * 4);
                }
            }
            As[kq * 4 + 0][row] = v.x;
            As[kq * 4 + 1][row] = v.y;
            As[kq * 4 + 2][row] = v.z;
            As[kq * 4 + 3][row] = v.w;
        }
        // ---- W tile -> Ws[k][n]
        if (BMODE == 0) {
            const int row = tid >> 2, wi = tid & 3;
            const int gn = n0 + row;
            float lo[4] = {0.f, 0.f, 0.f, 0.f}, hi[4] = {0.f, 0.f, 0.f, 0.f};
            if (gn < p.N) {
                const size_t blk = (size_t)gn * bpr + (k0 >> 5);
                const uint32_t w = reinterpret_cast<const uint32_t *>(p.qs + blk)[wi];
                const float dd = __half2float(p.ds[blk]);
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const uint32_t byte = (w >> (8 * t)) & 0xFFu;
                    lo[t] = ((float)(byte & 0xFu) - 8.0f) * dd;
                    hi[t] = ((float)(byte >> 4) - 8.0f) * dd;
                }
            }
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                Ws[wi * 4 + t][row] = lo[t];
                Ws[16 + wi * 4 + t][row] = hi[t];
            }
        } else {
#pragma unroll
            for (int it = 0; it < 2; ++it) {
                const int idx = tid + it * GB_THREADS;
                const int row = idx >> 3, kq = idx & 7;
                const int gn = n0 + row;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (gn < p.N) v = *reinterpret_cast<const float4 *>(p.wf + (size_t)gn * p.K + k0 + kq * 4);
                Ws[kq * 4 + 0][row] = v.x;
                Ws[kq * 4 + 1][row] = v.y;
                Ws[kq * 4 + 2][row] = v.z;
                Ws[kq * 4 + 3][row] = v.w;
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < GB_K; ++k) {
            const float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
            const float4 b = *reinterpret_cast<const float4 *>(&Ws[k][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) c[i][j] = fmaf(av[i], bv[j], c[i][j]);
        }
        __syncthreads();
    }
    // ---- epilogue
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int gm = m0 + ty * 4 + i;
        if (gm >= p.M) continue;
        if (EPI == EPI_SILU_MUL) {
#pragma unroll
            for (int j = 0; j < 4; j += 2) {
                const int gn = n0 + tx * 4 + j;
                if (gn + 1 < p.N) p.y[(size_t)gm * p.ldy + (gn >> 1)] = silu_f(c[i][j]) * c[i][j + 1];
            }
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int gn = n0 + tx * 4 + j;
                if (gn >= p.N) continue;
                float v = c[i][j] + (p.bias ? p.bias[gn] : 0.0f);
                if (EPI == EPI_RESIDUAL) v += p.res[(size_t)gm * p.ldy + gn];
                if (EPI == EPI_GELU) v = gelu_erf(v);
                p.y[(size_t)gm * p.ldy + gn] = v;
            }
        }
    }
}

template <int BMODE, int AMODE>
static void gemm_launch(const GemmArgs &p, int epi, cudaStream_t st) {
    dim3 grid((p.N + GB_N - 1) / GB_N, (p.M + GB_M - 1) / GB_M);
    switch (epi) {
        case EPI_NONE: gemm_kernel<BMODE, AMODE, EPI_NONE><<<grid, GB_THREADS, 0, st>>>(p); break;
        case EPI_RESIDUAL: gemm_kernel<BMODE, AMODE, EPI_RESIDUAL><<<grid, GB_THREADS, 0, st>>>(p); break;
        case EPI_SILU_MUL: gemm_kernel<BMODE, AMODE, EPI_SILU_MUL><<<grid, GB_THREADS, 0, st>>>(p); break;
        case EPI_GELU: gemm_kernel<BMODE, AMODE, EPI_GELU><<<grid, GB_THREADS, 0, st>>>(p); break;
        default: fail(VOX_EINVAL, "bad epilogue");
    }
    post_launch("gemm");
}

void launch_q4_gemm(const Q4Weight &w, const float *a, int M, float *y, int ldy, const float *bias,
                    const float *res, int epi, cudaStream_t st) {
    VOX_CHECK(w.K % 32 == 0, VOX_EINVAL, "q4_gemm: K=%d not a multiple of 32", w.K);
    if (M <= 0) return;
    GemmArgs p{};
    p.a = a; p.M = M; p.N = w.N; p.K = w.K; p.lda = w.K;
    p.qs = w.qs; p.ds = w.d; p.y = y; p.ldy = ldy; p.bias = bias; p.res = res;
    gemm_launch<0, 0>(p, epi, st);
}

void launch_conv2_gemm(const float *in, const float *w, const float *bias, float *out, int B, int T_in,
                       int T_out, int C_in, int C_out, cudaStream_t st, int t_off) {
    VOX_CHECK(C_in % 32 == 0, VOX_EINVAL, "conv2: C_in=%d not a multiple of 32", C_in);
    VOX_CHECK(t_off == 0 || B == 1, VOX_EINVAL, "conv2: a frame offset needs B == 1");
    if (B * T_out <= 0) return;
    GemmArgs p{};
    p.a = in; p.M = B * T_out; p.N = C_out; p.K = 3 * C_in; p.lda = 0;
    p.wf = w; p.y = out; p.ldy = C_out; p.bias = bias; p.res = nullptr;
    p.T_in = T_in; p.T_out = T_out; p.C_in = C_in; p.t_off = t_off;
    gemm_launch<1, 1>(p, EPI_GELU, st);
}

__global__ void transpose_mel_kernel(const float *__restrict__ in, float *__restrict__ out, int C, int T) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, t = t0 + threadIdx.x;
        tile[i][threadIdx.x] = (c < C && t < T) ? in[((size_t)b * C + c) * T + t] : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int t = t0 + i, c = c0 + threadIdx.x;
        if (t < T && c < C) out[((size_t)b * T + t) * C + c] = tile[threadIdx.x][i];
    }
}
void launch_transpose_mel(const float *in, float *out, int B, int C, int T, cudaStream_t st) {
    dim3 grid((T + 31) / 32, (C + 31) / 32, B), block(32, 8);
    transpose_mel_kernel<<<grid, block, 0, st>>>(in, out, C, T);
    post_launch("transpose_mel");
}

// =====================================================================================
// RMSNorm (reference rms_norm.rs:42-47, burn::nn::RmsNorm): y = x / sqrt(mean(x^2)+eps) * gamma,
// optionally times the precomputed ADA vector (1 + w2(gelu(w0 t))), model.rs:250-255.
// =====================================================================================
__global__ void rmsnorm_kernel(const float *__restrict__ x, const float *__restrict__ gamma,
                               const float *__restrict__ scale, float *__restrict__ y, int dim, float eps) {
    __shared__ float red[32];
    const float *xr = x + (size_t)blockIdx.x * dim;
    float *yr = y + (size_t)blockIdx.x * dim;
    float s = 0.0f;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) s = fmaf(xr[i], xr[i], s);
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0f;
        v = warp_sum(v);
        if (threadIdx.x == 0) red[0] = v;
    }
    __syncthreads();
    const float rms = sqrtf(red[0] / (float)dim + eps);
    for (int i = threadIdx.x; i < dim; i += blockDim.x) {
        float v = (xr[i] / rms) * gamma[i];
        if (scale) v *= scale[i];
        yr[i] = v;
    }
}

void launch_rmsnorm(const float *x, const float *gamma, const float *scale, float *y, int rows, int dim,
                    float eps, cudaStream_t st) {
    if (rows <= 0) return;
    rmsnorm_kernel<<<rows, 256, 0, st>>>(x, gamma, scale, y, dim, eps);
    post_launch("rmsnorm");
}

// =====================================================================================
// RoPE, interleaved pairs (reference rope.rs:103-141), tables built on the host as in rope.rs:35-64.
// =====================================================================================
__global__ void rope_inplace_kernel(float *buf, int ld, int q_off, int n_q, int k_off, int n_k, int hd,
                                    int seq, int pos0, const float *__restrict__ cos_t,
                                    const float *__restrict__ sin_t) {
    const int r = blockIdx.x;
    const int pos = pos0 + (r % seq);
    const int half = hd >> 1;
    float *row = buf + (size_t)r * ld;
    const int total = (n_q + n_k) * half;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int h = i / half, p = i - h * half;
        float *v = (h < n_q) ? row + q_off + h * hd + 2 * p : row + k_off + (h - n_q) * hd + 2 * p;
        const float c = cos_t[(size_t)pos * half + p], s = sin_t[(size_t)pos * half + p];
        const float xr = v[0], xi = v[1];
        v[0] = xr * c - xi * s;
        v[1] = xr * s + xi * c;
    }
}

void launch_rope_inplace(float *buf, int rows, int ld, int q_off, int n_q, int k_off, int n_k, int hd,
                         int seq, int pos0, const float *cos_t, const float *sin_t, cudaStream_t st) {
    if (rows <= 0) return;
    rope_inplace_kernel<<<rows, 256, 0, st>>>(buf, ld, q_off, n_q, k_off, n_k, hd, seq, pos0, cos_t, sin_t);
    post_launch("rope");
}

// =====================================================================================
// K4 (v1): encoder attention, causal + sliding window, flash-style online softmax in f32.
//   softmax(q k^T * scale + causal + (|i-j| > window -> -inf)) v   (model.rs:77-122, masking.rs:9-44)
// CTA = 32 queries of one (batch, head); 128 threads; thread (r = tid/4, c = tid%4) owns query row
// r, keys c, c+4, ... of each 64-key tile and a quarter of the head dimension of the output.
// Only the causal band is visited (<= window+1 keys per query).
// =====================================================================================
constexpr int EA_BQ = 32, EA_BK = 64, EA_THREADS = 128;

template <int HD>
__global__ void __launch_bounds__(EA_THREADS)
enc_attention_kernel(const float *__restrict__ qkv, float *__restrict__ out, int S, int H, int ld, int q_off,
                     int k_off, int v_off, int window, float scale) {
    extern __shared__ __align__(16) float sm[];
    float *Qs = sm;                          // [32][HD+1]  (odd strides: rows map to distinct banks)
    float *Ks = Qs + EA_BQ * (HD + 1);       // [64][HD+1]
    float *Vs = Ks + EA_BK * (HD + 1);       // [64][HD]
    float *Ps = Vs + EA_BK * HD;             // [32][65]
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * EA_BQ;
    const int tid = threadIdx.x, r = tid >> 2, c = tid & 3;
    constexpr int DQ = HD / 4;
    const float *base = qkv + (size_t)b * S * ld;
    for (int i = tid; i < EA_BQ * HD; i += EA_THREADS) {
        const int rr = i / HD, d = i - rr * HD;
        const int gi = q0 + rr;
        Qs[rr * (HD + 1) + d] = gi < S ? base[(size_t)gi * ld + q_off + h * HD + d] : 0.0f;
    }
    const int gi = q0 + r;
    float o[DQ];
#pragma unroll
    for (int d = 0; d < DQ; ++d) o[d] = 0.0f;
    float m_run = -INFINITY, l_run = 0.0f;
    const int q_last = min(q0 + EA_BQ - 1, S - 1);
    int j_begin = q0 - window;
    if (j_begin < 0) j_begin = 0;
    j_begin = (j_begin / EA_BK) * EA_BK;
    for (int j0 = j_begin; j0 <= q_last; j0 += EA_BK) {
        __syncthreads();
        for (int i = tid; i < EA_BK * HD; i += EA_THREADS) {
            const int kk = i / HD, d = i - kk * HD;
            const int gj = j0 + kk;
            float kv = 0.0f, vv = 0.0f;
            if (gj < S) {
                kv = base[(size_t)gj * ld + k_off + h * HD + d];
                vv = base[(size_t)gj * ld + v_off + h * HD + d];
            }
            Ks[kk * (HD + 1) + d] = kv;
            Vs[kk * HD + d] = vv;
        }
        __syncthreads();
        float s[16];
        float m_t = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
            const int kk = c + 4 * jj;
            const int gj = j0 + kk;
            const float *qr = Qs + r * (HD + 1);
            const float *kr = Ks + kk * (HD + 1);
            float acc = 0.0f;
#pragma unroll 16
            for (int d = 0; d < HD; ++d) acc = fmaf(qr[d], kr[d], acc);
            const bool valid = (gj < S) && (gj <= gi) && (gi - gj <= window);
            s[jj] = valid ? acc * scale : -INFINITY;
            m_t = fmaxf(m_t, s[jj]);
        }
        m_t = fmaxf(m_t, __shfl_xor_sync(0xffffffffu, m_t, 1));
        m_t = fmaxf(m_t, __shfl_xor_sync(0xffffffffu, m_t, 2));
        const float m_new = fmaxf(m_run, m_t);
        float alpha = 1.0f, psum = 0.0f;
        if (m_new == -INFINITY) {
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) Ps[r * (EA_BK + 1) + c + 4 * jj] = 0.0f;
        } else {
            alpha = expf(m_run - m_new);
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) {
                const float pv = expf(s[jj] - m_new);
                psum += pv;
                Ps[r * (EA_BK + 1) + c + 4 * jj] = pv;
            }
        }
        psum += __shfl_xor_sync(0xffffffffu, psum, 1);
        psum += __shfl_xor_sync(0xffffffffu, psum, 2);
        l_run = l_run * alpha + psum;
        m_run = m_new;
#pragma unroll
        for (int d = 0; d < DQ; ++d) o[d] *= alpha;
        __syncwarp();
        for (int kk = 0; kk < EA_BK; ++kk) {
            const float pv = Ps[r * (EA_BK + 1) + kk];
            const float *vr = Vs + kk * HD + c;  // thread c owns head dims d = 4 i + c: conflict-free V reads
#pragma unroll
            for (int d = 0; d < DQ; ++d) o[d] = fmaf(pv, vr[4 * d], o[d]);
        }
    }
    if (gi < S) {
        const float inv = 1.0f / l_run;
        float *orow = out + ((size_t)b * S + gi) * (H * HD) + h * HD + c;
#pragma unroll
        for (int d = 0; d < DQ; ++d) orow[4 * d] = o[d] * inv;
    }
}

void launch_enc_attention(const float *qkv, float *out, int B, int S, int H, int hd, int ld, int q_off,
                          int k_off, int v_off, int window, float scale, cudaStream_t st) {
    if (S <= 0) return;
    dim3 grid((S + EA_BQ - 1) / EA_BQ, H, B);
    const size_t smem = (size_t)(EA_BQ * (hd + 1) + EA_BK * (hd + 1) + EA_BK * hd + EA_BQ * (EA_BK + 1)) * sizeof(float);
#define ENC_ATTN_CASE(HD)                                                                                   \
    case HD: {                                                                                              \
        static SmemAttr attr;                                                                               \
        smem_attr_check(ensure_dyn_smem(enc_attention_kernel<HD>, smem, attr), "enc_attention");              \
        enc_attention_kernel<HD><<<grid, EA_THREADS, smem, st>>>(qkv, out, S, H, ld, q_off, k_off, v_off,   \
                                                                 window, scale);                            \
        break;                                                                                              \
    }
    switch (hd) {
        ENC_ATTN_CASE(32)
        ENC_ATTN_CASE(64)
        ENC_ATTN_CASE(128)
        default: fail(VOX_EINVAL, fmt("enc_attention: unsupported head_dim %d", hd));
    }
#undef ENC_ATTN_CASE
    post_launch("enc_attention");
}

// =====================================================================================
// Decoder: RoPE + KV append (kv_cache.rs:116-142; K cached post-RoPE) and GQA attention over the
// cache without materialising the repeated K/V (model.rs:125-197).  Positions come from a device
// counter so the same CUDA graph can be replayed for every step.
// =====================================================================================
__global__ void dec_rope_append_kernel(float *qkv, int M, int ld, int H, int Hkv, int hd, const KvView kv,
                                       const float *__restrict__ cos_t, const float *__restrict__ sin_t) {
    const int i = blockIdx.x, b = blockIdx.y;
    const int pos = kv.pos[b] + i;
    if (pos >= kv.max_seq()) return;
    const int half = hd >> 1;
    float *row = qkv + ((size_t)b * M + i) * ld;
    const float *cr = cos_t + (size_t)pos * half, *sr = sin_t + (size_t)pos * half;
    for (int t = threadIdx.x; t < H * half; t += blockDim.x) {
        const int h = t / half, p = t - h * half;
        float *v = row + h * hd + 2 * p;
        const float xr = v[0], xi = v[1];
        v[0] = xr * cr[p] - xi * sr[p];
        v[1] = xr * sr[p] + xi * cr[p];
    }
    const float *krow = row + H * hd;
    const float *vrow = krow + Hkv * hd;
    for (int t = threadIdx.x; t < Hkv * half; t += blockDim.x) {
        const int h = t / half, p = t - h * half;
        const float xr = krow[h * hd + 2 * p], xi = krow[h * hd + 2 * p + 1];
        float *dst = kv.k + kv_index(kv, b, Hkv, h, pos, hd) + 2 * p;
        dst[0] = xr * cr[p] - xi * sr[p];
        dst[1] = xr * sr[p] + xi * cr[p];
    }
    for (int t = threadIdx.x; t < Hkv * hd; t += blockDim.x) {
        const int h = t / hd, d = t - h * hd;
        kv.v[kv_index(kv, b, Hkv, h, pos, hd) + d] = vrow[t];
    }
}

void launch_dec_rope_append(float *qkv, int B, int M, int ld, int H, int Hkv, int hd, const KvView &kv,
                            const float *cos_t, const float *sin_t, cudaStream_t st) {
    dim3 grid(M, B);
    dec_rope_append_kernel<<<grid, 256, 0, st>>>(qkv, M, ld, H, Hkv, hd, kv, cos_t, sin_t);
    post_launch("dec_rope_append");
}

// grid (Hkv, M, B); block = 32 * (H/Hkv): one warp per query head of the group.
__global__ void dec_attention_kernel(const float *__restrict__ qkv, int M, int ld, int H, int Hkv, int hd, const KvView kv,
                                     int window, float scale, float *__restrict__ out) {
    extern __shared__ float sm[];
    const int kvh = blockIdx.x, i = blockIdx.y, b = blockIdx.z;
    const int G = H / Hkv;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pos = kv.pos[b] + i;
    const int max_seq = kv.max_seq();
    if (pos >= max_seq) return;
    float *qsm = sm + warp * hd;                        // [G][hd]
    float *sc = sm + G * hd + (size_t)warp * max_seq;   // [G][max_seq]
    const int h = kvh * G + warp;
    const float *qrow = qkv + ((size_t)b * M + i) * ld + h * hd;
    for (int d = lane; d < hd; d += 32) qsm[d] = qrow[d];
    __syncwarp();
    const int j_lo = pos - window > 0 ? pos - window : 0;
    float mx = -INFINITY;
    for (int j = j_lo + lane; j <= pos; j += 32) {
        const float4 *kr = reinterpret_cast<const float4 *>(kv.k + kv_index(kv, b, Hkv, kvh, j, hd));
        const float4 *q4 = reinterpret_cast<const float4 *>(qsm);
        float acc = 0.0f;
        for (int d = 0; d < (hd >> 2); ++d) {
            const float4 kk = kr[d];
            const float4 qv = q4[d];
            acc = fmaf(qv.x, kk.x, acc);
            acc = fmaf(qv.y, kk.y, acc);
            acc = fmaf(qv.z, kk.z, acc);
            acc = fmaf(qv.w, kk.w, acc);
        }
        acc *= scale;
        sc[j] = acc;
        mx = fmaxf(mx, acc);
    }
    mx = warp_max(mx);
    float sum = 0.0f;
    for (int j = j_lo + lane; j <= pos; j += 32) {
        const float pv = expf(sc[j] - mx);
        sc[j] = pv;
        sum += pv;
    }
    sum = warp_sum(sum);
    __syncwarp();
    const float inv = 1.0f / sum;
    float *orow = out + ((size_t)b * M + i) * (H * hd) + h * hd;
    for (int d = lane; d < hd; d += 32) {
        float acc = 0.0f;
        for (int j = j_lo; j <= pos; ++j) acc = fmaf(sc[j], kv.v[kv_index(kv, b, Hkv, kvh, j, hd) + d], acc);
        orow[d] = acc * inv;
    }
}

void launch_dec_attention(const float *qkv, int B, int M, int ld, int H, int Hkv, int hd, const KvView &kv, int window,
                          float scale, float *out, cudaStream_t st) {
    const int G = H / Hkv;
    dim3 grid(Hkv, M, B);
    const size_t smem = (size_t)G * (hd + kv.max_seq()) * sizeof(float);
    VOX_CHECK(smem <= 200 * 1024, VOX_EINVAL, "dec_attention: max_seq %d too large for the v1 kernel", kv.max_seq());
    static SmemAttr attr;
    if (smem > 48 * 1024) smem_attr_check(ensure_dyn_smem(dec_attention_kernel, smem, attr), "dec_attention");
    dec_attention_kernel<<<grid, 32 * G, smem, st>>>(qkv, M, ld, H, Hkv, hd, kv, window, scale, out);
    post_launch("dec_attention");
}

// =====================================================================================
// Embedding gather from the Q4 table + audio add (model.rs:584-618, 942-948), device-side ids.
// =====================================================================================
__global__ void embed_kernel(const uint4 *__restrict__ qs, const __half *__restrict__ ds, int K,
                             const int *__restrict__ ids, const float *__restrict__ audio, int audio_seq, int M,
                             const int *__restrict__ pos_ptr, float *__restrict__ x, float *__restrict__ ssq_out,
                             const int rows_total, const float *const *__restrict__ audio_rows) {
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");  // PDL: next kernel may prefetch weights
    const int i = blockIdx.x, b = blockIdx.y;
    const int r = b * M + i;
    const int id = ids[r];
    const int bpr = K >> 5;
    const float *arow = nullptr;
    if (audio_rows) {
        arow = audio_rows[b] ? audio_rows[b] + (size_t)i * K : nullptr;
    } else if (audio) {
        const int pos = (pos_ptr ? pos_ptr[b] : 0) + i;
        arow = audio + ((size_t)b * audio_seq + pos) * K;
    }
    for (int t = threadIdx.x; t < bpr * 16; t += blockDim.x) {
        const int blk = t >> 4, j = t & 15;
        const uint8_t byte = reinterpret_cast<const uint8_t *>(qs + (size_t)id * bpr + blk)[j];
        const float dd = __half2float(ds[(size_t)id * bpr + blk]);
        const int k = blk * 32 + j;
        float lo = ((float)(byte & 0xF) - 8.0f) * dd;
        float hi = ((float)(byte >> 4) - 8.0f) * dd;
        if (arow) {
            lo = arow[k] + lo;
            hi = arow[k + 16] + hi;
        }
        x[(size_t)r * K + k] = lo;
        x[(size_t)r * K + k + 16] = hi;
    }
    if (ssq_out) {  // per-16-element sums of squares for the consumer's fused RMSNorm (fixed order)
        __syncthreads();
        for (int t = threadIdx.x; t < (K >> 4); t += blockDim.x) {
            const float *p = x + (size_t)r * K + 16 * t;
            float s = 0.0f;
#pragma unroll
            for (int j = 0; j < 16; ++j) s = fmaf(p[j], p[j], s);
            ssq_out[(size_t)t * rows_total + r] = s;
        }
    }
}

void launch_embed(const Q4Weight &emb, const int *ids, const float *audio, int audio_seq, int B, int M,
                  const int *pos_ptr, float *x, float *ssq_out, cudaStream_t st, const float *const *audio_rows) {
    dim3 grid(M, B);
    embed_kernel<<<grid, 256, 0, st>>>(emb.qs, emb.d, emb.K, ids, audio, audio_seq, M, pos_ptr, x, ssq_out, B * M, audio_rows);
    post_launch("embed");
}

// =====================================================================================
// Greedy argmax, lowest index wins ties (reference: Burn argmax + into_scalar, model.rs:922,957).
// =====================================================================================
__global__ void argmax_kernel(const float *__restrict__ logits, int V, int *tok, int *out_ids, int out_ld,
                              const int *__restrict__ out_pos_ptr) {
    __shared__ float sv[32];
    __shared__ int si[32];
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
    const int b = blockIdx.x;
    const float *row = logits + (size_t)b * V;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
        const float v = row[i];
        if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    }
    if (bi == 0x7fffffff) bi = 0;  // all NaN/-inf: index 0
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int nw = blockDim.x >> 5;
        best = threadIdx.x < nw ? sv[threadIdx.x] : -INFINITY;
        bi = threadIdx.x < nw ? si[threadIdx.x] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (threadIdx.x == 0) {
            tok[b] = bi;
            if (out_ids) out_ids[(size_t)b * out_ld + out_pos_ptr[b]] = bi;
        }
    }
}

void launch_argmax(const float *logits, int B, int V, int *tok, int *out_ids, int out_ld,
                   const int *out_pos_ptr, cudaStream_t st) {
    argmax_kernel<<<B, 1024, 0, st>>>(logits, V, tok, out_ids, out_ld, out_pos_ptr);
    post_launch("argmax");
}

__global__ void argmax_multi_kernel(const float *__restrict__ logits, int V, int *tok, int *out_ids, int out_ld,
                                    const int *__restrict__ out_pos_ptr, float *svals, int *sidx, int *counters) {
    __shared__ float sv[32];
    __shared__ int si[32];
    __shared__ int is_last;
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
    const int part = blockIdx.x, b = blockIdx.y;
    const int per = (V + ARGMAX_PARTS - 1) / ARGMAX_PARTS;
    const int i0 = part * per, i1 = min(V, i0 + per);
    const float *row = logits + (size_t)b * V;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
        const float v = row[i];
        if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    }
    auto combine = [](float &bv, int &bx, float ov, int ox) {
        if (ov > bv || (ov == bv && ox < bx)) { bv = ov; bx = ox; }
    };
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int nw = blockDim.x >> 5;
        best = threadIdx.x < nw ? sv[threadIdx.x] : -INFINITY;
        bi = threadIdx.x < nw ? si[threadIdx.x] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
        if (threadIdx.x == 0) {
            svals[b * ARGMAX_PARTS + part] = best;
            sidx[b * ARGMAX_PARTS + part] = bi;
            __threadfence();
            const int old = atomicAdd(&counters[b], 1);
            is_last = (old == ARGMAX_PARTS - 1);
            if (is_last) counters[b] = 0;
        }
    }
    __syncthreads();
    if (is_last && threadIdx.x < 32) {
        __threadfence();
        best = -INFINITY;
        bi = 0x7fffffff;
        for (int p = threadIdx.x; p < ARGMAX_PARTS; p += 32)
            combine(best, bi, __ldcg(svals + b * ARGMAX_PARTS + p), __ldcg(sidx + b * ARGMAX_PARTS + p));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
        if (threadIdx.x == 0) {
            if (bi == 0x7fffffff) bi = 0;
            tok[b] = bi;
            if (out_ids) out_ids[(size_t)b * out_ld + out_pos_ptr[b]] = bi;
        }
    }
}

void launch_argmax_multi(const float *logits, int B, int V, int *tok, int *out_ids, int out_ld,
                         const int *out_pos_ptr, float *scratch_vals, int *scratch_idx, int *counters,
                         cudaStream_t st) {
    dim3 grid(ARGMAX_PARTS, B);
    argmax_multi_kernel<<<grid, 256, 0, st>>>(logits, V, tok, out_ids, out_ld, out_pos_ptr, scratch_vals, scratch_idx, counters);
    post_launch("argmax_multi");
}

__global__ void advance_kernel(int *a, int da, int *b, int db, int n) {
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
    const int i = threadIdx.x;
    if (i < n) {
        if (a) a[i] += da;
        if (b) b[i] += db;
    }
}
void launch_advance(int *a, int da, int *b, int db, int n, cudaStream_t st) {
    advance_kernel<<<1, 64, 0, st>>>(a, da, b, db, n);
    post_launch("advance");
}

__global__ void gather_last_kernel(const float *__restrict__ src, float *__restrict__ dst, int M, int dim) {
    const int b = blockIdx.x;
    const float *s = src + ((size_t)b * M + (M - 1)) * dim;
    for (int i = threadIdx.x; i < dim; i += blockDim.x) dst[(size_t)b * dim + i] = s[i];
}
void launch_gather_last(const float *src, float *dst, int B, int M, int dim, cudaStream_t st) {
    gather_last_kernel<<<B, 256, 0, st>>>(src, dst, M, dim);
    post_launch("gather_last");
}

// reshape_encoder_output (adapter.rs:108-122): drop S % factor tail rows, view [S/f, dim*f].
__global__ void reshape_rows_kernel(const float *__restrict__ src, float *__restrict__ dst, int S, int S_out,
                                    int dim, int factor) {
    const int so = blockIdx.x, b = blockIdx.y;
    const float *s = src + ((size_t)b * S + (size_t)so * factor) * dim;
    float *d = dst + ((size_t)b * S_out + so) * dim * factor;
    for (int i = threadIdx.x; i < dim * factor; i += blockDim.x) d[i] = s[i];
}
void launch_reshape_rows(const float *src, float *dst, int B, int S, int S_out, int dim, int factor,
                         cudaStream_t st) {
    if (S_out <= 0) return;
    dim3 grid(S_out, B);
    reshape_rows_kernel<<<grid, 256, 0, st>>>(src, dst, S, S_out, dim, factor);
    post_launch("reshape_rows");
}

__global__ void mul_vec_kernel(const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = a[i] * b[i];
}
void launch_mul_vec(const float *a, const float *b, float *out, size_t n, cudaStream_t st) {
    mul_vec_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, b, out, n);
    post_launch("mul_vec");
}

__global__ void gelu_kernel(float *x, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = gelu_erf(x[i]);
}
void launch_gelu(float *x, size_t n, cudaStream_t st) {
    if (!n) return;
    gelu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, n);
    post_launch("gelu");
}

// =====================================================================================
// K1: log-mel front-end (reference src/audio/mel.rs:128-257).  CTA = 8 frames; the reflect-padded,
// Hann-windowed frames are staged in shared memory (128-bit global reads where aligned); thread k
// computes DFT bin k of all 8 frames with a 400-entry twiddle table (index k*n mod 400); the 201-bin
// power spectrum stays in shared memory for the sparse triangular filterbank, log10, clamp, scale.
// =====================================================================================
constexpr int MEL_FR = 8, MEL_THREADS = 256, MEL_NFFT = 400, MEL_HOP = 160, MEL_NFREQ = 201, MEL_NMEL = 128;

__global__ void __launch_bounds__(MEL_THREADS)
mel_kernel(const float *__restrict__ samples, size_t n, size_t sample_stride, const float *__restrict__ window,
           const float *__restrict__ fb_vals, const int *__restrict__ fb_start, const int *__restrict__ fb_len,
           int fb_stride, float *__restrict__ out, int frames, int layout, int frame0) {
    __shared__ float ws[MEL_FR][MEL_NFFT];
    __shared__ __align__(16) float sp[(MEL_FR - 1) * MEL_HOP + MEL_NFFT];
    __shared__ float ct[MEL_NFFT], stt[MEL_NFFT];
    __shared__ float pw[MEL_FR][MEL_NFREQ + 3];
    const int b = blockIdx.y;
    const int f0 = frame0 + blockIdx.x * MEL_FR;   // frames [frame0, frames) of the signal (streaming: only the new ones)
    const float *sig = samples + (size_t)b * sample_stride;
    const long long nn = (long long)n;
    for (int i = threadIdx.x; i < MEL_NFFT; i += MEL_THREADS) {
        float s, c;
        sincospif(2.0f * (float)i / (float)MEL_NFFT, &s, &c);
        ct[i] = c;
        stt[i] = s;
    }
    // the CTA's 8 frames read one contiguous span of the signal ([160 f0 - 200, 160 (f0 + 7) + 200) = 1520 samples):
    // stage it ONCE in shared memory -- 128-bit loads where the span lies inside the signal, reflected indices
    // (torch.stft center=True, mel.rs:190-205) only at the two ends -- then window the frames out of shared memory
    {
        const long long span0 = (long long)f0 * MEL_HOP - MEL_NFFT / 2;
        constexpr int SPAN = (MEL_FR - 1) * MEL_HOP + MEL_NFFT;   // 1520
        static_assert(SPAN % 4 == 0, "span is float4-sized");
        const bool interior = span0 >= 0 && span0 + SPAN <= nn && ((reinterpret_cast<uintptr_t>(sig + span0) & 15) == 0);
        if (interior) {
            const float4 *src4 = reinterpret_cast<const float4 *>(sig + span0);
            for (int i = threadIdx.x; i < SPAN / 4; i += MEL_THREADS) reinterpret_cast<float4 *>(sp)[i] = src4[i];
        } else {
            for (int i = threadIdx.x; i < SPAN; i += MEL_THREADS) {
                long long src = span0 + i;
                if (src < 0) { src = -src; if (src > nn - 1) src = nn > 0 ? nn - 1 : 0; }
                else if (src >= nn) { src = 2 * nn - 2 - src; if (src < 0) src = 0; }
                sp[i] = nn > 0 ? sig[src] : 0.0f;
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < MEL_FR * MEL_NFFT; i += MEL_THREADS) {
        const int f = i / MEL_NFFT, j = i - f * MEL_NFFT;
        ws[f][j] = (f0 + f < frames) ? sp[f * MEL_HOP + j] * window[j] : 0.0f;
    }
    __syncthreads();
    if (threadIdx.x < MEL_NFREQ) {
        const int k = threadIdx.x;
        float re[MEL_FR], im[MEL_FR];
#pragma unroll
        for (int f = 0; f < MEL_FR; ++f) re[f] = im[f] = 0.0f;
        int idx = 0;
        for (int j = 0; j < MEL_NFFT; ++j) {
            const float c = ct[idx], s = stt[idx];
#pragma unroll
            for (int f = 0; f < MEL_FR; ++f) {
                const float v = ws[f][j];
                re[f] = fmaf(v, c, re[f]);
                im[f] = fmaf(-v, s, im[f]);
            }
            idx += k;
            if (idx >= MEL_NFFT) idx -= MEL_NFFT;
        }
#pragma unroll
        for (int f = 0; f < MEL_FR; ++f) pw[f][k] = re[f] * re[f] + im[f] * im[f];
    }
    __syncthreads();
    const float min_val = 1.5f - 8.0f;
    for (int i = threadIdx.x; i < MEL_FR * MEL_NMEL; i += MEL_THREADS) {
        const int f = i / MEL_NMEL, m = i - f * MEL_NMEL;
        if (f0 + f >= frames) continue;
        const int st = fb_start[m], ln = fb_len[m];
        const float *fv = fb_vals + (size_t)m * fb_stride;
        float acc = 0.0f;
        for (int j = 0; j < ln; ++j) acc += fv[j] * pw[f][st + j];
        float v = log10f(fmaxf(acc, 1e-10f));
        v = fmaxf(v, min_val);
        v = (v + 4.0f) / 4.0f;
        if (layout == 0) out[((size_t)b * frames + f0 + f) * MEL_NMEL + m] = v;
        else out[((size_t)b * MEL_NMEL + m) * frames + f0 + f] = v;
    }
}

void launch_mel(const float *samples, int B, size_t n, size_t sample_stride, const float *window,
                const float *fb_vals, const int *fb_start, const int *fb_len, int fb_stride, float *out,
                int frames, int layout, cudaStream_t st, int frame0) {
    if (frames - frame0 <= 0 || B <= 0) return;
    dim3 grid((frames - frame0 + MEL_FR - 1) / MEL_FR, B);
    mel_kernel<<<grid, MEL_THREADS, 0, st>>>(samples, n, sample_stride, window, fb_vals, fb_start, fb_len,
                                             fb_stride, out, frames, layout, frame0);
    post_launch("mel");
}

// peak_normalize (io.rs:59-68) + pad_audio (pad.rs:89-103) on device.
// max|x| per stream: PK_BLOCKS CTAs per stream, float4 loads, one atomicMax per CTA on the float's bit pattern (|x| >= 0:
// unsigned order == float order, so the result is exact and independent of the arrival order).  The scale
// (target / max, or 1 when max < 1e-10: io.rs:61-63) is derived by the consumer, which also writes the padded copy.
constexpr int PK_BLOCKS = 64, PK_THREADS = 256;
__global__ void __launch_bounds__(PK_THREADS) peak_max_kernel(const float *__restrict__ in, size_t n, unsigned *__restrict__ max_bits) {
    __shared__ float red[PK_THREADS / 32];
    const float *s = in + (size_t)blockIdx.y * n;
    float mx = 0.0f;
    const size_t stride = (size_t)gridDim.x * PK_THREADS;
    if ((n & 3) == 0 && ((reinterpret_cast<uintptr_t>(s) & 15) == 0)) {
        const float4 *s4 = reinterpret_cast<const float4 *>(s);
        for (size_t i = (size_t)blockIdx.x * PK_THREADS + threadIdx.x; i < n / 4; i += stride) {
            const float4 v = s4[i];
            mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
        }
    } else {
        for (size_t i = (size_t)blockIdx.x * PK_THREADS + threadIdx.x; i < n; i += stride) mx = fmaxf(mx, fabsf(s[i]));
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < PK_THREADS / 32 ? red[threadIdx.x] : 0.0f;
        v = warp_max(v);
        if (threadIdx.x == 0) atomicMax(max_bits + blockIdx.y, __float_as_uint(v));
    }
}
__global__ void scale_pad_kernel(const float *__restrict__ in, size_t n, const float *__restrict__ max_abs, float target,
                                 int do_norm, float *__restrict__ out, size_t out_stride, size_t left, int vec4) {
    const int b = blockIdx.y;
    const float mx = max_abs[b];
    const float scale = (!do_norm || mx < 1e-10f) ? 1.0f : target / mx;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec4) {
        if (i >= n / 4) return;
        float4 v = reinterpret_cast<const float4 *>(in + (size_t)b * n)[i];
        if (do_norm) { v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale; }
        reinterpret_cast<float4 *>(out + (size_t)b * out_stride + left)[i] = v;
    } else {
        if (i >= n) return;
        const float v = in[(size_t)b * n + i];
        out[(size_t)b * out_stride + left + i] = do_norm ? v * scale : v;
    }
}

void launch_peak_normalize_pad(const float *in, int B, size_t n, float target, int do_norm, float *out,
                               size_t out_stride, size_t left, float *scale_buf, cudaStream_t st) {
    cudaMemsetAsync(out, 0, sizeof(float) * out_stride * B, st);
    cudaMemsetAsync(scale_buf, 0, sizeof(float) * B, st);
    peak_max_kernel<<<dim3(PK_BLOCKS, B), PK_THREADS, 0, st>>>(in, n, reinterpret_cast<unsigned *>(scale_buf));
    post_launch("peak_max");
    const int vec4 = (n % 4 == 0 && left % 4 == 0 && out_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(out) & 15) == 0) ? 1 : 0;
    const size_t work = vec4 ? n / 4 : n;
    dim3 grid((unsigned)((work + 255) / 256), B);
    scale_pad_kernel<<<grid, 256, 0, st>>>(in, n, scale_buf, target, do_norm, out, out_stride, left, vec4);
    post_launch("scale_pad");
}

}  // namespace vox
