// gemm_tc5.cu -- K3: Q4_0 dequant-GEMM on the Hopper tensor cores (wgmma) for encoder / prefill sized problems:
//   Y[M_tok, N] = X[M_tok, K] . W[N, K]^T  (+ epilogue).
// Reference arithmetic: src/gguf/shader_naive.wgsl:31-98 (w = (q-8)*d in f32, f32 accumulate).
//
// f32-grade accuracy on f16 tensor cores ("2 x 2 split, 3 products"): wgmma has no f32-input MMA, so
//   w * 2^8  = w_hi + w_lo     f16 pieces, exact: (q-8)*d has <= 14 significant bits; hi = the 11-bit Veltkamp head of the f32
//                              product, lo = the exact tail; their f16 bit patterns are assembled with shifts and masks
//                              (g5_pack_f16x2) -- no half2 arithmetic and no conversion instructions (d' = d * 2^8 keeps lo
//                              out of the subnormal range)
//   x * 2^s_t = x_h + x_m      f16 pieces, 22 bits; s_t = per-token power of two that puts the row maximum in [2^7, 2^8)
// and the product is accumulated in f32 registers from the three largest terms
//   w_hi x_h + w_hi x_m + w_lo x_h            (dropped: w_lo x_m ~ 2^-22 |w||x|, the f32 rounding level)
// i.e. 3 f16 MMAs per 16-wide K step.  The epilogue multiplies token column t by 2^-(s_t + 8).  Measured against the
// oracle in tests/.
//
// "Swap-AB" tiling: the wgmma M dimension runs over output features, the N dimension over tokens, so a CTA owns
// Y[tok0:tok0+128, f0:f0+128]^T, split over its four warpgroups as 64 features x 64 tokens each (32 f32 accumulators
// per thread):
//   * A operand (weights): each thread dequantises one half Q4 block per 64-wide K chunk into two f16 K-major tiles in
//     shared memory (no-swizzle "interleaved" layout: 8x16-byte core matrices);
//   * B operand (tokens): the activation producer (split_tiles_kernel) already wrote x_h/x_m as f16 tiles in exactly that
//     shared-memory layout, so one 16 KB 1-D bulk copy per piece and chunk fetches them -- no tensor maps;
//   * a three-stage ring of (W, X) stages: the X copy of k-step i+1 is issued while k-step i dequantises, and wgmma
//     groups of k-step i stay in flight while k-step i+1 dequantises (one CTA barrier per k-step);
//   * epilogue straight from the accumulator registers; bias / residual / GELU / SiLU*up fused.
#include <cuda_fp16.h>

#include "common.h"
#include "kernels.h"

namespace vox {

void tc_count_launch(const char *name);

namespace {

constexpr int G5_WGS = 4;                                 // warpgroups: dequantisers, MMA issuers and epilogue alike
constexpr int G5_THREADS = G5_WGS * 128;
constexpr int G5_BM = 128;   // features per CTA
constexpr int G5_BN = 128;   // tokens per CTA
constexpr int G5_BK = 64;    // K per pipeline stage
constexpr int G5_TILE_BYTES = G5_BM * G5_BK * 2;          // 16 KB: one f16 operand tile (W or X: G5_BN == G5_BM)
constexpr int G5_PIECES = 2;                              // w_hi, w_lo and x_h, x_m
constexpr int G5_STAGES = 3;
constexpr int G5_STAGE_BYTES = 2 * G5_PIECES * G5_TILE_BYTES;   // W pieces, then X pieces
constexpr int G5_SMEM_BYTES = G5_STAGES * G5_STAGE_BYTES;       // 192 KB of the H100's 227 KB per block
constexpr float G5_WSCALE = 256.0f;                       // weights enter the MMA times 2^8 (see header)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "G5_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra G5_DONE;\n"
        "bra G5_WAIT;\n"
        "G5_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// wgmma shared-memory descriptor, K-major, no swizzle (layout type 0): core matrix = 8 rows x 16 bytes stored as 128
// contiguous bytes; LBO = byte distance between the two 8-element K chunks of one MMA, SBO = byte distance between
// consecutive 8-row groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}
// D[64 x 64] (f32, registers) += A[64 x 16] . B[16 x 64], A and B f16 K-major in shared memory
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
        "%32, %33, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(1)
        : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMA window
__device__ __forceinline__ void acc_fence(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// f16x2 bit pattern of two floats v0', v1' that are (value * 2^-112) of numbers exactly representable in f16 -- normal,
// subnormal or zero: with the exponent re-biased by the 2^-112 factor, the f16 exponent/mantissa field of v is simply bits
// 13..27 of v' (an f32 denormal v' lands on the matching f16 denormal), so no conversion instruction is needed.
__device__ __forceinline__ uint32_t g5_pack_f16x2(const float v0, const float v1) {
    const uint32_t b0 = __float_as_uint(v0), b1 = __float_as_uint(v1);
    const uint32_t em = ((b0 >> 13) & 0x00007FFFu) | ((b1 << 3) & 0x7FFF0000u);
    const uint32_t sg = ((b0 >> 16) & 0x00008000u) | (b1 & 0x80000000u);
    return em | sg;
}

struct G5Args {
    const uint4 *qs;      // row-major Q4 planes (kernels.h Q4Weight)
    const __half *ds;
    int N, K, M;          // M = tokens
    const __half *xt;         // [2][TT][KC][8][128][8] tiled f16 splits of X * 2^s_t (zero padded rows)
    const float *oscale;      // [TT*128] per-token output scale 2^-(s_t + 8)
    int TT, KC;
    float *y;
    int ldy;
    const float *bias, *res;
    // deterministic split-K (grid.z slices of KCs k-steps): partial tiles [z][tile][tok 128][feat 128],
    // the last CTA of a tile to arrive (ticket) adds them in slice order and runs the epilogue
    int SK, KCs;
    float *partial;
    int *counters;
};

template <int EPI>
__global__ void __launch_bounds__(G5_THREADS, 1) gemm_tc5_kernel(const G5Args a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ __align__(8) uint64_t full_bar[G5_STAGES];   // X pieces of a stage landed
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int f0 = blockIdx.x * G5_BM, tt = blockIdx.y, tok0 = tt * G5_BN;
    const int bpr = a.K >> 5;
    const int kc_begin = blockIdx.z * a.KCs, kc_end = min(a.KC, kc_begin + a.KCs), nk = kc_end - kc_begin;
    const size_t xt_piece = (size_t)a.TT * a.KC * (G5_TILE_BYTES / 2);  // elements per split piece

    auto fetch_x = [&](int it) {   // both X pieces of k-step kc_begin + it into stage it % G5_STAGES (one thread)
        const int s = it % G5_STAGES;
        unsigned char *dst = smem + (size_t)s * G5_STAGE_BYTES + G5_PIECES * G5_TILE_BYTES;
        mbar_expect_tx(&full_bar[s], G5_PIECES * G5_TILE_BYTES);
#pragma unroll
        for (int p = 0; p < G5_PIECES; ++p) {
            const __half *src = a.xt + p * xt_piece + ((size_t)tt * a.KC + kc_begin + it) * (G5_TILE_BYTES / 2);
            bulk_g2s(dst + p * G5_TILE_BYTES, src, G5_TILE_BYTES, &full_bar[s]);
        }
    };
    if (tid == 0) {
        for (int s = 0; s < G5_STAGES; ++s) mbar_init(&full_bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        if (nk > 0) fetch_x(0);
    }
    __syncthreads();

    // dequantisation: thread -> (feature row, Q4 block of the 64-wide chunk, nibble half)
    const int drow = tid >> 2, dblk = (tid >> 1) & 1, dhalf = tid & 1;
    const int gn = f0 + drow;
    // MMA: warpgroup -> 64 features (fq) x 64 tokens (tq) of the CTA tile
    const int fq = wg & 1, tq = wg >> 1;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;

    // this thread's Q4 block of the first k-step (rows beyond N: nibble 8 = weight 0, scale 0)
    uint4 q_cur = make_uint4(0x88888888u, 0x88888888u, 0x88888888u, 0x88888888u);
    __half d_cur = __float2half(0.0f);
    if (gn < a.N && nk > 0) {
        const size_t blk = (size_t)gn * bpr + (size_t)kc_begin * 2 + dblk;
        q_cur = __ldg(a.qs + blk);
        d_cur = __ldg(a.ds + blk);
    }
    for (int it = 0; it < nk; ++it) {
        const int kc = kc_begin + it, s = it % G5_STAGES;
        unsigned char *stage = smem + (size_t)s * G5_STAGE_BYTES;
        const uint4 q = q_cur;
        // d * 2^8 (the weights' MMA scale) * 2^-112 (f16 <- f32 exponent re-bias, see g5_pack_f16x2): exact power-of-two
        // scalings of the f16 block scale (one conversion per block; f32 denormals are NOT flushed in this file)
        const float dd = __half2float(d_cur) * G5_WSCALE * 1.92592994438723585305597794258492732e-34f;  // 2^-112
        if (gn < a.N && kc + 1 < kc_end) {  // next k-step's block: its L2 latency hides behind this step
            const size_t blk = (size_t)gn * bpr + (size_t)(kc + 1) * 2 + dblk;
            q_cur = __ldg(a.qs + blk);
            d_cur = __ldg(a.ds + blk);
        }
        // 16 weights of the block: low nibbles (elements 0..15, dhalf = 0) or high nibbles (16..31), as f16 hi + lo, all
        // on the FMA and ALU pipes: nibble -> float by OR-ing 0x4B000000 (2^23 + n), w' = (n - 8) * d'' in f32, Veltkamp
        // split hi' = RN_11bit(w') (c = w' * 8193; hi' = c - (c - w')), lo' = w' - hi' (exact), and the f16 bit patterns
        // of hi' * 2^112, lo' * 2^112 by shifts and masks (both are exactly representable: no rounding to do).
        const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
        uint32_t ph[8], pl[8];
#pragma unroll
        for (int wi = 0; wi < 4; ++wi) {
            const uint32_t nib = dhalf ? (w4[wi] >> 4) : w4[wi];
            float hi[4], lo[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const uint32_t n = (nib >> (8 * t)) & 0xFu;
                // _rn intrinsics: the splitting must not be contracted into FMAs
                const float w = __fmul_rn(__fsub_rn(__uint_as_float(0x4B000000u | n), 8388616.0f), dd);
                const float c = __fmul_rn(w, 8193.0f);
                hi[t] = __fsub_rn(c, __fsub_rn(c, w));
                lo[t] = __fsub_rn(w, hi[t]);
            }
            ph[wi * 2 + 0] = g5_pack_f16x2(hi[0], hi[1]);
            ph[wi * 2 + 1] = g5_pack_f16x2(hi[2], hi[3]);
            pl[wi * 2 + 0] = g5_pack_f16x2(lo[0], lo[1]);
            pl[wi * 2 + 1] = g5_pack_f16x2(lo[2], lo[3]);
        }
        // Stage s was last read by k-step it-3.  After this wait the warpgroup's MMAs up to k-step it-2 have retired;
        // every other warpgroup waited the same way at it-1 before the barrier this thread has passed.
        wgmma_wait<1>();
        // tile layout: [8 k-chunks of 8 elements][128 rows][16 bytes]; this thread owns k-chunks dblk*4 + dhalf*2 + {0,1}
        unsigned char *thi = stage, *tlo = stage + G5_TILE_BYTES;
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int off = (dblk * 4 + dhalf * 2 + c) * (G5_BM * 16) + drow * 16;
            *reinterpret_cast<uint4 *>(thi + off) = make_uint4(ph[4 * c + 0], ph[4 * c + 1], ph[4 * c + 2], ph[4 * c + 3]);
            *reinterpret_cast<uint4 *>(tlo + off) = make_uint4(pl[4 * c + 0], pl[4 * c + 1], pl[4 * c + 2], pl[4 * c + 3]);
        }
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");  // generic writes -> async (wgmma) reads
        __syncthreads();   // W of k-step it complete; every warpgroup's MMAs up to k-step it-2 retired
        if (tid == 0 && it + 1 < nk) fetch_x(it + 1);   // into the stage k-step it-2 read
        mbar_wait(&full_bar[s], (uint32_t)((it / G5_STAGES) & 1));   // X tiles landed
        const uint32_t wbase = smem_u32(stage) + fq * 64 * 16, xbase = smem_u32(stage + G5_PIECES * G5_TILE_BYTES) + tq * 64 * 16;
        const uint32_t lbo = G5_BM * 16, sbo = 128;   // K-chunk stride, 8-row group stride (W and X alike)
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < G5_BK / 16; ++ks) {
            const uint32_t koff = (uint32_t)ks * 2u * lbo;
            const uint64_t whi = gmma_desc(wbase + 0 * G5_TILE_BYTES + koff, lbo, sbo);
            const uint64_t wlo = gmma_desc(wbase + 1 * G5_TILE_BYTES + koff, lbo, sbo);
            const uint64_t xh = gmma_desc(xbase + 0 * G5_TILE_BYTES + koff, lbo, sbo);
            const uint64_t xm = gmma_desc(xbase + 1 * G5_TILE_BYTES + koff, lbo, sbo);
            // smallest terms first
            wgmma_m64n64k16(acc, wlo, xh);
            wgmma_m64n64k16(acc, whi, xm);
            wgmma_m64n64k16(acc, whi, xh);
        }
        wgmma_commit();
        acc_fence(acc);
    }
    wgmma_wait<0>();
    acc_fence(acc);

    // ---- epilogue.  Accumulator i of this thread: feature row fr(i), token column tc(i) of the CTA tile
    // (wgmma D fragment: warp w of the warpgroup holds rows 16w..16w+15, lane -> row lane/4 (+8), column pair lane%4)
    {
        __shared__ int is_last;
        const int frow = fq * 64 + (warp & 3) * 16 + (lane >> 2);
        const int tcol = tq * 64 + (lane & 3) * 2;
        auto fr = [&](int i) { return frow + ((i >> 1) & 1) * 8; };
        auto tc = [&](int i) { return tcol + (i >> 2) * 8 + (i & 1); };
        auto emit = [&](float (&r)[32]) {   // bias / residual / activation of the 32 accumulators in r
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int feat = f0 + fr(i), tok = tok0 + tc(i);
                float v = r[i] * a.oscale[tok];
                if (EPI == EPI_SILU_MUL) {
                    // features (2j, 2j+1) = (gate, up) sit in lanes 4 apart
                    const float other = __shfl_xor_sync(0xffffffffu, v, 4);
                    if (((lane >> 2) & 1) == 0 && tok < a.M && feat + 1 < a.N)
                        a.y[(size_t)tok * a.ldy + (feat >> 1)] = (v / (1.0f + expf(-v))) * other;
                } else if (tok < a.M && feat < a.N) {
                    if (a.bias) v += a.bias[feat];
                    if (EPI == EPI_RESIDUAL) v += a.res[(size_t)tok * a.ldy + feat];
                    if (EPI == EPI_GELU) v = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
                    a.y[(size_t)tok * a.ldy + feat] = v;
                }
            }
        };
        if (a.SK <= 1) {
            emit(acc);
        } else {
            // publish this slice's tile, take a ticket; the last arriver sums the slices in order
            const int tile_id = blockIdx.y * gridDim.x + blockIdx.x, n_tile = gridDim.x * gridDim.y;
            float *ptile = a.partial + ((size_t)blockIdx.z * n_tile + tile_id) * (G5_BM * G5_BN);
#pragma unroll
            for (int i = 0; i < 32; ++i) __stcg(ptile + (size_t)tc(i) * G5_BM + fr(i), acc[i]);
            __syncthreads();
            if (tid == 0) {
                __threadfence();
                const int old = atomicAdd(&a.counters[tile_id], 1);
                const int last = (old == a.SK - 1);
                if (last) {
                    a.counters[tile_id] = 0;
                    __threadfence();
                }
                is_last = last;
            }
            __syncthreads();
            if (is_last != 0) {
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    float v = 0.0f;
                    for (int z = 0; z < a.SK; ++z)
                        v += __ldcg(a.partial + ((size_t)z * n_tile + tile_id) * (G5_BM * G5_BN) + (size_t)tc(i) * G5_BM + fr(i));
                    acc[i] = v;
                }
                emit(acc);
            }
        }
    }
}

// X (f32, row-major [M][K]) -> two f16 pieces of X * 2^s_t in the wgmma operand tile layout, optionally through RMSNorm
// (x / sqrt(mean(x^2)+eps) * gamma (* ada)); s_t = per-token power of two putting the row maximum in [2^7, 2^8);
// oscale[t] = 2^-(s_t + 8) undoes it (and the weights' 2^8) in the GEMM epilogue.  CTA = 8 token rows; rows >= M are
// written as zeros.
__global__ void __launch_bounds__(256) split_tiles_kernel(const float *__restrict__ x, int M, int K, const float *__restrict__ gamma,
                                                          const float *__restrict__ ada, float eps, __half *__restrict__ xt,
                                                          float *__restrict__ oscale, int TT, int KC, int BN) {
    __shared__ float ssq_part[32][8], max_part[32][8];
    __shared__ float rms_s[8], sc_s[8];
    const int r8 = threadIdx.x & 7, cth = threadIdx.x >> 3;  // cth: 0..31 strides over the 16-byte chunks
    const int row = blockIdx.x * 8 + r8;
    const int nchunk = K >> 3;
    const bool valid = row < M;
    const float *xr = x + (size_t)(valid ? row : 0) * K;
    {   // pass 1: sum of squares (RMSNorm) and max |x * gamma * ada| (the row maximum after the norm is this / rms)
        float ssq = 0.0f, mx = 0.0f;
        if (valid)
            for (int c = cth; c < nchunk; c += 32) {
                const float4 v0 = *reinterpret_cast<const float4 *>(xr + c * 8);
                const float4 v1 = *reinterpret_cast<const float4 *>(xr + c * 8 + 4);
                float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    ssq = fmaf(v[e], v[e], ssq);
                    float g = v[e];
                    if (gamma) {
                        g *= gamma[c * 8 + e];
                        if (ada) g *= ada[c * 8 + e];
                    }
                    mx = fmaxf(mx, fabsf(g));
                }
            }
        ssq_part[cth][r8] = ssq;
        max_part[cth][r8] = mx;
        __syncthreads();
        if (threadIdx.x < 8) {
            float s = 0.0f, m = 0.0f;
            for (int i = 0; i < 32; ++i) {
                s += ssq_part[i][threadIdx.x];
                m = fmaxf(m, max_part[i][threadIdx.x]);
            }
            const float rms = gamma ? sqrtf(s / (float)K + eps) : 1.0f;
            rms_s[threadIdx.x] = rms;
            m = m / rms * 1.0001f;  // the split below rounds (v / rms) * gamma slightly differently: stay below 2^8
            int e = (int)((__float_as_uint(m) >> 23) & 0xFF) - 127;
            if (!(m > 0.0f) || m > 3.0e38f) e = 7;   // all-zero (or non-finite) row: scale 1
            e = e < -100 ? -100 : (e > 100 ? 100 : e);
            sc_s[threadIdx.x] = __uint_as_float((uint32_t)(7 - e + 127) << 23);            // 2^(7 - e)
            const int grow = blockIdx.x * 8 + threadIdx.x;
            oscale[grow] = __uint_as_float((uint32_t)(e - 7 - 8 + 127) << 23);              // 2^(e - 7) / 2^8
        }
        __syncthreads();
    }
    const float rms = rms_s[r8], sc = sc_s[r8];
    const int tt = row / BN, rin = row % BN;
    const size_t tile_el = (size_t)BN * G5_BK;   // f16 elements of one (token tile, k-step) tile
    const size_t piece = (size_t)TT * KC * tile_el;
    for (int c = cth; c < nchunk; c += 32) {
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (valid) {
            const float4 v0 = *reinterpret_cast<const float4 *>(xr + c * 8);
            const float4 v1 = *reinterpret_cast<const float4 *>(xr + c * 8 + 4);
            v[0] = v0.x; v[1] = v0.y; v[2] = v0.z; v[3] = v0.w; v[4] = v1.x; v[5] = v1.y; v[6] = v1.z; v[7] = v1.w;
            if (gamma) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    v[e] = (v[e] / rms) * gamma[c * 8 + e];
                    if (ada) v[e] *= ada[c * 8 + e];
                }
            }
        }
        uint32_t p[2][4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float f0 = v[2 * e] * sc, f1 = v[2 * e + 1] * sc;   // power-of-two scale: exact
            const __half2 h = __floats2half2_rn(f0, f1);
            const float2 hf = __half22float2(h);
            const __half2 m = __floats2half2_rn(f0 - hf.x, f1 - hf.y);
            p[0][e] = *reinterpret_cast<const uint32_t *>(&h);
            p[1][e] = *reinterpret_cast<const uint32_t *>(&m);
        }
        // tile (tt, kc = c/8), chunk-in-tile c%8, row rin: [8][BN][16 B]
        const size_t off = ((size_t)tt * KC + (c >> 3)) * tile_el + (size_t)((c & 7) * BN + rin) * 8;
#pragma unroll
        for (int s = 0; s < G5_PIECES; ++s)
            *reinterpret_cast<uint4 *>(xt + s * piece + off) = make_uint4(p[s][0], p[s][1], p[s][2], p[s][3]);
    }
}

}  // namespace

bool gemm_tc5_supported(const Q4Weight &w, int M) { return w.N % G5_BM == 0 && w.K % G5_BK == 0 && M >= 1; }

// f16 elements of the split buffer: two pieces of tiles + the per-token output scales (floats) behind them
static size_t g5_tiles_elems(int M, int K) {
    const size_t TT = (size_t)(M + G5_BN - 1) / G5_BN;
    return G5_PIECES * TT * (size_t)(K / G5_BK) * ((size_t)G5_BN * G5_BK);
}
size_t gemm_tc5_split_elems(int M, int K) {
    const size_t TT = (size_t)(M + G5_BN - 1) / G5_BN;
    return g5_tiles_elems(M, K) + 2 * TT * G5_BN + 16;
}
static float *g5_oscale_ptr(void *xt, int M, int K) {
    size_t off = g5_tiles_elems(M, K) * 2;          // bytes
    off = (off + 15) & ~(size_t)15;
    return reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(xt) + off);
}

// x [M][K] f32 -> xt (f16 pieces, tile layout; per-token scales behind them); rows padded to a multiple of 128 with zeros
void launch_split_tiles(const float *x, int M, int K, const float *gamma, const float *ada, float eps, void *xt,
                        cudaStream_t st) {
    VOX_CHECK(K % G5_BK == 0, VOX_EINVAL, "split_tiles: K=%d not a multiple of 64", K);
    const int TT = (M + G5_BN - 1) / G5_BN, KC = K / G5_BK;
    split_tiles_kernel<<<TT * (G5_BN / 8), 256, 0, st>>>(x, M, K, gamma, ada, eps, (__half *)xt, g5_oscale_ptr(xt, M, K), TT, KC,
                                                         G5_BN);
    tc_count_launch("split_tiles");
}

void launch_q4_gemm_tc5(const Q4Weight &w, const void *xt, int M, float *y, int ldy, const float *bias, const float *res,
                        int epi, const GemmWork *gw, cudaStream_t st) {
    VOX_CHECK(gemm_tc5_supported(w, M), VOX_EINVAL, "gemm_tc5: unsupported shape N=%d K=%d", w.N, w.K);
    G5Args a{};
    a.qs = w.qs;
    a.ds = w.d;
    a.N = w.N;
    a.K = w.K;
    a.M = M;
    a.xt = (const __half *)xt;
    a.oscale = g5_oscale_ptr(const_cast<void *>(xt), M, w.K);
    a.TT = (M + G5_BN - 1) / G5_BN;
    a.KC = w.K / G5_BK;
    a.y = y;
    a.ldy = ldy;
    a.bias = bias;
    a.res = res;
    const size_t smem = (size_t)G5_SMEM_BYTES;
    // split K when the output tiles alone cannot fill the GPU (single-stream encode: N = 1280 -> 50 tiles;
    // prefill: 38 tokens -> one token tile)
    const int tiles = (w.N / G5_BM) * a.TT;
    int SK = 1;
    if (gw && gw->partial && gw->counters && tiles < VOX_NUM_SMS * 2 / 3) {
        SK = VOX_NUM_SMS / tiles;
        SK = SK > 8 ? 8 : SK;
        while (SK > 1 && a.KC / SK < 4) --SK;
        while (SK > 1 && ((size_t)SK * tiles * G5_BM * G5_BN > gw->partial_floats || tiles > gw->n_counters)) --SK;
    }
    a.KCs = (a.KC + SK - 1) / SK;
    SK = (a.KC + a.KCs - 1) / a.KCs;
    a.SK = SK;
    a.partial = SK > 1 ? gw->partial : nullptr;
    a.counters = SK > 1 ? gw->counters : nullptr;
    dim3 grid(w.N / G5_BM, a.TT, SK);
#define G5_CASE(E)                                                                      \
    case E: {                                                                           \
        static SmemAttr attr;                                                           \
        smem_attr_check(ensure_dyn_smem(gemm_tc5_kernel<E>, smem, attr), "gemm_tc5");   \
        gemm_tc5_kernel<E><<<grid, G5_THREADS, smem, st>>>(a);                          \
        break;                                                                          \
    }
    switch (epi) {
        G5_CASE(EPI_NONE)
        G5_CASE(EPI_RESIDUAL)
        G5_CASE(EPI_SILU_MUL)
        G5_CASE(EPI_GELU)
        default: fail(VOX_EINVAL, "bad epilogue");
    }
#undef G5_CASE
    tc_count_launch("gemm_tc5");
}

}  // namespace vox
