// matvec_tc.cu -- K2-TC: Q4_0 dequant + matvec for M <= 8 tokens with the *dequant arithmetic* moved
// onto the tensor cores (mma.sync.m16n8k16, f16 x f16 -> f32), optionally fused with the RMSNorm
// (+ ADA scale) of its input, weights streamed by TMA bulk copies, deterministic split-K.
//
// Why: the SIMT kernel (kernels.cu K2) needs ~4 issue slots per weight (SHF, LOP3, I2FP, FFMA);
// by the data sheet an H100 SXM streams ~6 T weights/s from HBM (3.35 TB/s / 0.5625 B) and issues ~33 T
// lane-instr/s (132 SMs x 128 lanes x 1.98 GHz), so a SIMT single-token decode is issue-bound, not HBM-bound,
// as soon as anything else shares the issue slots.  Here a Q4 nibble n reaches the MMA as the f16 *subnormal*
// n * 2^-24 (nibble in bits 0-3 of a 16-bit lane) or 16 n * 2^-24 (bits 4-7): one LOP3 isolates two weights,
// no int->float conversion, no multiply (scripts/mma_denorm_test.cu verifies on hardware that HMMA treats these
// inputs exactly).
// Same arithmetic as the reference (src/gguf/shader.wgsl:96-127), re-associated:
//
//   y[m,n] = sum_b d[n,b] * ( sum_{k in b} q[n,k] x[m,k]  -  8 sum_{k in b} x[m,k] )
//
// * inner sums over one 32-weight block = two MMAs (low nibbles, high nibbles) with f32 accumulate;
// * the 32 activations of a block are scaled by a per-block power of two (block max -> [2^7,2^8))
//   and split into two f16 pieces hi = f16(x), mid = f16(x - hi): 22 mantissa bits -- below the f32
//   rounding of the dot product itself; products n*hi are exact in f32;
// * the per-block f16 scale d is applied to the f32 block sum in registers (it can not be folded into
//   the MMA: (q-8)*d needs 15 mantissa bits), exactly once per block like the reference;
// * NORM variant: x := ((x / sqrt(mean(x^2)+eps)) * gamma) * ada   (reference rms_norm.rs:42-47 +
//   model.rs:250-255) applied while staging; mean(x^2) comes from per-tile partial sums that the
//   producing kernel's residual epilogue left behind (fixed summation order), so no extra launch
//   and no extra pass over x;
// * split-K: grid.y CTAs share a row tile, each writes its partial sums, the last one to arrive
//   (atomic ticket) adds them in slice order and runs the epilogue => bitwise deterministic.
//
// Weight layout ("TC layout", built at load from the GGUF blocks, same 18 B / 32 weights):
//   qs_tc : uint4 [T = N/16 tiles][P = K/64 block pairs][32 lanes]
//           lane (g = lane/4, t = lane%4): .x = word t of (row 16T+g,   block 2P)
//                                          .y = word t of (row 16T+g+8, block 2P)
//                                          .z/.w = the same for block 2P+1
//           => a (tile, K-slice) is one contiguous chunk for a 1-D TMA bulk copy and each lane's
//              128-bit shared-memory read already holds its m16n8k16 A-fragment source words.
//   d_tc  : uint2 [T][P][8]  = halves {d(g,2P), d(g+8,2P), d(g,2P+1), d(g+8,2P+1)}
// MMA K index <-> block element (low-nibble MMA; high-nibble MMA adds 16):
//   kcol 2t -> 4t, 2t+1 -> 4t+2, 2t+8 -> 4t+1, 2t+9 -> 4t+3   (B fragments are staged to match).
#include <cuda_fp16.h>

#include <cstdlib>

#include "common.h"
#include "kernels.h"

namespace vox {

void tc_count_launch(const char *name);
void set_tc_pdl(bool on);

namespace {

inline void cuda_check_tc(cudaError_t e, const char *what) {
    if (e != cudaSuccess) fail(VOX_ECUDA, fmt("CUDA error: %s: %s", what, cudaGetErrorString(e)));
}

constexpr int TC_WARPS = 8;
constexpr int TC_THREADS = TC_WARPS * 32;

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t a0, const uint32_t a1, const uint32_t a2,
                                         const uint32_t a3, const uint32_t b0, const uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}

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
        "MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MBAR_DONE;\n"
        "bra MBAR_WAIT;\n"
        "MBAR_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (bytes % 16 == 0)
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// Programmatic dependent launch: let the next kernel in the stream start its prologue (weight
// prefetch) now; block until the previous kernel's results are visible.  No-ops when the kernel was
// launched without the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }

struct TcArgs {
    const uint4 *qs_tc;
    const uint2 *d_tc;
    int N, K, n_tiles, n_pairs;
    const float *x;
    float *y;
    int ldy;
    const float *bias, *res;
    // fused RMSNorm of the input
    const float *gamma, *ada;
    float eps;
    const float *ssq_in;  // [ssq_in_parts][M] partial sums of squares of x (nullptr: computed here)
    int ssq_in_parts;
    float *ssq_out;       // EPI_RESIDUAL: [n_tiles][M] partial sums of squares of the new rows
    // work decomposition
    int S, Ps, TG, nbuf;
    float *partial;       // [S][M][ldp]
    int ldp;
    int *counters;        // [n_tiles], zero between launches
};

// Effective activation value (after the optional fused RMSNorm).
// `rinv` = 1 / sqrt(mean(x^2)+eps): the reference divides (x / rms); multiplying by the reciprocal
// differs by <= 1 ulp per element and removes ~10 instructions per element from the staging pass.
__device__ __forceinline__ float4 eff4(const float4 v, const float rinv, const float *gamma, const float *ada, const int k) {
    if (!gamma) return v;
    const float4 g = *reinterpret_cast<const float4 *>(gamma + k);
    float4 o = make_float4((v.x * rinv) * g.x, (v.y * rinv) * g.y, (v.z * rinv) * g.z, (v.w * rinv) * g.w);
    if (ada) {
        const float4 a = *reinterpret_cast<const float4 *>(ada + k);
        o.x *= a.x; o.y *= a.y; o.z *= a.z; o.w *= a.w;
    }
    return o;
}

// Stage the activation side of blocks [b0, b0+nb) into shared memory:
//   bf   : uint2  [nb][2 (nibble half j)][2M cols][4 t]  B fragments {b0,b1} of lane (g = col, t)
//   off2 : float2 [nb][M]   { -8 * sum_{k in block} x ,  2^24 / block scale }
// Column c = 2*token + split (0 = hi, 1 = mid).  One work item = (block, token, t): elements
// 4t..4t+3 and 16+4t..16+4t+3; the four t-items of a block sit in adjacent lanes so the block sum and
// block max are 2-step shuffles.  Two items per thread are loaded before either is processed.
template <int M>
__device__ __forceinline__ void tc_stage(const TcArgs &a, const int b0, const int nb, const float *__restrict__ rms,
                                         uint2 *__restrict__ bf, float2 *__restrict__ off2) {
    const int items = nb * M * 4;
    constexpr int U = 2;
    for (int base = 0; base < items; base += TC_THREADS * U) {
        float4 lo[U], hi[U];
        int mm[U], bl[U];
        bool act[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = base + u * TC_THREADS + threadIdx.x;
            act[u] = i < items;
            mm[u] = act[u] ? (i >> 2) % M : 0;
            bl[u] = act[u] ? (i >> 2) / M : 0;
            const int kb = (b0 + bl[u]) * 32, t = i & 3;
            lo[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            hi[u] = lo[u];
            if (act[u] && kb < a.K) {
                lo[u] = *reinterpret_cast<const float4 *>(a.x + (size_t)mm[u] * a.K + kb + 4 * t);
                hi[u] = *reinterpret_cast<const float4 *>(a.x + (size_t)mm[u] * a.K + kb + 16 + 4 * t);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = base + u * TC_THREADS + threadIdx.x;
            const int t = i & 3, m = mm[u];
            const int kb = (b0 + bl[u]) * 32;
            float4 l = lo[u], h = hi[u];
            if (act[u] && kb < a.K) {
                l = eff4(l, rms[m], a.gamma, a.ada, kb + 4 * t);
                h = eff4(h, rms[m], a.gamma, a.ada, kb + 16 + 4 * t);
            }
            float bs = ((l.x + l.y) + (l.z + l.w)) + ((h.x + h.y) + (h.z + h.w));
            float bm = fmaxf(fmaxf(fmaxf(fabsf(l.x), fabsf(l.y)), fmaxf(fabsf(l.z), fabsf(l.w))),
                             fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fmaxf(fabsf(h.z), fabsf(h.w))));
            bs += __shfl_xor_sync(0xffffffffu, bs, 1);
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 1));
            bs += __shfl_xor_sync(0xffffffffu, bs, 2);
            bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 2));
            if (!act[u]) continue;
            // power-of-two block scale: block max -> [2^7, 2^8)
            int e = (int)((__float_as_uint(bm) >> 23) & 0xFF) - 127;
            if (!(bm > 0.0f) || bm > 3.0e38f) e = 7;  // all-zero (or non-finite) block: scale 1
            e = e < -100 ? -100 : (e > 100 ? 100 : e);
            const float s = __uint_as_float((uint32_t)(7 - e + 127) << 23);
            const float inv = __uint_as_float((uint32_t)(17 + e + 127) << 23);  // 2^24 / s
            const float ev[8] = {l.x * s, l.y * s, l.z * s, l.w * s,
                                 h.x * s * 0.0625f, h.y * s * 0.0625f, h.z * s * 0.0625f, h.w * s * 0.0625f};
            float hh[8], md[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                hh[q] = __half2float(__float2half_rn(ev[q]));
                md[q] = ev[q] - hh[q];
            }
            // j = 0: b0 = {elem 4t, 4t+2}, b1 = {4t+1, 4t+3};  j = 1: same on the (x/16) high half
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int o = 4 * j;
                uint2 fh, fm;
                fh.x = pack_h2(hh[o + 0], hh[o + 2]);
                fh.y = pack_h2(hh[o + 1], hh[o + 3]);
                fm.x = pack_h2(md[o + 0], md[o + 2]);
                fm.y = pack_h2(md[o + 1], md[o + 3]);
                uint2 *dst = bf + ((size_t)(bl[u] * 2 + j) * (2 * M)) * 4;
                dst[(2 * m + 0) * 4 + t] = fh;
                dst[(2 * m + 1) * 4 + t] = fm;
            }
            if (t == 0) off2[bl[u] * M + m] = make_float2(-8.0f * bs, inv);
        }
    }
}

template <int M, int EPI>
__device__ __forceinline__ void tc_epilogue(const TcArgs &a, const int tile, const float *__restrict__ vals /*[16][M]*/,
                                            float *__restrict__ sq /*[16*M] smem*/) {
    // vals[r*M + tok] = full dot products of tile row r.  Must be called by all threads of the CTA.
    if (EPI == EPI_SILU_MUL) {
        for (int i = threadIdx.x; i < 8 * M; i += TC_THREADS) {
            const int pr = i / M, tok = i - pr * M;
            const float g = vals[(2 * pr) * M + tok], u = vals[(2 * pr + 1) * M + tok];
            const int row = tile * 16 + 2 * pr;
            if (row + 1 < a.N) a.y[(size_t)tok * a.ldy + (row >> 1)] = (g / (1.0f + expf(-g))) * u;
        }
    } else {
        for (int i = threadIdx.x; i < 16 * M; i += TC_THREADS) {
            const int r = i / M, tok = i - r * M;
            const int row = tile * 16 + r;
            float v = 0.0f;
            if (row < a.N) {
                v = vals[i] + (a.bias ? a.bias[row] : 0.0f);
                if (EPI == EPI_RESIDUAL) v += a.res[(size_t)tok * a.ldy + row];
                if (EPI == EPI_GELU) v = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
                a.y[(size_t)tok * a.ldy + row] = v;
            }
            if (EPI == EPI_RESIDUAL && a.ssq_out) sq[i] = v * v;
        }
        if (EPI == EPI_RESIDUAL && a.ssq_out) {
            __syncthreads();
            if (threadIdx.x < M) {
                float s = 0.0f;
#pragma unroll
                for (int r = 0; r < 16; ++r) s += sq[r * M + threadIdx.x];
                a.ssq_out[(size_t)tile * M + threadIdx.x] = s;
            }
        }
    }
}

// EPI semantics as in kernels.h (Epi).  grid = (tile groups, K slices).
template <int M, int EPI>
__global__ void __launch_bounds__(TC_THREADS) q4_matvec_tc_kernel(const TcArgs a) {
    constexpr int CG = (M + 3) / 4;  // column groups of 8 (= 4 tokens x 2 splits)
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *rms = reinterpret_cast<float *>(smem_raw);                  // [8] reciprocal rms per token
    int *flag = reinterpret_cast<int *>(rms + 8);                       // [1] (+3 pad)
    float *stat = rms + 12;                                             // [TC_WARPS][M] fallback ssq partials
    float *red = stat + TC_WARPS * M;                                   // [TC_WARPS][16 rows][M]
    float *vals = red + TC_WARPS * 16 * M;                              // [16][M] reduced tile
    float *sq = vals + 16 * M;                                          // [16][M]
    float2 *off2 = reinterpret_cast<float2 *>(sq + 16 * M);            // [2*Ps][M]
    uint2 *bf = reinterpret_cast<uint2 *>(off2 + (size_t)a.Ps * 2 * M); // [2*Ps][2][2M][4]
    const int slice = blockIdx.y;
    const int p_begin = slice * a.Ps;
    const int np = min(a.Ps, a.n_pairs - p_begin);
    const uint32_t tile_q_bytes = (uint32_t)np * 512u, tile_d_bytes = (uint32_t)np * 64u;
    const uint32_t tile_bytes = (uint32_t)a.Ps * 576u;  // buffer stride (slot sized for a full slice)
    size_t woff = (size_t)(reinterpret_cast<unsigned char *>(bf + (size_t)a.Ps * 2 * 2 * 2 * M * 4) - smem_raw);
    woff = (woff + 127) & ~(size_t)127;
    unsigned char *wbuf = smem_raw + woff;
    uint64_t *mbar = reinterpret_cast<uint64_t *>(wbuf + (size_t)a.nbuf * tile_bytes);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int tile0 = blockIdx.x * a.TG;
    const int tile1 = min(a.n_tiles, tile0 + a.TG);

    auto issue_tile = [&](int tile, int buf) {  // one thread
        mbar_expect_tx(&mbar[buf], tile_q_bytes + tile_d_bytes);
        unsigned char *dst = wbuf + (size_t)buf * tile_bytes;
        bulk_g2s(dst, a.qs_tc + ((size_t)tile * a.n_pairs + p_begin) * 32, tile_q_bytes, &mbar[buf]);
        bulk_g2s(dst + tile_q_bytes, a.d_tc + ((size_t)tile * a.n_pairs + p_begin) * 8, tile_d_bytes, &mbar[buf]);
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < a.nbuf; ++i) mbar_init(&mbar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    // the weights do not depend on the previous kernel: start streaming the first tile now, let the
    // next kernel begin its own prefetch, and only then wait for our input activations
    if (threadIdx.x == 0) issue_tile(tile0, 0);
    pdl_trigger();
    pdl_wait();

    // ---- row statistics for the fused RMSNorm
    if (a.gamma) {
        if (a.ssq_in) {
            if (warp < M) {
                float s = 0.0f;
                for (int i = lane; i < a.ssq_in_parts; i += 32) s += a.ssq_in[(size_t)i * M + warp];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                if (lane == 0) rms[warp] = 1.0f / sqrtf(s / (float)a.K + a.eps);
            }
        } else {
            const int kq = a.K >> 2;
#pragma unroll
            for (int m = 0; m < M; ++m) {
                float ssq = 0.0f;
                for (int i = threadIdx.x; i < kq; i += TC_THREADS) {
                    const float4 v = *reinterpret_cast<const float4 *>(a.x + (size_t)m * a.K + 4 * i);
                    ssq = fmaf(v.x, v.x, ssq); ssq = fmaf(v.y, v.y, ssq); ssq = fmaf(v.z, v.z, ssq); ssq = fmaf(v.w, v.w, ssq);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) ssq += __shfl_xor_sync(0xffffffffu, ssq, o);
                if (lane == 0) stat[warp * M + m] = ssq;
            }
            __syncthreads();
            if (threadIdx.x < M) {
                float s = 0.0f;
#pragma unroll
                for (int w = 0; w < TC_WARPS; ++w) s += stat[w * M + threadIdx.x];
                rms[threadIdx.x] = 1.0f / sqrtf(s / (float)a.K + a.eps);
            }
        }
        __syncthreads();
    }
    tc_stage<M>(a, p_begin * 2, np * 2, rms, bf, off2);
    __syncthreads();

    int it = 0;
    for (int tile = tile0; tile < tile1; ++tile, ++it) {
        const int buf = a.nbuf == 2 ? (it & 1) : 0;
        const uint32_t parity = a.nbuf == 2 ? ((it >> 1) & 1) : (it & 1);
        if (a.nbuf == 2 && threadIdx.x == 0 && tile + 1 < tile1) {
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
            issue_tile(tile + 1, buf ^ 1);  // buffer buf^1 was released by the barriers ending iteration it-1
        }
        const uint4 *wq_s = reinterpret_cast<const uint4 *>(wbuf + (size_t)buf * tile_bytes) + lane;
        const uint2 *wd_s = reinterpret_cast<const uint2 *>(wbuf + (size_t)buf * tile_bytes + tile_q_bytes) + g;
        mbar_wait(&mbar[buf], parity);
        float acc[CG][2];
#pragma unroll
        for (int c = 0; c < CG; ++c) acc[c][0] = acc[c][1] = 0.0f;
#pragma unroll 2
        for (int pp = warp; pp < np; pp += TC_WARPS) {
            const uint4 wq = wq_s[(size_t)pp * 32];
            const uint2 wd = wd_s[(size_t)pp * 8];
            const uint32_t words[2][2] = {{wq.x, wq.y}, {wq.z, wq.w}};
            const __half2 dlo = *reinterpret_cast<const __half2 *>(&wd.x);
            const __half2 dhi = *reinterpret_cast<const __half2 *>(&wd.y);
            const float dsc[2][2] = {{__low2float(dlo), __high2float(dlo)}, {__low2float(dhi), __high2float(dhi)}};
#pragma unroll
            for (int bb = 0; bb < 2; ++bb) {
                const int bl = pp * 2 + bb;  // block index within the slice
                const uint32_t wg = words[bb][0], wg8 = words[bb][1];
                const uint32_t sg = wg >> 8, sg8 = wg8 >> 8;
                const uint32_t a_lo[4] = {wg & 0x000F000Fu, wg8 & 0x000F000Fu, sg & 0x000F000Fu, sg8 & 0x000F000Fu};
                const uint32_t a_hi[4] = {wg & 0x00F000F0u, wg8 & 0x00F000F0u, sg & 0x00F000F0u, sg8 & 0x00F000F0u};
                const uint2 *bfb = bf + (size_t)(bl * 2) * (2 * M) * 4;
#pragma unroll
                for (int c = 0; c < CG; ++c) {
                    const int col = c * 8 + g;
                    uint2 blo = make_uint2(0u, 0u), bhi = blo;
                    if (col < 2 * M) {
                        blo = bfb[col * 4 + t];
                        bhi = bfb[(2 * M + col) * 4 + t];
                    }
                    float cc[4] = {0.f, 0.f, 0.f, 0.f};
                    mma16816(cc, a_lo[0], a_lo[1], a_lo[2], a_lo[3], blo.x, blo.y);
                    mma16816(cc, a_hi[0], a_hi[1], a_hi[2], a_hi[3], bhi.x, bhi.y);
                    // thread holds (row g | g+8) x (cols 2t, 2t+1) = token 4c+t, splits hi+mid
                    const int tok = c * 4 + t;
                    const float2 o = tok < M ? off2[bl * M + tok] : make_float2(0.0f, 0.0f);
                    acc[c][0] = fmaf(dsc[bb][0], fmaf(cc[0] + cc[1], o.y, o.x), acc[c][0]);
                    acc[c][1] = fmaf(dsc[bb][1], fmaf(cc[2] + cc[3], o.y, o.x), acc[c][1]);
                }
            }
        }
        // ---- cross-warp reduction of the CTA's K range
#pragma unroll
        for (int c = 0; c < CG; ++c) {
            const int tok = c * 4 + t;
            if (tok < M) {
                red[(warp * 16 + g) * M + tok] = acc[c][0];
                red[(warp * 16 + g + 8) * M + tok] = acc[c][1];
            }
        }
        __syncthreads();  // also: every warp is done reading weight buffer `buf`
        for (int i = threadIdx.x; i < 16 * M; i += TC_THREADS) {
            float s = 0.0f;
#pragma unroll
            for (int w = 0; w < TC_WARPS; ++w) s += red[w * 16 * M + i];
            vals[i] = s;
        }
        __syncthreads();
        if (a.S == 1) {
            tc_epilogue<M, EPI>(a, tile, vals, sq);
        } else {
            // deterministic split-K: publish partials, last CTA to arrive sums them in slice order
            for (int i = threadIdx.x; i < 16 * M; i += TC_THREADS) {
                const int r = i / M, tok = i - r * M;
                __stcg(a.partial + ((size_t)slice * M + tok) * a.ldp + tile * 16 + r, vals[i]);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                // release: the barrier orders every thread's partial stores before this fence
                // (fences are cumulative), so one gpu-scope fence per CTA is enough
                __threadfence();
                const int old = atomicAdd(&a.counters[tile], 1);
                const int last = (old == a.S - 1);
                if (last) {
                    a.counters[tile] = 0;  // all slices have arrived: reset for the next launch
                    __threadfence();       // acquire side: the other slices' partials are now visible in L2
                }
                *flag = last;
            }
            __syncthreads();
            if (*flag) {
                for (int i = threadIdx.x; i < 16 * M; i += TC_THREADS) {
                    const int r = i / M, tok = i - r * M;
                    float s = 0.0f;
                    for (int sl = 0; sl < a.S; ++sl) s += __ldcg(a.partial + ((size_t)sl * M + tok) * a.ldp + tile * 16 + r);
                    vals[i] = s;
                }
                __syncthreads();
                tc_epilogue<M, EPI>(a, tile, vals, sq);
            }
        }
        if (a.nbuf == 1 && tile + 1 < tile1) {
            __syncthreads();
            if (threadIdx.x == 0) {
                asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
                issue_tile(tile + 1, 0);
            }
        } else {
            __syncthreads();  // vals / sq / red are reused by the next tile
        }
    }
}

// programmatic dependent launch between consecutive decode kernels (VOX_PDL=0 disables)
bool g_tc_pdl = !(getenv("VOX_PDL") && getenv("VOX_PDL")[0] == '0');

template <int M, int EPI>
void tc_launch_t(TcArgs a, const TcWork *wk, cudaStream_t st) {
    // ---- work decomposition
    // tuning knobs (environment, read once): VOX_TC_PS = K pairs per slice for M > 4,
    // VOX_TC_CTAS = target resident CTAs per SM when several tokens share the staging
    static const int env_ps = getenv("VOX_TC_PS") ? atoi(getenv("VOX_TC_PS")) : 0;
    static const int env_ctas = getenv("VOX_TC_CTAS") ? atoi(getenv("VOX_TC_CTAS")) : 0;
    const int ps_max = M <= 2 ? 64 : (M <= 4 ? 32 : (env_ps > 0 ? env_ps : 16));
    int S = 1;
    if (wk && wk->partial && wk->counters) S = (a.n_pairs + ps_max - 1) / ps_max;
    int Ps = (a.n_pairs + S - 1) / S;
    S = (a.n_pairs + Ps - 1) / Ps;
    if (S > 1) {
        VOX_CHECK((size_t)S * M * a.n_tiles * 16 <= wk->partial_floats && a.n_tiles <= wk->n_counters, VOX_EINVAL,
                  "q4_matvec_tc: split-K scratch too small (S=%d, N=%d)", S, a.N);
    }
    const size_t slice_bytes = (size_t)Ps * 576;
    int TG = (int)((20 * 1024 + slice_bytes - 1) / slice_bytes);
    TG = TG < 1 ? 1 : (TG > 4 ? 4 : TG);
    // the activation staging is per CTA: with several tokens it is a sizeable share of the work, so
    // give each CTA enough tiles to amortise it while keeping ~4 CTAs per SM in flight
    if (M > 2) {
        const int ctas = env_ctas > 0 ? env_ctas : 4;
        const int tg_occ = (int)(((size_t)a.n_tiles * S + VOX_NUM_SMS * ctas - 1) / (VOX_NUM_SMS * ctas));
        if (tg_occ > TG) TG = tg_occ > 16 ? 16 : tg_occ;
    }
    while (TG > 1 && (size_t)((a.n_tiles + TG - 1) / TG) * S < 2 * VOX_NUM_SMS) --TG;
    const int nbuf = TG > 1 ? 2 : 1;
    const size_t misc = (12 + TC_WARPS * M + TC_WARPS * 16 * M + 2 * 16 * M) * sizeof(float);
    const size_t act = misc + (size_t)Ps * 2 * M * sizeof(float2) + (size_t)Ps * 2 * 2 * 2 * M * 4 * sizeof(uint2);
    const size_t smem = act + 128 + (size_t)nbuf * slice_bytes + 64;
    VOX_CHECK(smem <= 200 * 1024, VOX_EINVAL, "q4_matvec_tc: shared memory %zu too large (K=%d, M=%d)", smem, a.K, M);
    static SmemAttr smem_attr;
    cuda_check_tc(ensure_dyn_smem(q4_matvec_tc_kernel<M, EPI>, 208 * 1024, smem_attr), "cudaFuncSetAttribute(q4_matvec_tc)");
    a.S = S;
    a.Ps = Ps;
    a.TG = TG;
    a.nbuf = nbuf;
    a.ldp = a.n_tiles * 16;
    a.partial = S > 1 ? wk->partial : nullptr;
    a.counters = S > 1 ? wk->counters : nullptr;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((a.n_tiles + TG - 1) / TG, S);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g_tc_pdl ? 1 : 0;
    cuda_check_tc(cudaLaunchKernelEx(&cfg, q4_matvec_tc_kernel<M, EPI>, a), "cudaLaunchKernelEx(q4_matvec_tc)");
    tc_count_launch("q4_matvec_tc");
}

template <int M>
void tc_launch_m(const TcArgs &a, const TcWork *wk, int epi, cudaStream_t st) {
    switch (epi) {
        case EPI_NONE: tc_launch_t<M, EPI_NONE>(a, wk, st); break;
        case EPI_RESIDUAL: tc_launch_t<M, EPI_RESIDUAL>(a, wk, st); break;
        case EPI_SILU_MUL: tc_launch_t<M, EPI_SILU_MUL>(a, wk, st); break;
        case EPI_GELU: tc_launch_t<M, EPI_GELU>(a, wk, st); break;
        default: fail(VOX_EINVAL, "bad epilogue");
    }
}

}  // namespace

void set_tc_pdl(bool on) { g_tc_pdl = on; }

void launch_q4_matvec_tc_ex(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                            const float *res, int epi, const float *gamma, const float *ada, float eps,
                            const TcWork *wk, cudaStream_t st) {
    VOX_CHECK(w.qs_tc != nullptr, VOX_EINVAL, "q4_matvec_tc: weight has no tensor-core layout");
    VOX_CHECK(M >= 1 && M <= 8, VOX_EINVAL, "q4_matvec_tc: M=%d out of range", M);
    VOX_CHECK(w.K % 32 == 0, VOX_EINVAL, "q4_matvec_tc: K=%d not a multiple of 32", w.K);
    TcArgs a{};
    a.qs_tc = w.qs_tc;
    a.d_tc = w.d_tc;
    a.N = w.N;
    a.K = w.K;
    a.n_tiles = (w.N + 15) / 16;
    a.n_pairs = (w.K / 32 + 1) / 2;
    a.x = x;
    a.y = y;
    a.ldy = ldy;
    a.bias = bias;
    a.res = res;
    a.gamma = gamma;
    a.ada = ada;
    a.eps = eps;
    a.ssq_in = (gamma && wk) ? wk->ssq_in : nullptr;
    a.ssq_in_parts = wk ? wk->ssq_in_parts : 0;
    a.ssq_out = (epi == EPI_RESIDUAL && wk) ? wk->ssq_out : nullptr;
    switch (M) {
        case 1: tc_launch_m<1>(a, wk, epi, st); break;
        case 2: tc_launch_m<2>(a, wk, epi, st); break;
        case 3: tc_launch_m<3>(a, wk, epi, st); break;
        case 4: tc_launch_m<4>(a, wk, epi, st); break;
        case 5: tc_launch_m<5>(a, wk, epi, st); break;
        case 6: tc_launch_m<6>(a, wk, epi, st); break;
        case 7: tc_launch_m<7>(a, wk, epi, st); break;
        default: tc_launch_m<8>(a, wk, epi, st); break;
    }
}

void launch_q4_matvec_tc_norm(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                              const float *res, int epi, const float *gamma, const float *ada, float eps,
                              cudaStream_t st) {
    launch_q4_matvec_tc_ex(w, x, M, y, ldy, bias, res, epi, gamma, ada, eps, nullptr, st);
}

void launch_q4_matvec_tc(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                         const float *res, int epi, cudaStream_t st) {
    launch_q4_matvec_tc_ex(w, x, M, y, ldy, bias, res, epi, nullptr, nullptr, 0.0f, nullptr, st);
}

}  // namespace vox
