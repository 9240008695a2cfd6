// enc_attn_tc.cu -- K4-TC: encoder attention (causal + sliding window) on the tensor cores with
// f32-grade accuracy.  Reference: src/gguf/model.rs:77-122 (softmax(q k^T * scale + mask) v) and
// masking.rs:9-44 (key j visible to query i iff j <= i and i - j <= window).
//
// Flash-attention-2 data flow with mma.sync.m16n8k16 (f16 x f16 -> f32):
//   CTA = 64 queries of one (stream, head), 4 warps x 16 query rows; key tiles of 64.
//   Every f32 operand is split into two f16 pieces  x = hi + lo  (hi = f16(x), lo = f16(x - hi))
//   and every product is three MMAs  hi.hi + hi.lo + lo.hi  with f32 accumulation.  The pieces carry
//   22 mantissa bits only while lo stays in f16's normal range and hi below 65504, so each operand is
//   first scaled by an exact power of two that brings its largest magnitude into [2^14, 2^15):
//   Q per query row, K per key tile, P (in [0, 1]) by 2^15, and V by the running maximum over the
//   key tiles the CTA has loaded (o is only ever scaled down, so it cannot overflow).  Keys no query
//   of the CTA can see are loaded as zeros and do not count towards these maxima.  The S tile's
//   factors are undone with `scale`, V's and P's as o is rescaled and stored.  So, whatever the
//   overall scale of the operands, the representation error and the dropped lo.lo term are 2^-22
//   relative to each operand, or 2^-39 relative to the largest Q of its row, K of its tile or V the
//   CTA has loaded, whichever is larger: elements far below the largest in the same tile or block
//   lose relative precision (tests/test_attention_ref.py models this arithmetic and bounds it; the
//   SIMT kernel K4 in kernels.cu is the f32 cross-check).
//   S = Q K^T : A = Q fragments (registers, loaded once), B = K tile [key][dim] from shared memory
//               (ldmatrix, rows padded to 72 halves: conflict-free);
//   online softmax in f32 registers (scale and mask applied to the f32 scores, exp in f32);
//   O += P V  : A = P re-used straight from the S accumulator layout, B = V tile [key][dim] through
//               ldmatrix.trans.
// Only the causal band is visited (the reference builds two S x S masks on the host per layer).
#include <cuda_fp16.h>

#include <cfloat>

#include "common.h"
#include "kernels.h"

namespace vox {

void tc_count_launch(const char *name);

namespace {

constexpr int ET_BQ = 64, ET_BK = 64, ET_THREADS = 128;
constexpr float P_SCALE = 32768.0f;  // 2^15: softmax probabilities are split as P * 2^15
constexpr int ET_PAD = 8;  // halves of row padding: row stride = HD + 8 halves (144 B for HD = 64)

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t b0, const uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void *p) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void *p) {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(a));
}
// (x, y) -> f16x2 hi piece and f16x2 lo piece
__device__ __forceinline__ void split2(const float x, const float y, uint32_t &hi, uint32_t &lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x - hf.x, y - hf.y);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}
// 2^k for k in [-126, 127]
__device__ __forceinline__ float pow2f(const int k) { return __uint_as_float((uint32_t)(k + 127) << 23); }
// k such that 2^k maps m = max |x| into [2^14, 2^15), clamped to [-126, 126] so that 2^k and 2^-k are normal;
// `keep` when m is 0 or not finite
__device__ __forceinline__ int split_exp(const float m, const int keep) {
    const int e = (int)((__float_as_uint(m) >> 23) & 0xff);
    if (!(m > 0.0f) || e == 0xff) return keep;
    return min(max(14 - (e - 127), -126), 126);
}
__device__ __forceinline__ float absmax4(const float a, const float b, const float c, const float d) {
    return fmaxf(fmaxf(fabsf(a), fabsf(b)), fmaxf(fabsf(c), fabsf(d)));
}

template <int HD>
__global__ void __launch_bounds__(ET_THREADS)
enc_attention_tc_kernel(const float *__restrict__ qkv, float *__restrict__ out, const int S_grid, const int H, const int ld,
                        const int q_off, const int k_off, const int v_off, const int window, const float scale,
                        const int *__restrict__ seg) {
    constexpr int STR = HD + ET_PAD;  // halves per shared-memory row
    constexpr int KS = HD / 16;       // k-steps of Q K^T
    constexpr int ND = HD / 8;        // n-tiles of the output
    constexpr int RL = HD / 4;        // threads per key row of the tile load (one float4 each)
    constexpr int IT = ET_BK * RL / ET_THREADS;  // key rows each thread loads per tile
    __shared__ __align__(16) __half Kh[ET_BK * STR], Kl[ET_BK * STR], Vh[ET_BK * STR], Vl[ET_BK * STR];
    __shared__ float tile_max[2][ET_THREADS / 32];  // per-warp max |k|, max |v| of the tile being loaded
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * ET_BQ;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    // stream b's rows [row0, row0 + S): the segment table's, or b * S_grid.. of a uniform batch
    const int row0 = seg ? seg[b] : b * S_grid, S = seg ? seg[b + 1] - row0 : S_grid;
    if (q0 >= S) return;   // the grid covers the longest segment
    const float *base = qkv + (size_t)row0 * ld;

    // ---- Q fragments (A operand), hi and lo pieces: rows q0 + 16*warp + {g, g+8}, each row scaled by its power of two
    //      (a row's elements sit in the 4 lanes of a quad)
    const int qr0 = q0 + warp * 16 + g, qr1 = qr0 + 8;
    float2 qv[KS][4];
    float qm0 = 0.0f, qm1 = 0.0f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
        qv[ks][0] = qv[ks][1] = qv[ks][2] = qv[ks][3] = make_float2(0.f, 0.f);
        if (qr0 < S) {
            const float *r = base + (size_t)qr0 * ld + q_off + h * HD + ks * 16 + 2 * t;
            qv[ks][0] = *reinterpret_cast<const float2 *>(r);
            qv[ks][2] = *reinterpret_cast<const float2 *>(r + 8);
        }
        if (qr1 < S) {
            const float *r = base + (size_t)qr1 * ld + q_off + h * HD + ks * 16 + 2 * t;
            qv[ks][1] = *reinterpret_cast<const float2 *>(r);
            qv[ks][3] = *reinterpret_cast<const float2 *>(r + 8);
        }
        qm0 = fmaxf(qm0, absmax4(qv[ks][0].x, qv[ks][0].y, qv[ks][2].x, qv[ks][2].y));
        qm1 = fmaxf(qm1, absmax4(qv[ks][1].x, qv[ks][1].y, qv[ks][3].x, qv[ks][3].y));
    }
#pragma unroll
    for (int x = 1; x <= 2; x <<= 1) {
        qm0 = fmaxf(qm0, __shfl_xor_sync(0xffffffffu, qm0, x));
        qm1 = fmaxf(qm1, __shfl_xor_sync(0xffffffffu, qm1, x));
    }
    const int eq0 = split_exp(qm0, 0), eq1 = split_exp(qm1, 0);
    const float fq[4] = {pow2f(eq0), pow2f(eq1), pow2f(eq0), pow2f(eq1)};
    // the rows' score factors: scale and the rows' Q powers of two undone (exactly: powers of two)
    const float sc0 = scale * pow2f(-eq0), sc1 = scale * pow2f(-eq1);
    uint32_t qh[KS][4], ql[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int a = 0; a < 4; ++a) split2(qv[ks][a].x * fq[a], qv[ks][a].y * fq[a], qh[ks][a], ql[ks][a]);

    float o[ND][4];
#pragma unroll
    for (int n = 0; n < ND; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.0f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};
    int ev_run = 126;  // o holds P V * 2^(15 + ev_run): P scaled by 2^15, V by the running power of two (never raised)

    const int q_last = min(q0 + ET_BQ - 1, S - 1);
    const int key_lo = q0 - window;  // keys [key_lo, q_last]: the keys some query of this CTA can see
    int j_begin = key_lo;
    if (j_begin < 0) j_begin = 0;
    j_begin = (j_begin / ET_BK) * ET_BK;
    for (int j0 = j_begin; j0 <= q_last; j0 += ET_BK) {
        __syncthreads();  // previous tile fully consumed
        // ---- K, V tile: f32 global -> f16 hi/lo shared, [key][dim]; K scaled by the tile's power of two, V by the running
        //      one.  Keys outside [key_lo, q_last] load as zeros.  A first pass takes the block-wide maxima; the split
        //      pass reads the tile again (from L1).
        float km = 0.0f, vm = 0.0f;
#pragma unroll 2
        for (int it = 0; it < IT; ++it) {
            const int i = tid + it * ET_THREADS;
            const int kk = i / RL, d4 = (i - kk * RL) * 4;
            if (j0 + kk >= key_lo && j0 + kk <= q_last) {
                const float *r = base + (size_t)(j0 + kk) * ld + h * HD + d4;
                const float4 kv = *reinterpret_cast<const float4 *>(r + k_off), vv = *reinterpret_cast<const float4 *>(r + v_off);
                km = fmaxf(km, absmax4(kv.x, kv.y, kv.z, kv.w));
                vm = fmaxf(vm, absmax4(vv.x, vv.y, vv.z, vv.w));
            }
        }
#pragma unroll
        for (int x = 16; x > 0; x >>= 1) {
            km = fmaxf(km, __shfl_xor_sync(0xffffffffu, km, x));
            vm = fmaxf(vm, __shfl_xor_sync(0xffffffffu, vm, x));
        }
        if (lane == 0) {
            tile_max[0][warp] = km;
            tile_max[1][warp] = vm;
        }
        __syncthreads();
        // V's power of two only falls (an all-zero tile keeps it): o is never scaled up
        const int ek = split_exp(fmaxf(fmaxf(tile_max[0][0], tile_max[0][1]), fmaxf(tile_max[0][2], tile_max[0][3])), 0);
        const int ev = min(ev_run, split_exp(fmaxf(fmaxf(tile_max[1][0], tile_max[1][1]), fmaxf(tile_max[1][2], tile_max[1][3])), ev_run));
        const float fk = pow2f(ek), fv = pow2f(ev);
#pragma unroll 2
        for (int it = 0; it < IT; ++it) {
            const int i = tid + it * ET_THREADS;
            const int kk = i / RL, d4 = (i - kk * RL) * 4;
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (j0 + kk >= key_lo && j0 + kk <= q_last) {
                const float *r = base + (size_t)(j0 + kk) * ld + h * HD + d4;
                kv = *reinterpret_cast<const float4 *>(r + k_off);
                vv = *reinterpret_cast<const float4 *>(r + v_off);
            }
            uint2 a, bq;
            split2(kv.x * fk, kv.y * fk, a.x, bq.x);
            split2(kv.z * fk, kv.w * fk, a.y, bq.y);
            *reinterpret_cast<uint2 *>(&Kh[kk * STR + d4]) = a;
            *reinterpret_cast<uint2 *>(&Kl[kk * STR + d4]) = bq;
            split2(vv.x * fv, vv.y * fv, a.x, bq.x);
            split2(vv.z * fv, vv.w * fv, a.y, bq.y);
            *reinterpret_cast<uint2 *>(&Vh[kk * STR + d4]) = a;
            *reinterpret_cast<uint2 *>(&Vl[kk * STR + d4]) = bq;
        }
        // the rows' score factors for this tile: scale and the row's and the tile's powers of two undone (exactly)
        const float st0 = sc0 * pow2f(-ek), st1 = sc1 * pow2f(-ek);
        __syncthreads();

        // ---- S = Q K^T (16 x 64 per warp), three MMAs per product
        float s[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.0f;
#pragma unroll
            for (int kp = 0; kp < KS / 2; ++kp) {
                // matrices: dims [32kp, +8), [+8, +16), [+16, +24), [+24, +32) of keys 8n .. 8n+7
                uint32_t kh[4], kl[4];
                const int roff = (n * 8 + (lane & 7)) * STR + kp * 32 + 8 * (lane >> 3);
                ldsm_x4(kh, &Kh[roff]);
                ldsm_x4(kl, &Kl[roff]);
                mma16816(s[n], qh[2 * kp], kh[0], kh[1]);
                mma16816(s[n], qh[2 * kp], kl[0], kl[1]);
                mma16816(s[n], ql[2 * kp], kh[0], kh[1]);
                mma16816(s[n], qh[2 * kp + 1], kh[2], kh[3]);
                mma16816(s[n], qh[2 * kp + 1], kl[2], kl[3]);
                mma16816(s[n], ql[2 * kp + 1], kh[2], kh[3]);
            }
        }
        // ---- scale (powers of two undone), mask, online softmax (rows g and g+8; a row's
        //      64 scores live in the 4 lanes of a quad)
        float m_t[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int gi = (e < 2) ? qr0 : qr1;
                const int gj = j0 + n * 8 + 2 * t + (e & 1);
                const bool valid = (gj < S) && (gj <= gi) && (gi - gj <= window);
                s[n][e] = valid ? s[n][e] * ((e < 2) ? st0 : st1) : -INFINITY;
                m_t[e >> 1] = fmaxf(m_t[e >> 1], s[n][e]);
            }
        }
        float alpha[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            m_t[r] = fmaxf(m_t[r], __shfl_xor_sync(0xffffffffu, m_t[r], 1));
            m_t[r] = fmaxf(m_t[r], __shfl_xor_sync(0xffffffffu, m_t[r], 2));
            const float m_new = fmaxf(m_run[r], m_t[r]);
            alpha[r] = (m_new == -INFINITY) ? 1.0f : expf(m_run[r] - m_new);
            m_run[r] = m_new;
        }
        float psum[2] = {0.0f, 0.0f};
        uint32_t ph[4][4], pl[4][4];  // P as A fragments: k-step j = key n-tiles 2j, 2j+1
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            float pv[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float mr = m_run[e >> 1];
                pv[e] = (mr == -INFINITY) ? 0.0f : expf(s[n][e] - mr);
                psum[e >> 1] += pv[e];
            }
            // C layout {row g: c0 c1, row g+8: c2 c3} of n-tile n -> A regs {a0, a1} (n even) or {a2, a3} (n odd).
            // P in [0, 1] is split as P * 2^15: its lo piece stays in f16's normal range down to P = 2^-18
            split2(pv[0] * P_SCALE, pv[1] * P_SCALE, ph[n >> 1][(n & 1) * 2 + 0], pl[n >> 1][(n & 1) * 2 + 0]);
            split2(pv[2] * P_SCALE, pv[3] * P_SCALE, ph[n >> 1][(n & 1) * 2 + 1], pl[n >> 1][(n & 1) * 2 + 1]);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + psum[r];  // quad-partial sums; reduced at the end
        // o moves to this tile's V power of two with the softmax rescale
        const int dv = ev - ev_run;  // in [-239, 0]: two exact power-of-two factors
        const float r0 = alpha[0] * pow2f(dv / 2) * pow2f(dv - dv / 2), r1 = alpha[1] * pow2f(dv / 2) * pow2f(dv - dv / 2);
        ev_run = ev;
#pragma unroll
        for (int n = 0; n < ND; ++n) {
            o[n][0] *= r0;
            o[n][1] *= r0;
            o[n][2] *= r1;
            o[n][3] *= r1;
        }
        // ---- O += P V
#pragma unroll
        for (int n = 0; n < ND; ++n) {
#pragma unroll
            for (int kp = 0; kp < 2; ++kp) {
                // matrices (transposed on load): keys [32kp, +8), [+8, +16), [+16, +24), [+24, +32) x dims 8n .. 8n+7
                uint32_t vh[4], vl[4];
                const int roff = (kp * 32 + (lane & 7) + 8 * (lane >> 3)) * STR + n * 8;
                ldsm_x4_t(vh, &Vh[roff]);
                ldsm_x4_t(vl, &Vl[roff]);
                mma16816(o[n], ph[2 * kp], vh[0], vh[1]);
                mma16816(o[n], ph[2 * kp], vl[0], vl[1]);
                mma16816(o[n], pl[2 * kp], vh[0], vh[1]);
                mma16816(o[n], ph[2 * kp + 1], vh[2], vh[3]);
                mma16816(o[n], ph[2 * kp + 1], vl[2], vl[3]);
                mma16816(o[n], pl[2 * kp + 1], vh[2], vh[3]);
            }
        }
    }
    // ---- normalise and store
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
    const int eo = -(15 + ev_run);  // undo P's and V's powers of two (eo in [-141, 98]: two exact factors)
    const float fo0 = pow2f(eo / 2), fo1 = pow2f(eo - eo / 2);
#pragma unroll
    for (int n = 0; n < ND; ++n) {
        if (qr0 < S)
            *reinterpret_cast<float2 *>(out + ((size_t)row0 + qr0) * (H * HD) + h * HD + n * 8 + 2 * t) =
                make_float2(o[n][0] * inv0 * fo0 * fo1, o[n][1] * inv0 * fo0 * fo1);
        if (qr1 < S)
            *reinterpret_cast<float2 *>(out + ((size_t)row0 + qr1) * (H * HD) + h * HD + n * 8 + 2 * t) =
                make_float2(o[n][2] * inv1 * fo0 * fo1, o[n][3] * inv1 * fo0 * fo1);
    }
}

}  // namespace

bool enc_attention_tc_supported(int hd, int ld, int q_off, int k_off, int v_off) {
    return (hd == 32 || hd == 64) && ld % 4 == 0 && q_off % 4 == 0 && k_off % 4 == 0 && v_off % 4 == 0;
}

void launch_enc_attention_tc(const float *qkv, float *out, int B, int S, int H, int hd, int ld, int q_off, int k_off,
                             int v_off, int window, float scale, cudaStream_t st, const int *seg) {
    if (S <= 0) return;
    VOX_CHECK(enc_attention_tc_supported(hd, ld, q_off, k_off, v_off), VOX_EINVAL, "enc_attention_tc: unsupported shape");
    dim3 grid((S + ET_BQ - 1) / ET_BQ, H, B);
    if (hd == 64) enc_attention_tc_kernel<64><<<grid, ET_THREADS, 0, st>>>(qkv, out, S, H, ld, q_off, k_off, v_off, window, scale, seg);
    else enc_attention_tc_kernel<32><<<grid, ET_THREADS, 0, st>>>(qkv, out, S, H, ld, q_off, k_off, v_off, window, scale, seg);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) fail(VOX_ECUDA, fmt("CUDA error: enc_attention_tc launch: %s", cudaGetErrorString(e)));
    tc_count_launch("enc_attention_tc");
}

}  // namespace vox
