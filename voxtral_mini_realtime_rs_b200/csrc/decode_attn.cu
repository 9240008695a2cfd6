// decode_attn.cu -- single-token decoder attention, fused with RoPE and the KV-cache append
// (reference src/gguf/model.rs:125-197 forward_with_cache for q_len = 1, rope.rs:103-141,
// kv_cache.rs:116-142).  One CTA per (kv head, stream): the 4 query heads of a GQA group share one
// pass over K and V (the reference materialises the x4 repeat), 8 warps split the keys, each lane
// owns hd/32 consecutive head dims, online softmax per (warp, head), merged through shared memory.
// K and V are read exactly once per kv head with 512-byte coalesced requests.
#include <cfloat>

#include "common.h"
#include "kernels.h"

namespace vox {

void tc_count_launch(const char *name);

namespace {

constexpr int DA_WARPS = 8;
constexpr int DA_THREADS = DA_WARPS * 32;

template <int G, int DPL, bool RING, typename KV>
__global__ void __launch_bounds__(DA_THREADS)
dec_attn_fused_kernel(const float *__restrict__ qkv, const int ld, const int H, const int Hkv, const KvView kv, const int window,
                      const float scale, const RopeView rope, float *__restrict__ out) {
    constexpr int HD = DPL * 32;
    __shared__ float qs[G][HD];
    __shared__ float kvs[2][HD];
    __shared__ float red_m[DA_WARPS][G], red_l[DA_WARPS][G];
    __shared__ float red_acc[DA_WARPS][G][HD];
    __shared__ int pts[64];  // this row's page table (first 64 slots = 1024 positions; beyond: global)
    // let the next kernel (the wo matvec) start prefetching its weights while we run
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
    const int kvh = blockIdx.x, b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pos = kv.pos[b];
    if (!RING && pos >= kv.max_seq()) return;
    for (int i = threadIdx.x; i < 64 && i < kv.max_pages; i += DA_THREADS) pts[i] = kv.page_table[(size_t)b * kv.max_pages + i];
    const float *row = qkv + (size_t)b * ld;  // M = 1: one row per stream
    // ---- load q (G heads), k, v of this group; RoPE q and k; append k, v at `pos`
    for (int i = threadIdx.x; i < G * HD; i += DA_THREADS) qs[i / HD][i % HD] = row[(kvh * G + i / HD) * HD + i % HD];
    for (int i = threadIdx.x; i < HD; i += DA_THREADS) {
        kvs[0][i] = row[H * HD + kvh * HD + i];
        kvs[1][i] = row[(H + Hkv) * HD + kvh * HD + i];
    }
    __syncthreads();
    const int half = HD / 2;
    for (int i = threadIdx.x; i < (G + 1) * half; i += DA_THREADS) {
        const int h = i / half, p = i - h * half;
        float *v = (h < G) ? &qs[h][2 * p] : &kvs[0][2 * p];
        const size_t rr = (size_t)(RING ? pos % rope.rows : pos) * half + p;
        const float c = rope.cos_t[rr], s = rope.sin_t[rr];
        const float xr = v[0], xi = v[1];
        v[0] = xr * c - xi * s;
        v[1] = xr * s + xi * c;
    }
    __syncthreads();
    if constexpr (kv_type_of<KV>() == KvType::Q8) {
        // the whole head vector is in kvs: a thread per 16-element block of K, then of V
        constexpr int NB = HD / KV_Q8_BLOCK;
        if (threadIdx.x < 2 * NB) {
            const int kv_i = threadIdx.x / NB, blk = threadIdx.x - kv_i * NB;
            const KvQ8Row r = kv_q8_row<RING>(kv_ptr<int8_t>(kv_i ? kv.v : kv.k), kv, b, Hkv, kvh, pos, HD);
            kv_q8_store16(r.q + blk * KV_Q8_BLOCK, r.d + blk, &kvs[kv_i][blk * KV_Q8_BLOCK]);
        }
    } else {
        const size_t at = kv_index<RING>(kv, b, Hkv, kvh, pos, HD);
        for (int i = threadIdx.x; i < HD; i += DA_THREADS) {
            kv_store(kv_ptr<KV>(kv.k) + at + i, kvs[0][i]);
            kv_store(kv_ptr<KV>(kv.v) + at + i, kvs[1][i]);
        }
    }
    __syncthreads();  // the CTA's own global writes are visible to all its threads after the barrier

    float q[G][DPL];
#pragma unroll
    for (int h = 0; h < G; ++h)
#pragma unroll
        for (int i = 0; i < DPL; ++i) q[h][i] = qs[h][lane * DPL + i];
    float m_run[G], l_run[G], acc[G][DPL];
#pragma unroll
    for (int h = 0; h < G; ++h) {
        m_run[h] = -INFINITY;
        l_run[h] = 0.0f;
#pragma unroll
        for (int i = 0; i < DPL; ++i) acc[h][i] = 0.0f;
    }
    const int j_lo = pos - window > 0 ? pos - window : 0;
    for (int j = j_lo + warp; j <= pos; j += DA_WARPS) {
        float kk[DPL], vv[DPL];
        const int pg = RING ? (j / KV_PAGE) % kv.max_pages : j / KV_PAGE;
        const int phys = pg < 64 ? pts[pg] : kv.page_table[(size_t)b * kv.max_pages + pg];
        if constexpr (kv_type_of<KV>() == KvType::Q8) {
            // this lane's DPL dims lie in one scale block
            const KvQ8Row kr = kv_q8_at(kv_ptr<int8_t>(kv.k), (size_t)phys * Hkv + kvh, j % KV_PAGE, HD);
            const KvQ8Row vr = kv_q8_at(kv_ptr<int8_t>(kv.v), (size_t)phys * Hkv + kvh, j % KV_PAGE, HD);
            const float kd = __half2float(kr.d[lane * DPL / KV_Q8_BLOCK]), vd = __half2float(vr.d[lane * DPL / KV_Q8_BLOCK]);
#pragma unroll
            for (int i = 0; i < DPL; ++i) {
                kk[i] = kv_q8_load(kr.q[lane * DPL + i], kd);
                vv[i] = kv_q8_load(vr.q[lane * DPL + i], vd);
            }
        } else {
            const size_t at = (((size_t)phys * Hkv + kvh) * KV_PAGE + (j % KV_PAGE)) * HD + lane * DPL;
            const KV *kr = kv_ptr<KV>(kv.k) + at;
            const KV *vr = kv_ptr<KV>(kv.v) + at;
#pragma unroll
            for (int i = 0; i < DPL; ++i) {
                kk[i] = kv_load(kr[i]);
                vv[i] = kv_load(vr[i]);
            }
        }
        float s[G];
#pragma unroll
        for (int h = 0; h < G; ++h) {
            float d = 0.0f;
#pragma unroll
            for (int i = 0; i < DPL; ++i) d = fmaf(q[h][i], kk[i], d);
            s[h] = d;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int h = 0; h < G; ++h) s[h] += __shfl_xor_sync(0xffffffffu, s[h], o);
#pragma unroll
        for (int h = 0; h < G; ++h) {
            const float sc = s[h] * scale;
            const float m_new = fmaxf(m_run[h], sc);
            const float alpha = expf(m_run[h] - m_new);  // exp(-inf) = 0 on the first key
            const float p = expf(sc - m_new);
            l_run[h] = l_run[h] * alpha + p;
            m_run[h] = m_new;
#pragma unroll
            for (int i = 0; i < DPL; ++i) acc[h][i] = fmaf(p, vv[i], acc[h][i] * alpha);
        }
    }
    // ---- merge the warps' partial softmax states
#pragma unroll
    for (int h = 0; h < G; ++h) {
        if (lane == 0) {
            red_m[warp][h] = m_run[h];
            red_l[warp][h] = l_run[h];
        }
#pragma unroll
        for (int i = 0; i < DPL; ++i) red_acc[warp][h][lane * DPL + i] = acc[h][i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G * HD; i += DA_THREADS) {
        const int h = i / HD, d = i - h * HD;
        float mx = -INFINITY;
#pragma unroll
        for (int w = 0; w < DA_WARPS; ++w) mx = fmaxf(mx, red_m[w][h]);
        float num = 0.0f, den = 0.0f;
#pragma unroll
        for (int w = 0; w < DA_WARPS; ++w) {
            const float f = (red_m[w][h] == -INFINITY) ? 0.0f : expf(red_m[w][h] - mx);
            num = fmaf(red_acc[w][h][d], f, num);
            den = fmaf(red_l[w][h], f, den);
        }
        out[(size_t)b * (H * HD) + (kvh * G + h) * HD + d] = num / den;
    }
}

template <int G, bool RING, typename KV>
void launch_g(int dpl, dim3 grid, cudaStream_t st, const float *qkv, int ld, int H, int Hkv, const KvView &kv, int window,
              float scale, const RopeView &rope, float *out) {
    switch (dpl) {
        case 1: dec_attn_fused_kernel<G, 1, RING, KV><<<grid, DA_THREADS, 0, st>>>(qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 2: dec_attn_fused_kernel<G, 2, RING, KV><<<grid, DA_THREADS, 0, st>>>(qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 4: dec_attn_fused_kernel<G, 4, RING, KV><<<grid, DA_THREADS, 0, st>>>(qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        default: fail(VOX_EINVAL, "dec_attn_fused: unsupported head_dim");
    }
}

}  // namespace

bool dec_attn_fused_supported(int H, int Hkv, int hd) {
    const int G = H / Hkv;
    return (hd == 32 || hd == 64 || hd == 128) && (G == 1 || G == 2 || G == 4) && H % Hkv == 0;
}

void launch_dec_attn_fused(float *qkv, int B, int ld, int H, int Hkv, int hd, const KvView &kv, int window, float scale,
                           const RopeView &rope, float *out, cudaStream_t st) {
    VOX_CHECK(dec_attn_fused_supported(H, Hkv, hd), VOX_EINVAL, "dec_attn_fused: unsupported shape");
    // the key at pos - window must still be in the ring after the append at pos
    if (kv.ring)
        VOX_CHECK(window < kv.max_seq(), VOX_EINVAL, "dec_attn_fused: window %d does not fit the KV ring of %d", window,
                  kv.max_seq());
    const int G = H / Hkv, dpl = hd / 32;
    dim3 grid(Hkv, B);
    if (kv.type == KvType::Q8) {
        switch (G * 2 + (kv.ring ? 1 : 0)) {
            case 2: launch_g<1, false, int8_t>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
            case 3: launch_g<1, true, int8_t>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
            case 4: launch_g<2, false, int8_t>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
            case 5: launch_g<2, true, int8_t>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
            case 8: launch_g<4, false, int8_t>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
            default: launch_g<4, true, int8_t>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        }
        tc_count_launch("dec_attn_fused");
        return;
    }
    const bool f16 = kv.type == KvType::F16;
    switch (G * 4 + (kv.ring ? 2 : 0) + (f16 ? 1 : 0)) {
        case 4: launch_g<1, false, float>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 5: launch_g<1, false, __half>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 6: launch_g<1, true, float>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 7: launch_g<1, true, __half>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 8: launch_g<2, false, float>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 9: launch_g<2, false, __half>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 10: launch_g<2, true, float>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 11: launch_g<2, true, __half>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 16: launch_g<4, false, float>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 17: launch_g<4, false, __half>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        case 18: launch_g<4, true, float>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
        default: launch_g<4, true, __half>(dpl, grid, st, qkv, ld, H, Hkv, kv, window, scale, rope, out); break;
    }
    tc_count_launch("dec_attn_fused");
}

}  // namespace vox
