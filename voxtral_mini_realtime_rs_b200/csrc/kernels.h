// kernels.h -- host-callable launchers for the sm_90a kernels (all asynchronous on `st`).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>

#include <cstdint>

namespace vox {

// SMs of the target GPU (H100 SXM): sizes grids and the split-K scratch of the GEMMs
constexpr int VOX_NUM_SMS = 132;

// Opt-in to more than 48 KB of dynamic shared memory.  The attribute is per (function, DEVICE), and the C ABI takes a
// device index, so one process can drive several GPUs: remember what was set per device (not per process), with
// atomics so that first use from two threads is safe (setting the same attribute twice is harmless).
struct SmemAttr {
    std::atomic<size_t> bytes[64];
};
template <typename F>
inline cudaError_t ensure_dyn_smem(F func, size_t bytes, SmemAttr &st) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (st.bytes[dev].load(std::memory_order_acquire) >= bytes) return cudaSuccess;
    e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) {
        size_t cur = st.bytes[dev].load(std::memory_order_relaxed);
        while (cur < bytes && !st.bytes[dev].compare_exchange_weak(cur, bytes, std::memory_order_release)) {}
    }
    return e;
}
void smem_attr_check(cudaError_t e, const char *what);  // throws vox::Error(VOX_ECUDA) on failure (kernels.cu)


// Repacked Q4_0 weight resident in HBM.  The 18-byte GGUF blocks {f16 d; u8 qs[16]} are split at
// load into a 16-byte-aligned nibble plane and an f16 scale plane (row-major by n, K-blocks
// contiguous) so that a warp reads 512 contiguous bytes per request.  Dequant rule unchanged:
// element i of a block = (qs[i] & 15) - 8, element i+16 = (qs[i] >> 4) - 8, times d.
struct Q4Weight {
    const uint4 *qs = nullptr;   // [N][K/32]
    const __half *d = nullptr;   // [N][K/32]
    // optional tensor-core ("TC") layout of the same blocks, see matvec_tc.cu
    const uint4 *qs_tc = nullptr;  // [N/16][K/64][32]
    const uint2 *d_tc = nullptr;   // [N/16][K/64][8]
    int N = 0, K = 0;
    // every block scale is finite with |d| < 32: the domain in which the wgmma GEMM's f16 split of (q-8)*d*2^8 is exact
    // (gemm_tc5.cu); set by upload_q4, which sees the scales on the host
    bool d_below_32 = false;
    size_t bytes() const { return (size_t)N * (K / 32) * 18; }
};

enum Epi : int {
    EPI_NONE = 0,      // y = acc (+bias)
    EPI_RESIDUAL = 1,  // y = res + acc (+bias)     (y may alias res)
    EPI_SILU_MUL = 2,  // rows (2i,2i+1) = (gate_i, up_i): y[:, i] = silu(gate) * up, ldy = N/2
    EPI_GELU = 3,      // y = gelu_erf(acc + bias)
};

// Per-row ADA scale: the rows of one call belong to streams, each at its own transcription delay.  Row r of a B x M
// problem is scaled by rows[r / m] + off (one pointer per stream, e.g. its [L][D] ADA set, off = layer * D).
// rows == nullptr: no ADA scale.
struct AdaRows {
    const float *const *rows = nullptr;
    int m = 1;
    size_t off = 0;
    __host__ __device__ const float *row(int r) const { return rows[r / m] + off; }
};

// y[M,N] = x[M,K] . W^T, M <= 8 (decode / batched decode): warp-per-row-pair, shuffle reduce.
void launch_q4_matvec(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                      const float *res, int epi, cudaStream_t st);
// Caller-owned scratch for the tensor-core matvec: split-K partial sums + tickets, and the per-tile
// sums of squares that residual epilogues leave behind for the next kernel's fused RMSNorm.
struct TcWork {
    float *partial = nullptr;      // [S][M][n_tiles*16]
    size_t partial_floats = 0;
    int *counters = nullptr;       // [n_counters], zero between launches
    int n_counters = 0;
    const float *ssq_in = nullptr; // [ssq_in_parts][M] partial sums of squares of the input rows
    int ssq_in_parts = 0;
    float *ssq_out = nullptr;      // [N/16][M], written by EPI_RESIDUAL epilogues
};
// same contract as launch_q4_matvec, dequant arithmetic on the tensor cores (mma.sync, f16 subnormal nibbles); needs
// the TC layout (w.qs_tc).  matvec_tc.cu.  gamma (+ optional ada_rows): RMSNorm of the input fused into the staging
// pass, x := ((x / sqrt(mean(x^2)+eps)) * gamma) * ada_rows.row(m).  wk (optional): split-K over K slices, fused-norm
// sums of squares.
void launch_q4_matvec_tc_ex(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                            const float *res, int epi, const float *gamma, float eps, const TcWork *wk, cudaStream_t st,
                            const AdaRows &ada_rows = AdaRows{});
// Split-K scratch sizes launch_q4_matvec_tc_ex needs for an N x K weight at up to 8 rows: partial_floats and n_counters
// are set, the pointers are left to the caller (counters zeroed).
TcWork q4_matvec_tc_work_size(int N, int K);
// Decoder KV cache of ONE layer as the attention kernels see it: PAGED (KVCache semantics of kv_cache.rs:52-142 --
// append at the stream's position, read keys 0..pos -- over fixed-size pages so that sessions of different ages
// share one pool).  Batch row b owns logical pages page_table[b][0..max_pages); logical position j lives at
//   pool + ((phys(b, j / KV_PAGE) * Hkv + kv_head) * KV_PAGE + j % KV_PAGE) * hd  (Q8: kv_q8_row below).
// Positions are per row (pos[b] = number of cached positions of row b = position of its next token): whole-utterance
// batches keep them equal, streaming sessions do not.
// ring: the page table row is a RING -- logical page lp lives in slot lp % max_pages and positions are unbounded (the
// sessions of an unbounded stream pool, stream.cu; safe while max_pages * KV_PAGE > window + the rows a prefill writes
// before reading).  The kernels take it as a template flag, so the non-ring code is the plain table walk.
constexpr int KV_PAGE = 16;
// Element type of the decoder KV cache, fixed for a session's lifetime (vox_session_create_ex kv_dtype): f32, IEEE
// binary16 (__half), or Q8: int8 with one f16 scale per 16 consecutive head dims (int8_t).  Kernels take the C++ type
// as a template parameter KV next to RING; every load and store of a cached K or V element goes through kv_load /
// kv_store and the kv_q8_* helpers below, the one place the formats are decided.
enum class KvType : uint8_t { F32 = 0, F16 = 1, Q8 = 2 };
// Q8 pages: each (page, kv head) unit holds its values [KV_PAGE][hd] int8 and then their scales [KV_PAGE][hd / 16] f16,
// contiguous -- 2304 bytes at hd 128, 576 at hd 32, both multiples of 16, so one unit's rows and scales stage with
// 16-byte copies.  Scale block i of a row covers its head dims [16i, 16i + 16).
constexpr int KV_Q8_BLOCK = 16;
// bytes of one (page, kv head) unit: KV_PAGE positions of hd values
__host__ __device__ constexpr size_t kv_unit_bytes(KvType t, int hd) {
    return t == KvType::Q8 ? (size_t)KV_PAGE * hd + (size_t)KV_PAGE * (hd / KV_Q8_BLOCK) * 2
                           : (size_t)KV_PAGE * hd * (t == KvType::F16 ? 2 : 4);
}
template <typename KV> __host__ __device__ constexpr KvType kv_type_of() {
    return sizeof(KV) == 1 ? KvType::Q8 : (sizeof(KV) == 2 ? KvType::F16 : KvType::F32);
}
// Base address of a KV page pool, typed by its element: kv_pool sets the member of the pool's KvType, kv_ptr<KV> reads
// the member of the kernel's KV (the same type: a kernel instantiation is chosen by the view's KvType).
union KvPool {
    float *f32 = nullptr;
    __half *f16;
    int8_t *q8;   // byte address of the pool's (page, kv head) units
};
inline KvPool kv_pool(void *p, KvType t) {
    KvPool r;
    if (t == KvType::F16) r.f16 = static_cast<__half *>(p);
    else if (t == KvType::Q8) r.q8 = static_cast<int8_t *>(p);
    else r.f32 = static_cast<float *>(p);
    return r;
}
template <typename KV> __host__ __device__ __forceinline__ KV *kv_ptr(const KvPool &p);
template <> __host__ __device__ __forceinline__ float *kv_ptr<float>(const KvPool &p) { return p.f32; }
template <> __host__ __device__ __forceinline__ __half *kv_ptr<__half>(const KvPool &p) { return p.f16; }
template <> __host__ __device__ __forceinline__ int8_t *kv_ptr<int8_t>(const KvPool &p) { return p.q8; }
template <typename KV> __host__ __device__ __forceinline__ KV *kv_ptr(const volatile KvPool &p);
template <> __host__ __device__ __forceinline__ float *kv_ptr<float>(const volatile KvPool &p) { return p.f32; }
template <> __host__ __device__ __forceinline__ __half *kv_ptr<__half>(const volatile KvPool &p) { return p.f16; }
template <> __host__ __device__ __forceinline__ int8_t *kv_ptr<int8_t>(const volatile KvPool &p) { return p.q8; }
// Q8 storage rule of one block x[0..16) (include/voxtral.h VOX_DTYPE_KV_Q8):
//   a = max |x_i|, d = f16_rn(min(a / 127, 65504)), q_i = clamp(rint(x_i / d), -127, 127) (q_i = 0 when d == 0);
//   a block holding a NaN stores d = NaN and q_i = 0.  Decoded value: (float)d * q_i, exact in f32.
// The host mirror (DecoderKv::read) decodes with the same product.
inline float kv_q8_decode_host(const int8_t q, const __half d) { return __half2float(d) * (float)q; }
struct KvView {
    KvPool k, v;                       // [n_pages][Hkv][KV_PAGE][hd] of `type`
    const int *page_table = nullptr;   // [B][max_pages] physical page ids
    int max_pages = 0;                 // logical pages per row; capacity = max_pages * KV_PAGE positions (ring: slots)
    bool ring = false;
    KvType type = KvType::F32;
    const int *pos = nullptr;          // [B]
    __host__ __device__ int max_seq() const { return max_pages * KV_PAGE; }
};
#ifdef __CUDACC__
template <bool RING = false>
__device__ __forceinline__ size_t kv_index(const KvView &kv, const int b, const int Hkv, const int kvh, const int j, const int hd) {
    const int lp = j / KV_PAGE;
    const int phys = kv.page_table[(size_t)b * kv.max_pages + (RING ? lp % kv.max_pages : lp)];
    return (((size_t)phys * Hkv + kvh) * KV_PAGE + (j % KV_PAGE)) * hd;
}
// Stored value of x: f32 as is; f16 clamped to [-65504, 65504] (a value past the f16 range stores +-65504, never
// +-inf), then rounded to nearest even.  NaN fails both comparisons and stays NaN.
__device__ __forceinline__ float kv_clamp16(const float x) { return x > 65504.0f ? 65504.0f : (x < -65504.0f ? -65504.0f : x); }
__device__ __forceinline__ void kv_store(float *p, const float x) { *p = x; }
__device__ __forceinline__ void kv_store(__half *p, const float x) { *p = __float2half_rn(kv_clamp16(x)); }
// four consecutive elements (16-byte aligned for f32, 8-byte for f16)
__device__ __forceinline__ void kv_store4(float *p, const float4 x) { *reinterpret_cast<float4 *>(p) = x; }
__device__ __forceinline__ void kv_store4(__half *p, const float4 x) {
    const __half2 lo = __halves2half2(__float2half_rn(kv_clamp16(x.x)), __float2half_rn(kv_clamp16(x.y)));
    const __half2 hi = __halves2half2(__float2half_rn(kv_clamp16(x.z)), __float2half_rn(kv_clamp16(x.w)));
    uint2 u;
    u.x = *reinterpret_cast<const uint32_t *>(&lo);
    u.y = *reinterpret_cast<const uint32_t *>(&hi);
    *reinterpret_cast<uint2 *>(p) = u;
}
// exact widening to f32
__device__ __forceinline__ float kv_load(const float x) { return x; }
__device__ __forceinline__ float kv_load(const __half x) { return __half2float(x); }
// elements [4d, 4d + 4) of a row (16-byte aligned f32, 8-byte aligned f16)
__device__ __forceinline__ float4 kv_load4(const float *row, const int d) { return reinterpret_cast<const float4 *>(row)[d]; }
__device__ __forceinline__ float4 kv_load4(const __half *row, const int d) {
    const uint2 u = reinterpret_cast<const uint2 *>(row)[d];
    const float2 lo = __half22float2(*reinterpret_cast<const __half2 *>(&u.x));
    const float2 hi = __half22float2(*reinterpret_cast<const __half2 *>(&u.y));
    return make_float4(lo.x, lo.y, hi.x, hi.y);
}
// elements [4c, 4c + 8) of a row, c even (the shared-memory K tiles of decode_mega.cu: the row is 16-byte aligned)
__device__ __forceinline__ void kv_load8(const float *row, const int c, float4 &a, float4 &b) {
    a = reinterpret_cast<const float4 *>(row)[c];
    b = reinterpret_cast<const float4 *>(row)[c + 1];
}
__device__ __forceinline__ void kv_load8(const __half *row, const int c, float4 &a, float4 &b) {
    const uint4 u = reinterpret_cast<const uint4 *>(row)[c >> 1];
    const float2 f0 = __half22float2(*reinterpret_cast<const __half2 *>(&u.x));
    const float2 f1 = __half22float2(*reinterpret_cast<const __half2 *>(&u.y));
    const float2 f2 = __half22float2(*reinterpret_cast<const __half2 *>(&u.z));
    const float2 f3 = __half22float2(*reinterpret_cast<const __half2 *>(&u.w));
    a = make_float4(f0.x, f0.y, f1.x, f1.y);
    b = make_float4(f2.x, f2.y, f3.x, f3.y);
}
// ---- Q8: position j of (row b, kv head kvh) in a pool of (page, kv head) units (kv_unit_bytes): its hd values and
// its hd / 16 scales
struct KvQ8Row {
    int8_t *q;
    __half *d;
};
// row r of unit u = phys * Hkv + kv head
__device__ __forceinline__ KvQ8Row kv_q8_at(int8_t *pool, const size_t u, const int r, const int hd) {
    int8_t *unit = pool + u * kv_unit_bytes(KvType::Q8, hd);
    return KvQ8Row{unit + (size_t)r * hd, reinterpret_cast<__half *>(unit + (size_t)KV_PAGE * hd) + r * (hd / KV_Q8_BLOCK)};
}
template <bool RING = false>
__device__ __forceinline__ KvQ8Row kv_q8_row(int8_t *pool, const KvView &kv, const int b, const int Hkv, const int kvh, const int j,
                                             const int hd) {
    const int lp = j / KV_PAGE;
    const int phys = kv.page_table[(size_t)b * kv.max_pages + (RING ? lp % kv.max_pages : lp)];
    return kv_q8_at(pool, (size_t)phys * Hkv + kvh, j % KV_PAGE, hd);
}
// |x| as bits: ordered like the magnitudes, and any NaN compares above +inf (0x7f800000), so an integer max over a block
// is its absmax with NaN propagated
__device__ __forceinline__ unsigned kv_q8_abits(const float x) { return __float_as_uint(x) & 0x7fffffffu; }
__device__ __forceinline__ unsigned kv_q8_abits4(const float4 x) {
    return max(max(kv_q8_abits(x.x), kv_q8_abits(x.y)), max(kv_q8_abits(x.z), kv_q8_abits(x.w)));
}
// the block's scale from its absmax bits: f16_rn(min(a / 127, 65504)) (IEEE f32 division), NaN for a NaN block
__device__ __forceinline__ __half kv_q8_scale(const unsigned abits) {
    const float a = __uint_as_float(abits);
    return abits > 0x7f800000u ? __float2half_rn(a) : __float2half_rn(fminf(a / 127.0f, 65504.0f));
}
// q = clamp(rint(x / d), -127, 127); 0 when d is 0 or NaN
__device__ __forceinline__ int kv_q8_quant(const float x, const float d) {
    if (!(d > 0.0f)) return 0;
    return (int)fminf(fmaxf(rintf(x / d), -127.0f), 127.0f);
}
// four quantised values of scale d packed as the 4 bytes they are stored in
__device__ __forceinline__ uint32_t kv_q8_pack4(const float4 x, const float d) {
    return (uint32_t)(kv_q8_quant(x.x, d) & 0xff) | (uint32_t)(kv_q8_quant(x.y, d) & 0xff) << 8 |
           (uint32_t)(kv_q8_quant(x.z, d) & 0xff) << 16 | (uint32_t)(kv_q8_quant(x.w, d) & 0xff) << 24;
}
// stores one whole block x[0..16) at q (16-byte aligned) and its scale at *d
__device__ __forceinline__ void kv_q8_store16(int8_t *q, __half *d, const float *x) {
    unsigned ab = 0;
#pragma unroll
    for (int i = 0; i < KV_Q8_BLOCK; ++i) ab = max(ab, kv_q8_abits(x[i]));
    const __half dh = kv_q8_scale(ab);
    const float df = __half2float(dh);
    uint4 u;
    u.x = kv_q8_pack4(make_float4(x[0], x[1], x[2], x[3]), df);
    u.y = kv_q8_pack4(make_float4(x[4], x[5], x[6], x[7]), df);
    u.z = kv_q8_pack4(make_float4(x[8], x[9], x[10], x[11]), df);
    u.w = kv_q8_pack4(make_float4(x[12], x[13], x[14], x[15]), df);
    *reinterpret_cast<uint4 *>(q) = u;
    *d = dh;
}
// decoded value: (float)d * q, exact in f32
__device__ __forceinline__ float kv_q8_load(const int8_t q, const float d) { return d * (float)q; }
// four decoded values from their 4 stored bytes
__device__ __forceinline__ float4 kv_q8_load4(const uint32_t u, const float d) {
    return make_float4(d * (float)(int8_t)(u & 0xff), d * (float)(int8_t)((u >> 8) & 0xff), d * (float)(int8_t)((u >> 16) & 0xff),
                       d * (float)(int8_t)(u >> 24));
}
#endif
// Decoder RoPE tables as the kernels read them: cos / sin [rows][hd/2], position p at row p -- or, for a ring KvView, at
// row p % rows of an unbounded pool's small ring tables, whose rows the host fills for the positions of each launch.
struct RopeView {
    const float *cos_t = nullptr, *sin_t = nullptr;
    int rows = 0;
};
// single-token decoder attention fused with RoPE + KV append (decode_attn.cu); qkv rows [B][ld]
bool dec_attn_fused_supported(int H, int Hkv, int hd);
void launch_dec_attn_fused(float *qkv, int B, int ld, int H, int Hkv, int hd, const KvView &kv, int window, float scale,
                           const RopeView &rope, float *out, cudaStream_t st);
// y[M,N] = A[M,K] . W^T for any M (encoder / prefill): tiled SIMT GEMM, in-tile dequant.
void launch_q4_gemm(const Q4Weight &w, const float *a, int M, float *y, int ldy, const float *bias,
                    const float *res, int epi, cudaStream_t st);
// wgmma path (gemm_tc5.cu): X is first split into two f16 pieces laid out as wgmma operand tiles
// (optionally through RMSNorm), then Y = X . W^T with f32-grade accuracy on the tensor cores.
bool gemm_tc5_supported(const Q4Weight &w, int M);
size_t gemm_tc5_split_elems(int M, int K);  // f16 elements needed for the split buffer
void launch_split_tiles(const float *x, int M, int K, const float *gamma, float eps, void *xt, cudaStream_t st,
                        const AdaRows &ada_rows = AdaRows{});
// Caller-owned scratch for the GEMM's stream-K schedule: partial sums of tiles split across CTAs, summed in a fixed order
struct GemmWork {
    float *partial = nullptr;  // [2 per CTA][tokens of the tile][128 features]
    size_t partial_floats = 0;
    int *counters = nullptr;   // [n_counters] zero between launches
    int n_counters = 0;
};
void launch_q4_gemm_tc5(const Q4Weight &w, const void *xt, int M, float *y, int ldy, const float *bias, const float *res,
                        int epi, const GemmWork *gw, cudaStream_t st);
// GemmWork sizes launch_q4_gemm_tc5 needs (it refuses less), for any shape; pointers left to the caller
GemmWork gemm_tc5_work_size();

// Which Q4 kernels a caller lets launch_q4_linear choose: the tensor-core matvec for M <= 8 (else the SIMT matvec) and
// the wgmma GEMM for M > 8 (else the SIMT GEMM).
struct Q4Path {
    bool matvec_tc = true;
    bool gemm_tc = true;
};
// Caller-owned scratch of launch_q4_linear.
struct Q4Scratch {
    void *xt = nullptr;             // split tiles of the wgmma GEMM
    size_t xt_elems = 0;            // capacity of xt; M > 8 rows needing more (gemm_tc5_split_elems) take the SIMT GEMM
    const GemmWork *gw = nullptr;   // split tiles of the wgmma GEMM (required when xt is given)
    const TcWork *tc = nullptr;     // split-K and fused-norm sums of squares of the tensor-core matvec (null: neither)
};
// y = epi(norm(x) . W^T + bias) (+res) for any M: the one place that picks the Q4 kernel of a linear layer.
// gamma (optional) selects the RMSNorm (+ per-row ADA scale `ada_rows`) of the input.  It is fused into the wgmma
// GEMM's operand split, or into the tensor-core matvec when sc.tc carries ssq_in; otherwise it runs as launch_rmsnorm
// into `tmp` ([M][K]) ahead of the matvec / SIMT GEMM.
void launch_q4_linear(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias, const float *res,
                      int epi, const float *gamma, float eps, float *tmp, const Q4Scratch &sc, const Q4Path &path,
                      cudaStream_t st, const AdaRows &ada_rows = AdaRows{});
// conv1 / conv2 as implicit GEMM: in [B][T_in][C_in] time-major, W [C_out][3*C_in] (k = tap*C_in + c),
// stride 2, pad 1, + bias, GELU -> out [B][T_out][C_out].
// t_off (B == 1 only): compute conv outputs t_off .. t_off+T_out-1 into out[0..T_out) -- the incremental form used by
// the streaming session; input rows outside [0, T_in) are the zero padding.  in0 (B == 1 only): absolute input row of
// in[0] (a streaming buffer that has slid past the start of the signal); T_in stays the absolute input length.
void launch_conv2_gemm(const float *in, const float *w, const float *bias, float *out, int B, int T_in,
                       int T_out, int C_in, int C_out, cudaStream_t st, int t_off = 0, int in0 = 0);
// [B][C][T] -> [B][T][C]
void launch_transpose_mel(const float *in, float *out, int B, int C, int T, cudaStream_t st);
// y = x / sqrt(mean(x^2)+eps) * gamma (* ada_rows.row(r), the optional per-row ADA vector)
void launch_rmsnorm(const float *x, const float *gamma, float *y, int rows, int dim, float eps, cudaStream_t st,
                    const AdaRows &ada_rows = AdaRows{});
// in-place interleaved-pair RoPE on q (n_q heads) and k (n_k heads) inside a fused row buffer;
// row r has position pos0 + (r % seq).  cos/sin: [max_pos][hd/2].
// seg (device, optional): rows of streams of different lengths packed one after the other, stream s's rows
// [seg[s], seg[s+1]) for s < n_seg; row r then has position pos0 + r - (start of its stream), and seq is unused.
void launch_rope_inplace(float *buf, int rows, int ld, int q_off, int n_q, int k_off, int n_k, int hd,
                         int seq, int pos0, const float *cos_t, const float *sin_t, cudaStream_t st,
                         const int *seg = nullptr, int n_seg = 0);
// encoder attention: causal + sliding window (|i-j| <= window), per (batch, head); qkv rows
// [B*S][ld] with q at q_off, k at k_off, v at v_off; out [B*S][H*hd].
// seg (device, optional): stream b's rows are [seg[b], seg[b+1]) of qkv and out instead of [b*S, (b+1)*S), and S is the
// longest stream's length; a stream's band never reaches into another stream's rows.
void launch_enc_attention(const float *qkv, float *out, int B, int S, int H, int hd, int ld, int q_off,
                          int k_off, int v_off, int window, float scale, cudaStream_t st, const int *seg = nullptr);
// same contract on the tensor cores (enc_attn_tc.cu): mma.sync with two-piece f16 operands, each operand scaled by a
// power of two first (Q per row, K per key tile, V by the running tile maximum, P by 2^15), so 22-bit pieces at any
// overall operand scale (relative to the largest element of the row, tile or block: enc_attn_tc.cu); hd 32 or 64,
// ld and the offsets multiples of 4, qkv 16-byte aligned
bool enc_attention_tc_supported(int hd, int ld, int q_off, int k_off, int v_off);
void launch_enc_attention_tc(const float *qkv, float *out, int B, int S, int H, int hd, int ld, int q_off,
                             int k_off, int v_off, int window, float scale, cudaStream_t st, const int *seg = nullptr);
// decoder: RoPE q in place, RoPE k -> Kcache, v -> Vcache at positions kv.pos[b] + i.
// qkv rows [B*M][ld].
void launch_dec_rope_append(float *qkv, int B, int M, int ld, int H, int Hkv, int hd, const KvView &kv,
                            const RopeView &rope, cudaStream_t st);
// decoder GQA attention over the cache (keys 0..kv.pos[b]+i, window), out [B*M][H*hd].  dec_attention_check throws
// what launch_dec_attention refuses (shared memory, head_dim, a ring that cannot hold window + M positions), so a caller
// can refuse before it launches dec_rope_append.
void dec_attention_check(int M, int H, int Hkv, int hd, const KvView &kv, int window);
void launch_dec_attention(const float *qkv, int B, int M, int ld, int H, int Hkv, int hd, const KvView &kv, int window,
                          float scale, float *out, cudaStream_t st);
// x[r][:] = audio[audio_off[b] + (pos[b] + i)*K ..] + dequant(E[ids[r]]),  r = b*M + i; without audio (nullptr) the
// embedding alone.  audio_off [B]: element offset of row b's stream's position 0, signed (an unbounded stream pool's
// buffer slides past it).
// ssq_out (optional): [K/16][B*M] per-16-element sums of squares of the written rows (TcWork::ssq_in)
void launch_embed(const Q4Weight &emb, const int *ids, const float *audio, const int64_t *audio_off, int B, int M,
                  const int *pos, float *x, float *ssq_out, cudaStream_t st);
// greedy argmax (lowest index wins ties) over logits [B][V]; writes tok[b] and, if out_ids,
// out_ids[b*out_ld + out_pos[b]]
void launch_argmax(const float *logits, int B, int V, int *tok, int *out_ids, int out_ld,
                   const int *out_pos_ptr, cudaStream_t st);
// multi-CTA variant: ARGMAX_PARTS CTAs per row, last one to arrive (atomic ticket) reduces the partial
// results in fixed order; scratch: vals/idx [B][ARGMAX_PARTS], counters [B] zero between launches
constexpr int ARGMAX_PARTS = 64;
void launch_argmax_multi(const float *logits, int B, int V, int *tok, int *out_ids, int out_ld,
                         const int *out_pos_ptr, float *scratch_vals, int *scratch_idx, int *counters,
                         cudaStream_t st);
// Token confidences (vox_session_set_top_k): per row b, the k most likely ids of logits [B][V] (descending logit, the
// lower id first on equal logits -- so ids[0] is the greedy argmax) and their log-probabilities logit - logsumexp(row),
// in f32 at temperature 1.  ARGMAX_PARTS CTAs per row; the last to arrive (atomic ticket) merges the partial
// (max, sum of exp) pairs and top-k lists in fixed order, so the result is bitwise reproducible.  Row b's result goes to
// position out_pos[b] - 1 (the argmax and the step counters have run): ids / logprobs [B][out_ld][TOPK_MAX], entries
// [0, k).  scratch: m/l [B][ARGMAX_PARTS], vals/idx [B][ARGMAX_PARTS][TOPK_MAX], counters [B] zero between launches.
constexpr int TOPK_MAX = 8;   // VOX_MAX_TOP_K
struct ScoreWork {
    float *m = nullptr, *l = nullptr, *vals = nullptr;
    int *idx = nullptr, *counters = nullptr;
};
void launch_token_scores(const float *logits, int B, int V, int k, const int *out_pos_ptr, int out_ld, int *top_ids,
                         float *top_logprobs, const ScoreWork &w, cudaStream_t st);
// Beam search (vox_session_set_beam, beam.cu): the W beams of stream s (of b) run as rows w * b + s of the decode step.
// After each step (token scores at k >= W have run), launch_beam_select takes, per stream, the W best of the candidates
// (live rank j, one of its row's top-W ids) by score cum[j] + (double)logprob descending, then parent rank ascending,
// then id ascending; writes the new ranks' rows, cum and d_tok, and each row's (token, parent row) at its output
// position out_pos - 1.  The first child of a surviving parent keeps the parent's row; the other children take the rows
// of the ranks without children.  launch_beam_fork then gives every row whose parent row q differs from itself q's
// page-table entries of the full pages below its next write position and a copy of the filled part of q's current page.
// launch_beam_traceback walks the parent rows back from the last position: ids [b][W][n] and scores [b][W] in rank
// order; rank 0's ids into out rows [0, b); with top_ids (non-null), rank 0's token scores gathered into rows [0, b).
// s0 / out_stride: the launch walks streams s0 .. s0 + b - 1 (ids relative to stream s0, scores absolute) and writes
// stream s's rank-0 ids and scores into row s * out_stride -- the stream's first beam row when its beams are rows
// s * W .. s * W + W - 1 (streams of different lengths, one launch per output length).
constexpr int BEAM_MAX = 8;   // VOX_MAX_BEAM (the top-k list holds the W candidates of a row: BEAM_MAX <= TOPK_MAX)
struct BeamWork {
    int *rank_row = nullptr;                        // [b][W] row holding each rank
    double *cum = nullptr;                          // [b][W] summed log-probability of each rank
    int *src = nullptr;                             // [rows] parent row of each row's beam (== row: nothing to fork)
    int *hist_tok = nullptr, *hist_par = nullptr;   // [rows][out_ld] token and parent row per output position
};
void launch_beam_select(const int *top_ids, const float *top_lp, const int *out_pos, int out_ld, int b, int W, int n_live,
                        const BeamWork &w, int *tok, cudaStream_t st);
// kc / vc: KV page pools of element type `type`, layer_bytes bytes per layer
void launch_beam_fork(void *kc, void *vc, KvType type, size_t layer_bytes, int layers, int *page_table, int max_pages,
                      const int *pos, const int *src, int rows, int Hkv, int hd, cudaStream_t st);
void launch_beam_traceback(const BeamWork &w, int b, int W, int n, int out_ld, int *ids, double *scores, int *out,
                           int *top_ids, float *top_lp, cudaStream_t st, int s0 = 0, int out_stride = 1);
// Phrase boosting (vox_session_set_bias, bias.cu).  Stream s's list: n_phrases[s] phrases, phrase i of lens[...] ids at
// ids + (s * BIAS_MAX_PHRASES + i) * BIAS_MAX_LEN with boost boosts[s * BIAS_MAX_PHRASES + i]; its history: the last
// hist[s][BIAS_HIST] (<= BIAS_HIST) text ids it emitted, oldest first, in hist[s][0..).  Every stream's list sits at a
// fixed offset, so a captured step reads whatever list is set when it replays.
constexpr int BIAS_MAX_PHRASES = 256;   // VOX_MAX_BIAS_PHRASES
constexpr int BIAS_MAX_LEN = 16;        // VOX_MAX_BIAS_LEN
constexpr int BIAS_FIRST_TEXT_ID = 1000;   // VOX_FIRST_TEXT_ID: lower ids never enter a history
constexpr int BIAS_HIST = BIAS_MAX_LEN - 1;   // a phrase's longest matched prefix
struct BiasLists {
    int *ids = nullptr;        // [streams][BIAS_MAX_PHRASES][BIAS_MAX_LEN]
    int *lens = nullptr;       // [streams][BIAS_MAX_PHRASES]
    float *boosts = nullptr;   // [streams][BIAS_MAX_PHRASES]
    int *n_phrases = nullptr;  // [streams]
    int *hist = nullptr;       // [streams][BIAS_HIST + 1]: ids, then their count
};
// After the step's argmax and counter advance, per row r of stream row_stream[r] with a non-empty list: the argmax of
// fl32(logit(t) + boost(t)) (lowest id on ties) over the greedy id tok[r] and the ids the list offers after the stream's
// history, into tok[r] and out_ids[r * out_ld + out_pos[r] - 1]; a winner >= BIAS_FIRST_TEXT_ID joins the history.
// One CTA per row; a row whose stream has no list leaves at once.
void launch_bias_select(const float *logits, int B, int V, const int *row_stream, const BiasLists &lists, int *tok, int *out_ids,
                        int out_ld, const int *out_pos, cudaStream_t st);
// a[i] += da; b[i] += db for i < n  (device-side per-row step counters for graph replay)
void launch_advance(int *a, int da, int *b, int db, int n, cudaStream_t st);
// gather rows: dst[b][:] = src[b*M + (M-1)][:]
void launch_gather_last(const float *src, float *dst, int B, int M, int dim, cudaStream_t st);
// reshape_encoder_output is a pure view when S % factor == 0; otherwise rows are re-packed
void launch_reshape_rows(const float *src, float *dst, int B, int S, int S_out, int dim, int factor,
                         cudaStream_t st);
// out[i] = a[i] * b[i]
void launch_mul_vec(const float *a, const float *b, float *out, size_t n, cudaStream_t st);

// mel: samples [B][n] device -> log-mel; layout 0 [B][frames][128], 1 [B][128][frames]
// frames [frame0, frames) are computed.  B == 1 streaming buffers that slide: samples[0] is absolute sample sample0 (a
// multiple of 4 keeps the aligned interior path) and out row 0 is absolute frame out0; n stays the absolute length.
void launch_mel(const float *samples, int B, size_t n, size_t sample_stride, const float *window,
                const float *fb_vals, const int *fb_start, const int *fb_len, int fb_stride, float *out,
                int frames, int layout, cudaStream_t st, int frame0 = 0, size_t sample0 = 0, int out0 = 0);
// peak normalisation on device: per stream max|x| then scale (target/max), skip if max < 1e-10;
// writes into a padded buffer at offset left (rest pre-zeroed by caller)
void launch_peak_normalize_pad(const float *in, int B, size_t n, float target, int do_norm, float *out,
                               size_t out_stride, size_t left, float *scale_buf, cudaStream_t st);

uint64_t kernel_launch_count();
// kernels executed through CUDA-graph replays (or, negative, captured-not-executed launches)
void add_graph_launches(int64_t n);

}  // namespace vox
