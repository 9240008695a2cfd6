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
    size_t bytes() const { return (size_t)N * (K / 32) * 18; }
};

enum Epi : int {
    EPI_NONE = 0,      // y = acc (+bias)
    EPI_RESIDUAL = 1,  // y = res + acc (+bias)     (y may alias res)
    EPI_SILU_MUL = 2,  // rows (2i,2i+1) = (gate_i, up_i): y[:, i] = silu(gate) * up, ldy = N/2
    EPI_GELU = 3,      // y = gelu_erf(acc + bias)
};

// y[M,N] = x[M,K] . W^T, M <= 8 (decode / batched decode): warp-per-row-pair, shuffle reduce.
void launch_q4_matvec(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                      const float *res, int epi, cudaStream_t st);
// same contract, dequant arithmetic on the tensor cores (mma.sync, f16 subnormal nibbles); needs the
// TC layout (w.qs_tc).  matvec_tc.cu
void launch_q4_matvec_tc(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                         const float *res, int epi, cudaStream_t st);
// Session-owned scratch for the tensor-core matvec: split-K partial sums + tickets, and the per-tile
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
void launch_q4_matvec_tc_ex(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                            const float *res, int epi, const float *gamma, const float *ada, float eps,
                            const TcWork *wk, cudaStream_t st);
// ... with the RMSNorm (+ optional ADA scale) of the input fused into the staging pass:
// x := ((x / sqrt(mean(x^2)+eps)) * gamma) * ada
void launch_q4_matvec_tc_norm(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                              const float *res, int epi, const float *gamma, const float *ada, float eps,
                              cudaStream_t st);
// Decoder KV cache of ONE layer as the attention kernels see it: PAGED (KVCache semantics of kv_cache.rs:52-142 --
// append at the stream's position, read keys 0..pos -- over fixed-size pages so that sessions of different ages
// share one pool).  Batch row b owns logical pages page_table[b][0..max_pages); logical position j lives at
//   pool + ((phys(b, j / KV_PAGE) * Hkv + kv_head) * KV_PAGE + j % KV_PAGE) * hd.
// Positions are per row (pos[b] = number of cached positions of row b = position of its next token): whole-utterance
// batches keep them equal, streaming sessions do not.
constexpr int KV_PAGE = 16;
struct KvView {
    float *k = nullptr, *v = nullptr;  // [n_pages][Hkv][KV_PAGE][hd]
    const int *page_table = nullptr;   // [B][max_pages] physical page ids
    int max_pages = 0;                 // logical pages per row; capacity = max_pages * KV_PAGE positions
    const int *pos = nullptr;          // [B]
    __host__ __device__ int max_seq() const { return max_pages * KV_PAGE; }
};
#ifdef __CUDACC__
__device__ __forceinline__ size_t kv_index(const KvView &kv, const int b, const int Hkv, const int kvh, const int j, const int hd) {
    const int phys = kv.page_table[(size_t)b * kv.max_pages + (j / KV_PAGE)];
    return (((size_t)phys * Hkv + kvh) * KV_PAGE + (j % KV_PAGE)) * hd;
}
#endif
// single-token decoder attention fused with RoPE + KV append (decode_attn.cu); qkv rows [B][ld]
bool dec_attn_fused_supported(int H, int Hkv, int hd);
void launch_dec_attn_fused(float *qkv, int B, int ld, int H, int Hkv, int hd, const KvView &kv, int window, float scale,
                           const float *cos_t, const float *sin_t, float *out, cudaStream_t st);
// y[M,N] = A[M,K] . W^T for any M (encoder / prefill): tiled SIMT GEMM, in-tile dequant.
void launch_q4_gemm(const Q4Weight &w, const float *a, int M, float *y, int ldy, const float *bias,
                    const float *res, int epi, cudaStream_t st);
// wgmma path (gemm_tc5.cu): X is first split into two f16 pieces laid out as wgmma operand tiles
// (optionally through RMSNorm), then Y = X . W^T with f32-grade accuracy on the tensor cores.
bool gemm_tc5_supported(const Q4Weight &w, int M);
size_t gemm_tc5_split_elems(int M, int K);  // f16 elements needed for the split buffer
void launch_split_tiles(const float *x, int M, int K, const float *gamma, const float *ada, float eps, void *xt,
                        cudaStream_t st);
// Caller-owned scratch for the GEMM's deterministic split-K (used when N/128 x M/128 tiles cannot fill the GPU)
struct GemmWork {
    float *partial = nullptr;  // [slices][tiles][128][128]
    size_t partial_floats = 0;
    int *counters = nullptr;   // [n_counters] zero between launches
    int n_counters = 0;
};
void launch_q4_gemm_tc5(const Q4Weight &w, const void *xt, int M, float *y, int ldy, const float *bias, const float *res,
                        int epi, const GemmWork *gw, cudaStream_t st);
// conv1 / conv2 as implicit GEMM: in [B][T_in][C_in] time-major, W [C_out][3*C_in] (k = tap*C_in + c),
// stride 2, pad 1, + bias, GELU -> out [B][T_out][C_out].
// t_off (B == 1 only): compute conv outputs t_off .. t_off+T_out-1 into out[0..T_out) -- the incremental form used by
// the streaming session; input rows outside [0, T_in) are the zero padding.
void launch_conv2_gemm(const float *in, const float *w, const float *bias, float *out, int B, int T_in,
                       int T_out, int C_in, int C_out, cudaStream_t st, int t_off = 0);
// [B][C][T] -> [B][T][C]
void launch_transpose_mel(const float *in, float *out, int B, int C, int T, cudaStream_t st);
// y = x / sqrt(mean(x^2)+eps) * gamma (* scale, optional ADA vector)
void launch_rmsnorm(const float *x, const float *gamma, const float *scale, float *y, int rows, int dim,
                    float eps, cudaStream_t st);
// in-place interleaved-pair RoPE on q (n_q heads) and k (n_k heads) inside a fused row buffer;
// row r has position pos0 + (r % seq).  cos/sin: [max_pos][hd/2].
void launch_rope_inplace(float *buf, int rows, int ld, int q_off, int n_q, int k_off, int n_k, int hd,
                         int seq, int pos0, const float *cos_t, const float *sin_t, cudaStream_t st);
// encoder attention: causal + sliding window (|i-j| <= window), per (batch, head); qkv rows
// [B*S][ld] with q at q_off, k at k_off, v at v_off; out [B*S][H*hd].
void launch_enc_attention(const float *qkv, float *out, int B, int S, int H, int hd, int ld, int q_off,
                          int k_off, int v_off, int window, float scale, cudaStream_t st);
// same contract on the tensor cores (enc_attn_tc.cu): mma.sync with two-piece f16 operands, f32-grade accuracy
bool enc_attention_tc_supported(int hd, int ld, int q_off, int k_off, int v_off);
void launch_enc_attention_tc(const float *qkv, float *out, int B, int S, int H, int hd, int ld, int q_off,
                             int k_off, int v_off, int window, float scale, cudaStream_t st);
// decoder: RoPE q in place, RoPE k -> Kcache, v -> Vcache at positions kv.pos[b] + i.
// qkv rows [B*M][ld].
void launch_dec_rope_append(float *qkv, int B, int M, int ld, int H, int Hkv, int hd, const KvView &kv,
                            const float *cos_t, const float *sin_t, cudaStream_t st);
// decoder GQA attention over the cache (keys 0..kv.pos[b]+i, window), out [B*M][H*hd].
void launch_dec_attention(const float *qkv, int B, int M, int ld, int H, int Hkv, int hd, const KvView &kv, int window,
                          float scale, float *out, cudaStream_t st);
// x[r][:] = audio_row(b, pos[b] + i) + dequant(E[ids[r]]),  r = b*M + i; the audio row is audio_rows[b] + i*K when the
// pointer table is given (streaming sessions: one pointer per row), else audio + (b*audio_seq + pos[b] + i)*K, else 0
// (pos == nullptr: position 0).
// ssq_out (optional): [K/16][B*M] per-16-element sums of squares of the written rows (TcWork::ssq_in)
void launch_embed(const Q4Weight &emb, const int *ids, const float *audio, int audio_seq, int B, int M,
                  const int *pos, float *x, float *ssq_out, cudaStream_t st, const float *const *audio_rows = nullptr);
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
// a[i] += da; b[i] += db for i < n  (device-side per-row step counters for graph replay)
void launch_advance(int *a, int da, int *b, int db, int n, cudaStream_t st);
// gather rows: dst[b][:] = src[b*M + (M-1)][:]
void launch_gather_last(const float *src, float *dst, int B, int M, int dim, cudaStream_t st);
// reshape_encoder_output is a pure view when S % factor == 0; otherwise rows are re-packed
void launch_reshape_rows(const float *src, float *dst, int B, int S, int S_out, int dim, int factor,
                         cudaStream_t st);
// out[i] = a[i] * b[i]
void launch_mul_vec(const float *a, const float *b, float *out, size_t n, cudaStream_t st);
// GELU in place
void launch_gelu(float *x, size_t n, cudaStream_t st);

// mel: samples [B][n] device -> log-mel; layout 0 [B][frames][128], 1 [B][128][frames]
void launch_mel(const float *samples, int B, size_t n, size_t sample_stride, const float *window,
                const float *fb_vals, const int *fb_start, const int *fb_len, int fb_stride, float *out,
                int frames, int layout, cudaStream_t st, int frame0 = 0);  // frames [frame0, frames) are computed
// peak normalisation on device: per stream max|x| then scale (target/max), skip if max < 1e-10;
// writes into a padded buffer at offset left (rest pre-zeroed by caller)
void launch_peak_normalize_pad(const float *in, int B, size_t n, float target, int do_norm, float *out,
                               size_t out_stride, size_t left, float *scale_buf, cudaStream_t st);

uint64_t kernel_launch_count();
// kernels executed through CUDA-graph replays (or, negative, captured-not-executed launches)
void add_graph_launches(int64_t n);

}  // namespace vox
