/* voxtral.h -- C ABI of libvoxtral_b200.so
 *
 * H100-native (sm_90a) replacement for the Q4_0 GGUF hot path of
 * TrevorS/voxtral-mini-realtime-rs.  The reference exposes no C FFI; its seams are the Rust
 * functions cited beside each entry point below (paths relative to the reference repo).  A Rust
 * `extern "C"` binding for this header is shown in INTEGRATION.md.
 *
 * Conventions
 *   - every function returns int32 status: VOX_OK (0) or a VOX_E* code; vox_last_error() returns a
 *     thread-local message for the last failure on the calling thread.  No exceptions or panics
 *     cross the boundary (the reference panics via expect()/assert_eq!, src/gguf/op.rs:92-100,166).
 *   - handles are opaque; plain pointers + sizes only; pointers are HOST memory unless the
 *     parameter name ends in `_dev`.  `stream` parameters are `cudaStream_t` passed as void*
 *     (NULL = the handle's own stream).
 *   - thread-compatibility: one thread per handle at a time; different sessions may run
 *     concurrently (they own their stream, KV cache and workspace).
 *   - there is NO CPU fallback: every compute entry point fails with VOX_ECUDA if no sm_90
 *     device / driver is available.
 */
#ifndef VOXTRAL_H
#define VOXTRAL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VOX_OK 0
#define VOX_EINVAL 1    /* bad argument / shape mismatch          */
#define VOX_EIO 2       /* file / parse error                     */
#define VOX_ENOTFOUND 3 /* tensor or key not found                */
#define VOX_ECUDA 4     /* CUDA runtime / launch / no device      */
#define VOX_ENOMEM 5
#define VOX_EFORMAT 6   /* unsupported dtype / version            */
#define VOX_ECAPACITY 7 /* caller buffer too small                */

#define VOX_DTYPE_F32 0 /* GgmlDtype, src/gguf/reader.rs:18-49 */
#define VOX_DTYPE_F16 1
#define VOX_DTYPE_Q4_0 2
/* decoder KV cache only (vox_session_create_ex): int8 with an f16 scale per 16 head dims.  Outside GGML's type table,
 * so it never collides with a vox_gguf_tensor_info code (GGUF's Q8_0, type 8, has blocks of 32 and rounds differently). */
#define VOX_DTYPE_KV_Q8 100

const char *vox_last_error(void);
int32_t vox_version(void);
/* number of visible CUDA devices (0 if none / no driver) */
int32_t vox_device_count(void);

/* ------------------------------------------------------------------ GGUF reader
 * GgufReader + ShardedCursor, src/gguf/reader.rs:88-314 */
typedef struct vox_gguf vox_gguf;
int32_t vox_gguf_open(const char *path, vox_gguf **out);                       /* Q4ModelLoader::from_file loader.rs:82 */
int32_t vox_gguf_open_shards(const void *const *bufs, const size_t *lens, size_t n_shards,
                             vox_gguf **out);                                    /* from_bytes / from_shards loader.rs:92,101; buffers are borrowed */
int32_t vox_gguf_version(const vox_gguf *g, uint32_t *version);                /* reader.rs:191 */
int32_t vox_gguf_tensor_count(const vox_gguf *g, uint64_t *count);             /* reader.rs:196 */
int32_t vox_gguf_tensor_name(const vox_gguf *g, uint64_t index, const char **name); /* tensor_names reader.rs:206 */
int32_t vox_gguf_tensor_info(const vox_gguf *g, const char *name, uint32_t *dtype, uint32_t *ndim,
                             uint64_t dims[4] /* GGUF order, as stored */, uint64_t *nbytes); /* reader.rs:201 */
int32_t vox_gguf_tensor_data(vox_gguf *g, const char *name, void *dst, size_t cap); /* reader.rs:211-223 */
void vox_gguf_close(vox_gguf *g);

/* ------------------------------------------------------------------ audio plumbing (host) */
int32_t vox_peak_normalize(float *samples, size_t n, float target_peak);       /* AudioBuffer::peak_normalize io.rs:59-68 */
typedef struct {
    uint32_t sample_rate;            /* 16000 */
    uint32_t n_left_pad_tokens;      /* 76    */
    float frame_rate;                /* 12.5  */
    uint32_t extra_right_pad_tokens; /* 17    */
} vox_pad_config;                    /* PadConfig pad.rs:20-46 */
void vox_pad_config_default(vox_pad_config *cfg);
size_t vox_pad_audio_len(size_t n, const vox_pad_config *cfg /* NULL = default */);
int32_t vox_pad_audio(const float *in, size_t n, const vox_pad_config *cfg, float *out, size_t cap,
                      size_t *out_len);                                          /* pad_audio pad.rs:89-103 */
typedef struct {
    size_t start_sample, end_sample, index;
    int32_t is_last;
} vox_chunk;                                                                     /* AudioChunk chunk.rs:71-83 */
int32_t vox_chunk_plan(size_t n_samples, size_t max_mel_frames, size_t overlap_frames,
                       vox_chunk *out, size_t cap, size_t *n_chunks);            /* chunk_audio chunk.rs:122-166 */
int32_t vox_time_embedding(float t, int32_t dim, float *out);                    /* TimeEmbedding::embed time_embedding.rs:41-71 */
/* Streaming-session bookkeeping (SURVEY 8(f)-1; the incremental forms of mel.rs:175-182, conv.rs:47-48,
 * adapter.rs:115-121, model.rs:883-960): how far each stage can advance once `n_samples` samples of the PADDED
 * signal are known (`ended` != 0: the right padding is in, the stream is complete).  An output is counted only
 * when every input it reads is final, so the counts never have to be revised:
 * out[0] log-mel frames, out[1] conv1 frames, out[2] encoder frames, out[3] audio embeddings (decoder positions
 * with audio), out[4] token ids that can be emitted.  Checked against oracle/streaming.py. */
int32_t vox_stream_progress(size_t n_samples, int32_t ended, int32_t reshape_factor, int32_t prefix_len, int64_t out[5]);

/* ------------------------------------------------------------------ mel front-end (GPU)
 * MelSpectrogram::{new, num_frames, compute_log}, src/audio/mel.rs:73,175,128 */
typedef struct vox_mel vox_mel;
int32_t vox_mel_create(int32_t device, vox_mel **out);
size_t vox_mel_num_frames(size_t n_samples);
/* host in / host out, [frames][128] row-major like Vec<Vec<f32>> */
int32_t vox_mel_compute_log(vox_mel *mel, const float *samples, size_t n, float *out, size_t cap_floats);
/* device in / device out; layout 0 = [frames][128], 1 = [128][frames] (the [1,128,T] tensor the
 * callers build by transposing, transcribe.rs:295-305) */
int32_t vox_mel_compute_log_dev(vox_mel *mel, const float *samples_dev, size_t n, float *out_dev,
                                int32_t layout, void *stream);
int32_t vox_mel_filterbank(const vox_mel *mel, float *out /* [128][201] */);   /* create_mel_filterbank mel.rs:288-339 */
int32_t vox_mel_window(const vox_mel *mel, float *out /* [400] */);            /* hann_window mel.rs:345-349 */
void vox_mel_free(vox_mel *mel);

/* ------------------------------------------------------------------ Q4 operator seam
 * Q4Tensor (tensor.rs:16-113), Q4Linear (linear.rs:17-40), q4_matmul (op.rs:86-137) */
typedef struct vox_q4 vox_q4;
int32_t vox_q4_tensor_create(const uint8_t *q4_bytes, size_t nbytes, int64_t n, int64_t k,
                             int32_t device, vox_q4 **out);                      /* from_q4_bytes tensor.rs:35-71 */
int32_t vox_q4_tensor_shape(const vox_q4 *w, int64_t *n, int64_t *k);
int32_t vox_q4_tensor_dequantize(const vox_q4 *w, float *out /* [n*k] host */); /* dequantize tensor.rs:83-113 */
/* y[b,m,:] = x[b,m,:] . W^T (+ bias); x [B,M,K] contiguous f32, y [B,M,N]; async on `stream`.
 * A handle owns its split-K / operand-staging scratch: launches on ONE handle must be ordered (one stream, or
 * event-ordered streams) -- the call is not reentrant per handle; distinct handles are independent. */
int32_t vox_q4_matmul(const vox_q4 *w, const float *x_dev, float *y_dev, int32_t b, int32_t m,
                      const float *bias_dev /* nullable */, void *stream);
/* host-buffer convenience (H2D, kernel, D2H, sync) -- what benches/q4_ops.rs:76-91 times */
int32_t vox_q4_matmul_host(const vox_q4 *w, const float *x, float *y, int32_t b, int32_t m,
                           const float *bias /* nullable */);
/* One linear layer of the model in any of its fused forms, on the kernel vox_q4_set_matvec_mode selects:
 *   y[r,:] = epi(norm(x[r,:]) . W^T + bias) (+ res[r,:])
 * x [rows][K] contiguous f32 (must not overlap y); y and res rows are ldy floats apart; res may equal y (in place).
 * epi: VOX_EPI_* below.  SiLU*up reads output features (2i, 2i+1) as (gate_i, up_i) and writes N/2 columns.
 * gamma_dev (nullable) selects the RMSNorm x / sqrt(mean(x^2) + eps) * gamma; ada_dev (nullable, needs gamma) is a
 * device array of device pointers to K floats each: row r is further scaled by ada_dev[r / ada_m].  gamma and every
 * ADA vector must be 16-byte aligned.
 * ssq_in_dev (nullable, needs gamma): [ceil(K/16)][rows] partial sums of squares of x, each over 16 consecutive
 * elements, from which the tensor-core matvec takes the norm.  ssq_out_dev (nullable, residual only):
 * [ceil(N/16)][rows], written with the same partial sums of the new y rows.  Both need the tensor-core matvec
 * (rows <= 8, mode bit 0 clear).  Refused with VOX_EINVAL (vox_last_error says why): rows < 1, an unknown epi, a
 * residual without res or res with another epi, SiLU*up with an odd N, ldy < N/2 or a bias, any other epi with
 * ldy < N, ADA without gamma or ada_m < 1, ssq_in without gamma, ssq_out without a residual, and either ssq pointer
 * when the call would not run the tensor-core matvec.  The unfused norm goes through a [rows][K] scratch the handle
 * owns; same reentrancy rule as vox_q4_matmul. */
#define VOX_EPI_NONE 0
#define VOX_EPI_RESIDUAL 1
#define VOX_EPI_SILU_MUL 2
#define VOX_EPI_GELU 3
int32_t vox_q4_linear(const vox_q4 *w, const float *x_dev, float *y_dev, int32_t rows, int32_t ldy,
                      const float *bias_dev, const float *res_dev, int32_t epi, const float *gamma_dev, float eps,
                      const float *const *ada_dev, int32_t ada_m, const float *ssq_in_dev, float *ssq_out_dev,
                      void *stream);
void vox_q4_tensor_free(vox_q4 *w);

/* ------------------------------------------------------------------ attention operator seam
 * Encoder attention (model.rs:77-122, masking.rs:9-107): for every (stream, head), query i attends to key j iff
 * j <= i and i - j <= window, out = softmax(scale * q k^T) v.  All pointers are device pointers.
 *   VOX_ATTN_ENC_TC   K4-TC (enc_attn_tc.cu), the encoder's production kernel;
 *   VOX_ATTN_ENC_SIMT K4 (kernels.cu), its f32 SIMT cross-check;
 *   VOX_ATTN_STREAM   K4-S (stream.cu), the streaming pools' attention over per-session K/V rings.
 * Encoder kernels: stream t's rows are b * s + [0, s), or seg[t] .. seg[t + 1] - 1 when seg ([b + 1] ints) is given
 * (then s is the longest stream); row r's q, k and v of head hh start at qkv + r * ld + {q,k,v}_off + hh * hd, and its
 * output at out + r * h * hd + hh * hd.
 * Ring kernel: row r (r < rows) is query position row_pos[r] of session row_slot[r]; its q of head hh starts at
 * qkv + r * ld + hh * hd; key position p of that session is slot p % ring of k_ring / v_ring, [slots][ring][h * hd];
 * its output is out + r * h * hd + hh * hd.  The caller keeps every key a row can see in the ring.
 * The named kernel runs and no other.  Refused with VOX_EINVAL (vox_last_error says why): an unknown kernel, a null
 * pointer the kernel reads, b, s, rows or h below 1, a negative window, operands that do not fit in ld; K4-TC: hd not
 * 32 or 64, ld or an offset not a multiple of 4, qkv not 16-byte aligned; K4: hd not 32, 64 or 128; K4-S: hd not 32,
 * 64 or 128, ring < 1 or window >= ring. */
#define VOX_ATTN_ENC_TC 0
#define VOX_ATTN_ENC_SIMT 1
#define VOX_ATTN_STREAM 2
typedef struct vox_attn_args {
    const float *qkv;
    int32_t ld;
    int32_t q_off, k_off, v_off;          /* encoder kernels */
    int32_t b, s, h, hd;                  /* b and s: encoder kernels */
    const int32_t *seg;                   /* encoder kernels, nullable */
    int32_t rows;                         /* ring kernel */
    const int32_t *row_slot, *row_pos;    /* ring kernel, [rows] each */
    const float *k_ring, *v_ring;         /* ring kernel */
    int32_t ring;                         /* ring kernel */
    int32_t window;
    float scale;
    float *out;
} vox_attn_args;
int32_t vox_attention(int32_t device, int32_t kernel, const vox_attn_args *args, void *stream);

/* Decoder attention (model.rs:125-197, rope.rs:103-141, kv_cache.rs:116-142) over one layer's paged K/V cache.  Row
 * r = bb * m + i (bb < b, i < m) is position pos[bb] + i of stream bb; its q of head hh, k and v of kv head g start at
 * qkv + r * ld + hh * hd, + (h + g) * hd and + (h + hkv + g) * hd.  The call rotates q and k by the RoPE row of the
 * position (row p of cos / sin [rope_rows][hd / 2], or p % rope_rows for a ring), appends k after RoPE and v to the
 * cache at that position, and writes out + r * h * hd + hh * hd = softmax(scale q k^T) v over the keys
 * max(0, p - window) .. p of kv head hh / (h / hkv).  All pointers are device pointers.
 *   VOX_DEC_ATTN_FUSED   K5 (decode_attn.cu): one launch fused with RoPE and the append, m == 1; qkv is left unchanged;
 *   VOX_DEC_ATTN_PREFILL K5 prefill (kernels.cu): dec_rope_append, which rotates q in place, then dec_attention.
 * Cache: kv_dtype VOX_DTYPE_F32, VOX_DTYPE_F16 or VOX_DTYPE_KV_Q8, each value stored by the rule of
 * vox_session_create_ex.  k_pool / v_pool are [pages][hkv] units of 16 positions: [16][hd] values, and for q8 [16][hd]
 * int8 followed by [16][hd / 16] f16 scales.  Position p of stream bb is slot p % 16 of physical page
 * page_table[bb * max_pages + p / 16], or with ring != 0 page_table[bb * max_pages + (p / 16) % max_pages], so that
 * positions are unbounded.
 * The named kernel runs and no other.  Refused with VOX_EINVAL (vox_last_error says why), before any launch: an unknown
 * kernel or kv_dtype, a null pointer the kernel reads, b, m, h, hkv, hd, max_pages or rope_rows below 1, h % hkv != 0,
 * ld < (h + 2 hkv) hd, a negative window; fused: m != 1 or a shape it has no instantiation for (hd 32, 64 or 128,
 * h / hkv 1, 2 or 4), a ring with window >= 16 max_pages; prefill: hd not a multiple of 4 (16 for q8), shared memory
 * 4 (h / hkv) (hd + 16 max_pages) above 200 KB, a ring with window + m > 16 max_pages; without a ring, a negative
 * pos[bb] or pos[bb] + m above 16 max_pages or rope_rows (pos is downloaded to check). */
#define VOX_DEC_ATTN_FUSED 0
#define VOX_DEC_ATTN_PREFILL 1
typedef struct vox_dec_attn_args {
    float *qkv;                           /* [b * m][ld]; prefill rotates its q columns in place */
    int32_t ld;
    int32_t b, m, h, hkv, hd;
    int32_t kv_dtype;
    void *k_pool, *v_pool;
    const int32_t *page_table;            /* [b][max_pages] */
    int32_t max_pages;
    int32_t ring;
    const int32_t *pos;                   /* [b] */
    const float *cos, *sin;               /* [rope_rows][hd / 2] */
    int32_t rope_rows;
    int32_t window;
    float scale;
    float *out;                           /* [b * m][h * hd] */
} vox_dec_attn_args;
int32_t vox_dec_attention(int32_t device, int32_t kernel, const vox_dec_attn_args *args, void *stream);

/* kernel selection of the operator seam (bit mask, default 0): bit 0 = SIMT warp-reduce matvec instead of
 * the tensor-core-assisted one (M <= 8); bit 1 = SIMT tiled GEMM instead of the wgmma GEMM (M > 8).
 * All implement the same contract; exposed for A/B measurement and parity tests. */
int32_t vox_q4_set_matvec_mode(int32_t mode);

/* small device-memory helpers so that non-CUDA callers (ctypes, Rust) can drive the *_dev calls */
int32_t vox_dev_malloc(int32_t device, size_t bytes, void **ptr_dev);
int32_t vox_dev_free(int32_t device, void *ptr_dev);
int32_t vox_dev_upload(int32_t device, void *dst_dev, const void *src, size_t bytes);
int32_t vox_dev_download(int32_t device, void *dst, const void *src_dev, size_t bytes);
int32_t vox_dev_sync(int32_t device);
/* cudaProfilerStart/Stop, for `ncu --profile-from-start off` captures of a region */
int32_t vox_profiler_start(void);
int32_t vox_profiler_stop(void);
/* page-locked host memory for the end-to-end (host-buffer) path */
int32_t vox_host_alloc_pinned(size_t bytes, void **ptr);
int32_t vox_host_free_pinned(void *ptr);
/* CUDA-event timing of `iters` back-to-back vox_q4_matmul launches cycling over `n_weights`
 * tensors (L2-defeating rotation, SURVEY 8d); returns average ms per launch */
int32_t vox_q4_matmul_bench(const vox_q4 *const *weights, int32_t n_weights, int32_t m,
                            int32_t iters, int32_t warmup, float *avg_ms);

/* ------------------------------------------------------------------ model
 * Q4ModelLoader::load (loader.rs:109-128) -> Q4VoxtralModel (model.rs:759-989) */
typedef struct vox_model vox_model;
typedef struct {
    int32_t n_mels, enc_dim, enc_layers, enc_heads, enc_head_dim, enc_ffn, enc_window;
    int32_t dec_dim, dec_layers, dec_heads, dec_kv_heads, dec_head_dim, dec_ffn, dec_window;
    int32_t vocab, t_cond_dim, reshape_factor, prefix_len;
    uint64_t q4_bytes;        /* raw Q4 payload bytes in the file                 */
    uint64_t device_bytes;    /* bytes resident in HBM after repack               */
    uint64_t decode_step_bytes; /* algorithmic Q4 bytes read per single-token step */
} vox_model_info;
int32_t vox_model_load_gguf(const char *path, int32_t device, vox_model **out);
int32_t vox_model_load_gguf_handle(vox_gguf *g, int32_t device, vox_model **out);
int32_t vox_model_get_info(const vox_model *m, vox_model_info *info);
void vox_model_free(vox_model *m);

/* ------------------------------------------------------------------ session
 * caller-owned mutable state (LayerCaches kv_cache.rs:208-259 + workspace + stream). */
typedef struct vox_session vox_session;
typedef struct vox_tokenizer vox_tokenizer;   /* the tokenizer section below */
typedef struct {
    float preprocess_ms; /* pad + H2D + mel                       (e2e_bench.rs:147-149) */
    float encode_ms;     /* conv + encoder + adapter              (e2e_bench.rs:161-167) */
    float decode_ms;     /* prefill + autoregressive loop         (e2e_bench.rs:170-232) */
    float total_ms;
    float prefill_ms;    /* part of decode_ms: 38-token prefill + first argmax */
    int32_t decode_tokens; /* per stream: seq_len - 38 */
    int32_t seq_len;
} vox_timings;
/* max_batch concurrent streams, up to max_mel_frames mel frames per stream */
int32_t vox_session_create(vox_model *m, int32_t max_batch, int32_t max_mel_frames, vox_session **out);
/* Decoder KV cache element type, chosen at creation and fixed for the session's (or pool's) lifetime.
 *   VOX_DTYPE_F32 (what vox_session_create / vox_stream_pool_create use): K after RoPE and V are cached as computed.
 *   VOX_DTYPE_F16: half the KV memory and half the attention's K/V traffic.  K after RoPE and V are stored as IEEE
 *     binary16: each value is clamped to [-65504, 65504], then rounded to nearest even, so a value outside the f16 range
 *     stores +-65504, never +-inf; NaN stays NaN.  Every attention path (prefill, decode step, persistent kernel,
 *     per-op paths) reads the stored values, including the current position's own key and value, widens them exactly to
 *     f32 and computes as with an f32 cache, so all paths compute the same function.  Nothing else changes:
 *     activations, logits, weights, the encoder and its K/V rings, token scores, beams and bias work as before.
 *   VOX_DTYPE_KV_Q8: 1.125 bytes per cached value, 9/32 of the f32 KV memory and 9/16 of the f16.  Each block of 16
 *     consecutive head dims x[0..16) of one (position, kv head) vector (f32: K after RoPE, or V) is stored as
 *       a   = max_i |x_i|
 *       d   = f16_rn(min(a / 127, 65504))          (a / 127 an f32 division; f16_rn rounds to nearest even)
 *       q_i = 0 if d == 0, else clamp(rint(x_i / (float)d), -127, 127)
 *                                                  (f32 division; rint to nearest even; -128 is never stored)
 *     A block holding a NaN stores d = NaN and q_i = 0: the whole block decodes to NaN.  The decoded value is
 *     (float)d * q_i, exact in f32.  As for f16, every attention path reads the decoded values, including the current
 *     position's own key and value, and computes as with an f32 cache holding them; vox_session_debug_read("kv_k<l>" /
 *     "kv_v<l>") returns them as f32.  Nothing else changes.
 *   Any other kv_dtype: VOX_EINVAL, and *out is left untouched. */
int32_t vox_session_create_ex(vox_model *m, int32_t max_batch, int32_t max_mel_frames, int32_t kv_dtype, vox_session **out);
/* bytes of device memory the session allocated (all of it at creation; the first set_top_k / set_beam / set_bias and
 * the debug captures add their buffers) -- for sizing servers without querying the shared device */
int32_t vox_session_device_bytes(const vox_session *s, uint64_t *bytes);
/* TimeEmbedding::embed(delay) + the 26 ADA scale vectors (model.rs:250-255), once per session: every stream at
 * delay_tokens (80 ms each; 6.0 when the session is created) */
int32_t vox_session_set_delay(vox_session *s, float delay_tokens);
/* stream i of every later call (encode/prefill/decode/transcribe/generate_step/forward_streaming) is conditioned on
 * delays[i], i < b; streams >= b keep theirs.  vox_session_set_delay(d) sets every stream to d.
 * 1 <= b <= max_batch and every delay finite and >= 0, else VOX_EINVAL; VOX_ECUDA without a device.  Each stream keeps
 * its own ADA vectors (2 x layers x dec_dim floats, 639 KB at production geometry).  A call whose rows all have one
 * delay runs the shared-vector kernels; rows at different delays still share one weight sweep per decode step (the
 * kernels read each row's own ADA vectors). */
int32_t vox_session_set_delays(vox_session *s, const float *delays, int32_t b);
/* encode_audio (model.rs:783-788): mel [B,128,T] host -> audio_embeds [B,S,dec_dim] host (nullable);
 * seq_len = S.  The embeddings also stay resident in the session for vox_prefill/decode. */
int32_t vox_encode_audio(vox_session *s, const float *mel, int32_t b, int32_t t_frames,
                         float *audio_embeds /* nullable */, size_t cap_floats, int32_t *seq_len);
/* transcribe_streaming (model.rs:873-963): mel [B,128,T] host -> out_ids [B][n_out], n_out = S-38
 * (0 when S<38).  Equal-length streams per call (the reference is batch 1; vox_transcribe_pcm_ragged takes streams of
 * different lengths). */
int32_t vox_transcribe_streaming(vox_session *s, const float *mel, int32_t b, int32_t t_frames,
                                 int32_t *out_ids, size_t cap_ids, int32_t *n_out, vox_timings *tm);
/* full pipeline from PCM (transcribe.rs:187-318 per chunk): samples [B][n] host, optional
 * peak_normalize(0.95), pad_audio, GPU mel, encode, decode -> ids */
int32_t vox_transcribe_pcm(vox_session *s, const float *samples, int32_t b, size_t n,
                           int32_t peak_normalize, int32_t *out_ids, size_t cap_ids, int32_t *n_out,
                           vox_timings *tm);
/* Streams of different lengths in one call.  samples: stream s's lens[s] samples follow stream s-1's (host, 16 kHz).
 * Each stream is handled exactly as vox_transcribe_pcm handles a single stream: optional peak_normalize(0.95) over its
 * own samples, pad_audio, log-mel, encode, 38-position prefill, greedy (or beam) decode.
 * out_ids: stream s's n_out[s] ids follow stream s-1's; n_out[s] = max(0, S4_s - 38), where S4_s follows from lens[s]
 * alone (pad_audio length -> mel frames -> two stride-2 convolutions -> / reshape_factor).
 *   - Arguments: VOX_EINVAL unless 1 <= b <= max_batch (b * W <= max_batch at beam width W > 1), every lens[s] >= 1
 *     and every stream's mel frames <= max_mel_frames; VOX_ECAPACITY when cap_ids < sum of n_out.  All of these are
 *     checked on the host before any device work; a refused call leaves the session as it was.
 *   - Equal lengths: when every lens[s] is equal the call is vox_transcribe_pcm of the same [b][n] array, bit for bit
 *     (ids, token scores, n-best).
 *   - Work: the encoder runs over the sum of the streams' frames, not b x the longest.  The decoder's rows are the
 *     streams sorted by decreasing n_out, and a stream's rows leave the decode step after its last token, so the step's
 *     cost follows the streams still running.  A stream with n_out = 0 takes no decoder rows; n_out = 1 takes the
 *     prefill only.
 *   - Per-stream settings: vox_session_set_delays applies stream i's delay to stream i of the call.  With
 *     vox_session_set_top_k(k), vox_session_token_scores returns stream s's n_out[s] x k entries after those of stream
 *     s-1, with *b = b and *n = sum of n_out (for equal lengths the [b][n][k] layout).  vox_session_nbest likewise:
 *     stream s's W hypotheses of n_out[s] ids each after stream s-1's, scores [b][W].
 *   - Timings: seq_len and decode_tokens are the longest stream's (the positions actually run).
 *   - Like a beam call, the call leaves the decoder cache empty (vox_session_cache_len 0). */
int32_t vox_transcribe_pcm_ragged(vox_session *s, const float *samples, const size_t *lens, int32_t b,
                                  int32_t peak_normalize, int32_t *out_ids, size_t cap_ids,
                                  int32_t *n_out /* [b] */, vox_timings *tm);
/* same, samples already resident in HBM ([B][n] device); used for the device-resident bench leg */
int32_t vox_transcribe_pcm_dev(vox_session *s, const float *samples_dev, int32_t b, size_t n,
                               int32_t *out_ids, size_t cap_ids, int32_t *n_out, vox_timings *tm);
/* incremental API: generate_step_with_cache (model.rs:857-867): ids [B][M] -> logits [B][M][vocab]
 * host; appends to the session's decoder KV cache (vox_session_reset clears it). */
int32_t vox_generate_step_with_cache(vox_session *s, const int32_t *ids, int32_t b, int32_t m,
                                     float *logits, size_t cap_floats);
/* forward_streaming (model.rs:801-814): teacher-forced full pass from mel: decoder inputs = audio_embeds + embed(ids),
 * ids [B][S] with S = the sequence length vox_encode_audio would report; logits [B][S][vocab] host.  Leaves the
 * decoder KV cache filled with the S positions.  (Parity/debug entry: it ships every logit to the host.) */
int32_t vox_forward_streaming(vox_session *s, const float *mel, int32_t b, int32_t t_frames, const int32_t *ids,
                              int32_t n_ids, float *logits, size_t cap_floats);
/* Device-side incremental decode (the production form of generate_step_with_cache, model.rs:857-867: same graph, but
 * the greedy argmax (model.rs:922, 957) stays on the device and feeds the next step instead of shipping
 * [B][M][vocab] logits to the host).
 * vox_prefill: ids [B][M] at cache positions len..len+M-1; add_audio != 0 adds the session's audio embeddings of
 * those positions (after vox_encode_audio; model.rs:894-903); next_tok [B] (nullable) = argmax of the last row.
 * After vox_transcribe_pcm_ragged, row i reads the call's stream i (caller order), B must be its stream count and
 * only positions every stream has are allowed (those of the shortest stream), else VOX_EINVAL; the same for
 * vox_decode_step.
 * vox_decode_step: one position; tok [B] NULL = use the device-side token left by the previous call;
 * next_tok NULL with tok NULL = fully asynchronous (no host sync). */
int32_t vox_prefill(vox_session *s, const int32_t *ids, int32_t b, int32_t m, int32_t add_audio, int32_t *next_tok);
int32_t vox_decode_step(vox_session *s, const int32_t *tok /* nullable */, int32_t b, int32_t add_audio,
                        int32_t *next_tok /* nullable */);
/* Token confidences.  k = 0 (the default) turns them off; 1 <= k <= VOX_MAX_TOP_K turns them on for every later
 * vox_transcribe_streaming, vox_transcribe_pcm, vox_transcribe_pcm_dev, vox_prefill and vox_decode_step; any other k is
 * VOX_EINVAL.  For each emitted token the device keeps the k most likely ids (descending logit, the lower id first on
 * equal logits, so top_ids[0] is the emitted greedy id) and their log-probabilities logit - logsumexp(logits) (f32,
 * temperature 1).  The ids do not change.  Costs one extra kernel launch per prefill and decode step, and
 * 2 x max_batch x (KV capacity) x 8 x 4 bytes of device memory from the first k > 0. */
#define VOX_MAX_TOP_K 8
int32_t vox_session_set_top_k(vox_session *s, int32_t k);
/* The scores of the last transcribe call ([b][n][k], n = its n_out) or of the last vox_prefill / vox_decode_step
 * ([b][1][k], the position that call emitted), row-major in top_ids / top_logprobs (cap elements each).  Synchronises the
 * session's stream.  Both buffers NULL: only *b, *n, *k are set.  VOX_EINVAL if that call ran with k = 0, VOX_ECAPACITY
 * if cap < b * n * k. */
int32_t vox_session_token_scores(vox_session *s, int32_t *top_ids, float *top_logprobs, size_t cap, int32_t *b,
                                 int32_t *n, int32_t *k);
/* Beam search for vox_transcribe_streaming, vox_transcribe_pcm and vox_transcribe_pcm_dev: width W in
 * [1, VOX_MAX_BEAM] beams per stream, else VOX_EINVAL.  W = 1 (the default) is the greedy path, unchanged.
 *   - After the prefill the beam list holds one entry, the prefix, with score 0.  At each emitted position every live
 *     beam j offers its W most likely tokens (the token-score order, see vox_session_set_top_k) with log-probability
 *     lp; a candidate's score is cum[j] + (double)lp, summed in f64 on the device.  The new beam list is the W best
 *     candidates ordered by score descending, then parent rank j ascending, then token id ascending.  That order is the
 *     beam ranking.
 *   - Every position emits exactly one token, so every hypothesis has n_out tokens and no length penalty applies.  The
 *     call returns the rank-0 hypothesis in out_ids; vox_session_nbest returns all W in rank order.
 *   - The W beams of stream s run as W rows of the batched decode step, so b * W <= max_batch, else VOX_EINVAL.  Each
 *     stream's delay applies to all of its beams.
 *   - With token confidences on (k > 0), vox_session_token_scores returns, for the rank-0 hypothesis, the top-k of the
 *     distribution each of its tokens was chosen from; top_ids[0] need not be the emitted id.
 *   - While W > 1, vox_prefill and vox_decode_step return VOX_EINVAL (no incremental beam search).  A beam call leaves
 *     the decoder cache empty (vox_session_cache_len 0).  Streaming pools always decode greedily. */
#define VOX_MAX_BEAM 8
int32_t vox_session_set_beam(vox_session *s, int32_t width);
/* The n-best list of the last transcribe call: ids [b][w][n] (n = its n_out) and summed log-probabilities scores [b][w]
 * (descending per stream); ids needs cap >= b * w * n elements and scores b * w.  Synchronises the session's stream.  Both
 * buffers NULL: only *b, *w, *n are set.  VOX_EINVAL if that call ran at width 1, VOX_ECAPACITY if cap is short. */
int32_t vox_session_nbest(vox_session *s, int32_t *ids, double *scores, size_t cap, int32_t *b, int32_t *w, int32_t *n);
/* Phrase boosting (custom vocabulary) for greedy decoding: vox_transcribe_streaming, vox_transcribe_pcm,
 * vox_transcribe_pcm_ragged, vox_transcribe_pcm_dev, vox_prefill, vox_decode_step and streaming pools.
 *   - A stream's bias list holds up to VOX_MAX_BIAS_PHRASES phrases.  A phrase is 1 to VOX_MAX_BIAS_LEN token ids, each
 *     in [VOX_FIRST_TEXT_ID, vocab), with a boost b > 0 (finite, in logit units).  A word's ids depend on its leading
 *     space, so a list may hold both forms; vox_session_set_bias_text builds them from words.
 *   - The stream's history h is the sequence of text ids (>= VOX_FIRST_TEXT_ID) it has emitted since the history was
 *     last cleared; lower (special) ids, [STREAMING_PAD] among them, never enter it.  The history is cleared whenever the
 *     decoder cache is emptied (every transcribe call, vox_session_reset, a pool session's prefill) and when the stream's
 *     list is set.
 *   - At every position the stream emits (the prefill's output included), candidate id t gets
 *         boost(t) = max { b_i : phrase i, 0 <= j < len_i, the last j ids of h equal phrase_i[0..j), phrase_i[j] = t }
 *     or 0 when no phrase offers t: the first id of every phrase is always offered, a continuation only while the
 *     history ends in the phrase's prefix.  The emitted id is the argmax of (float)(logit(t) + boost(t)) over the whole
 *     vocabulary, the lowest id winning a tie: the greedy rule applied to boosted logits.  The logits themselves are
 *     unchanged (vox_session_debug_read "logits", token scores: top_ids[0] is the unboosted argmax and need not be the
 *     emitted id).
 *   - With no list (the default) a stream decodes exactly as before.  While some stream of a session has a list, every
 *     prefill and decode step costs one extra kernel launch; device memory (about 18 KB per stream) is allocated by the
 *     first non-empty list.
 *   - A transcribe call at beam width > 1 while any stream has a list returns VOX_EINVAL before any device work.
 *     vox_generate_step_with_cache and vox_forward_streaming emit nothing and are unaffected.
 * Phrase p is ids[off_p .. off_p + lens[p]) with off_p = lens[0] + ... + lens[p-1]; n_phrases = 0 clears the list.
 * stream in [0, max_batch), or -1 for every stream.  VOX_EINVAL for an unknown stream, n_phrases outside
 * [0, VOX_MAX_BIAS_PHRASES], a length outside [1, VOX_MAX_BIAS_LEN], an id outside [VOX_FIRST_TEXT_ID, vocab), a boost
 * that is not finite and > 0, or NULL buffers with n_phrases > 0; a refused call changes nothing. */
#define VOX_FIRST_TEXT_ID 1000
#define VOX_MAX_BIAS_PHRASES 256
#define VOX_MAX_BIAS_LEN 16
int32_t vox_session_set_bias(vox_session *s, int32_t stream, const int32_t *ids, const int32_t *lens, const float *boosts,
                             int32_t n_phrases);
/* vox_session_set_bias with the phrases given as words: phrases[p] is NUL-terminated UTF-8, boosts[p] its boost.
 * Expansion rule (the whole contract): phrase p gives the id phrase vox_tokenizer_encode(p), then the id phrase
 * vox_tokenizer_encode(" " + p) unless p starts with White_Space (a word in running text carries its leading space); the
 * second form is dropped when it equals the first.  Both forms get boosts[p].  The forms go in phrase order, and the
 * result goes to vox_session_set_bias unchanged: the same replacement of the stream's list, history clearing and device
 * rule.  No other variant is added: case ("Zurich" / "zurich"), plural or other spellings are separate phrases the caller
 * lists.  n_phrases = 0 clears the list (t, phrases and boosts may then be NULL).
 * VOX_EINVAL, changing nothing, for an empty phrase, a NULL phrase or buffer, invalid UTF-8, a form longer than
 * VOX_MAX_BIAS_LEN ids (the message names the phrase index), more than VOX_MAX_BIAS_PHRASES forms after expansion, and
 * every case vox_session_set_bias refuses (a form id outside the model's vocabulary, a boost that is not finite and > 0,
 * an unknown stream); VOX_EFORMAT for a tokenizer that cannot encode (vox_tokenizer_encode).  All of it is checked on the
 * host before any device work. */
int32_t vox_session_set_bias_text(vox_session *s, int32_t stream, const vox_tokenizer *t, const char *const *phrases,
                                  const float *boosts, int32_t n_phrases);
int32_t vox_session_cache_len(const vox_session *s, int32_t *len);             /* LayerCaches::seq_len */
int32_t vox_session_reset(vox_session *s);                                       /* LayerCaches::reset  */
/* debugging / parity: copy an internal activation by name ("enc_out","audio_embeds","conv","enc<i>",
 * "logits","ada") to host; "mega_trace" = SM-clock phase stamps of the last persistent decode step
 * (6 floats per phase, microseconds); "mega_epoch" = {persistent-kernel launches the host has counted
 * since the last epoch re-base, the device epoch} (equal between calls); "mega_attn" = the attention
 * tiling of each persistent launch of the last decode step, 4 floats per launch {rows, token capacity,
 * keys per K/V tile, key chunks per (stream, kv head)} (none after a per-op step); "kv_k<l>" / "kv_v<l>" = decoder layer l's
 * cached K (after RoPE) or V for the rows of the last call, positions [0, cache length), as f32 [row][pos][kv_head][hd]
 * (an f16 cache widened exactly; not on the ring-indexed sessions of an unbounded stream pool); "mel" = the log-mel of
 * the last call that started from PCM (vox_transcribe_pcm, _dev, _ragged): time-major [sum of the streams' frames][128],
 * stream after stream (each stream's frames = vox_mel_num_frames(its padded length)); after a call that took its mel
 * from the caller (vox_encode_audio, vox_transcribe_streaming), that mel as [B][128][T]; VOX_ENOTFOUND before either;
 * "pcm_pad" = the normalised, padded signal of each stream of the last PCM call (vox_pad_audio_len samples per stream),
 * stream after stream; VOX_ENOTFOUND unless the last such call started from PCM; names of the form "<switch>_on|_off|_auto" (graph, tc, gemm_tc |
 * gemm_simt, enc_attn_tc | enc_attn_simt, mega, capture) flip a kernel-selection switch and return no
 * data (INTEGRATION.md section 5) */
int32_t vox_session_debug_read(vox_session *s, const char *what, float *out, size_t cap_floats,
                               size_t *n_floats);
/* per-kernel-family launch counter since creation (for bench.py's gpu_launches) */
int32_t vox_session_launch_count(const vox_session *s, uint64_t *launches);
void vox_session_free(vox_session *s);

/* ------------------------------------------------------------------ streaming sessions (SURVEY 8(f)-1)
 * The reference has the pieces (Q4AudioEncoder::forward_with_cache model.rs:437-452, encode_audio_with_cache
 * model.rs:790-799, KVCache::apply_sliding_window kv_cache.rs:176-203) but its CLI transcribes whole utterances.
 * A pool is one GPU worker for up to max_sessions live sessions: audio is pushed in arbitrary pieces, vox_stream_tick
 * advances every session as far as its audio allows -- incremental log-mel, conv stem with carried frames, encoder
 * layers over per-layer K/V rings (absolute positions; keys older than the sliding window are overwritten), adapter,
 * and ONE batched decoder step for all sessions that can take one (rows at different positions, paged KV) -- and
 * every token is available as soon as its inputs are final.  The ids equal vox_transcribe_pcm's of the same audio.
 * Samples must already be peak-normalised if the caller wants io.rs:59-68 semantics (it needs the whole utterance). */
typedef struct vox_stream_pool vox_stream_pool;
typedef struct {
    float gpu_ms;            /* device time of the tick (CUDA events)                 */
    int32_t live_sessions;   /* open and not yet drained after the tick               */
    int32_t mel_frames, encoder_rows, prefills, decode_steps, decode_rows;
} vox_stream_stats;
/* max_seconds in [1, 60]: sessions of up to that much audio, their whole history resident on the device.
 * max_seconds = 0: sessions of ANY length.  Both attentions are sliding-window, so a session keeps only what it can
 * still read -- decoder KV as a per-session ring of pages covering the decoder window, the encoder K/V rings, RoPE rows
 * computed for the positions in flight, and 30 s of padded audio in its PCM / mel / conv / audio-embedding buffers --
 * fixed when the pool is created.  push_pcm then fails with VOX_ECAPACITY while the audio not yet consumed by a tick
 * would exceed those 30 s; encode_chunk is not available.  Absolute positions stay int32: ~248 days of audio. */
int32_t vox_stream_pool_create(vox_model *m, int32_t max_sessions, float max_seconds, vox_stream_pool **out);
/* kv_dtype as vox_session_create_ex: every session of the pool shares its page pool, so they share the element type.
 * An unbounded pool's state is dominated by the decoder KV ring; VOX_DTYPE_F16 halves it and VOX_DTYPE_KV_Q8 takes it to
 * 9/32 of f32 (INTEGRATION.md section 3b). */
int32_t vox_stream_pool_create_ex(vox_model *m, int32_t max_sessions, float max_seconds, int32_t kv_dtype,
                                  vox_stream_pool **out);
/* bytes of device memory the pool allocated (its session's arena, which holds every per-session buffer) */
int32_t vox_stream_pool_device_bytes(const vox_stream_pool *p, uint64_t *bytes);
int32_t vox_stream_open(vox_stream_pool *p, int32_t *session);
/* the session's transcription delay in tokens (80 ms each); default 6.0 on vox_stream_open.  Only before the session's
 * 38-position prefill has run (vox_stream_session_info.decoder_positions == 0), else VOX_EINVAL; also VOX_EINVAL for an
 * unknown session or a delay that is not finite and >= 0.  VOX_ECUDA without a device, before the arguments are checked.
 * Sessions at different delays share one decode step. */
int32_t vox_stream_set_delay(vox_stream_pool *p, int32_t session, float delay_tokens);
/* the session's bias list (see vox_session_set_bias), same arguments and errors; VOX_EINVAL for a session that is not
 * open.  It takes effect at the session's next decoder position and clears its history; vox_stream_open empties it. */
int32_t vox_stream_set_bias(vox_stream_pool *p, int32_t session, const int32_t *ids, const int32_t *lens, const float *boosts,
                            int32_t n_phrases);
/* the session's bias list from words: vox_session_set_bias_text's expansion, then vox_stream_set_bias */
int32_t vox_stream_set_bias_text(vox_stream_pool *p, int32_t session, const vox_tokenizer *t, const char *const *phrases,
                                 const float *boosts, int32_t n_phrases);
int32_t vox_stream_push_pcm(vox_stream_pool *p, int32_t session, const float *samples, size_t n);
int32_t vox_stream_finish(vox_stream_pool *p, int32_t session);        /* end of utterance: right padding, pad.rs:89-103 */
int32_t vox_stream_tick(vox_stream_pool *p, vox_stream_stats *stats /* nullable */);
/* ids emitted since the last poll; *done != 0 once the finished session has emitted everything */
int32_t vox_stream_poll_ids(vox_stream_pool *p, int32_t session, int32_t *ids, size_t cap, size_t *n, int32_t *done);
/* token confidences (see vox_session_set_top_k) for every session of the pool: one batched step serves them all, so k is
 * pool-wide and can change only while no session is open (else VOX_EINVAL); VOX_EINVAL for k outside [0, VOX_MAX_TOP_K]. */
int32_t vox_stream_pool_set_top_k(vox_stream_pool *p, int32_t k);
/* vox_stream_poll_ids plus the scores of the same n <= cap tokens, [n][k] in top_ids / top_logprobs (cap * k elements
 * each).  VOX_EINVAL while the pool's k is 0.  Both poll functions drop the tokens they return, with their scores. */
int32_t vox_stream_poll_scored(vox_stream_pool *p, int32_t session, int32_t *ids, int32_t *top_ids, float *top_logprobs,
                               size_t cap, size_t *n, int32_t *done);
/* parity/debug: audio embeddings produced so far, [n][dec_dim] host.  Fails (VOX_ECAPACITY) once an unbounded session
 * has evicted its first rows: use vox_stream_audio_embeds_range. */
int32_t vox_stream_audio_embeds(vox_stream_pool *p, int32_t session, float *out, size_t cap_floats, int32_t *n);
/* audio embeddings [first, first + n) (absolute indices), [n][dec_dim] host.  VOX_ECAPACITY when `first` is no longer
 * resident (see vox_stream_session_info.first_audio_embed), VOX_EINVAL past the embeddings produced so far. */
int32_t vox_stream_audio_embeds_range(vox_stream_pool *p, int32_t session, int64_t first, int64_t n, float *out,
                                      size_t cap_floats);
/* log-mel frames [first, first + n) (absolute frame indices of the padded stream), [n][128] host: the frames the
 * encoder's conv stem read.  VOX_ECAPACITY when `first` is no longer resident (an unbounded session keeps the frames
 * its conv stem still reads, and slides them out when its buffer is full), VOX_EINVAL past
 * vox_stream_session_info.mel_frames. */
int32_t vox_stream_mel_range(vox_stream_pool *p, int32_t session, int64_t first, int64_t n, float *out, size_t cap_floats);
/* a struct tag (not a typedef): the function below has the same name */
struct vox_stream_session_info {
    int64_t samples;            /* padded signal samples known (left padding included; vox_stream_progress) */
    int64_t mel_frames, encoder_frames, audio_embeds;  /* final frames / embeddings produced */
    int64_t first_audio_embed;  /* first embedding still resident on the device */
    int64_t decoder_positions;  /* decoder positions cached (0 until the 38-position prefill has run) */
    int64_t ids_emitted;
    int32_t kv_pages;           /* decoder KV pages the session holds */
};
int32_t vox_stream_session_info(vox_stream_pool *p, int32_t session, struct vox_stream_session_info *out);
/* encode_audio_with_cache (model.rs:790-799) with upstream's semantics: one mel chunk [128][t_frames] (host) through the
 * conv stem on its own, the encoder layers over the session's K/V caches (RoPE / mask offsets = cached length), x4 stack
 * and adapter -> the chunk's S/4 embeddings [n][dec_dim] (host).  Chunk-wise alternative to push_pcm/tick; do not mix. */
int32_t vox_stream_encode_chunk(vox_stream_pool *p, int32_t session, const float *mel, int32_t t_frames, float *audio_embeds,
                                size_t cap_floats, int32_t *n);
int32_t vox_stream_close(vox_stream_pool *p, int32_t session);
void vox_stream_pool_free(vox_stream_pool *p);

/* ------------------------------------------------------------------ tokenizer (host)
 * VoxtralTokenizer, src/tokenizer/mod.rs:70-214 (vox_tokenizer is declared with the session) */
int32_t vox_tokenizer_from_file(const char *path, vox_tokenizer **out);         /* mod.rs:70  */
int32_t vox_tokenizer_from_json(const char *json, size_t len, vox_tokenizer **out); /* mod.rs:125 */
int32_t vox_tokenizer_decode(const vox_tokenizer *t, const uint32_t *ids, size_t n, char *buf,
                             size_t cap, size_t *written);                       /* mod.rs:170 */
int32_t vox_tokenizer_decode_token(const vox_tokenizer *t, uint32_t id, char *buf, size_t cap,
                                   size_t *written, int32_t *found);             /* mod.rs:194 */
int32_t vox_tokenizer_vocab_size(const vox_tokenizer *t, size_t *n);            /* mod.rs:211 */
/* Tekken encode (mistral_common's Tekkenizer.encode(text, bos=False, eos=False), tiktoken's encode with no special
 * tokens): UTF-8 text[len] -> text ids (>= VOX_FIRST_TEXT_ID) in ids[cap]; *n = ids needed.  ids NULL: only *n.
 * Special-token text such as "[INST]" is plain text; no Unicode normalisation (NFC and NFD text give different ids).
 * The ids decode back to the text: vox_tokenizer_decode(encode(s)) == s.  The rank table (the text ranks below
 * default_vocab_size - 1000, the lowest position winning for a repeated byte string) is built by the first call and kept;
 * concurrent calls on one handle are safe.
 * VOX_EINVAL invalid UTF-8 (overlong forms, surrogates, > U+10FFFF, truncated sequences); VOX_EFORMAT a pattern other
 * than Tekken's or a vocabulary without the 256 byte tokens (decoding still works); VOX_ECAPACITY cap < *n (and *n is
 * set). */
int32_t vox_tokenizer_encode(const vox_tokenizer *t, const char *text, size_t len, int32_t *ids, size_t cap, size_t *n);
void vox_tokenizer_free(vox_tokenizer *t);

#ifdef __cplusplus
}
#endif
#endif /* VOXTRAL_H */
