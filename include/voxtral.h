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
void vox_q4_tensor_free(vox_q4 *w);
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
/* TimeEmbedding::embed(delay) + the 26 ADA scale vectors (model.rs:250-255), once per session */
int32_t vox_session_set_delay(vox_session *s, float delay_tokens);
/* encode_audio (model.rs:783-788): mel [B,128,T] host -> audio_embeds [B,S,dec_dim] host (nullable);
 * seq_len = S.  The embeddings also stay resident in the session for vox_prefill/decode. */
int32_t vox_encode_audio(vox_session *s, const float *mel, int32_t b, int32_t t_frames,
                         float *audio_embeds /* nullable */, size_t cap_floats, int32_t *seq_len);
/* transcribe_streaming (model.rs:873-963): mel [B,128,T] host -> out_ids [B][n_out], n_out = S-38
 * (0 when S<38).  Equal-length streams per call (the reference is batch 1). */
int32_t vox_transcribe_streaming(vox_session *s, const float *mel, int32_t b, int32_t t_frames,
                                 int32_t *out_ids, size_t cap_ids, int32_t *n_out, vox_timings *tm);
/* full pipeline from PCM (transcribe.rs:187-318 per chunk): samples [B][n] host, optional
 * peak_normalize(0.95), pad_audio, GPU mel, encode, decode -> ids */
int32_t vox_transcribe_pcm(vox_session *s, const float *samples, int32_t b, size_t n,
                           int32_t peak_normalize, int32_t *out_ids, size_t cap_ids, int32_t *n_out,
                           vox_timings *tm);
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
 * vox_decode_step: one position; tok [B] NULL = use the device-side token left by the previous call;
 * next_tok NULL with tok NULL = fully asynchronous (no host sync). */
int32_t vox_prefill(vox_session *s, const int32_t *ids, int32_t b, int32_t m, int32_t add_audio, int32_t *next_tok);
int32_t vox_decode_step(vox_session *s, const int32_t *tok /* nullable */, int32_t b, int32_t add_audio,
                        int32_t *next_tok /* nullable */);
int32_t vox_session_cache_len(const vox_session *s, int32_t *len);             /* LayerCaches::seq_len */
int32_t vox_session_reset(vox_session *s);                                       /* LayerCaches::reset  */
/* debugging / parity: copy an internal activation by name ("enc_out","audio_embeds","conv","enc<i>",
 * "logits","ada") to host; "mega_trace" = SM-clock phase stamps of the last persistent decode step
 * (6 floats per phase, microseconds); names of the form "<switch>_on|_off|_auto" (graph, tc, pdl, gemm_tc |
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
int32_t vox_stream_pool_create(vox_model *m, int32_t max_sessions, float max_seconds, vox_stream_pool **out);
int32_t vox_stream_open(vox_stream_pool *p, int32_t *session);
int32_t vox_stream_push_pcm(vox_stream_pool *p, int32_t session, const float *samples, size_t n);
int32_t vox_stream_finish(vox_stream_pool *p, int32_t session);        /* end of utterance: right padding, pad.rs:89-103 */
int32_t vox_stream_tick(vox_stream_pool *p, vox_stream_stats *stats /* nullable */);
/* ids emitted since the last poll; *done != 0 once the finished session has emitted everything */
int32_t vox_stream_poll_ids(vox_stream_pool *p, int32_t session, int32_t *ids, size_t cap, size_t *n, int32_t *done);
/* parity/debug: audio embeddings produced so far, [n][dec_dim] host */
int32_t vox_stream_audio_embeds(vox_stream_pool *p, int32_t session, float *out, size_t cap_floats, int32_t *n);
/* encode_audio_with_cache (model.rs:790-799) with upstream's semantics: one mel chunk [128][t_frames] (host) through the
 * conv stem on its own, the encoder layers over the session's K/V caches (RoPE / mask offsets = cached length), x4 stack
 * and adapter -> the chunk's S/4 embeddings [n][dec_dim] (host).  Chunk-wise alternative to push_pcm/tick; do not mix. */
int32_t vox_stream_encode_chunk(vox_stream_pool *p, int32_t session, const float *mel, int32_t t_frames, float *audio_embeds,
                                size_t cap_floats, int32_t *n);
int32_t vox_stream_close(vox_stream_pool *p, int32_t session);
void vox_stream_pool_free(vox_stream_pool *p);

/* ------------------------------------------------------------------ tokenizer (host)
 * VoxtralTokenizer, src/tokenizer/mod.rs:70-214 */
typedef struct vox_tokenizer vox_tokenizer;
int32_t vox_tokenizer_from_file(const char *path, vox_tokenizer **out);         /* mod.rs:70  */
int32_t vox_tokenizer_from_json(const char *json, size_t len, vox_tokenizer **out); /* mod.rs:125 */
int32_t vox_tokenizer_decode(const vox_tokenizer *t, const uint32_t *ids, size_t n, char *buf,
                             size_t cap, size_t *written);                       /* mod.rs:170 */
int32_t vox_tokenizer_decode_token(const vox_tokenizer *t, uint32_t id, char *buf, size_t cap,
                                   size_t *written, int32_t *found);             /* mod.rs:194 */
int32_t vox_tokenizer_vocab_size(const vox_tokenizer *t, size_t *n);            /* mod.rs:211 */
void vox_tokenizer_free(vox_tokenizer *t);

#ifdef __cplusplus
}
#endif
#endif /* VOXTRAL_H */
