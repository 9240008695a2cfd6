// rust/voxtral_sys.rs -- raw `extern "C"` bindings for include/voxtral.h (libvoxtral_b200.so).
//
// SOURCE ONLY: there is no Rust toolchain in the build environment (SURVEY F1), so this file has never been compiled;
// it is the `src/b200/sys.rs` a maintainer of TrevorS/voxtral-mini-realtime-rs would add behind a `b200` cargo feature
// (Cargo.toml: `b200 = []`; build.rs: `println!("cargo:rustc-link-lib=dylib=voxtral_b200")`).  INTEGRATION.md shows the
// safe wrapper (`mod.rs`) and the call-site changes in src/bin/transcribe.rs.  tests/test_host_abi.py checks that every
// function declared here is exported by the library with the same name.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_void};

#[repr(C)] pub struct vox_gguf { _p: [u8; 0] }
#[repr(C)] pub struct vox_model { _p: [u8; 0] }
#[repr(C)] pub struct vox_session { _p: [u8; 0] }
#[repr(C)] pub struct vox_q4 { _p: [u8; 0] }
#[repr(C)] pub struct vox_mel { _p: [u8; 0] }
#[repr(C)] pub struct vox_tokenizer { _p: [u8; 0] }
#[repr(C)] pub struct vox_stream_pool { _p: [u8; 0] }

// decoder KV cache element types (vox_session_create_ex / vox_stream_pool_create_ex kv_dtype)
pub const VOX_DTYPE_F32: i32 = 0;
pub const VOX_DTYPE_F16: i32 = 1;
pub const VOX_DTYPE_KV_Q8: i32 = 100;   // int8 with an f16 scale per 16 head dims (include/voxtral.h)

#[repr(C)] #[derive(Default, Clone, Copy)]
pub struct vox_timings {
    pub preprocess_ms: f32, pub encode_ms: f32, pub decode_ms: f32, pub total_ms: f32,
    pub prefill_ms: f32, pub decode_tokens: i32, pub seq_len: i32,
}
#[repr(C)] #[derive(Default, Clone, Copy)]
pub struct vox_stream_stats {
    pub gpu_ms: f32, pub live_sessions: i32, pub mel_frames: i32, pub encoder_rows: i32,
    pub prefills: i32, pub decode_steps: i32, pub decode_rows: i32,
}
#[repr(C)] #[derive(Clone, Copy, Default)]
pub struct vox_stream_session_info {
    pub samples: i64, pub mel_frames: i64, pub encoder_frames: i64, pub audio_embeds: i64,
    pub first_audio_embed: i64, pub decoder_positions: i64, pub ids_emitted: i64, pub kv_pages: i32,
}
#[repr(C)] #[derive(Clone, Copy)]
pub struct vox_pad_config { pub sample_rate: u32, pub n_left_pad_tokens: u32, pub frame_rate: f32,
                            pub extra_right_pad_tokens: u32 }

extern "C" {
    pub fn vox_last_error() -> *const c_char;
    // src/gguf/reader.rs + loader.rs
    pub fn vox_gguf_open(path: *const c_char, out: *mut *mut vox_gguf) -> i32;
    pub fn vox_gguf_open_shards(bufs: *const *const c_void, lens: *const usize, n: usize,
                                out: *mut *mut vox_gguf) -> i32;
    pub fn vox_gguf_close(g: *mut vox_gguf);
    pub fn vox_model_load_gguf(path: *const c_char, device: i32, out: *mut *mut vox_model) -> i32;
    pub fn vox_model_load_gguf_handle(g: *mut vox_gguf, device: i32, out: *mut *mut vox_model) -> i32;
    pub fn vox_model_free(m: *mut vox_model);
    // src/gguf/model.rs
    pub fn vox_session_create(m: *mut vox_model, max_batch: i32, max_mel_frames: i32,
                              out: *mut *mut vox_session) -> i32;
    // kv_dtype: VOX_DTYPE_F32 (0), VOX_DTYPE_F16 (1) or VOX_DTYPE_KV_Q8 (100), the decoder KV cache's element type
    pub fn vox_session_create_ex(m: *mut vox_model, max_batch: i32, max_mel_frames: i32, kv_dtype: i32,
                                 out: *mut *mut vox_session) -> i32;
    pub fn vox_session_device_bytes(s: *const vox_session, bytes: *mut u64) -> i32;
    pub fn vox_session_set_delay(s: *mut vox_session, delay_tokens: f32) -> i32;
    pub fn vox_session_set_delays(s: *mut vox_session, delays: *const f32, b: i32) -> i32;
    pub fn vox_encode_audio(s: *mut vox_session, mel: *const f32, b: i32, t: i32,
                            audio_embeds: *mut f32, cap: usize, seq_len: *mut i32) -> i32;
    pub fn vox_transcribe_streaming(s: *mut vox_session, mel: *const f32, b: i32, t: i32,
                                    out_ids: *mut i32, cap: usize, n_out: *mut i32,
                                    tm: *mut vox_timings) -> i32;
    pub fn vox_transcribe_pcm(s: *mut vox_session, samples: *const f32, b: i32, n: usize,
                              peak_normalize: i32, out_ids: *mut i32, cap: usize, n_out: *mut i32,
                              tm: *mut vox_timings) -> i32;
    pub fn vox_transcribe_pcm_ragged(s: *mut vox_session, samples: *const f32, lens: *const usize, b: i32,
                                     peak_normalize: i32, out_ids: *mut i32, cap: usize,
                                     n_out: *mut i32, tm: *mut vox_timings) -> i32;
    pub fn vox_generate_step_with_cache(s: *mut vox_session, ids: *const i32, b: i32, m: i32,
                                        logits: *mut f32, cap: usize) -> i32;
    // forward_streaming (model.rs:801-814) and the device-side incremental decode (model.rs:857-867 without the
    // logits round trip)
    pub fn vox_forward_streaming(s: *mut vox_session, mel: *const f32, b: i32, t: i32, ids: *const i32, n_ids: i32,
                                 logits: *mut f32, cap: usize) -> i32;
    pub fn vox_prefill(s: *mut vox_session, ids: *const i32, b: i32, m: i32, add_audio: i32, next_tok: *mut i32) -> i32;
    pub fn vox_decode_step(s: *mut vox_session, tok: *const i32, b: i32, add_audio: i32, next_tok: *mut i32) -> i32;
    pub fn vox_session_reset(s: *mut vox_session) -> i32;
    // token confidences: top-k ids and log-probabilities of every emitted token (k <= VOX_MAX_TOP_K = 8; 0 = off)
    pub fn vox_session_set_top_k(s: *mut vox_session, k: i32) -> i32;
    pub fn vox_session_token_scores(s: *mut vox_session, top_ids: *mut i32, top_logprobs: *mut f32, cap: usize,
                                    b: *mut i32, n: *mut i32, k: *mut i32) -> i32;
    // beam search of the transcribe calls (width <= VOX_MAX_BEAM = 8; 1 = greedy) and its n-best list
    pub fn vox_session_set_beam(s: *mut vox_session, width: i32) -> i32;
    pub fn vox_session_nbest(s: *mut vox_session, ids: *mut i32, scores: *mut f64, cap: usize, b: *mut i32, w: *mut i32,
                             n: *mut i32) -> i32;
    // phrase boosting (custom vocabulary): phrase p is ids[off_p .. off_p + lens[p]); stream -1 = every stream;
    // n_phrases = 0 clears
    pub fn vox_session_set_bias(s: *mut vox_session, stream: i32, ids: *const i32, lens: *const i32, boosts: *const f32,
                                n_phrases: i32) -> i32;
    // the same from words (NUL-terminated UTF-8): each word and its leading-space form (include/voxtral.h)
    pub fn vox_session_set_bias_text(s: *mut vox_session, stream: i32, t: *const vox_tokenizer, phrases: *const *const c_char,
                                     boosts: *const f32, n_phrases: i32) -> i32;
    pub fn vox_session_free(s: *mut vox_session);
    // src/gguf/{tensor,linear,op}.rs
    pub fn vox_q4_tensor_create(bytes: *const u8, nbytes: usize, n: i64, k: i64, device: i32,
                                out: *mut *mut vox_q4) -> i32;
    pub fn vox_q4_matmul(w: *const vox_q4, x_dev: *const f32, y_dev: *mut f32, b: i32, m: i32,
                         bias_dev: *const f32, stream: *mut c_void) -> i32;
    pub fn vox_q4_matmul_host(w: *const vox_q4, x: *const f32, y: *mut f32, b: i32, m: i32,
                              bias: *const f32) -> i32;
    pub fn vox_q4_tensor_free(w: *mut vox_q4);
    // src/audio/{mel,pad,io}.rs, src/models/time_embedding.rs
    pub fn vox_mel_create(device: i32, out: *mut *mut vox_mel) -> i32;
    pub fn vox_mel_num_frames(n: usize) -> usize;
    pub fn vox_mel_compute_log(m: *mut vox_mel, samples: *const f32, n: usize, out: *mut f32, cap: usize) -> i32;
    pub fn vox_mel_free(m: *mut vox_mel);
    pub fn vox_peak_normalize(samples: *mut f32, n: usize, target: f32) -> i32;
    pub fn vox_pad_audio_len(n: usize, cfg: *const vox_pad_config) -> usize;
    pub fn vox_pad_audio(inp: *const f32, n: usize, cfg: *const vox_pad_config, out: *mut f32,
                         cap: usize, out_len: *mut usize) -> i32;
    pub fn vox_time_embedding(t: f32, dim: i32, out: *mut f32) -> i32;
    pub fn vox_stream_progress(n_samples: usize, ended: i32, reshape_factor: i32, prefix_len: i32, out: *mut i64) -> i32;
    // streaming sessions: Q4AudioEncoder::forward_with_cache (model.rs:437-452), encode_audio_with_cache (790-799)
    pub fn vox_stream_pool_create(m: *mut vox_model, max_sessions: i32, max_seconds: f32, out: *mut *mut vox_stream_pool) -> i32;
    pub fn vox_stream_pool_create_ex(m: *mut vox_model, max_sessions: i32, max_seconds: f32, kv_dtype: i32,
                                     out: *mut *mut vox_stream_pool) -> i32;
    pub fn vox_stream_pool_device_bytes(p: *const vox_stream_pool, bytes: *mut u64) -> i32;
    pub fn vox_stream_open(p: *mut vox_stream_pool, session: *mut i32) -> i32;
    pub fn vox_stream_set_delay(p: *mut vox_stream_pool, session: i32, delay_tokens: f32) -> i32;
    pub fn vox_stream_set_bias(p: *mut vox_stream_pool, session: i32, ids: *const i32, lens: *const i32, boosts: *const f32,
                               n_phrases: i32) -> i32;
    pub fn vox_stream_set_bias_text(p: *mut vox_stream_pool, session: i32, t: *const vox_tokenizer,
                                    phrases: *const *const c_char, boosts: *const f32, n_phrases: i32) -> i32;
    pub fn vox_stream_push_pcm(p: *mut vox_stream_pool, session: i32, samples: *const f32, n: usize) -> i32;
    pub fn vox_stream_finish(p: *mut vox_stream_pool, session: i32) -> i32;
    pub fn vox_stream_tick(p: *mut vox_stream_pool, stats: *mut vox_stream_stats) -> i32;
    pub fn vox_stream_poll_ids(p: *mut vox_stream_pool, session: i32, ids: *mut i32, cap: usize, n: *mut usize, done: *mut i32) -> i32;
    pub fn vox_stream_pool_set_top_k(p: *mut vox_stream_pool, k: i32) -> i32;
    pub fn vox_stream_poll_scored(p: *mut vox_stream_pool, session: i32, ids: *mut i32, top_ids: *mut i32, top_logprobs: *mut f32,
                                  cap: usize, n: *mut usize, done: *mut i32) -> i32;
    // max_seconds = 0: sessions of any length (include/voxtral.h)
    pub fn vox_stream_audio_embeds_range(p: *mut vox_stream_pool, session: i32, first: i64, n: i64, out: *mut f32,
                                         cap: usize) -> i32;
    pub fn vox_stream_mel_range(p: *mut vox_stream_pool, session: i32, first: i64, n: i64, out: *mut f32, cap: usize) -> i32;
    pub fn vox_stream_session_info(p: *mut vox_stream_pool, session: i32, out: *mut vox_stream_session_info) -> i32;
    pub fn vox_stream_encode_chunk(p: *mut vox_stream_pool, session: i32, mel: *const f32, t_frames: i32, audio_embeds: *mut f32,
                                   cap: usize, n: *mut i32) -> i32;
    pub fn vox_stream_close(p: *mut vox_stream_pool, session: i32) -> i32;
    pub fn vox_stream_pool_free(p: *mut vox_stream_pool);
    // src/tokenizer/mod.rs
    pub fn vox_tokenizer_from_file(path: *const c_char, out: *mut *mut vox_tokenizer) -> i32;
    pub fn vox_tokenizer_decode(t: *const vox_tokenizer, ids: *const u32, n: usize, buf: *mut c_char,
                                cap: usize, written: *mut usize) -> i32;
    pub fn vox_tokenizer_free(t: *mut vox_tokenizer);
    // Tekken encode, which the crate's tokenizer lacks: UTF-8 text -> text ids; ids NULL: only *n
    pub fn vox_tokenizer_encode(t: *const vox_tokenizer, text: *const c_char, len: usize, ids: *mut i32, cap: usize,
                                n: *mut usize) -> i32;
}
