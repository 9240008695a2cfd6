// model.h -- Q4 Voxtral model resident in HBM + per-session state.
// Mirrors Q4ModelLoader (reference src/gguf/loader.rs) and Q4VoxtralModel (src/gguf/model.rs).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <string>
#include <tuple>
#include <vector>

#include "audio_host.h"
#include "gguf.h"
#include "decode_mega.h"
#include "encoder.h"
#include "kernels.h"
#include "kv_cache.h"
#include "token_select.h"

namespace vox {

void cuda_check(cudaError_t e, const char *what);
#define CUDA_OK(x) ::vox::cuda_check((x), #x)

// Owns device allocations of one device.
struct DeviceArena {
    int device = 0;
    std::vector<void *> ptrs;
    size_t total = 0;
    void *alloc(size_t bytes);
    template <typename T>
    T *alloc_n(size_t n) { return (T *)alloc(n * sizeof(T)); }
    template <typename T>
    T *upload(const T *host, size_t n) {
        T *d = alloc_n<T>(n);
        CUDA_OK(cudaMemcpy(d, host, n * sizeof(T), cudaMemcpyHostToDevice));
        return d;
    }
    void release();
    ~DeviceArena() { release(); }
};

// Allocates the buffers of a split-K scratch (TcWork, GemmWork) whose sizes are set; the tickets start at zero.
template <typename Work>
void alloc_split_k(DeviceArena &arena, Work &w) {
    w.partial = arena.alloc_n<float>(w.partial_floats);
    w.counters = arena.alloc_n<int>(w.n_counters);
    CUDA_OK(cudaMemset(w.counters, 0, sizeof(int) * w.n_counters));
}

// Mel constants on device (window + sparse filterbank).
struct MelTables {
    float *window = nullptr;
    float *fb_vals = nullptr;
    int *fb_start = nullptr, *fb_len = nullptr;
    int fb_stride = 0;
    std::vector<float> fb_dense, window_host;
    void build(DeviceArena &arena);
};

struct EncLayerW {
    float *attn_norm = nullptr, *ffn_norm = nullptr;
    Q4Weight wqkv, wo, w13, w2;
    float *bqkv = nullptr, *bo = nullptr, *b2 = nullptr;
};
struct DecLayerW {
    float *attn_norm = nullptr, *ffn_norm = nullptr;
    Q4Weight ada0, ada2, wqkv, wo, w13, w2;
};

struct Model {
    int device = 0;
    vox_model_info info{};
    float rope_theta = 1e6f, norm_eps = 1e-5f;
    DeviceArena arena;
    // encoder
    float *conv1_w = nullptr, *conv1_b = nullptr, *conv2_w = nullptr, *conv2_b = nullptr;
    std::vector<EncLayerW> enc;
    float *enc_norm = nullptr;
    Q4Weight adapter0, adapter2, tok_emb;
    std::vector<DecLayerW> dec;
    float *dec_norm = nullptr;
    float *enc_cos = nullptr, *enc_sin = nullptr, *dec_cos = nullptr, *dec_sin = nullptr;
    int enc_rope_len = 4096, dec_rope_len = 16384;  // loader.rs:196, 284
    MelTables mel;
    RopeView dec_rope() const { return RopeView{dec_cos, dec_sin, dec_rope_len}; }

    static Model *load(const Gguf &g, int device);
};

// RoPE rows [p0, p0 + n) of head dim hd (RoPEConfig::init, rope.rs:35-64, f32 throughout: cos/sin((float)p * inv_freq)):
// the model's tables and the ring tables of unbounded stream pools are both filled by this one function.
void rope_rows(int hd, float theta, int64_t p0, int n, float *cos_out, float *sin_out);

// Repack raw GGUF Q4_0 blocks of one or more [N_i, K] matrices into the device layout.
// interleave=true: two parts with equal N, rows (2i, 2i+1) = (a_i, b_i).
Q4Weight upload_q4(DeviceArena &arena, const std::vector<const uint8_t *> &raw, const std::vector<int> &n_rows,
                   int K, bool interleave, bool tc_layout = false);

// transcription delay of a new session or stream session, in tokens of 80 ms: the CLI default --delay 6
// (transcribe.rs:49-51)
constexpr float kDefaultDelay = 6.0f;

// Everything a captured decode step depends on that is chosen on the host: a step captured under another key launches
// other kernels or reads another op table.
struct StepKey {
    int rows = 0, top_k = 0, beam_w = 1;
    bool matvec_tc = true, gemm_tc = true, use_mega = true, bias = false;
    auto tie() const { return std::tie(rows, top_k, beam_w, matvec_tc, gemm_tc, use_mega, bias); }
    bool operator==(const StepKey &o) const { return tie() == o.tie(); }
};
struct StepGraph {
    StepKey key;
    cudaGraphExec_t exec = nullptr;
    uint64_t nodes = 0;            // kernel launches per replay
    unsigned mega_launches = 0;    // persistent-kernel launches per replay
};

struct Session {
    Model *m = nullptr;
    int max_batch = 0, M_max = 0;
    cudaStream_t st = nullptr;
    DeviceArena arena;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    // audio encoder (encoder.h): its buffers, the embeddings of the last encode, the debug capture
    AudioEncoder enc;
    // read on the host only (argument checks, step counts, debug reads), never by a launch: rows of the last call's
    // logits
    int cur_B = 0;
    // decoder
    DecoderKv kv;                         // of max_batch rows (vox_session_create_ex kv_dtype)
    RopeView dec_rope;                    // the model's tables, or an unbounded stream pool's ring
    float *x_dec = nullptr, *h_dec = nullptr, *qkv_dec = nullptr, *attn_dec = nullptr, *act_dec = nullptr;
    float *last_h = nullptr, *logits = nullptr;
    float *logits_all = nullptr;
    size_t logits_all_cap = 0;
    // per-stream transcription delay (vox_session_set_delays): stream i's ADA set at ada_sets + i * ada_set_floats(),
    // {ADA scale [L][D], ffn_norm x ADA scale [L][D]} (the latter for the persistent decode kernel)
    std::vector<float> delays;
    float *ada_sets = nullptr, *t_embed = nullptr, *ada_tmp = nullptr;
    size_t ada_set_floats() const { return (size_t)2 * m->info.dec_layers * m->info.dec_dim; }
    // row i of a launch reads its stream's ADA set and audio embeddings through the tables [max_batch] bind_rows
    // fills: the ADA set pointers (kernels.h AdaRows, the persistent kernel's ffn_ada_rows) and the audio offsets (launch_embed)
    const float **d_ada_rows = nullptr, **d_fga_rows = nullptr;
    int64_t *d_audio_off = nullptr;
    std::vector<int> bound_streams;     // what the tables hold, per row
    std::vector<int64_t> bound_offs;
    int *d_pos = nullptr, *d_outpos = nullptr, *d_tok = nullptr, *d_ids = nullptr, *d_out = nullptr;
    int out_ld = 0;     // row pitch of d_out and of the per-output buffers: kv.capacity()
    int cache_len = 0;  // host mirror of d_pos[] (all rows equal) for the incremental API
    // the stream of each decoder row while a transcribe call runs whose rows are not its streams in order (beams, a
    // ragged call's sorted streams), or the slot of each row of a stream pool's launch; empty: row r belongs to stream r
    std::vector<int> row_streams;
    // token scores, beam search, phrase boosting and the record of the last call's results (token_select.h)
    TokenSelect sel;
    // sel.set_bias, and a new binding of rows once it has created the row table
    void set_bias(int stream, const int32_t *ids, const int32_t *lens, const float *boosts, int n);
    // host mirror of d_outpos[] (the stream pool's session aside): outputs per row since reset (incremental calls /
    // transcribe)
    std::vector<int> out_rows;
    StepGraph step_graph;   // the offline transcription's decode step, captured once per key and replayed
    bool use_graph = true;
    // scratch of the fused decode path: split-K partials + tickets, per-tile sums of squares of the
    // residual stream (consumed by the next kernel's fused RMSNorm), multi-CTA argmax scratch
    TcWork tc_split;  // split-K only; tc_work() adds the sums of squares
    float *ssq_x = nullptr;
    float *am_vals = nullptr;
    int *am_idx = nullptr, *am_cnt = nullptr;
    TcWork tc_work(bool norm_in, bool ssq_out) const;
    // persistent decode-step kernel (decode_mega.h): its op table, scratch, launches and step epoch.  VOX_MEGA=0 (or
    // debug "mega_off") selects the per-op launches.
    bool use_mega = true;
    DecodeMega mega;
    bool fused_decode(int rows) const;
    void *xt_buf = nullptr;   // f16 split tiles feeding the wgmma GEMM
    size_t xt_elems = 0;
    GemmWork gemm_work;       // split-K scratch of the wgmma GEMM
    // tensor-core matvec for M <= 8 (VOX_MATVEC=simt disables), wgmma GEMM for M > 8 (VOX_GEMM=simt disables)
    Q4Path path;

    // kv_ring: each row's decoder KV is a ring of pages (DecoderKv::create), and positions are unbounded (stream pools
    // with no length limit; the pool owner points dec_rope at its RoPE ring)
    // kv_type: element type of the decoder KV cache
    static Session *create(Model *m, int max_batch, int max_mel_frames, bool kv_ring = false, KvType kv_type = KvType::F32);
    ~Session();
    // every stream at `delay` (tokens of 80 ms)
    void set_delay(float delay);
    // stream i at delays[i] for i < b; streams >= b keep theirs
    void set_delays(const float *delays, int b);
    void set_stream_delay(int stream, float delay);
    // the per-row tables of launches over rows [0, B), as row_streams maps them to streams: each row's stream's ADA set
    // and audio offset.  Runs at the start of every prefill, decode step and teacher-forced pass.  Launch-free, and
    // copy-free when no row's stream or offset has changed (so it may run inside a stream capture); a delay change
    // rewrites the sets in place and needs no new binding.
    void bind_rows(int B);
    // launch_q4_linear with the session's GEMM scratch and path choice; `gamma`, `tmp`, `tc` and `ada_rows` as there
    void linear(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias, const float *res,
                int epi, const float *gamma = nullptr, float *tmp = nullptr, const TcWork *tc = nullptr,
                const AdaRows &ada_rows = AdaRows{});
    bool decoder_forward(int B, int M);
    void lm_head_rows(int rows, bool norm_pending, float *dst);
    // teacher-forced pass over ids [b][M] (+ the audio embeddings at positions *d_pos.. when with_audio): logits of every
    // row into dst [b * M][vocab], positions advanced by M
    void forward_logits(int b, int M, const int *ids_host, bool with_audio, float *dst);
    // host-side preparation a decode step over R rows depends on (bind_rows, the persistent kernel's op table); returns the step's persistent-kernel launches, 0 on the per-op path.  Copy- and sync-free when
    // the last step had the same shape, so that it may run under stream capture.
    unsigned prepare_step(int R);
    // returns prepare_step(B), the persistent-kernel launches it issues (mega counts them unless it is capturing)
    unsigned decode_step(int B, bool add_audio = true);
    // `n` decode steps over R rows, each one `step()`: CUDA-graph replay of one captured step when use_graph, else eager
    template <class Step> void run_steps(int R, int n, Step step);
    // generic prefill over ids [B][M] at positions *d_pos.. (+ audio rows when add_audio): KV append, lm_head of the
    // last row, argmax -> d_tok (device feedback) and d_out; advances the device counters
    void prefill(int B, int M, const int *ids_host, bool add_audio);
    // the incremental API after argument validation: vox_prefill over ids_host [b][M], or vox_decode_step (ids_host
    // nullptr, M = 1) over rows [0, b); then advances cache_len, out_rows and the positions vox_session_token_scores
    // reads
    void step_incremental(int b, int M, const int *ids_host, bool add_audio);
    void check_batch(int b) const;
    void check_ids(const int32_t *ids, size_t n) const;
    // encodes the B streams of T mel frames in enc.mel_tm, then runs prefill + loop; returns tokens per stream.  `total`:
    // the getters report the counts over all streams (vox_transcribe_pcm_ragged at equal lengths)
    int transcribe_from_mel(int B, int T, int32_t *out_ids, size_t cap_ids, vox_timings *tm, bool total = false);
    // vox_transcribe_pcm_ragged after its argument checks: b streams of lens[s] host samples, one after the other;
    // n_out[s] ids of stream s after those of stream s - 1 in out_ids.  Records ev[0..4] like the other transcribe calls.
    void transcribe_ragged(const float *samples, const size_t *lens, int b, int normalize, int32_t *out_ids,
                           int32_t *n_out, vox_timings *tm);
    void reset();
    // re-bases the persistent kernel's step epoch once it has advanced far (see reset)
    void rebase_epoch() { mega.rebase_epoch(st); }
};

}  // namespace vox
