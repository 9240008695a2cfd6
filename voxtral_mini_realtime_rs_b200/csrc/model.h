// model.h -- Q4 Voxtral model resident in HBM + per-session state.
// Mirrors Q4ModelLoader (reference src/gguf/loader.rs) and Q4VoxtralModel (src/gguf/model.rs).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>
#include <vector>

#include "audio_host.h"
#include "gguf.h"
#include "decode_mega.h"
#include "kernels.h"

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

    static Model *load(const Gguf &g, int device);
};

// Repack raw GGUF Q4_0 blocks of one or more [N_i, K] matrices into the device layout.
// interleave=true: two parts with equal N, rows (2i, 2i+1) = (a_i, b_i).
Q4Weight upload_q4(DeviceArena &arena, const std::vector<const uint8_t *> &raw, const std::vector<int> &n_rows,
                   int K, bool interleave, bool tc_layout = false);

struct Session {
    Model *m = nullptr;
    int max_batch = 0, max_mel_frames = 0;
    int T1_max = 0, S_max = 0, S4_max = 0, M_max = 0;
    cudaStream_t st = nullptr;
    DeviceArena arena;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    // audio
    float *pcm = nullptr, *pcm_pad = nullptr, *peak_scale = nullptr;
    size_t pcm_cap = 0, pcm_pad_cap = 0;
    float *mel = nullptr;     // [B][128][T] as handed in by callers (reference layout)
    float *mel_tm = nullptr;  // [B][T][128] time-major copy consumed by the conv1 implicit GEMM
    // encoder workspace
    float *h1 = nullptr, *x_enc = nullptr, *h_enc = nullptr, *qkv_enc = nullptr, *attn_enc = nullptr, *act_enc = nullptr;
    float *packed = nullptr, *adapter_h = nullptr, *audio = nullptr;
    int cur_B = 0, cur_S = 0, cur_S4 = 0;
    // decoder
    // decoder KV cache: page pools [L][n_pages][Hkv][KV_PAGE][hd] + per-row page tables (kernels.h KvView).  Whole-
    // utterance batches use the identity mapping (row b owns pages b*max_pages..); streaming sessions allocate pages
    float *kc = nullptr, *vc = nullptr;
    int kv_max_pages = 0, kv_n_pages = 0;
    int *d_page_table = nullptr;          // [max_batch][kv_max_pages]
    std::vector<int> page_table_host;
    size_t kv_layer_stride() const { return (size_t)kv_n_pages * m->info.dec_kv_heads * KV_PAGE * m->info.dec_head_dim; }
    KvView kv_view(int layer) const;
    float *x_dec = nullptr, *h_dec = nullptr, *qkv_dec = nullptr, *attn_dec = nullptr, *act_dec = nullptr;
    float *last_h = nullptr, *logits = nullptr;
    float *logits_all = nullptr;
    size_t logits_all_cap = 0;
    float *ada = nullptr, *t_embed = nullptr, *ada_tmp = nullptr;
    float *ffn_gamma_ada = nullptr;  // [L][D] ffn_norm weight x ADA scale (persistent decode kernel)
    bool delay_set = false;
    int *d_pos = nullptr, *d_outpos = nullptr, *d_tok = nullptr, *d_ids = nullptr, *d_out = nullptr;
    int out_ld = 0;
    int cache_len = 0;  // host mirror of d_pos[] (all rows equal) for the incremental API
    // streaming pool (stream.cu): rows of a step belong to sessions of different ages -- no d_out history, audio
    // embeddings through a per-row pointer table (decode) or a per-launch base pointer (single-session prefill)
    bool stream_mode = false;
    const float *const *audio_rows_dev = nullptr;
    const float *audio_base = nullptr;
    cudaGraphExec_t step_graph = nullptr;
    int step_graph_B = 0, step_graph_S4 = 0;
    uint64_t step_graph_nodes = 0;
    bool use_graph = true;
    // scratch of the fused decode path: split-K partials + tickets, per-tile sums of squares of the
    // residual stream (consumed by the next kernel's fused RMSNorm), multi-CTA argmax scratch
    float *tc_partial = nullptr;
    size_t tc_partial_floats = 0;
    int *tc_counters = nullptr;
    int tc_n_counters = 0;
    float *ssq_x = nullptr;
    float *am_vals = nullptr;
    int *am_idx = nullptr, *am_cnt = nullptr;
    TcWork tc_work(bool norm_in, bool ssq_out) const;
    // persistent decode-step kernel (decode_mega.cu): op table per batch size, grid barrier words,
    // per-CTA argmax candidates.  VOX_MEGA=0 (or debug "mega_off") selects the per-op launches.
    bool use_mega = true;
    int mega_min_B = 1;  // smallest batch that uses the persistent kernel (every batch size does)
    int mega_B = 0, mega_grid = 0, mega_n_ops = 0, mega_ops_cap = 0;
    MegaPlan mega_plan;
    std::vector<MegaOp> mega_ops_host;
    MegaOp *mega_ops = nullptr;
    unsigned *mega_bar = nullptr;
    float *mega_am_vals = nullptr;
    int *mega_am_idx = nullptr;
    float *mega_att_acc = nullptr, *mega_att_ml = nullptr;  // key-chunk softmax states (MG_ATTN -> MG_ATTN_MERGE)
    int mega_att_units = 0;
    int *mega_att_flags = nullptr, *mega_epoch = nullptr;
    unsigned mega_steps_host = 0;  // decode steps since the device epoch was last re-based (Session::reset)
    // activation fragments (decode_mega.cu frag_build): residual stream x norm weight, attention output, SwiGLU output
    uint2 *mega_xf_bf = nullptr, *mega_af_bf = nullptr, *mega_cf_bf = nullptr;
    float2 *mega_xf_off = nullptr, *mega_af_off = nullptr, *mega_cf_off = nullptr;
    size_t mega_xf_blocks = 0, mega_af_blocks = 0, mega_cf_blocks = 0;
    unsigned long long *mega_trace_w = nullptr;    // [16][6][8] (debug "mega_trace_w", VOX_MEGA_TRACE_ALL=1)
    unsigned long long *mega_trace_all = nullptr;  // [grid][mega_ops_cap][4] (debug "mega_trace_all", VOX_MEGA_TRACE_ALL=1)
    unsigned long long *mega_trace = nullptr;  // [mega_ops_cap][6] SM-clock stamps of CTA 0 (debug "mega_trace")
    bool mega_prepare(int B);
    bool fused_decode(int rows) const;
    void decode_step_mega(int b0, int B, bool add_audio);
    void *xt_buf = nullptr;   // f16 split tiles feeding the wgmma GEMM
    size_t xt_elems = 0;
    GemmWork gemm_work;       // split-K scratch of the wgmma GEMM
    bool use_enc_attn_tc = true;  // tensor-core encoder attention (VOX_ENC_ATTN=simt disables)
    bool use_gemm_tc = true;  // wgmma GEMM for M > 8 (VOX_GEMM=simt disables)
    // y = epi(norm(x) . W^T): RMSNorm fused into the operand split when the wgmma path applies,
    // else rmsnorm into `tmp` + linear()
    void linear_n(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias, const float *res, int epi,
                  const float *gamma, const float *ada, float *tmp);
    bool use_tc = true;  // tensor-core-assisted matvec for M <= 8 (VOX_MATVEC=simt disables)
    std::vector<float> enc_debug;  // per-layer captures when debugging is enabled
    bool debug_capture = false;
    float *dbg_layers = nullptr;   // [enc_layers][B*S][enc_dim]
    float *dbg_conv = nullptr;

    static Session *create(Model *m, int max_batch, int max_mel_frames);
    ~Session();
    void set_delay(float delay);
    // mel already on device, time-major, in s->mel_tm
    void encode(int B, int T);
    void linear(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias, const float *res,
                int epi);
    bool decoder_forward(int B, int M);
    void lm_head_rows(int rows, bool norm_pending, float *dst);
    void decode_step(int B, bool add_audio = true);
    // generic prefill over ids [B][M] at positions *d_pos.. (+ audio rows when add_audio): KV append, lm_head of the
    // last row, argmax -> d_tok (device feedback) and d_out; advances the counters
    void prefill(int B, int M, const int *ids_host, bool add_audio);
    // runs prefill + loop; returns tokens per stream
    int transcribe_from_mel(int B, int T, int32_t *out_ids, size_t cap_ids, vox_timings *tm, bool timed_pre);
    void reset();
};

}  // namespace vox
