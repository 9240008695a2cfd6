// stream.h -- pool of live streaming sessions sharing one GPU worker (stream.cu).
#pragma once
#include <cstdint>
#include <vector>

#include "model.h"

namespace vox {

// Padded audio an unbounded session keeps resident on the device: its PCM, mel, conv1, encoder-output and audio-embedding
// buffers hold this much and slide forward as the session advances.
constexpr float kResidentSeconds = 30.0f;

// K4-S: encoder attention of R rows, each at (session row_slot[r], absolute position row_pos[r]), over the sessions' K/V
// rings kr / vr [slot][ring][H*hd] (position p at p % ring): keys max(0, p - window) .. p.  q of row r at qkv + r * ld,
// out [R][H*hd].  hd in {32, 64, 128}.
void launch_stream_attn(const float *qkv, int R, int ld, int H, int hd, const int *row_slot, const int *row_pos, const float *kr,
                        const float *vr, int ring, int window, float scale, float *out, cudaStream_t st);

struct StreamPool {
    // Counters are absolute (since the session opened).  Every audio-side buffer of a session holds a window of rows
    // starting at absolute row *0 (pcm0, mel0, ...): always 0 in a bounded pool, whose buffers hold the whole stream.
    struct Slot {
        bool open = false, ended = false, drained = false;
        size_t n_samples = 0, n_audio = 0;        // padded samples known so far / audio samples pushed
        int n_mel = 0, n_c1 = 0, n_enc = 0, n_emb = 0;  // final frames produced per stage
        int pos = 0;                              // decoder positions cached (0: prefill pending)
        int last_tok = 0;
        std::vector<int32_t> ids;                 // emitted ids not yet polled
        std::vector<int32_t> top_ids;             // their scores, [ids.size()][s->sel.top_k] (pool top_k > 0)
        std::vector<float> top_lp;
        int64_t n_ids = 0;                        // ids emitted (positions >= 38)
        size_t pcm0 = 0;                          // absolute sample / frame / row of each buffer's row 0
        int mel0 = 0, c10 = 0, enc0 = 0, emb0 = 0;
    };
    Model *m = nullptr;
    Session *s = nullptr;       // private session: weights view, decoder state, workspaces, stream
    vox_pad_config pad{};
    int max_sessions = 0, max_new = 0, ring = 0;
    bool unbounded = false;     // created with max_seconds = 0: no length limit, fixed device state
    size_t cap_samples = 0;
    float *pcm = nullptr;       // [slot][cap_samples] padded signal
    float *enc_out = nullptr;   // [slot][S_max][enc_dim] encoder output frames (after the final norm)
    float *ek = nullptr, *ev = nullptr;  // encoder K/V rings [layer][slot][ring][H*hd], absolute position p at p % ring
    // unbounded pools: encoder RoPE rows [slot][ring][hd/2] (position p at p % ring, like the K/V rings) and the
    // decoder's RoPE ring (kernels.h RopeView), filled by the host for the positions each launch computes
    float *enc_rope_cos = nullptr, *enc_rope_sin = nullptr;
    float *dec_rope_cos = nullptr, *dec_rope_sin = nullptr;
    float *slide_tmp = nullptr;  // unbounded pools: bounce buffer of slide() (stream.cu), the size of the largest session buffer
    int *d_row_slot = nullptr, *d_row_pos = nullptr;
    std::vector<Slot> slots;

    // max_seconds in [1, 60]: sessions up to that long, all their state resident.  0: sessions of any length.
    // kv_type: element type of the decoder KV pages every session of the pool shares (Session::create)
    static StreamPool *create(Model *m, int max_sessions, float max_seconds, KvType kv_type = KvType::F32);
    ~StreamPool();
    int open();   // the new session runs at kDefaultDelay
    // the session's transcription delay (its own ADA set); only before its prefill has run
    void set_delay(int id, float delay);
    // session id's phrase list (Session::set_bias on its slot); open() empties it, and its prefill clears its history
    void set_bias(int id, const int32_t *ids, const int32_t *lens, const float *boosts, int n);
    void push(int id, const float *samples, size_t n);
    void finish(int id);
    void close(int id);
    void tick(vox_stream_stats *stats);
    // token confidences of every session (one batched step serves them all): only while no session is open
    void set_top_k(int k);
    // up to `cap` ids (and, when top_ids / top_lp are given, their [n][top_k] scores); what is returned is dropped
    size_t poll(int id, int32_t *ids, int32_t *top_ids, float *top_lp, size_t cap, bool *done);
    const float *audio_embeds(int id, int *n);   // device pointer [n][dec_dim]; fails once rows were evicted
    // device pointer to resident audio embeddings [first, first + n)
    const float *audio_embeds_range(int id, int64_t first, int64_t n);
    // device pointer to resident log-mel frames [first, first + n), [n][n_mels]
    const float *mel_range(int id, int64_t first, int64_t n);
    void session_info(int id, struct vox_stream_session_info *out);
    // encode_audio_with_cache (model.rs:790-799): one mel chunk [128][T] (host) through the conv stem ON ITS OWN (zero
    // padding at the chunk edges, as upstream) and the encoder layers over the session's K/V rings; returns the
    // chunk's S/4 audio embeddings (host, [n][dec_dim]).  For sessions driven chunk-wise instead of push()/tick().
    int encode_chunk(int id, const float *mel, int T, float *out, size_t cap_floats);

  private:
    Slot &slot(int id);
    void encoder_rows(int R);
    void upload_rows(const std::vector<int> &rows, bool with_tokens);
    void append_scores(Slot &sl, const int32_t *top_ids, const float *top_lp);
    int final_enc(const Slot &sl) const;
    void fill_rope(float *cos_d, float *sin_d, int hd, int rows, size_t row0, int64_t p0, int n);
};

}  // namespace vox
