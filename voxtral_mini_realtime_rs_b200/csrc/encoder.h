// encoder.h -- host side of the audio encoder (encoder.cu): PCM front end, conv stem, encoder layers, x4 reshape and
// adapter, with the workspace they run in and the audio embeddings they leave for the decoder.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <functional>
#include <vector>

#include "common.h"

namespace vox {

struct DeviceArena;
struct Model;
struct Session;

// What a transcribe call makes of one stream of n samples: the padded length (pad_audio), mel frames, audio positions
// after the two stride-2 convolutions and the reshape, and decoder outputs (positions after the prefix; 0 when shorter).
struct StreamGeom {
    size_t padded = 0;
    int frames = 0, S = 0, S4 = 0, n_out = 0;
};
StreamGeom stream_geometry(const vox_model_info &c, size_t n);

// A session's audio encoder.  Its buffers hold max_batch streams of up to max_mel_frames mel frames, uniform or packed
// one after the other; a stream pool uses them as one fixed region per slot instead (slot_mel, slot_conv1, slot_audio).
struct AudioEncoder {
    // the buffers from `arena` for max_batch streams of up to max_mel_frames frames; VOX_ENC_ATTN=simt selects the SIMT
    // encoder attention
    void create(DeviceArena &arena, const Model &m, int max_batch, int max_mel_frames);

    // PCM front end of b streams of lens[s] samples, in two steps around the caller's start event.  prepare_pcm sizes
    // the signal buffers (the input one only for host samples) and records `front`; pcm_to_mel copies host samples in
    // (one stream after the other), or reads device samples `dev` laid out the same way, then peak-normalises (when
    // `normalize`), pads and computes each stream's mel into mel_tm, packed one after the other.  Equal lengths run as
    // one batch, stream s's padded signal at s * padded; other lengths stream by stream, each padded signal 16-byte
    // aligned.
    void prepare_pcm(Session &s, const size_t *lens, int b, bool host);
    void pcm_to_mel(Session &s, const float *host, const float *dev, const size_t *lens, int b, int normalize);
    // a caller's mel [b][128][t] (host) into `mel` and its time-major copy into mel_tm; checks b and t first
    void upload_mel(Session &s, const float *mel, int b, int t);

    // Q4VoxtralModel::encode_audio (model.rs:783-788) of b streams of T[s] mel frames packed one after the other in
    // mel_tm: conv -> layers -> norm -> reshape x4 -> adapter into `audio`, stream after stream (audio_offs).  Equal
    // frame counts run as one batch.  Otherwise the convolutions run per stream (their zero padding is at each
    // stream's own ends), the layers' linears over all rows at once, RoPE and attention read the segment table d_seg,
    // and each stream keeps its own S / 4 embeddings: work follows the sum of the lengths, not b x the longest.
    void encode(Session &s, int b, const int *T);
    // The encoder layers over `rows` rows of x_enc, then the final norm into h_enc.  attn(layer) is the step between
    // the layer's wqkv and wo: RoPE and attention from qkv_enc into attn_enc.
    void layers(Session &s, int rows, const std::function<void(int)> &attn);
    // adapter0 with GELU into adapter_h, then adapter2 into dst: n rows of x4-stacked encoder frames to embeddings
    void adapt(Session &s, const float *src, int n, float *dst);
    // debug capture of the conv output and every layer's output (debug "capture_on"): allocated the first time
    void set_capture(Session &s, bool on);

    // a stream pool's slot `id`: its mel frames [max_mel_frames][n_mels], conv1 frames [T1_max][enc_dim] and audio
    // embeddings [S4_max][dec_dim]; set_slot_offset points the slot's decoder rows at its embeddings when the first
    // resident one is position `first` (negative offsets once the window has slid past position 0)
    float *slot_mel(int id) const;
    float *slot_conv1(int id) const;
    float *slot_audio(int id) const;
    void set_slot_offset(int id, int64_t first);

    const Model *m = nullptr;
    int max_batch = 0, max_mel_frames = 0;
    int T1_max = 0, S_max = 0, S4_max = 0;   // conv1 frames, encoder rows and audio positions of max_mel_frames
    bool use_attn_tc = true;                  // tensor-core encoder attention (debug "enc_attn_simt" / "enc_attn_tc")
    // front end
    float *pcm = nullptr, *pcm_pad = nullptr, *peak_scale = nullptr;
    size_t pcm_cap = 0, pcm_pad_cap = 0;
    float *mel = nullptr;     // [B][128][T] as handed in by callers (reference layout)
    float *mel_tm = nullptr;  // [B][T][128] time-major copy consumed by the conv1 implicit GEMM
    // front end of the last call that started from PCM or from a caller's mel, for the "mel" / "pcm_pad" debug reads:
    // per stream its mel frames (packed one after the other in mel_tm) and, from PCM, its padded length and offset in
    // pcm_pad; a mel call leaves `padded` empty and its [B][128][T] input in `mel`
    struct FrontEnd {
        std::vector<int> frames;
        std::vector<size_t> padded, pad_off;
    } front;
    // workspace
    float *h1 = nullptr, *x_enc = nullptr, *h_enc = nullptr, *qkv_enc = nullptr, *attn_enc = nullptr, *act_enc = nullptr;
    float *packed = nullptr, *adapter_h = nullptr;
    int *d_seg = nullptr;       // [max_batch + 1] encoder row of each stream's first frame (packed streams)
    std::vector<int> seg_host;
    // output: stream s's audio embedding of position p is at audio + audio_offs[s] + p * dec_dim, for the streams of the
    // last encode or the slots of a stream pool.  Read on the host only (argument checks, debug reads): `positions`
    // every stream of the last encode has embeddings for, its encoder rows, and its embeddings, all streams together.
    float *audio = nullptr;
    std::vector<int64_t> audio_offs;
    int positions = 0, rows = 0, audio_n = 0;
    // debug capture: [enc_layers][rows][enc_dim] and [rows][enc_dim] of the last encode
    bool capture = false;
    float *dbg_layers = nullptr, *dbg_conv = nullptr;

  private:
    void reserve_pcm(Session &s, size_t in_floats, size_t padded_floats);   // grows pcm / pcm_pad to hold that much
    void rope_attention(Session &s, int rows, int B, int S, const int *seg);
};

}  // namespace vox
