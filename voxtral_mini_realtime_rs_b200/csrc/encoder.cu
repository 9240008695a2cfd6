// encoder.cu -- host side of the audio encoder: buffers, PCM front end, encode and adapter (no kernels of its own).
#include "encoder.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <string>

#include "model.h"

namespace vox {

static int conv_out(int t) { return (t + 2 - 3) / 2 + 1; }  // conv.rs:47-48

StreamGeom stream_geometry(const vox_model_info &c, size_t n) {
    vox_pad_config pc;
    pad_config_default(&pc);
    StreamGeom g;
    g.padded = pad_audio_len(n, pc);
    const size_t frames = mel_num_frames(g.padded);
    g.frames = (int)std::min(frames, (size_t)1 << 30);
    g.S = conv_out(conv_out(g.frames));
    g.S4 = g.S / c.reshape_factor;
    g.n_out = std::max(0, g.S4 - c.prefix_len);
    return g;
}

void AudioEncoder::create(DeviceArena &arena, const Model &model, int max_batch_, int max_mel_frames_) {
    const vox_model_info &c = model.info;
    m = &model;
    max_batch = max_batch_;
    max_mel_frames = max_mel_frames_;
    T1_max = conv_out(max_mel_frames);
    S_max = conv_out(T1_max);
    S4_max = S_max / c.reshape_factor;
    VOX_CHECK(S_max <= m->enc_rope_len, VOX_EINVAL, "max_mel_frames %d exceeds the encoder RoPE table", max_mel_frames);
    const size_t B = max_batch;
    const int hdq = c.enc_heads * c.enc_head_dim;
    mel = arena.alloc_n<float>(B * c.n_mels * max_mel_frames);
    mel_tm = arena.alloc_n<float>(B * c.n_mels * max_mel_frames);
    peak_scale = arena.alloc_n<float>(B);
    h1 = arena.alloc_n<float>(B * T1_max * c.enc_dim);
    const size_t rows_max = B * S_max;
    x_enc = arena.alloc_n<float>(rows_max * c.enc_dim);
    h_enc = arena.alloc_n<float>(rows_max * c.enc_dim);
    qkv_enc = arena.alloc_n<float>(rows_max * 3 * hdq);
    attn_enc = arena.alloc_n<float>(rows_max * hdq);
    act_enc = arena.alloc_n<float>(rows_max * c.enc_ffn);
    const size_t rows4 = B * std::max(S4_max, 1);
    packed = arena.alloc_n<float>(rows4 * c.enc_dim * c.reshape_factor);
    adapter_h = arena.alloc_n<float>(rows4 * c.dec_dim);
    audio = arena.alloc_n<float>(rows4 * c.dec_dim);
    d_seg = arena.alloc_n<int>(B + 1);
    const char *av = getenv("VOX_ENC_ATTN");
    use_attn_tc = !(av && std::string(av) == "simt");
}

void AudioEncoder::reserve_pcm(Session &s, size_t in_floats, size_t padded_floats) {
    if (in_floats > pcm_cap) {
        pcm = s.arena.alloc_n<float>(in_floats);
        pcm_cap = in_floats;
    }
    if (padded_floats > pcm_pad_cap) {
        pcm_pad = s.arena.alloc_n<float>(padded_floats);
        pcm_pad_cap = padded_floats;
    }
}

static bool equal_lengths(const size_t *lens, int b) {
    return std::all_of(lens, lens + b, [&](size_t n) { return n == lens[0]; });
}

void AudioEncoder::prepare_pcm(Session &s, const size_t *lens, int b, bool host) {
    const bool uniform = equal_lengths(lens, b);
    FrontEnd f;
    size_t in = 0, pad = 0;
    for (int i = 0; i < b; ++i) {
        const StreamGeom g = stream_geometry(m->info, lens[i]);
        f.frames.push_back(g.frames);
        f.padded.push_back(g.padded);
        f.pad_off.push_back(pad);
        in += lens[i];
        pad += uniform ? g.padded : (g.padded + 3) / 4 * 4;   // packed: each stream's padded signal 16-byte aligned
    }
    reserve_pcm(s, host ? in : 0, pad);
    front = std::move(f);
}

void AudioEncoder::pcm_to_mel(Session &s, const float *host, const float *dev, const size_t *lens, int b, int normalize) {
    const MelTables &t = m->mel;
    const int n_mels = m->info.n_mels;
    vox_pad_config pc;
    pad_config_default(&pc);
    const size_t left = pad_left(pc);
    const std::vector<int> &T = front.frames;
    const std::vector<size_t> &padded = front.padded, &pad_off = front.pad_off;
    const float *src = dev;
    if (host) {
        size_t in = 0;
        for (int i = 0; i < b; ++i) in += lens[i];
        CUDA_OK(cudaMemcpyAsync(pcm, host, sizeof(float) * in, cudaMemcpyHostToDevice, s.st));
        src = pcm;
    }
    if (equal_lengths(lens, b)) {
        launch_peak_normalize_pad(src, b, lens[0], 0.95f, normalize, pcm_pad, padded[0], left, peak_scale, s.st);
        launch_mel(pcm_pad, b, padded[0], padded[0], t.window, t.fb_vals, t.fb_start, t.fb_len, t.fb_stride, mel_tm, T[0], 0,
                   s.st);
        return;
    }
    for (int i = 0, t0 = 0; i < b; src += lens[i], t0 += T[i], ++i) {
        launch_peak_normalize_pad(src, 1, lens[i], 0.95f, normalize, pcm_pad + pad_off[i], padded[i], left, peak_scale + i,
                                  s.st);
        launch_mel(pcm_pad + pad_off[i], 1, padded[i], padded[i], t.window, t.fb_vals, t.fb_start, t.fb_len, t.fb_stride,
                   mel_tm + (size_t)t0 * n_mels, T[i], 0, s.st);
    }
}

void AudioEncoder::upload_mel(Session &s, const float *host_mel, int b, int t) {
    const int n_mels = m->info.n_mels;
    s.check_batch(b);
    VOX_CHECK(t >= 1 && t <= max_mel_frames, VOX_EINVAL, "mel frames %d exceed session max_mel_frames %d", t, max_mel_frames);
    CUDA_OK(cudaSetDevice(m->device));
    front.frames.assign(b, t);
    front.padded.clear();
    front.pad_off.clear();
    CUDA_OK(cudaMemcpyAsync(mel, host_mel, sizeof(float) * (size_t)b * n_mels * t, cudaMemcpyHostToDevice, s.st));
    launch_transpose_mel(mel, mel_tm, b, n_mels, t, s.st);
}

void AudioEncoder::layers(Session &s, int n_rows, const std::function<void(int)> &attn) {
    const vox_model_info &c = m->info;
    const int d = c.enc_dim;
    for (int i = 0; i < c.enc_layers; ++i) {
        const EncLayerW &l = m->enc[i];
        s.linear(l.wqkv, x_enc, n_rows, qkv_enc, 3 * c.enc_heads * c.enc_head_dim, l.bqkv, nullptr, EPI_NONE, l.attn_norm, h_enc);
        attn(i);
        s.linear(l.wo, attn_enc, n_rows, x_enc, d, l.bo, x_enc, EPI_RESIDUAL);
        s.linear(l.w13, x_enc, n_rows, act_enc, c.enc_ffn, nullptr, nullptr, EPI_SILU_MUL, l.ffn_norm, h_enc);
        s.linear(l.w2, act_enc, n_rows, x_enc, d, l.b2, x_enc, EPI_RESIDUAL);
        if (capture && dbg_layers)
            CUDA_OK(cudaMemcpyAsync(dbg_layers + (size_t)i * n_rows * d, x_enc, sizeof(float) * n_rows * d,
                                    cudaMemcpyDeviceToDevice, s.st));
    }
    launch_rmsnorm(x_enc, m->enc_norm, h_enc, n_rows, d, m->norm_eps, s.st);
}

// RoPE and attention of B streams of up to S rows each: one after the other S rows apart, or, with a segment table
// `seg` (device, [B + 1]), packed at seg[b]
void AudioEncoder::rope_attention(Session &s, int n_rows, int B, int S, const int *seg) {
    const vox_model_info &c = m->info;
    const int H = c.enc_heads, hd = c.enc_head_dim, hdq = H * hd;
    const float scale = powf((float)hd, -0.5f);
    launch_rope_inplace(qkv_enc, n_rows, 3 * hdq, 0, H, hdq, H, hd, S, 0, m->enc_cos, m->enc_sin, s.st, seg, seg ? B : 0);
    const bool tc = use_attn_tc && enc_attention_tc_supported(hd, 3 * hdq, 0, hdq, 2 * hdq);
    (tc ? launch_enc_attention_tc : launch_enc_attention)(qkv_enc, attn_enc, B, S, H, hd, 3 * hdq, 0, hdq, 2 * hdq, c.enc_window,
                                                          scale, s.st, seg);
}

void AudioEncoder::encode(Session &s, int b, const int *T) {
    const vox_model_info &c = m->info;
    s.check_batch(b);
    for (int i = 0; i < b; ++i)
        VOX_CHECK(T[i] >= 1 && T[i] <= max_mel_frames, VOX_EINVAL, "mel frames %d exceed session max_mel_frames %d", T[i],
                  max_mel_frames);
    const int d = c.enc_dim, f = c.reshape_factor, D = c.dec_dim;
    const bool uniform = std::all_of(T, T + b, [&](int t) { return t == T[0]; });
    std::vector<int> T1(b), S(b), S4(b);
    seg_host.assign(b + 1, 0);
    audio_offs.resize(b);
    int S_long = 0, sum_T = 0, n = 0, S4_short = S4_max;
    for (int i = 0; i < b; ++i) {
        T1[i] = conv_out(T[i]);
        S[i] = conv_out(T1[i]);
        S4[i] = S[i] / f;
        seg_host[i + 1] = seg_host[i] + S[i];
        S_long = std::max(S_long, S[i]);
        S4_short = std::min(S4_short, S4[i]);
        sum_T += T[i];
        audio_offs[i] = (int64_t)n * D;
        n += S4[i];
    }
    const int n_rows = seg_host[b];
    // b <= max_batch streams of <= max_mel_frames frames: the scratch create() sized for max_batch uniform streams holds
    // them packed
    if (!(sum_T <= max_batch * max_mel_frames && n_rows <= max_batch * S_max))
        fail(VOX_EINVAL, "encode: packed streams exceed the session scratch");
    if (uniform) {
        // conv1 + GELU as implicit GEMM over the time-major mel [B][T][128] (K = 3*128)
        launch_conv2_gemm(mel_tm, m->conv1_w, m->conv1_b, h1, b, T[0], T1[0], c.n_mels, d, s.st);
        launch_conv2_gemm(h1, m->conv2_w, m->conv2_b, x_enc, b, T1[0], S[0], d, d, s.st);
    } else {
        CUDA_OK(cudaMemcpyAsync(d_seg, seg_host.data(), sizeof(int) * (b + 1), cudaMemcpyHostToDevice, s.st));
        for (int i = 0, t0 = 0, t1 = 0; i < b; t0 += T[i], t1 += T1[i], ++i) {
            launch_conv2_gemm(mel_tm + (size_t)t0 * c.n_mels, m->conv1_w, m->conv1_b, h1 + (size_t)t1 * d, 1, T[i], T1[i],
                              c.n_mels, d, s.st);
            launch_conv2_gemm(h1 + (size_t)t1 * d, m->conv2_w, m->conv2_b, x_enc + (size_t)seg_host[i] * d, 1, T1[i], S[i], d,
                              d, s.st);
        }
    }
    if (capture && dbg_conv)
        CUDA_OK(cudaMemcpyAsync(dbg_conv, x_enc, sizeof(float) * n_rows * d, cudaMemcpyDeviceToDevice, s.st));
    const int *seg = uniform ? nullptr : d_seg;
    layers(s, n_rows, [&](int) { rope_attention(s, n_rows, b, S_long, seg); });
    rows = n_rows;
    positions = S4_short;
    audio_n = n;
    if (n == 0) return;
    if (uniform) {
        launch_reshape_rows(h_enc, packed, b, S[0], S4[0], d, f, s.st);
    } else {
        for (int i = 0, o = 0; i < b; o += S4[i], ++i)
            launch_reshape_rows(h_enc + (size_t)seg_host[i] * d, packed + (size_t)o * d * f, 1, S[i], S4[i], d, f, s.st);
    }
    adapt(s, packed, n, audio);
}

void AudioEncoder::adapt(Session &s, const float *src, int n, float *dst) {
    const int D = m->info.dec_dim;
    s.linear(m->adapter0, src, n, adapter_h, D, nullptr, nullptr, EPI_GELU);
    s.linear(m->adapter2, adapter_h, n, dst, D, nullptr, nullptr, EPI_NONE);
}

void AudioEncoder::set_capture(Session &s, bool on) {
    const vox_model_info &c = m->info;
    if (on && !dbg_layers) {
        dbg_layers = s.arena.alloc_n<float>((size_t)c.enc_layers * max_batch * S_max * c.enc_dim);
        dbg_conv = s.arena.alloc_n<float>((size_t)max_batch * S_max * c.enc_dim);
    }
    capture = on;
}

float *AudioEncoder::slot_mel(int id) const { return mel_tm + (size_t)id * max_mel_frames * m->info.n_mels; }
float *AudioEncoder::slot_conv1(int id) const { return h1 + (size_t)id * T1_max * m->info.enc_dim; }
float *AudioEncoder::slot_audio(int id) const { return audio + (size_t)id * S4_max * m->info.dec_dim; }

void AudioEncoder::set_slot_offset(int id, int64_t first) {
    audio_offs.resize(max_batch);   // a stream pool's session never encodes: one offset per slot
    audio_offs[id] = ((int64_t)id * S4_max - first) * m->info.dec_dim;
}

}  // namespace vox
