// stream.cu -- true streaming sessions (SURVEY 8(f)-1): audio arrives in arbitrary pieces, every stage advances as far
// as its inputs are final, and every token is emitted as soon as it can be -- with the ids of the whole-utterance
// transcribe_streaming (reference src/gguf/model.rs:873-963).  The reference ships the building blocks but no driver:
//   Q4AudioEncoder::forward_with_cache   model.rs:437-452   (encoder layers over a KV cache)
//   encode_audio_with_cache              model.rs:790-799
//   KVCache::apply_sliding_window        kv_cache.rs:176-203 (unused upstream; it would re-base positions)
// What a session carries (the test-side incremental restatement tests/test_oracle_streaming.py checks derives the table):
//   samples (the padded signal so far) -> log-mel frames (final once samples < 160 i + 200 are known) -> conv1 / conv2
//   frames (k3 s2 p1: output t needs input 2t+1) -> 32 encoder layers over a per-layer K/V RING of window + slack
//   positions (absolute positions for RoPE and the causal / sliding-window masks; keys older than the window are simply
//   overwritten) -> x4 frame stack + adapter -> one decoder position per 160 ms of audio, greedy ids.
// Unbounded pools (max_seconds = 0) keep every stage's state fixed: the audio-side buffers are windows that slide
// forward (slide() below), the decoder KV of a session is a ring of pages covering the decoder window (kernels.h KvView),
// and RoPE rows come from small ring tables the host fills for the positions in flight.
// Continuous batching: one pool = one GPU worker.  A tick gathers the new encoder frames of ALL live sessions into one
// row batch (the linears do not care which session a row belongs to; RoPE / ring append / attention take a per-row
// (session, absolute position)), and all sessions that can take a decoder step share ONE decode step -- rows at
// different positions, KV pages from one pool (kernels.h KvView).
#include "stream.h"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "common.h"

namespace vox {

namespace {

constexpr int SA_WARPS = 4, SA_THREADS = SA_WARPS * 32;
// rows of an unbounded pool's decoder RoPE ring: rows of one decoder launch must not meet in it (tick() defers a row
// whose position collides with another row's), which is rare with a ring this long
constexpr int kDecRopeRing = 4096;

// RoPE(q) in place, RoPE(k) and v into the row's session ring at slot (pos % ring).  qkv rows [R][3*HQ].
__global__ void stream_rope_append_kernel(float *__restrict__ qkv, const int ld, const int H, const int hd,
                                          const int *__restrict__ row_slot, const int *__restrict__ row_pos, float *__restrict__ kr,
                                          float *__restrict__ vr, const int ring, const float *__restrict__ cos_t,
                                          const float *__restrict__ sin_t, const bool rope_ring) {
    const int r = blockIdx.x;
    const int slot = row_slot[r], pos = row_pos[r];
    const int half = hd >> 1, HQ = H * hd;
    float *row = qkv + (size_t)r * ld;
    // RoPE row: the model's table at `pos`, or (rope_ring) the session's ring row, which sits where its K/V row does
    const size_t rr = rope_ring ? ((size_t)slot * ring + (pos % ring)) * half : (size_t)pos * half;
    const float *cr = cos_t + rr, *sr = sin_t + rr;
    float *kdst = kr + ((size_t)slot * ring + (pos % ring)) * HQ;
    float *vdst = vr + ((size_t)slot * ring + (pos % ring)) * HQ;
    for (int i = threadIdx.x; i < H * half; i += blockDim.x) {
        const int h = i / half, p = i - h * half;
        float *q = row + h * hd + 2 * p;
        const float c = cr[p], s = sr[p];
        const float qr = q[0], qi = q[1];
        q[0] = qr * c - qi * s;
        q[1] = qr * s + qi * c;
        const float *k = row + HQ + h * hd + 2 * p;
        kdst[h * hd + 2 * p] = k[0] * c - k[1] * s;
        kdst[h * hd + 2 * p + 1] = k[0] * s + k[1] * c;
    }
    for (int i = threadIdx.x; i < HQ; i += blockDim.x) vdst[i] = row[2 * HQ + i];
}

// Encoder attention of one (head, row) over the session's K/V ring: keys max(0, pos - window) .. pos (causal + sliding
// window with the cache offset, masking.rs:50-107), online softmax per warp, merged through shared memory.
template <int DPL>
__global__ void __launch_bounds__(SA_THREADS)
stream_enc_attn_kernel(const float *__restrict__ qkv, const int ld, const int H, const int *__restrict__ row_slot,
                       const int *__restrict__ row_pos, const float *__restrict__ kr, const float *__restrict__ vr, const int ring,
                       const int window, const float scale, float *__restrict__ out) {
    constexpr int HD = DPL * 32;
    __shared__ float red_m[SA_WARPS], red_l[SA_WARPS];
    __shared__ float red_acc[SA_WARPS][HD];
    const int h = blockIdx.x, r = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slot = row_slot[r], pos = row_pos[r];
    const int HQ = H * HD;
    float q[DPL];
#pragma unroll
    for (int i = 0; i < DPL; ++i) q[i] = qkv[(size_t)r * ld + h * HD + lane * DPL + i];
    float m_run = -INFINITY, l_run = 0.0f, acc[DPL];
#pragma unroll
    for (int i = 0; i < DPL; ++i) acc[i] = 0.0f;
    const int j_lo = pos - window > 0 ? pos - window : 0;
    const float *kb = kr + (size_t)slot * ring * HQ + h * HD + lane * DPL;
    const float *vb = vr + (size_t)slot * ring * HQ + h * HD + lane * DPL;
    for (int j = j_lo + warp; j <= pos; j += SA_WARPS) {
        const size_t at = (size_t)(j % ring) * HQ;
        float kk[DPL], vv[DPL];
#pragma unroll
        for (int i = 0; i < DPL; ++i) {
            kk[i] = kb[at + i];
            vv[i] = vb[at + i];
        }
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < DPL; ++i) s = fmaf(q[i], kk[i], s);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        s *= scale;
        const float m_new = fmaxf(m_run, s);
        const float alpha = expf(m_run - m_new);
        const float p = expf(s - m_new);
        l_run = l_run * alpha + p;
        m_run = m_new;
#pragma unroll
        for (int i = 0; i < DPL; ++i) acc[i] = fmaf(p, vv[i], acc[i] * alpha);
    }
    if (lane == 0) {
        red_m[warp] = m_run;
        red_l[warp] = l_run;
    }
#pragma unroll
    for (int i = 0; i < DPL; ++i) red_acc[warp][lane * DPL + i] = acc[i];
    __syncthreads();
    for (int d = threadIdx.x; d < HD; d += SA_THREADS) {
        float mx = -INFINITY;
#pragma unroll
        for (int w = 0; w < SA_WARPS; ++w) mx = fmaxf(mx, red_m[w]);
        float num = 0.0f, den = 0.0f;
#pragma unroll
        for (int w = 0; w < SA_WARPS; ++w) {
            const float f = (red_m[w] == -INFINITY) ? 0.0f : expf(red_m[w] - mx);
            num = fmaf(red_acc[w][d], f, num);
            den = fmaf(red_l[w], f, den);
        }
        out[(size_t)r * HQ + h * HD + d] = num / den;
    }
}

}  // namespace

void launch_stream_attn(const float *qkv, int R, int ld, int H, int hd, const int *row_slot, const int *row_pos, const float *kr,
                        const float *vr, int ring, int window, float scale, float *out, cudaStream_t st) {
    dim3 grid(H, R);
    switch (hd / 32) {
        case 1: stream_enc_attn_kernel<1><<<grid, SA_THREADS, 0, st>>>(qkv, ld, H, row_slot, row_pos, kr, vr, ring, window, scale, out); break;
        case 2: stream_enc_attn_kernel<2><<<grid, SA_THREADS, 0, st>>>(qkv, ld, H, row_slot, row_pos, kr, vr, ring, window, scale, out); break;
        case 4: stream_enc_attn_kernel<4><<<grid, SA_THREADS, 0, st>>>(qkv, ld, H, row_slot, row_pos, kr, vr, ring, window, scale, out); break;
        default: fail(VOX_EINVAL, "stream attention: unsupported head_dim");
    }
    cuda_check(cudaGetLastError(), "stream_enc_attn launch");
}

namespace {

int conv_out(int t) { return t > 0 ? (t + 2 - 3) / 2 + 1 : 0; }

// Slides a session buffer of `cap` rows of `row` floats whose row 0 is absolute row `base` so that rows up to `end`
// fit: rows [keep, valid) move to the front and `base` becomes `keep`.  Nothing moves while `end` already fits (always,
// in a bounded pool).  Overlapping moves bounce through `tmp` (as large as any session buffer): two copies at most.
// zero_tail: the rows after the moved ones are cleared (the PCM buffer's right padding is read as zeros).
template <typename I>
void slide(float *buf, size_t row, int64_t cap, I &base, int64_t keep, int64_t valid, int64_t end, bool zero_tail, float *tmp,
           cudaStream_t st) {
    if (end - (int64_t)base <= cap) return;
    VOX_CHECK(keep >= (int64_t)base && keep <= valid && end - keep <= cap, VOX_ECAPACITY,
              "stream buffer of %lld rows cannot hold rows %lld..%lld", (long long)cap, (long long)keep, (long long)end);
    const int64_t shift = keep - (int64_t)base, n = valid - keep;
    const size_t bytes = sizeof(float) * (size_t)n * row;
    if (n > 0 && n <= shift) {
        CUDA_OK(cudaMemcpyAsync(buf, buf + (size_t)shift * row, bytes, cudaMemcpyDeviceToDevice, st));
    } else if (n > 0) {
        CUDA_OK(cudaMemcpyAsync(tmp, buf + (size_t)shift * row, bytes, cudaMemcpyDeviceToDevice, st));
        CUDA_OK(cudaMemcpyAsync(buf, tmp, bytes, cudaMemcpyDeviceToDevice, st));
    }
    if (zero_tail) CUDA_OK(cudaMemsetAsync(buf + (size_t)n * row, 0, sizeof(float) * (size_t)(cap - n) * row, st));
    base = (I)keep;
}

// first sample the next mel frame reads (its window starts 200 samples left of 160 t), down to a multiple of 4: the
// mel kernel's aligned interior path needs the buffer start aligned like the signal
size_t pcm_keep(int n_mel) { return (size_t)std::max<int64_t>(0, (int64_t)n_mel * 160 - 200) & ~(size_t)3; }

}  // namespace

// ======================================================================================================
StreamPool *StreamPool::create(Model *m, int max_sessions, float max_seconds, KvType kv_type) {
    VOX_CHECK(max_sessions >= 1 && max_sessions <= 64, VOX_EINVAL, "max_sessions %d out of range [1,64]", max_sessions);
    const bool unbounded = max_seconds == 0.0f;
    VOX_CHECK(unbounded || (max_seconds >= 1.0f && max_seconds <= 60.0f), VOX_EINVAL,
              "max_seconds %.1f out of range [1,60] (encoder RoPE table: %d frames), or 0 for sessions of any length", max_seconds,
              m->enc_rope_len);
    const vox_model_info &c = m->info;
    vox_pad_config pc;
    pad_config_default(&pc);
    StreamPool *p = new StreamPool();
    try {
        p->m = m;
        p->pad = pc;
        p->max_sessions = max_sessions;
        p->unbounded = unbounded;
        p->cap_samples = pad_audio_len((size_t)std::ceil((unbounded ? kResidentSeconds : max_seconds) * 16000.0f), pc);
        const int cap_mel = (int)mel_num_frames(p->cap_samples);
        // unbounded: the frame buffers get a few frames beyond the resident audio for the rows their consumers still read
        p->s = Session::create(m, max_sessions, unbounded ? cap_mel + 16 : cap_mel, unbounded, kv_type);
        Session *s = p->s;
        VOX_CHECK(s->enc.S_max <= m->enc_rope_len, VOX_EINVAL, "max_seconds exceeds the encoder RoPE table");
        p->max_new = 256;
        p->ring = c.enc_window + p->max_new;
        const int HQ = c.enc_heads * c.enc_head_dim;
        const size_t B = max_sessions;
        p->pcm = s->arena.alloc_n<float>(B * p->cap_samples);
        p->enc_out = s->arena.alloc_n<float>(B * s->enc.S_max * c.enc_dim);
        const size_t ring_elems = (size_t)c.enc_layers * B * p->ring * HQ;
        p->ek = s->arena.alloc_n<float>(ring_elems);
        p->ev = s->arena.alloc_n<float>(ring_elems);
        const size_t max_rows = (size_t)B * p->max_new;
        p->d_row_slot = s->arena.alloc_n<int>(max_rows);
        p->d_row_pos = s->arena.alloc_n<int>(max_rows);
        if (unbounded) {
            const size_t enc_rows = B * p->ring * (c.enc_head_dim / 2), dec_rows = (size_t)kDecRopeRing * (c.dec_head_dim / 2);
            p->enc_rope_cos = s->arena.alloc_n<float>(enc_rows);
            p->enc_rope_sin = s->arena.alloc_n<float>(enc_rows);
            p->dec_rope_cos = s->arena.alloc_n<float>(dec_rows);
            p->dec_rope_sin = s->arena.alloc_n<float>(dec_rows);
            s->dec_rope = RopeView{p->dec_rope_cos, p->dec_rope_sin, kDecRopeRing};
            const AudioEncoder &e = s->enc;
            const size_t most = std::max({p->cap_samples, (size_t)e.max_mel_frames * c.n_mels, (size_t)e.T1_max * c.enc_dim,
                                          (size_t)e.S_max * c.enc_dim, (size_t)e.S4_max * c.dec_dim});
            p->slide_tmp = s->arena.alloc_n<float>(most);
        }
        p->slots.resize(max_sessions);
    } catch (...) {
        delete p;
        throw;
    }
    return p;
}

StreamPool::~StreamPool() { delete s; }

int StreamPool::open() {
    for (int i = 0; i < max_sessions; ++i)
        if (!slots[i].open) {
            Slot &sl = slots[i];
            sl = Slot();
            sl.open = true;
            // the left padding of pad_audio (pad.rs:89-93) is part of the stream
            sl.n_samples = pad_left(pad);
            CUDA_OK(cudaSetDevice(m->device));
            CUDA_OK(cudaMemsetAsync(pcm + (size_t)i * cap_samples, 0, sizeof(float) * cap_samples, s->st));
            s->set_stream_delay(i, kDefaultDelay);   // a reused slot does not inherit the previous session's delay ...
            if (s->sel.bias_n[i] > 0) s->set_bias(i, nullptr, nullptr, nullptr, 0);   // ... or its phrase list
            return i;
        }
    fail(VOX_ECAPACITY, fmt("all %d stream sessions are in use", max_sessions));
}

void StreamPool::set_delay(int id, float delay) {
    const Slot &sl = slot(id);
    VOX_CHECK(sl.pos == 0, VOX_EINVAL, "stream session %d: the delay can only change before its prefill has run", id);
    VOX_CHECK(std::isfinite(delay) && delay >= 0.0f, VOX_EINVAL, "delay %g must be finite and >= 0", delay);
    CUDA_OK(cudaSetDevice(m->device));
    s->set_stream_delay(id, delay);
}

void StreamPool::set_bias(int id, const int32_t *ids, const int32_t *lens, const float *boosts, int n) {
    slot(id);
    s->set_bias(id, ids, lens, boosts, n);
}

StreamPool::Slot &StreamPool::slot(int id) {
    VOX_CHECK(id >= 0 && id < max_sessions && slots[id].open, VOX_EINVAL, "stream session %d is not open", id);
    return slots[id];
}

void StreamPool::push(int id, const float *samples, size_t n) {
    Slot &sl = slot(id);
    VOX_CHECK(!sl.ended, VOX_EINVAL, "stream session %d already finished", id);
    const size_t worst = sl.n_samples + n + pad_right(pad, sl.n_samples + n);  // right padding included, should finish() follow
    if (unbounded)
        VOX_CHECK(worst - pcm_keep(sl.n_mel) <= cap_samples, VOX_ECAPACITY,
                  "stream session %d: %zu samples not yet consumed exceed the resident %.0f s; call vox_stream_tick first", id,
                  sl.n_samples + n - pcm_keep(sl.n_mel), kResidentSeconds);
    else
        VOX_CHECK(worst <= cap_samples, VOX_ECAPACITY, "stream session %d: %zu samples exceed the pool's max_seconds", id, sl.n_audio + n);
    CUDA_OK(cudaSetDevice(m->device));
    float *buf = pcm + (size_t)id * cap_samples;
    slide(buf, 1, (int64_t)cap_samples, sl.pcm0, (int64_t)pcm_keep(sl.n_mel), (int64_t)sl.n_samples, (int64_t)worst, true, slide_tmp, s->st);
    if (n) CUDA_OK(cudaMemcpyAsync(buf + (sl.n_samples - sl.pcm0), samples, sizeof(float) * n, cudaMemcpyHostToDevice, s->st));
    CUDA_OK(cudaStreamSynchronize(s->st));  // `samples` is caller memory
    sl.n_samples += n;
    sl.n_audio += n;
}

void StreamPool::finish(int id) {
    Slot &sl = slot(id);
    VOX_CHECK(!sl.ended, VOX_EINVAL, "stream session %d already finished", id);
    sl.n_samples += pad_right(pad, sl.n_samples);  // zeros: the buffer was cleared at open()
    sl.ended = true;
}

void StreamPool::close(int id) {
    Slot &sl = slot(id);
    s->kv.release(id);
    sl = Slot();
}

void StreamPool::set_top_k(int k) {
    for (int i = 0; i < max_sessions; ++i)
        VOX_CHECK(!slots[i].open, VOX_EINVAL, "top_k of a stream pool can only change while no session is open (session %d is)", i);
    s->sel.set_top_k(k);
}

size_t StreamPool::poll(int id, int32_t *ids, int32_t *top_ids, float *top_lp, size_t cap, bool *done) {
    Slot &sl = slot(id);
    const size_t n = std::min(cap, sl.ids.size()), nk = n * (size_t)s->sel.top_k;
    if (n) memcpy(ids, sl.ids.data(), sizeof(int32_t) * n);
    if (nk && top_ids) memcpy(top_ids, sl.top_ids.data(), sizeof(int32_t) * nk);
    if (nk && top_lp) memcpy(top_lp, sl.top_lp.data(), sizeof(float) * nk);
    sl.ids.erase(sl.ids.begin(), sl.ids.begin() + n);  // polled ids are dropped: host memory stays bounded
    sl.top_ids.erase(sl.top_ids.begin(), sl.top_ids.begin() + nk);
    sl.top_lp.erase(sl.top_lp.begin(), sl.top_lp.begin() + nk);
    if (done) *done = sl.ended && sl.drained && sl.ids.empty();
    return n;
}

// Encoder layers over `R` gathered rows in s->enc.x_enc (Q4EncoderLayer::forward_with_cache, model.rs:300-315).
void StreamPool::encoder_rows(int R) {
    const vox_model_info &c = m->info;
    const int HQ = c.enc_heads * c.enc_head_dim;
    const float scale = powf((float)c.enc_head_dim, -0.5f);
    const size_t ring_stride = (size_t)max_sessions * ring * HQ;
    s->enc.layers(*s, R, [&](int i) {
        stream_rope_append_kernel<<<R, 256, 0, s->st>>>(s->enc.qkv_enc, 3 * HQ, c.enc_heads, c.enc_head_dim, d_row_slot, d_row_pos,
                                                        ek + i * ring_stride, ev + i * ring_stride, ring,
                                                        unbounded ? enc_rope_cos : m->enc_cos, unbounded ? enc_rope_sin : m->enc_sin,
                                                        unbounded);
        cuda_check(cudaGetLastError(), "stream_rope_append launch");
        launch_stream_attn(s->enc.qkv_enc, R, 3 * HQ, c.enc_heads, c.enc_head_dim, d_row_slot, d_row_pos, ek + i * ring_stride,
                           ev + i * ring_stride, ring, c.enc_window, scale, s->enc.attn_enc, s->st);
    });
}

// rows[i] = slot id of batch row i: page tables, positions and fed-back tokens of this launch; the rows' slots and
// their audio offsets for the session to bind (Session::bind_rows: ADA sets and audio embeddings)
void StreamPool::upload_rows(const std::vector<int> &rows, bool with_tokens) {
    const int nb = (int)rows.size();
    std::vector<int> pos(nb), tok(nb), zero(nb, 0);
    for (int i = 0; i < nb; ++i) {
        const Slot &sl = slots[rows[i]];
        pos[i] = sl.pos;
        tok[i] = sl.last_tok;
        s->enc.set_slot_offset(rows[i], sl.emb0);
    }
    s->row_streams = rows;
    s->kv.bind(rows, s->st);
    CUDA_OK(cudaMemcpyAsync(s->d_pos, pos.data(), sizeof(int) * nb, cudaMemcpyHostToDevice, s->st));
    CUDA_OK(cudaMemcpyAsync(s->d_outpos, zero.data(), sizeof(int) * nb, cudaMemcpyHostToDevice, s->st));
    if (with_tokens) CUDA_OK(cudaMemcpyAsync(s->d_tok, tok.data(), sizeof(int) * nb, cudaMemcpyHostToDevice, s->st));
    CUDA_OK(cudaStreamSynchronize(s->st));  // the staging vectors die with this frame
}

void StreamPool::tick(vox_stream_stats *st_out) {
    const vox_model_info &c = m->info;
    CUDA_OK(cudaSetDevice(m->device));
    const int d = c.enc_dim, D = c.dec_dim, rf = c.reshape_factor, P = c.prefix_len;
    AudioEncoder &e = s->enc;
    vox_stream_stats stats{};
    s->rebase_epoch();  // between ticks: no decode step is in flight
    cudaEvent_t e0 = s->ev[0], e1 = s->ev[1];
    CUDA_OK(cudaEventRecord(e0, s->st));
    bool more = true;
    while (more) {
        more = false;
        // ---- front end: mel -> conv1 -> conv2 for every session, new encoder rows gathered into s->enc.x_enc
        std::vector<int> row_slot, row_pos;
        struct Span { int slot, r0, n; };
        std::vector<Span> spans;
        for (int id = 0; id < max_sessions; ++id) {
            Slot &sl = slots[id];
            if (!sl.open || sl.drained) continue;
            int64_t tg[5];
            stream_progress(sl.n_samples, sl.ended, rf, P, tg);
            const int mel_t = (int)tg[0], c1_t = (int)tg[1];
            int enc_t = (int)tg[2];
            if (enc_t - sl.n_enc > max_new) {  // bounded by the ring slack: the rest in the next pass
                enc_t = sl.n_enc + max_new;
                more = true;
            }
            float *mel_s = e.slot_mel(id), *c1_s = e.slot_conv1(id);
            // each buffer keeps from the first row its consumer still reads: conv1 output t reads mel 2t-1..2t+1, conv2
            // output t reads conv1 2t-1..2t+1
            if (mel_t > sl.n_mel) {
                slide(mel_s, c.n_mels, e.max_mel_frames, sl.mel0, std::max(0, 2 * sl.n_c1 - 1), sl.n_mel, mel_t, false, slide_tmp, s->st);
                launch_mel(pcm + (size_t)id * cap_samples, 1, sl.n_samples, cap_samples, m->mel.window, m->mel.fb_vals, m->mel.fb_start,
                           m->mel.fb_len, m->mel.fb_stride, mel_s, mel_t, 0, s->st, sl.n_mel, sl.pcm0, sl.mel0);
                stats.mel_frames += mel_t - sl.n_mel;
                sl.n_mel = mel_t;
            }
            if (c1_t > sl.n_c1) {
                slide(c1_s, d, e.T1_max, sl.c10, std::max(0, 2 * sl.n_enc - 1), sl.n_c1, c1_t, false, slide_tmp, s->st);
                launch_conv2_gemm(mel_s, m->conv1_w, m->conv1_b, c1_s + (size_t)(sl.n_c1 - sl.c10) * d, 1, sl.n_mel, c1_t - sl.n_c1, c.n_mels,
                                  d, s->st, sl.n_c1, sl.mel0);
                sl.n_c1 = c1_t;
            }
            const int n_new = enc_t - sl.n_enc;
            if (n_new > 0) {
                const int r0 = (int)row_slot.size();
                launch_conv2_gemm(c1_s, m->conv2_w, m->conv2_b, e.x_enc + (size_t)r0 * d, 1, sl.n_c1, n_new, d, d, s->st, sl.n_enc,
                                  sl.c10);
                if (unbounded)
                    fill_rope(enc_rope_cos, enc_rope_sin, c.enc_head_dim, ring, (size_t)id * ring, sl.n_enc, n_new);
                for (int i = 0; i < n_new; ++i) {
                    row_slot.push_back(id);
                    row_pos.push_back(sl.n_enc + i);
                }
                spans.push_back({id, r0, n_new});
            }
        }
        // ---- encoder layers over all new rows at once (KV rings), final norm, scatter to the sessions
        const int R = (int)row_slot.size();
        if (R > 0) {
            CUDA_OK(cudaMemcpyAsync(d_row_slot, row_slot.data(), sizeof(int) * R, cudaMemcpyHostToDevice, s->st));
            CUDA_OK(cudaMemcpyAsync(d_row_pos, row_pos.data(), sizeof(int) * R, cudaMemcpyHostToDevice, s->st));
            CUDA_OK(cudaStreamSynchronize(s->st));
            encoder_rows(R);
            stats.encoder_rows += R;
            for (const Span &sp : spans) {
                Slot &sl = slots[sp.slot];
                float *eo = enc_out + (size_t)sp.slot * e.S_max * d;
                slide(eo, d, e.S_max, sl.enc0, (int64_t)sl.n_emb * rf, sl.n_enc, sl.n_enc + sp.n, false, slide_tmp, s->st);
                CUDA_OK(cudaMemcpyAsync(eo + (size_t)(sl.n_enc - sl.enc0) * d, e.h_enc + (size_t)sp.r0 * d,
                                        sizeof(float) * (size_t)sp.n * d, cudaMemcpyDeviceToDevice, s->st));
                sl.n_enc += sp.n;
            }
        }
        // ---- x4 frame stack + adapter (adapter.rs:108-122, model.rs:745-749): 4 consecutive frames are contiguous
        for (int id = 0; id < max_sessions; ++id) {
            Slot &sl = slots[id];
            if (!sl.open || sl.drained) continue;
            const int emb_t = sl.n_enc / rf, n_new = emb_t - sl.n_emb;
            if (n_new <= 0) continue;
            const float *src = enc_out + ((size_t)id * e.S_max + ((size_t)sl.n_emb * rf - sl.enc0)) * d;
            // embeddings stay resident for audio_embeds_range as long as they can: when the buffer is full, the older
            // half goes -- never one the decoder has still to read (position pos reads embedding pos)
            float *emb = e.slot_audio(id);
            slide(emb, D, e.S4_max, sl.emb0, std::min<int64_t>(sl.pos, emb_t - e.S4_max / 2), sl.n_emb, emb_t, false, slide_tmp, s->st);
            e.adapt(*s, src, n_new, emb + (size_t)(sl.n_emb - sl.emb0) * D);
            sl.n_emb = emb_t;
        }
        // ---- decoder: prefill of sessions whose 38 prefix positions have their audio (model.rs:883-923)
        for (int id = 0; id < max_sessions; ++id) {
            Slot &sl = slots[id];
            if (!sl.open || sl.drained || sl.pos != 0 || sl.n_emb < P) continue;
            VOX_CHECK(sl.emb0 == 0, VOX_ECAPACITY, "stream session %d: prefill embeddings were evicted", id);
            s->kv.reserve(id, P + 1);
            if (unbounded) fill_rope(dec_rope_cos, dec_rope_sin, c.dec_head_dim, kDecRopeRing, 0, 0, P);
            upload_rows({id}, false);
            s->sel.clear_bias_history(id, s->st);   // the slot's decoder cache starts empty
            std::vector<int> prefix((size_t)P, 32);
            prefix[0] = 1;
            s->prefill(1, P, prefix.data(), true);
            int tok = 0;
            std::vector<int32_t> top((size_t)s->sel.top_k);
            std::vector<float> lp((size_t)s->sel.top_k);
            CUDA_OK(cudaMemcpyAsync(&tok, s->d_tok, sizeof(int), cudaMemcpyDeviceToHost, s->st));
            s->sel.fetch_rows(1, top.data(), lp.data(), s->st);
            CUDA_OK(cudaStreamSynchronize(s->st));
            sl.last_tok = tok;
            sl.ids.push_back(tok);
            append_scores(sl, top.data(), lp.data());
            sl.n_ids += 1;
            sl.pos = P;  // cached positions; the next step is position P and consumes audio[P]
            stats.prefills += 1;
        }
        // ---- decoder steps: every session with a pending position shares one step (model.rs:938-960)
        for (;;) {
            std::vector<int> rows;
            for (int id = 0; id < max_sessions; ++id) {
                Slot &sl = slots[id];
                if (!sl.open || sl.drained || sl.pos < P) continue;
                // position p = sl.pos consumes audio[p]; the offline loop stops before the last embedding (model.rs:938)
                // (sl.pos = cached positions = index of the next position's audio embedding)
                const int last = sl.ended ? std::min(sl.n_emb - 1, final_enc(sl) / rf - 2) : sl.n_emb - 1;
                if (sl.pos > last) continue;
                // a RoPE ring row serves one position per launch: a row whose position meets another's waits for the
                // next step of this loop
                bool clash = false;
                for (int o : rows) clash |= unbounded && slots[o].pos != sl.pos && slots[o].pos % kDecRopeRing == sl.pos % kDecRopeRing;
                if (!clash) rows.push_back(id);
            }
            if (rows.empty()) break;
            for (int id : rows) {
                s->kv.reserve(id, slots[id].pos + 1);
                if (unbounded) fill_rope(dec_rope_cos, dec_rope_sin, c.dec_head_dim, kDecRopeRing, 0, slots[id].pos, 1);
            }
            upload_rows(rows, true);   // every row's output position starts at 0: its token and scores land there
            s->decode_step((int)rows.size(), true);
            std::vector<int> toks(rows.size());
            std::vector<int32_t> top(rows.size() * s->sel.top_k);
            std::vector<float> lp(rows.size() * s->sel.top_k);
            CUDA_OK(cudaMemcpyAsync(toks.data(), s->d_tok, sizeof(int) * rows.size(), cudaMemcpyDeviceToHost, s->st));
            s->sel.fetch_rows((int)rows.size(), top.data(), lp.data(), s->st);
            CUDA_OK(cudaStreamSynchronize(s->st));
            for (size_t i = 0; i < rows.size(); ++i) {
                Slot &sl = slots[rows[i]];
                sl.last_tok = toks[i];
                sl.ids.push_back(toks[i]);
                append_scores(sl, top.data() + i * s->sel.top_k, lp.data() + i * s->sel.top_k);
                sl.n_ids += 1;
                sl.pos += 1;
            }
            stats.decode_steps += 1;
            stats.decode_rows += (int)rows.size();
        }
        for (int id = 0; id < max_sessions; ++id) {
            Slot &sl = slots[id];
            if (!sl.open || sl.drained || !sl.ended) continue;
            int64_t tg[5];
            stream_progress(sl.n_samples, true, rf, P, tg);
            if (sl.n_enc == (int)tg[2] && sl.n_emb == (int)tg[3] && sl.n_ids == tg[4]) sl.drained = true;
        }
    }
    CUDA_OK(cudaEventRecord(e1, s->st));
    CUDA_OK(cudaEventSynchronize(e1));
    float ms = 0.0f;
    CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    stats.gpu_ms = ms;
    for (int id = 0; id < max_sessions; ++id)
        if (slots[id].open && !slots[id].drained) stats.live_sessions += 1;
    if (st_out) *st_out = stats;
}

// Q4VoxtralModel::encode_audio_with_cache (model.rs:790-799) = Q4AudioEncoder::forward_with_cache (437-452: conv stem on
// the chunk alone, layers extend the caches) + reshape_encoder_output + adapter.
int StreamPool::encode_chunk(int id, const float *mel, int T, float *out, size_t cap) {
    const vox_model_info &c = m->info;
    Slot &sl = slot(id);
    VOX_CHECK(!unbounded, VOX_EINVAL, "encode_chunk needs a pool with max_seconds > 0 (its output region is linear)");
    VOX_CHECK(sl.n_samples == pad_left(pad) && sl.n_audio == 0, VOX_EINVAL, "stream session %d is fed by push(): do not mix with encode_chunk", id);
    AudioEncoder &e = s->enc;
    VOX_CHECK(T >= 1 && T <= e.max_mel_frames, VOX_EINVAL, "mel chunk of %d frames exceeds the pool's capacity %d", T, e.max_mel_frames);
    CUDA_OK(cudaSetDevice(m->device));
    const int d = c.enc_dim, D = c.dec_dim, rf = c.reshape_factor;
    const int T1 = conv_out(T), S = conv_out(T1), S4 = S / rf;
    VOX_CHECK(sl.n_enc + S <= m->enc_rope_len, VOX_ECAPACITY, "encoder positions %d exceed the RoPE table (%d)", sl.n_enc + S, m->enc_rope_len);
    VOX_CHECK(cap >= (size_t)S4 * D, VOX_ECAPACITY, "audio_embeds capacity %zu < %zu", cap, (size_t)S4 * D);
    e.upload_mel(*s, mel, 1, T);
    launch_conv2_gemm(e.mel_tm, m->conv1_w, m->conv1_b, e.h1, 1, T, T1, c.n_mels, d, s->st);
    // rows beyond the ring slack go through the layers in several passes; the conv output of the whole chunk waits in
    // the session's (otherwise unused in chunk mode) encoder-output region
    float *conv = enc_out + (size_t)id * e.S_max * d;
    launch_conv2_gemm(e.h1, m->conv2_w, m->conv2_b, conv, 1, T1, S, d, d, s->st);
    for (int r0 = 0; r0 < S; r0 += max_new) {
        const int R = std::min(max_new, S - r0);
        std::vector<int> rs(R, id), rp(R);
        for (int i = 0; i < R; ++i) rp[i] = sl.n_enc + r0 + i;
        CUDA_OK(cudaMemcpyAsync(e.x_enc, conv + (size_t)r0 * d, sizeof(float) * (size_t)R * d, cudaMemcpyDeviceToDevice, s->st));
        CUDA_OK(cudaMemcpyAsync(d_row_slot, rs.data(), sizeof(int) * R, cudaMemcpyHostToDevice, s->st));
        CUDA_OK(cudaMemcpyAsync(d_row_pos, rp.data(), sizeof(int) * R, cudaMemcpyHostToDevice, s->st));
        CUDA_OK(cudaStreamSynchronize(s->st));
        encoder_rows(R);
        CUDA_OK(cudaMemcpyAsync(e.packed + (size_t)r0 * d, e.h_enc, sizeof(float) * (size_t)R * d, cudaMemcpyDeviceToDevice, s->st));
    }
    sl.n_enc += S;
    if (S4 > 0) {
        e.adapt(*s, e.packed, S4, e.audio);
        CUDA_OK(cudaMemcpyAsync(out, e.audio, sizeof(float) * (size_t)S4 * D, cudaMemcpyDeviceToHost, s->st));
    }
    CUDA_OK(cudaStreamSynchronize(s->st));
    return S4;
}

int StreamPool::final_enc(const Slot &sl) const {
    int64_t tg[5];
    stream_progress(sl.n_samples, true, m->info.reshape_factor, m->info.prefix_len, tg);
    return (int)tg[2];
}

const float *StreamPool::audio_embeds(int id, int *n) {
    Slot &sl = slot(id);
    VOX_CHECK(sl.emb0 == 0, VOX_ECAPACITY, "stream session %d: audio embeddings before %d were evicted; use vox_stream_audio_embeds_range",
              id, sl.emb0);
    *n = sl.n_emb;
    return s->enc.slot_audio(id);
}

const float *StreamPool::audio_embeds_range(int id, int64_t first, int64_t n) {
    Slot &sl = slot(id);
    VOX_CHECK(first >= 0 && n >= 0 && first + n <= sl.n_emb, VOX_EINVAL, "stream session %d: audio embeddings [%lld, %lld) not produced yet (%d so far)",
              id, (long long)first, (long long)(first + n), sl.n_emb);
    VOX_CHECK(first >= sl.emb0, VOX_ECAPACITY, "stream session %d: audio embedding %lld is no longer resident (first resident: %d)", id,
              (long long)first, sl.emb0);
    return s->enc.slot_audio(id) + (size_t)(first - sl.emb0) * m->info.dec_dim;
}

const float *StreamPool::mel_range(int id, int64_t first, int64_t n) {
    Slot &sl = slot(id);
    VOX_CHECK(first >= 0 && n >= 0 && first + n <= sl.n_mel, VOX_EINVAL, "stream session %d: mel frames [%lld, %lld) not produced yet (%d so far)",
              id, (long long)first, (long long)(first + n), sl.n_mel);
    VOX_CHECK(first >= sl.mel0, VOX_ECAPACITY, "stream session %d: mel frame %lld is no longer resident (first resident: %d)", id,
              (long long)first, sl.mel0);
    return s->enc.slot_mel(id) + (size_t)(first - sl.mel0) * m->info.n_mels;
}

void StreamPool::session_info(int id, struct vox_stream_session_info *out) {
    const Slot &sl = slot(id);
    *out = {};
    out->samples = (int64_t)sl.n_samples;
    out->mel_frames = sl.n_mel;
    out->encoder_frames = sl.n_enc;
    out->audio_embeds = sl.n_emb;
    out->first_audio_embed = sl.emb0;
    out->decoder_positions = sl.pos;
    out->ids_emitted = sl.n_ids;
    out->kv_pages = s->kv.pages(id);
}

void StreamPool::append_scores(Slot &sl, const int32_t *top_ids, const float *top_lp) {
    sl.top_ids.insert(sl.top_ids.end(), top_ids, top_ids + s->sel.top_k);
    sl.top_lp.insert(sl.top_lp.end(), top_lp, top_lp + s->sel.top_k);
}

// RoPE rows of positions [p0, p0 + n) into a ring table of `rows` rows starting at row `row0`: position p at row p % rows
void StreamPool::fill_rope(float *cos_d, float *sin_d, int hd, int rows, size_t row0, int64_t p0, int n) {
    const int half = hd / 2;
    std::vector<float> cv((size_t)n * half), sv((size_t)n * half);
    rope_rows(hd, m->rope_theta, p0, n, cv.data(), sv.data());
    for (int i = 0; i < n;) {
        const int r = (int)((p0 + i) % rows), len = std::min(n - i, rows - r);
        const size_t at = (row0 + r) * half;
        CUDA_OK(cudaMemcpyAsync(cos_d + at, cv.data() + (size_t)i * half, sizeof(float) * len * half, cudaMemcpyHostToDevice, s->st));
        CUDA_OK(cudaMemcpyAsync(sin_d + at, sv.data() + (size_t)i * half, sizeof(float) * len * half, cudaMemcpyHostToDevice, s->st));
        i += len;
    }
    // (an asynchronous copy from pageable memory has consumed its source when it returns)
}

}  // namespace vox
