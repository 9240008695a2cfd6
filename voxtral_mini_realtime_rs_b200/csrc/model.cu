// model.cu -- GGUF -> HBM loader (with load-time Q4 repack) and the session that runs
// encode_audio / prefill / decode on one CUDA stream.  Graph semantics follow the reference's
// src/gguf/model.rs (cited per function); nothing here is a translation of its Burn code.
#include "model.h"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "common.h"

namespace vox {

void cuda_check(cudaError_t e, const char *what) {
    if (e != cudaSuccess) fail(VOX_ECUDA, fmt("CUDA error: %s: %s", what, cudaGetErrorString(e)));
}

void *DeviceArena::alloc(size_t bytes) {
    if (bytes == 0) bytes = 16;
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) fail(VOX_ENOMEM, fmt("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)));
    ptrs.push_back(p);
    total += bytes;
    return p;
}

void DeviceArena::release() {
    for (void *p : ptrs) cudaFree(p);
    ptrs.clear();
    total = 0;
}

void MelTables::build(DeviceArena &arena) {
    fb_dense.resize((size_t)kMelBins * kMelFreqs);
    mel_filterbank(fb_dense.data());
    window_host.resize(kMelNfft);
    hann_window(kMelNfft, window_host.data());
    // sparse spans: [start, start+len) covers every non-zero of the dense row, in ascending bin
    // order so the sum equals the reference's dense sequential sum (adding 0.0 is exact).
    std::vector<int> start(kMelBins), len(kMelBins);
    int maxlen = 1;
    for (int m = 0; m < kMelBins; ++m) {
        int lo = kMelFreqs, hi = -1;
        for (int j = 0; j < kMelFreqs; ++j)
            if (fb_dense[(size_t)m * kMelFreqs + j] != 0.0f) { lo = std::min(lo, j); hi = std::max(hi, j); }
        if (hi < 0) { lo = 0; hi = -1; }
        start[m] = lo;
        len[m] = hi - lo + 1;
        maxlen = std::max(maxlen, len[m]);
    }
    fb_stride = maxlen;
    std::vector<float> vals((size_t)kMelBins * maxlen, 0.0f);
    for (int m = 0; m < kMelBins; ++m)
        for (int j = 0; j < len[m]; ++j) vals[(size_t)m * maxlen + j] = fb_dense[(size_t)m * kMelFreqs + start[m] + j];
    window = arena.upload(window_host.data(), window_host.size());
    fb_vals = arena.upload(vals.data(), vals.size());
    fb_start = arena.upload(start.data(), start.size());
    fb_len = arena.upload(len.data(), len.size());
}

static void build_tc_layout(DeviceArena &arena, Q4Weight &w, const std::vector<uint8_t> &qs,
                            const std::vector<uint16_t> &ds);

Q4Weight upload_q4(DeviceArena &arena, const std::vector<const uint8_t *> &raw, const std::vector<int> &n_rows,
                   int K, bool interleave, bool tc_layout) {
    VOX_CHECK(K % 32 == 0, VOX_EINVAL, "Q4 weight with K=%d (not a multiple of 32)", K);
    const int bpr = K / 32;
    int N = 0;
    for (int n : n_rows) N += n;
    if (interleave) VOX_CHECK(raw.size() == 2 && n_rows[0] == n_rows[1], VOX_EINVAL, "interleave needs two equal parts");
    std::vector<uint8_t> qs((size_t)N * bpr * 16);
    std::vector<uint16_t> ds((size_t)N * bpr);
    int row_base = 0;
    for (size_t p = 0; p < raw.size(); ++p) {
        for (int r = 0; r < n_rows[p]; ++r) {
            const int dst_row = interleave ? 2 * r + (int)p : row_base + r;
            const uint8_t *src = raw[p] + (size_t)r * bpr * 18;
            uint8_t *qd = qs.data() + (size_t)dst_row * bpr * 16;
            uint16_t *dd = ds.data() + (size_t)dst_row * bpr;
            for (int b = 0; b < bpr; ++b) {
                memcpy(dd + b, src + (size_t)b * 18, 2);
                memcpy(qd + (size_t)b * 16, src + (size_t)b * 18 + 2, 16);
            }
        }
        row_base += n_rows[p];
    }
    Q4Weight w;
    w.N = N;
    w.K = K;
    // f16 bits: |d| < 32 <=> exponent field < 16 (0x5000 = 32.0); inf and NaN fail too
    w.d_below_32 = std::all_of(ds.begin(), ds.end(), [](uint16_t h) { return (h & 0x7FFFu) < 0x5000u; });
    w.qs = (const uint4 *)arena.upload(qs.data(), qs.size());
    w.d = (const __half *)arena.upload(ds.data(), ds.size());
    if (tc_layout) build_tc_layout(arena, w, qs, ds);
    return w;
}

// TC layout (matvec_tc.cu): tiles of 16 rows x pairs of blocks; lane (g,t) of a tile/pair owns word t
// of rows g and g+8 of both blocks; scales grouped per g.  Rows / blocks beyond N / K are zero (d = 0).
static void build_tc_layout(DeviceArena &arena, Q4Weight &w, const std::vector<uint8_t> &qs,
                            const std::vector<uint16_t> &ds) {
    const int bpr = w.K / 32;
    const int n_tiles = (w.N + 15) / 16, n_pairs = (bpr + 1) / 2;
    std::vector<uint32_t> q((size_t)n_tiles * n_pairs * 32 * 4, 0u);
    std::vector<uint16_t> d((size_t)n_tiles * n_pairs * 8 * 4, 0);
    const uint32_t *src = reinterpret_cast<const uint32_t *>(qs.data());
    for (int T = 0; T < n_tiles; ++T)
        for (int P = 0; P < n_pairs; ++P) {
            uint32_t *qd = q.data() + ((size_t)T * n_pairs + P) * 128;
            uint16_t *dd = d.data() + ((size_t)T * n_pairs + P) * 32;
            for (int g = 0; g < 8; ++g)
                for (int bb = 0; bb < 2; ++bb) {
                    const int b = 2 * P + bb;
                    if (b >= bpr) continue;
                    for (int h = 0; h < 2; ++h) {
                        const int row = 16 * T + g + 8 * h;
                        if (row >= w.N) continue;
                        const size_t blk = (size_t)row * bpr + b;
                        for (int t = 0; t < 4; ++t) qd[(g * 4 + t) * 4 + bb * 2 + h] = src[blk * 4 + t];
                        dd[g * 4 + bb * 2 + h] = ds[blk];
                    }
                }
        }
    w.qs_tc = (const uint4 *)arena.upload(q.data(), q.size());
    w.d_tc = (const uint2 *)arena.upload(d.data(), d.size());
}

namespace {

const char *kEnc = "mm_streams_embeddings.embedding_module.whisper_encoder";
const char *kAdapter = "mm_streams_embeddings.embedding_module.audio_language_projection";
const char *kTokEmb = "mm_streams_embeddings.embedding_module.tok_embeddings.weight";
const char *kFinalNorm = "norm.weight";

float f16_to_f32(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 0x1Fu, man = h & 0x3FFu, bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else {
            int e = -1;
            do { e++; man <<= 1; } while ((man & 0x400u) == 0);
            man &= 0x3FFu;
            bits = sign | ((uint32_t)(127 - 15 - e) << 23) | (man << 13);
        }
    } else if (exp == 31) bits = sign | 0x7F800000u | (man << 13);
    else bits = sign | ((exp + 127 - 15) << 23) | (man << 13);
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

struct Loader {
    const Gguf &g;
    Model &m;
    uint64_t q4_bytes = 0;

    const GgufTensorInfo &info(const std::string &name) {
        const GgufTensorInfo *t = g.find(name);
        VOX_CHECK(t != nullptr, VOX_ENOTFOUND, "Tensor '%s' not found in GGUF", name.c_str());
        return *t;
    }
    bool has(const std::string &name) { return g.find(name) != nullptr; }

    // load_f32_tensor (loader.rs:443-474): F32/F16 -> f32; shape checked.
    std::vector<float> f32(const std::string &name, const std::vector<int64_t> &shape) {
        const GgufTensorInfo &t = info(name);
        VOX_CHECK(t.dtype != VOX_DTYPE_Q4_0, VOX_EFORMAT, "Cannot load Q4_0 tensor '%s' as f32", name.c_str());
        VOX_CHECK(t.shape() == shape, VOX_EINVAL, "Tensor '%s' has unexpected shape", name.c_str());
        std::vector<uint8_t> raw((size_t)t.byte_size());
        g.read_tensor(t, raw.data());
        size_t n = (size_t)t.num_elements();
        std::vector<float> out(n);
        if (t.dtype == VOX_DTYPE_F32) memcpy(out.data(), raw.data(), n * 4);
        else
            for (size_t i = 0; i < n; ++i) {
                uint16_t h;
                memcpy(&h, raw.data() + 2 * i, 2);
                out[i] = f16_to_f32(h);
            }
        return out;
    }
    float *f32_dev(const std::string &name, const std::vector<int64_t> &shape) {
        std::vector<float> v = f32(name, shape);
        return m.arena.upload(v.data(), v.size());
    }
    // load_q4_linear (loader.rs:390-405): dtype must be Q4_0; shape [N,K] checked.
    std::vector<uint8_t> q4_raw(const std::string &name, int N, int K) {
        const GgufTensorInfo &t = info(name);
        VOX_CHECK(t.dtype == VOX_DTYPE_Q4_0, VOX_EFORMAT, "Expected Q4_0 for '%s', got dtype %u", name.c_str(), t.dtype);
        std::vector<int64_t> shp = t.shape();
        VOX_CHECK(shp.size() == 2 && shp[0] == N && shp[1] == K, VOX_EINVAL, "Tensor '%s' has unexpected shape (want [%d,%d])",
                  name.c_str(), N, K);
        std::vector<uint8_t> raw((size_t)t.byte_size());
        g.read_tensor(t, raw.data());
        q4_bytes += raw.size();
        return raw;
    }
    Q4Weight q4(const std::string &name, int N, int K, bool tc = false) {
        std::vector<uint8_t> raw = q4_raw(name, N, K);
        return upload_q4(m.arena, {raw.data()}, {N}, K, false, tc);
    }
    Q4Weight q4_concat(const std::vector<std::string> &names, const std::vector<int> &ns, int K, bool tc = false) {
        std::vector<std::vector<uint8_t>> raws;
        std::vector<const uint8_t *> ptrs;
        for (size_t i = 0; i < names.size(); ++i) raws.push_back(q4_raw(names[i], ns[i], K));
        for (auto &r : raws) ptrs.push_back(r.data());
        return upload_q4(m.arena, ptrs, ns, K, false, tc);
    }
    Q4Weight q4_interleave(const std::string &a, const std::string &b, int N, int K, bool tc = false) {
        std::vector<uint8_t> ra = q4_raw(a, N, K), rb = q4_raw(b, N, K);
        return upload_q4(m.arena, {ra.data(), rb.data()}, {N, N}, K, true, tc);
    }
    // optional bias (loader.rs:428-437): zeros when the tensor is absent
    std::vector<float> bias_or_zero(const std::string &name, int n) {
        if (has(name)) return f32(name, {n});
        return std::vector<float>((size_t)n, 0.0f);
    }
};

void build_rope(DeviceArena &arena, int hd, int max_seq, float theta, float **cos_d, float **sin_d) {
    const int half = hd / 2;
    std::vector<float> c((size_t)max_seq * half), s((size_t)max_seq * half);
    rope_rows(hd, theta, 0, max_seq, c.data(), s.data());
    *cos_d = arena.upload(c.data(), c.size());
    *sin_d = arena.upload(s.data(), s.size());
}

}  // namespace

void rope_rows(int hd, float theta, int64_t p0, int n, float *cos_out, float *sin_out) {
    const int half = hd / 2;
    std::vector<float> inv(half);
    for (int i = 0; i < half; ++i) inv[i] = 1.0f / powf(theta, (float)(2 * i) / (float)hd);
    for (int r = 0; r < n; ++r)
        for (int i = 0; i < half; ++i) {
            const float f = (float)(p0 + r) * inv[i];
            cos_out[(size_t)r * half + i] = cosf(f);
            sin_out[(size_t)r * half + i] = sinf(f);
        }
}

Model *Model::load(const Gguf &g, int device) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    VOX_CHECK(e == cudaSuccess && ndev > 0, VOX_ECUDA, "no CUDA device available (%s); this library has no CPU fallback",
              cudaGetErrorString(e));
    VOX_CHECK(device >= 0 && device < ndev, VOX_EINVAL, "device %d out of range (have %d)", device, ndev);
    CUDA_OK(cudaSetDevice(device));
    Model *mp = new Model();
    try {
        Model &m = *mp;
        m.device = device;
        m.arena.device = device;
        Loader L{g, m};
        vox_model_info &c = m.info;
        // ---- dims: optional voxtral.* KVs, else the reference defaults (config.rs:441-486) ----
        auto kv = [&](const char *k, int dflt) { uint32_t v; return g.kv_u32(k, &v) ? (int)v : dflt; };
        c.enc_layers = kv("voxtral.enc.n_layers", 32);
        c.enc_heads = kv("voxtral.enc.n_heads", 32);
        c.enc_head_dim = kv("voxtral.enc.head_dim", 64);
        c.enc_window = kv("voxtral.enc.sliding_window", 750);
        c.dec_layers = kv("voxtral.dec.n_layers", 26);
        c.dec_heads = kv("voxtral.dec.n_heads", 32);
        c.dec_kv_heads = kv("voxtral.dec.n_kv_heads", 8);
        c.dec_head_dim = kv("voxtral.dec.head_dim", 128);
        c.dec_window = kv("voxtral.dec.sliding_window", 8192);
        c.reshape_factor = kv("voxtral.reshape_factor", 4);
        c.prefix_len = 38;
        const std::string E = kEnc;
        {
            std::vector<int64_t> s = L.info(E + ".conv_layers.0.conv.weight").shape();
            VOX_CHECK(s.size() == 3 && s[2] == 3, VOX_EINVAL, "conv_layers.0 weight must be [C,mels,3]");
            c.enc_dim = (int)s[0];
            c.n_mels = (int)s[1];
            VOX_CHECK(c.n_mels == kMelBins, VOX_EINVAL, "n_mels=%d unsupported (mel front-end is 128-bin)", c.n_mels);
        }
        // shapes come from the file: check the rank before indexing and the range before dividing
        auto dim2 = [&](const std::string &name, int axis) {
            std::vector<int64_t> s = L.info(name).shape();
            VOX_CHECK(s.size() == 2, VOX_EINVAL, "Tensor '%s' must be 2-D (has %zu dims)", name.c_str(), s.size());
            VOX_CHECK(s[axis] >= 1 && s[axis] <= (1 << 24), VOX_EINVAL, "Tensor '%s' dim %d = %lld out of range", name.c_str(), axis,
                      (long long)s[axis]);
            return (int)s[axis];
        };
        c.enc_ffn = dim2(E + ".transformer.layers.0.feed_forward.w1.weight", 0);
        c.vocab = dim2(kTokEmb, 0);
        c.dec_dim = dim2(kTokEmb, 1);
        c.dec_ffn = dim2("layers.0.feed_forward.w1.weight", 0);
        c.t_cond_dim = dim2("layers.0.ada_rms_norm_t_cond.0.weight", 0);
        for (int v : {c.enc_layers, c.enc_heads, c.enc_head_dim, c.dec_layers, c.dec_heads, c.dec_kv_heads, c.dec_head_dim,
                      c.reshape_factor, c.enc_dim})
            VOX_CHECK(v >= 1 && v <= (1 << 20), VOX_EINVAL, "model dimension %d out of range (voxtral.* metadata)", v);
        VOX_CHECK(c.enc_window >= 0 && c.dec_window >= 0, VOX_EINVAL, "negative sliding window");
        VOX_CHECK(c.dec_heads % c.dec_kv_heads == 0, VOX_EINVAL, "dec_heads %% dec_kv_heads != 0");
        VOX_CHECK(c.enc_head_dim == 32 || c.enc_head_dim == 64 || c.enc_head_dim == 128, VOX_EINVAL,
                  "encoder head_dim %d unsupported", c.enc_head_dim);
        VOX_CHECK(c.dec_head_dim % 4 == 0, VOX_EINVAL, "decoder head_dim %d unsupported", c.dec_head_dim);

        const int d = c.enc_dim, hdq = c.enc_heads * c.enc_head_dim, D = c.dec_dim;
        // ---- conv downsampler (loader.rs:263-275), f32 ----
        {   // conv1 weights [o][c][tap] -> [o][tap*n_mels + c]: conv1 runs as an implicit GEMM on the
            // time-major mel like conv2
            std::vector<float> w = L.f32(E + ".conv_layers.0.conv.weight", {d, c.n_mels, 3});
            std::vector<float> r((size_t)d * 3 * c.n_mels);
            for (int o = 0; o < d; ++o)
                for (int ci = 0; ci < c.n_mels; ++ci)
                    for (int t = 0; t < 3; ++t)
                        r[(size_t)o * 3 * c.n_mels + (size_t)t * c.n_mels + ci] = w[((size_t)o * c.n_mels + ci) * 3 + t];
            m.conv1_w = m.arena.upload(r.data(), r.size());
        }
        m.conv1_b = L.f32_dev(E + ".conv_layers.0.conv.bias", {d});
        {
            std::vector<float> w = L.f32(E + ".conv_layers.1.conv.weight", {d, d, 3});
            std::vector<float> r((size_t)d * 3 * d);  // [o][tap*C + c] for the implicit GEMM
            for (int o = 0; o < d; ++o)
                for (int ci = 0; ci < d; ++ci)
                    for (int t = 0; t < 3; ++t) r[(size_t)o * 3 * d + (size_t)t * d + ci] = w[((size_t)o * d + ci) * 3 + t];
            m.conv2_w = m.arena.upload(r.data(), r.size());
        }
        m.conv2_b = L.f32_dev(E + ".conv_layers.1.conv.bias", {d});
        // ---- encoder layers (loader.rs:215-260) ----
        m.enc.resize(c.enc_layers);
        for (int i = 0; i < c.enc_layers; ++i) {
            const std::string p = E + ".transformer.layers." + std::to_string(i);
            EncLayerW &l = m.enc[i];
            l.attn_norm = L.f32_dev(p + ".attention_norm.weight", {d});
            l.ffn_norm = L.f32_dev(p + ".ffn_norm.weight", {d});
            l.wqkv = L.q4_concat({p + ".attention.wq.weight", p + ".attention.wk.weight", p + ".attention.wv.weight"},
                                 {hdq, hdq, hdq}, d);
            std::vector<float> bq = L.bias_or_zero(p + ".attention.wq.bias", hdq);
            std::vector<float> bv = L.bias_or_zero(p + ".attention.wv.bias", hdq);
            std::vector<float> bqkv((size_t)3 * hdq, 0.0f);  // wk has no bias (loader.rs:229)
            memcpy(bqkv.data(), bq.data(), sizeof(float) * hdq);
            memcpy(bqkv.data() + 2 * hdq, bv.data(), sizeof(float) * hdq);
            l.bqkv = m.arena.upload(bqkv.data(), bqkv.size());
            l.wo = L.q4(p + ".attention.wo.weight", d, hdq);
            std::vector<float> bo = L.bias_or_zero(p + ".attention.wo.bias", d);
            l.bo = m.arena.upload(bo.data(), bo.size());
            l.w13 = L.q4_interleave(p + ".feed_forward.w1.weight", p + ".feed_forward.w3.weight", c.enc_ffn, d);
            l.w2 = L.q4(p + ".feed_forward.w2.weight", d, c.enc_ffn);
            std::vector<float> b2 = L.bias_or_zero(p + ".feed_forward.w2.bias", d);
            l.b2 = m.arena.upload(b2.data(), b2.size());
        }
        m.enc_norm = L.f32_dev(E + ".transformer.norm.weight", {d});
        // ---- adapter (loader.rs:377-383) ----
        m.adapter0 = L.q4(std::string(kAdapter) + ".0.weight", D, d * c.reshape_factor);
        m.adapter2 = L.q4(std::string(kAdapter) + ".2.weight", D, D);
        // ---- tied embeddings / lm_head: kept Q4 on device (WASM-path semantics, model.rs:689) ----
        {
            const GgufTensorInfo &t = L.info(kTokEmb);
            VOX_CHECK(t.dtype == VOX_DTYPE_Q4_0, VOX_EFORMAT,
                      "tok_embeddings must be Q4_0 in this build (got dtype %u)", t.dtype);
            m.tok_emb = L.q4(kTokEmb, c.vocab, D, true);
        }
        // ---- decoder layers (loader.rs:329-375) ----
        const int qd = c.dec_heads * c.dec_head_dim, kvd = c.dec_kv_heads * c.dec_head_dim;
        m.dec.resize(c.dec_layers);
        uint64_t dec_q4 = 0;
        for (int j = 0; j < c.dec_layers; ++j) {
            const std::string p = "layers." + std::to_string(j);
            DecLayerW &l = m.dec[j];
            const uint64_t before = L.q4_bytes;
            l.ada0 = L.q4(p + ".ada_rms_norm_t_cond.0.weight", c.t_cond_dim, D);
            l.ada2 = L.q4(p + ".ada_rms_norm_t_cond.2.weight", D, c.t_cond_dim);
            l.attn_norm = L.f32_dev(p + ".attention_norm.weight", {D});
            l.ffn_norm = L.f32_dev(p + ".ffn_norm.weight", {D});
            l.wqkv = L.q4_concat({p + ".attention.wq.weight", p + ".attention.wk.weight", p + ".attention.wv.weight"},
                                 {qd, kvd, kvd}, D, true);
            l.wo = L.q4(p + ".attention.wo.weight", D, qd, true);
            l.w13 = L.q4_interleave(p + ".feed_forward.w1.weight", p + ".feed_forward.w3.weight", c.dec_ffn, D, true);
            l.w2 = L.q4(p + ".feed_forward.w2.weight", D, c.dec_ffn, true);
            dec_q4 += L.q4_bytes - before;
        }
        m.dec_norm = L.f32_dev(kFinalNorm, {D});
        build_rope(m.arena, c.enc_head_dim, m.enc_rope_len, m.rope_theta, &m.enc_cos, &m.enc_sin);
        build_rope(m.arena, c.dec_head_dim, m.dec_rope_len, m.rope_theta, &m.dec_cos, &m.dec_sin);
        m.mel.build(m.arena);
        c.q4_bytes = L.q4_bytes;
        c.device_bytes = m.arena.total;
        c.decode_step_bytes = dec_q4 + m.tok_emb.bytes();
        CUDA_OK(cudaDeviceSynchronize());
    } catch (...) {
        delete mp;
        throw;
    }
    return mp;
}

// ======================================================================================
// Session
// ======================================================================================
Session *Session::create(Model *m, int max_batch, int max_mel_frames, bool kv_ring, KvType kv_type) {
    VOX_CHECK(max_batch >= 1 && max_batch <= 64, VOX_EINVAL, "max_batch %d out of range [1,64]", max_batch);
    VOX_CHECK(max_mel_frames >= 16, VOX_EINVAL, "max_mel_frames %d too small", max_mel_frames);
    CUDA_OK(cudaSetDevice(m->device));
    Session *s = new Session();
    try {
        const vox_model_info &c = m->info;
        s->m = m;
        s->arena.device = m->device;
        s->max_batch = max_batch;
        s->M_max = std::max(c.prefix_len, 64);
        s->enc.create(s->arena, *m, max_batch, max_mel_frames);
        const int S_max = s->enc.S_max, S4_max = s->enc.S4_max;
        CUDA_OK(cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking));
        for (auto &e : s->ev) CUDA_OK(cudaEventCreate(&e));
        const size_t B = max_batch;
        // decoder
        s->kv.create(s->arena, c, max_batch, S4_max, s->M_max, kv_ring, kv_type);
        s->out_ld = s->kv.capacity();
        s->sel.create(s->arena, m->device, max_batch, s->out_ld, c.vocab);
        s->dec_rope = m->dec_rope();
        const size_t drows = B * s->M_max;
        const int qkvd = (c.dec_heads + 2 * c.dec_kv_heads) * c.dec_head_dim;
        s->x_dec = s->arena.alloc_n<float>(drows * c.dec_dim);
        s->h_dec = s->arena.alloc_n<float>(drows * c.dec_dim);
        s->qkv_dec = s->arena.alloc_n<float>(drows * qkvd);
        s->attn_dec = s->arena.alloc_n<float>(drows * c.dec_heads * c.dec_head_dim);
        s->act_dec = s->arena.alloc_n<float>(drows * c.dec_ffn);
        s->last_h = s->arena.alloc_n<float>(B * c.dec_dim);
        s->logits = s->arena.alloc_n<float>(B * c.vocab);
        s->ada_sets = s->arena.alloc_n<float>(B * s->ada_set_floats());
        s->delays.assign(B, 0.0f);
        s->d_ada_rows = (const float **)s->arena.alloc(sizeof(float *) * B);
        s->d_fga_rows = (const float **)s->arena.alloc(sizeof(float *) * B);
        s->d_audio_off = s->arena.alloc_n<int64_t>(B);
        s->t_embed = s->arena.alloc_n<float>(c.dec_dim);
        s->ada_tmp = s->arena.alloc_n<float>(c.t_cond_dim);
        s->d_pos = s->arena.alloc_n<int>(B);      // per row (kernels.h KvView::pos)
        s->d_outpos = s->arena.alloc_n<int>(B);
        s->d_tok = s->arena.alloc_n<int>(B);
        s->d_ids = s->arena.alloc_n<int>(drows);
        s->d_out = s->arena.alloc_n<int>(B * s->out_ld);
        {   // split-tile buffer of the wgmma GEMM: largest (rows, K) pair it is used with
            const int rows_e = max_batch * S_max, rows_d = max_batch * s->M_max;
            size_t e = 0;
            for (int K : {c.enc_dim, c.enc_heads * c.enc_head_dim, c.enc_ffn}) e = std::max(e, gemm_tc5_split_elems(rows_e, K / 64 * 64));
            e = std::max(e, gemm_tc5_split_elems(max_batch * std::max(S4_max, 1), c.enc_dim * c.reshape_factor / 64 * 64));
            for (int K : {c.dec_dim, c.dec_heads * c.dec_head_dim, c.dec_ffn}) e = std::max(e, gemm_tc5_split_elems(std::max(rows_d, max_batch * std::max(S4_max, 1)), K / 64 * 64));
            s->xt_elems = e;
            s->xt_buf = s->arena.alloc(e * 2);
            s->gemm_work = gemm_tc5_work_size();
            alloc_split_k(s->arena, s->gemm_work);
            const char *gv = getenv("VOX_GEMM");
            s->path.gemm_tc = !(gv && std::string(gv) == "simt");
            const char *tv = getenv("VOX_MATVEC");
            s->path.matvec_tc = !(tv && std::string(tv) == "simt");
        }
        {   // fused-decode scratch (see TcWork): split-K of the largest decoder / lm_head matvec
            std::vector<const Q4Weight *> ws{&m->tok_emb};
            for (const DecLayerW &l : m->dec) ws.insert(ws.end(), {&l.wqkv, &l.wo, &l.w13, &l.w2});
            for (const Q4Weight *w : ws) {
                const TcWork need = q4_matvec_tc_work_size(w->N, w->K);
                s->tc_split.partial_floats = std::max(s->tc_split.partial_floats, need.partial_floats);
                s->tc_split.n_counters = std::max(s->tc_split.n_counters, need.n_counters);
            }
            alloc_split_k(s->arena, s->tc_split);
            s->ssq_x = s->arena.alloc_n<float>((size_t)((c.dec_dim + 15) / 16) * 8);
            s->am_vals = s->arena.alloc_n<float>((size_t)max_batch * ARGMAX_PARTS);
            s->am_idx = s->arena.alloc_n<int>((size_t)max_batch * ARGMAX_PARTS);
            s->am_cnt = s->arena.alloc_n<int>(max_batch);
            CUDA_OK(cudaMemset(s->am_cnt, 0, sizeof(int) * max_batch));
        }
        const char *mv = getenv("VOX_MEGA");
        s->use_mega = !(mv && mv[0] == '0');
        s->mega.create(*s);
        CUDA_OK(cudaMemset(s->d_pos, 0, sizeof(int) * B));
        CUDA_OK(cudaMemset(s->d_outpos, 0, sizeof(int) * B));
        s->out_rows.assign(B, 0);
        s->set_delay(kDefaultDelay);
    } catch (...) {
        delete s;
        throw;
    }
    return s;
}

Session::~Session() {
    if (step_graph.exec) cudaGraphExecDestroy(step_graph.exec);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
}

void Session::linear(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias, const float *res,
                     int epi, const float *gamma, float *tmp, const TcWork *tc, const AdaRows &ada_rows) {
    launch_q4_linear(w, x, M, y, ldy, bias, res, epi, gamma, m->norm_eps, tmp, Q4Scratch{xt_buf, xt_elems, &gemm_work, tc},
                     path, st, ada_rows);
}

// TimeEmbedding::embed (time_embedding.rs:41-71) + the per-layer ADA scale
// 1 + w2(gelu(w0(t)))  (model.rs:250-255) into ada_dst [L][D], and ffn_norm x that scale into fga_dst [L][D].
static void compute_ada(Session &s, float delay, float *ada_dst, float *fga_dst) {
    const Model *m = s.m;
    const vox_model_info &c = m->info;
    std::vector<float> t(c.dec_dim);
    time_embedding(delay, c.dec_dim, t.data());
    CUDA_OK(cudaMemcpyAsync(s.t_embed, t.data(), sizeof(float) * c.dec_dim, cudaMemcpyHostToDevice, s.st));
    CUDA_OK(cudaStreamSynchronize(s.st));
    std::vector<float> ones(c.dec_dim, 1.0f);
    for (int j = 0; j < c.dec_layers; ++j) {
        float *dst = ada_dst + (size_t)j * c.dec_dim;
        CUDA_OK(cudaMemcpyAsync(dst, ones.data(), sizeof(float) * c.dec_dim, cudaMemcpyHostToDevice, s.st));
        launch_q4_matvec(m->dec[j].ada0, s.t_embed, 1, s.ada_tmp, c.t_cond_dim, nullptr, nullptr, EPI_GELU, s.st);
        // dst = 1 + w2 . gelu(...)   (residual epilogue onto the vector of ones)
        launch_q4_matvec(m->dec[j].ada2, s.ada_tmp, 1, dst, c.dec_dim, nullptr, dst, EPI_RESIDUAL, s.st);
        launch_mul_vec(m->dec[j].ffn_norm, dst, fga_dst + (size_t)j * c.dec_dim, c.dec_dim, s.st);
    }
    CUDA_OK(cudaStreamSynchronize(s.st));
}

// t is constant for a transcription: the vectors are computed once per delay, into stream 0's set, and copied to the
// other streams' sets.
void Session::set_delay(float delay) {
    CUDA_OK(cudaSetDevice(m->device));
    const size_t n = ada_set_floats();
    compute_ada(*this, delay, ada_sets, ada_sets + n / 2);
    delays[0] = delay;
    for (int i = 1; i < max_batch; ++i) {
        CUDA_OK(cudaMemcpyAsync(ada_sets + i * n, ada_sets, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
        delays[i] = delay;
    }
    CUDA_OK(cudaStreamSynchronize(st));
}

// delays are compared as values; set_delay accepts any float, so two NaNs count as one delay
static bool same_delay(float a, float b) { return a == b || (std::isnan(a) && std::isnan(b)); }

void Session::set_delays(const float *d, int b) {
    VOX_CHECK(b >= 1 && b <= max_batch, VOX_EINVAL, "set_delays: %d streams out of range [1,%d]", b, max_batch);
    for (int i = 0; i < b; ++i)
        VOX_CHECK(std::isfinite(d[i]) && d[i] >= 0.0f, VOX_EINVAL, "delay %g of stream %d must be finite and >= 0", d[i], i);
    CUDA_OK(cudaSetDevice(m->device));
    for (int i = 0; i < b; ++i) set_stream_delay(i, d[i]);
}

void Session::set_stream_delay(int i, float d) {
    if (same_delay(delays[i], d)) return;
    const size_t n = ada_set_floats();
    float *set = ada_sets + (size_t)i * n;
    int same = -1;   // another stream at this delay: copy its vectors (computed by the same launches: bitwise equal)
    for (int j = 0; j < max_batch && same < 0; ++j)
        if (j != i && same_delay(delays[j], d)) same = j;
    if (same >= 0) {
        CUDA_OK(cudaMemcpyAsync(set, ada_sets + (size_t)same * n, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
        CUDA_OK(cudaStreamSynchronize(st));
    } else {
        compute_ada(*this, d, set, set + n / 2);
    }
    delays[i] = d;
}

void Session::bind_rows(int B) {
    std::vector<int> streams(B);
    std::vector<int64_t> offs(B);
    for (int r = 0; r < B; ++r) {
        const int s = row_streams.empty() ? r : row_streams[r];
        streams[r] = s;
        offs[r] = s < (int)enc.audio_offs.size() ? enc.audio_offs[s] : 0;   // (a stream without embeddings reads none)
    }
    if (bound_streams.size() >= (size_t)B && std::equal(streams.begin(), streams.end(), bound_streams.begin()) &&
        std::equal(offs.begin(), offs.end(), bound_offs.begin()))
        return;
    std::vector<const float *> a(B), f(B);
    for (int r = 0; r < B; ++r) {
        a[r] = ada_sets + (size_t)streams[r] * ada_set_floats();
        f[r] = a[r] + ada_set_floats() / 2;
    }
    CUDA_OK(cudaMemcpyAsync(d_ada_rows, a.data(), sizeof(float *) * B, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(d_fga_rows, f.data(), sizeof(float *) * B, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyAsync(d_audio_off, offs.data(), sizeof(int64_t) * B, cudaMemcpyHostToDevice, st));
    sel.bind_rows(streams, st);
    CUDA_OK(cudaStreamSynchronize(st));   // the staging vectors die with this frame
    bound_streams = std::move(streams);
    bound_offs = std::move(offs);
}

void Session::check_batch(int b) const { VOX_CHECK(b >= 1 && b <= max_batch, VOX_EINVAL, "batch %d exceeds session max_batch %d", b, max_batch); }
void Session::check_ids(const int32_t *ids, size_t n) const {
    for (size_t i = 0; i < n; ++i) VOX_CHECK(ids[i] >= 0 && ids[i] < m->info.vocab, VOX_EINVAL, "token id %d out of range", ids[i]);
}

// Q4LanguageModel::forward_hidden_with_cache (model.rs:665-677) over x_dec [B*M][D]; positions
// *d_pos + i.  Leaves the final-normed hidden states in h_dec -- or, on the fused decode path, returns
// true and leaves the un-normed stream in x_dec for lm_head_rows().  Does not advance *d_pos.
bool Session::fused_decode(int rows) const { return path.matvec_tc && rows <= 8 && m->tok_emb.qs_tc != nullptr; }

TcWork Session::tc_work(bool norm_in, bool ssq_out_) const {
    TcWork w = tc_split;
    if (norm_in) {
        w.ssq_in = ssq_x;
        w.ssq_in_parts = (m->info.dec_dim + 15) / 16;
    }
    if (ssq_out_) w.ssq_out = ssq_x;
    return w;
}

bool Session::decoder_forward(int B, int M) {
    const vox_model_info &c = m->info;
    const int D = c.dec_dim, H = c.dec_heads, Hkv = c.dec_kv_heads, hd = c.dec_head_dim;
    const int qkvd = (H + 2 * Hkv) * hd, rows = B * M;
    const float scale = powf((float)hd, -0.5f);
    // decode-sized problems: RMSNorm fused into the consuming matvec, RoPE + KV append fused into the
    // attention kernel => 5 launches per layer instead of 8
    const bool fused = fused_decode(rows);
    const TcWork wk_norm = tc_work(true, false), wk_res = tc_work(false, true);
    const TcWork *tc_norm = fused ? &wk_norm : nullptr, *tc_res = fused ? &wk_res : nullptr;
    const bool fattn = fused && M == 1 && dec_attn_fused_supported(H, Hkv, hd);
    for (int j = 0; j < c.dec_layers; ++j) {
        const DecLayerW &l = m->dec[j];
        const KvView kvl = kv.view(j, d_pos);
        linear(l.wqkv, x_dec, rows, qkv_dec, qkvd, nullptr, nullptr, EPI_NONE, l.attn_norm, h_dec, tc_norm);
        if (fattn) {
            launch_dec_attn_fused(qkv_dec, B, qkvd, H, Hkv, hd, kvl, c.dec_window, scale, dec_rope, attn_dec, st);
        } else {
            launch_dec_rope_append(qkv_dec, B, M, qkvd, H, Hkv, hd, kvl, dec_rope, st);
            launch_dec_attention(qkv_dec, B, M, qkvd, H, Hkv, hd, kvl, c.dec_window, scale, attn_dec, st);
        }
        linear(l.wo, attn_dec, rows, x_dec, D, nullptr, x_dec, EPI_RESIDUAL, nullptr, nullptr, tc_res);
        linear(l.w13, x_dec, rows, act_dec, c.dec_ffn, nullptr, nullptr, EPI_SILU_MUL, l.ffn_norm, h_dec, tc_norm,
               AdaRows{d_ada_rows, M, (size_t)j * D});
        linear(l.w2, act_dec, rows, x_dec, D, nullptr, x_dec, EPI_RESIDUAL, nullptr, nullptr, tc_res);
    }
    if (!fused) launch_rmsnorm(x_dec, m->dec_norm, h_dec, rows, D, m->norm_eps, st);
    return fused;
}

// lm_head over `rows` decoder rows (model.rs:680-691); `norm_pending`: x_dec still needs the final
// RMSNorm (fused into the matvec), else h_dec already holds the normed hidden states.
void Session::lm_head_rows(int rows, bool norm_pending, float *dst) {
    const TcWork wk = tc_work(true, false);
    linear(m->tok_emb, norm_pending ? x_dec : h_dec, rows, dst, m->info.vocab, nullptr, nullptr, EPI_NONE,
           norm_pending ? m->dec_norm : nullptr, nullptr, norm_pending ? &wk : nullptr);
}

void Session::forward_logits(int b, int M, const int *ids_host, bool with_audio, float *dst) {
    bind_rows(b);
    CUDA_OK(cudaMemcpyAsync(d_ids, ids_host, sizeof(int) * (size_t)b * M, cudaMemcpyHostToDevice, st));
    launch_embed(m->tok_emb, d_ids, with_audio ? enc.audio : nullptr, d_audio_off, b, M, d_pos, x_dec,
                 fused_decode(b * M) ? ssq_x : nullptr, st);
    const bool pending = decoder_forward(b, M);
    lm_head_rows(b * M, pending, dst);
    launch_advance(d_pos, M, nullptr, 0, b, st);
    cache_len += M;
}

unsigned Session::prepare_step(int R) {
    bind_rows(R);
    // the persistent kernel runs the step as row groups of a fused-decode size
    return use_mega && fused_decode(1) ? mega.prepare(*this, R) : 0u;
}

// One autoregressive step for B streams (model.rs:938-960): embed(prev token) + audio[pos-1],
// 26 layers, lm_head, argmax, device-side feedback; all positions read from device counters.
unsigned Session::decode_step(int B, bool add_audio) {
    const unsigned mega_launches = prepare_step(B);
    mega.attn_log.clear();
    if (mega_launches > 0) mega.step(*this, B, add_audio);
    else {
        launch_embed(m->tok_emb, d_tok, add_audio ? enc.audio : nullptr, d_audio_off, B, 1, d_pos, x_dec,
                     fused_decode(B) ? ssq_x : nullptr, st);
        const bool pending = decoder_forward(B, 1);
        lm_head_rows(B, pending, logits);
        launch_argmax_multi(logits, B, m->info.vocab, d_tok, d_out, out_ld, d_outpos, am_vals, am_idx, am_cnt, st);
        launch_advance(d_pos, 1, d_outpos, 1, B, st);
    }
    sel.after_step(*this, B);   // over every row (every group of the persistent kernel's)
    return mega_launches;
}

void Session::set_bias(int stream, const int32_t *ids, const int32_t *lens, const float *boosts, int n) {
    if (sel.set_bias(stream, ids, lens, boosts, n, st)) bound_streams.clear();   // the next bind_rows fills the row table
}

// Prefill of M positions for B streams (model.rs:894-923 with M = 38; also the incremental vox_prefill).
void Session::prefill(int B, int M, const int *ids_host, bool add_audio) {
    const vox_model_info &c = m->info;
    bind_rows(B);
    CUDA_OK(cudaMemcpyAsync(d_ids, ids_host, sizeof(int) * (size_t)B * M, cudaMemcpyHostToDevice, st));
    launch_embed(m->tok_emb, d_ids, add_audio ? enc.audio : nullptr, d_audio_off, B, M, d_pos, x_dec,
                 fused_decode(B * M) ? ssq_x : nullptr, st);
    const bool pending = decoder_forward(B, M);
    if (pending) {   // decode-sized prefill (B*M <= 8): final norm still pending in x_dec
        launch_rmsnorm(x_dec, m->dec_norm, h_dec, B * M, c.dec_dim, m->norm_eps, st);
    }
    // lm_head on the last row only (the reference computes all M rows and keeps one)
    launch_gather_last(h_dec, last_h, B, M, c.dec_dim, st);
    linear(m->tok_emb, last_h, B, logits, c.vocab, nullptr, nullptr, EPI_NONE);
    launch_argmax(logits, B, c.vocab, d_tok, d_out, out_ld, d_outpos, st);
    launch_advance(d_pos, M, d_outpos, 1, B, st);
    sel.after_step(*this, B);
}

void Session::step_incremental(int b, int M, const int *ids_host, bool add_audio) {
    if (ids_host) prefill(b, M, ids_host, add_audio);
    else decode_step(b, add_audio);
    cache_len += M;
    sel.record_step(b, out_rows.data());   // each row's output just emitted
    for (int r = 0; r < b; ++r) ++out_rows[r];
}

void Session::reset() {
    CUDA_OK(cudaMemsetAsync(d_pos, 0, sizeof(int) * max_batch, st));
    CUDA_OK(cudaMemsetAsync(d_outpos, 0, sizeof(int) * max_batch, st));
    std::fill(out_rows.begin(), out_rows.end(), 0);
    cache_len = 0;
    kv.restore_identity(st);
    sel.clear_bias_history(-1, st);
    rebase_epoch();
}

// A replay reads the op table and the row tables (ADA sets, audio offsets) the host built: prepare_step re-builds them
// before the first replay (an incremental call or another encode in between may have changed them), and every other
// host-side choice the captured kernels depend on is in the key.  `step()` returns its persistent-kernel launches.
template <class Step>
void Session::run_steps(int R, int n, Step step) {
    if (n <= 0) return;
    prepare_step(R);
    const StepKey key{R, sel.top_k, sel.beam_w, path.matvec_tc, path.gemm_tc, use_mega, sel.bias_on()};
    if (use_graph && !(step_graph.exec && step_graph.key == key)) {
        // first step eagerly (also performs any one-time kernel attribute setup), then capture one step and replay it
        step();
        --n;
        if (step_graph.exec) { cudaGraphExecDestroy(step_graph.exec); step_graph.exec = nullptr; }
        if (n > 0) {
            cudaGraph_t graph = nullptr;
            const uint64_t before = kernel_launch_count();
            CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
            mega.capturing = true;   // captured, not executed: not counted
            try {
                step_graph.mega_launches = step();
            } catch (...) {
                mega.capturing = false;
                cudaStreamEndCapture(st, &graph);
                if (graph) cudaGraphDestroy(graph);
                throw;
            }
            mega.capturing = false;
            CUDA_OK(cudaStreamEndCapture(st, &graph));
            step_graph.nodes = kernel_launch_count() - before;
            add_graph_launches(-(int64_t)step_graph.nodes);  // captured, not executed
            cudaError_t e = cudaGraphInstantiate(&step_graph.exec, graph, 0);
            cudaGraphDestroy(graph);
            cuda_check(e, "cudaGraphInstantiate");
            step_graph.key = key;
        }
    }
    for (int i = 0; i < n; ++i) {
        if (!use_graph) { step(); continue; }
        CUDA_OK(cudaGraphLaunch(step_graph.exec, st));
        add_graph_launches((int64_t)step_graph.nodes);
        mega.launches += step_graph.mega_launches;
    }
}

namespace {
// the rows of a transcribe call map to their streams for that call only, also when it throws
struct RowStreams {
    Session *s;
    ~RowStreams() { s->row_streams.clear(); }
};
}  // namespace

// Q4VoxtralModel::transcribe_streaming (model.rs:873-963).  Expects the mel in enc.mel_tm; records
// ev[2] (after encode), ev[4] (after the prefill) and ev[3] (after decode) on the stream.  Returns tokens per stream.
int Session::transcribe_from_mel(int B, int T, int32_t *out_ids, size_t cap_ids, vox_timings *tm, bool total) {
    const vox_model_info &c = m->info;
    const int W = sel.beam_w, R = B * W;   // decode rows: beam w of stream s in row w * B + s
    sel.check_rows(B);
    RowStreams row_guard{this};
    if (W > 1)
        for (int r = 0; r < R; ++r) row_streams.push_back(r % B);
    const std::vector<int> frames(B, T);
    enc.encode(*this, B, frames.data());
    cur_B = B;
    CUDA_OK(cudaEventRecord(ev[2], st));
    const int S4 = enc.positions, P = c.prefix_len;
    int n_out = 0;
    if (S4 >= P) {
        n_out = S4 - P;
        VOX_CHECK(cap_ids >= (size_t)B * n_out, VOX_ECAPACITY, "out_ids capacity %zu < %d x %d", cap_ids, B, n_out);
        reset();
        // prefix = [BOS] + [STREAMING_PAD]*37 (model.rs:883-892)
        std::vector<int> prefix((size_t)B * P, 32);
        for (int b = 0; b < B; ++b) prefix[(size_t)b * P] = 1;
        prefill(B, P, prefix.data(), true);
        if (W > 1) {
            // beam rows w * B + s take stream s's step counters (and read its audio embeddings through row_streams); the
            // selection at position 0 has one live rank per stream (the prefix, score 0), whose top-W ids become the W
            // beams, and the fork hands the prefix's KV to the other rows
            for (int w = 1; w < W; ++w) {
                CUDA_OK(cudaMemcpyAsync(d_pos + w * B, d_pos, sizeof(int) * B, cudaMemcpyDeviceToDevice, st));
                CUDA_OK(cudaMemcpyAsync(d_outpos + w * B, d_outpos, sizeof(int) * B, cudaMemcpyDeviceToDevice, st));
            }
            std::vector<int> rank_row((size_t)B * W);
            for (int s = 0; s < B; ++s)
                for (int w = 0; w < W; ++w) rank_row[(size_t)s * W + w] = w * B + s;
            sel.beam_begin(*this, rank_row, B);
        }
        CUDA_OK(cudaEventRecord(ev[4], st));
        run_steps(R, S4 - P - 1, [&] {
            const unsigned launches = decode_step(R);
            if (W > 1) sel.beam_step(*this, B, W);
            return launches;
        });
        if (W > 1) sel.traceback(*this, std::vector<int>(B, n_out).data(), B, 1);
    } else if (W > 1) {
        sel.zero_nbest_scores(0, B, st);
    }
    if (S4 < P) CUDA_OK(cudaEventRecord(ev[4], st));
    CUDA_OK(cudaEventRecord(ev[3], st));
    std::vector<int> host((size_t)B * out_ld);
    if (n_out > 0) CUDA_OK(cudaMemcpyAsync(host.data(), d_out, sizeof(int) * host.size(), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b)
        for (int i = 0; i < n_out; ++i) out_ids[(size_t)b * n_out + i] = host[(size_t)b * out_ld + i];
    if (W > 1) {
        // the cache holds W hypotheses per stream, not one: the incremental API starts over, on the identity page table
        reset();
        CUDA_OK(cudaStreamSynchronize(st));
    } else {
        cache_len = n_out > 0 ? S4 - 1 : 0;
        if (S4 >= P)   // the prefill's output and one per step
            for (int b = 0; b < B; ++b) out_rows[b] = std::max(n_out, 1);
    }
    std::vector<int> order(B), n(B, n_out);   // stream b's rank 0 beam is row b, the traceback's ids are [B][W][n_out]
    for (int b = 0; b < B; ++b) order[b] = b;
    sel.record_transcribe(B, order.data(), n.data(), 1, total);
    if (tm) {
        tm->seq_len = S4;
        tm->decode_tokens = n_out;
    }
    return n_out;
}

// ======================================================================================
// Streams of different lengths in one call (vox_transcribe_pcm_ragged)
// ======================================================================================

// Streams sorted (stably) by decreasing output count own the rows: beams w of sorted stream i run in row i * W + w, so
// the streams that still need tokens are always the rows [0, R).  Every stream with output takes the prefill; then the
// steps run in segments, one per distinct output count, each over the rows still live.
//
// transcribe_from_mel is not this function at equal lengths, and moving it here would change what it costs and computes:
//   - it prefills b rows and replicates them to the beam rows (then beam_begin).  Here the rows are stream-major, so that the
//     live streams stay a prefix of the rows; a prefill row is then both a fork source and another stream's fork
//     destination, and all b * W rows take the prefill: the prefill GEMMs' M grows W-fold (38 -> 304 at 1 stream x 8
//     beams; not measured for that case).
//   - another beam row layout moves a beam into another group of 8 rows when b * W > 8.  The persistent kernel's
//     attn_chunks follows the group's row count, so the softmax merge order, and with it the low bits, would change.
void Session::transcribe_ragged(const float *samples, const size_t *lens, int b, int normalize, int32_t *out_ids,
                                int32_t *n_out, vox_timings *tm) {
    const vox_model_info &c = m->info;
    const int W = sel.beam_w, P = c.prefix_len;
    check_batch(b);
    sel.check_rows(b);
    std::vector<StreamGeom> g(b);
    for (int s = 0; s < b; ++s) {
        g[s] = stream_geometry(c, lens[s]);
        n_out[s] = g[s].n_out;
    }
    CUDA_OK(cudaSetDevice(m->device));
    enc.prepare_pcm(*this, lens, b, true);
    std::vector<int> order(b);
    for (int s = 0; s < b; ++s) order[s] = s;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return g[x].n_out > g[y].n_out; });
    int live = 0;
    while (live < b && g[order[live]].n_out > 0) ++live;
    std::vector<int> row0(b);   // stream s's rank 0 beam
    RowStreams row_guard{this};
    row_streams.assign((size_t)b * W, 0);
    for (int i = 0; i < b; ++i) {
        row0[order[i]] = i * W;
        for (int w = 0; w < W; ++w) row_streams[(size_t)i * W + w] = order[i];
    }

    CUDA_OK(cudaEventRecord(ev[0], st));
    enc.pcm_to_mel(*this, samples, nullptr, lens, b, normalize);
    CUDA_OK(cudaEventRecord(ev[1], st));
    enc.encode(*this, b, enc.front.frames.data());
    cur_B = b * W;   // the call's decoder rows, whose logits debug "logits" reads
    CUDA_OK(cudaEventRecord(ev[2], st));

    const int n_max = live > 0 ? g[order[0]].n_out : 0;
    reset();
    if (live > 0) {
        const int R0 = live * W;
        // prefix = [BOS] + [STREAMING_PAD]*37 (model.rs:883-892) in every row, each beam row of a stream included: the
        // first selection then reads one parent row per stream (its rank 0) and forks it into the others
        std::vector<int> prefix((size_t)R0 * P, 32);
        for (int r = 0; r < R0; ++r) prefix[(size_t)r * P] = 1;
        prefill(R0, P, prefix.data(), true);
        if (W > 1) {
            std::vector<int> rank_row(R0);
            for (int r = 0; r < R0; ++r) rank_row[r] = r;
            sel.beam_begin(*this, rank_row, live);
        }
        CUDA_OK(cudaEventRecord(ev[4], st));
        for (int t = 1; t < n_max;) {   // outputs [0, t) of every live stream are done
            int L = 0;
            while (L < live && g[order[L]].n_out > t) ++L;
            const int t_end = g[order[L - 1]].n_out;
            run_steps(L * W, t_end - t, [&] {
                const unsigned launches = decode_step(L * W);
                if (W > 1) sel.beam_step(*this, L, W);
                return launches;
            });
            t = t_end;
        }
        if (W > 1) {
            std::vector<int> n_sorted(live);
            for (int i = 0; i < live; ++i) n_sorted[i] = g[order[i]].n_out;
            sel.traceback(*this, n_sorted.data(), live, W);
        }
    } else {
        CUDA_OK(cudaEventRecord(ev[4], st));
    }
    CUDA_OK(cudaEventRecord(ev[3], st));

    if (W > 1 && live < b) sel.zero_nbest_scores(live, b, st);   // a stream without output has no hypotheses

    // ids back in the caller's stream order: stream s's outputs are in the row of its rank 0 beam, row0[s]
    std::vector<int> host((size_t)live * W * out_ld);
    if (live > 0) CUDA_OK(cudaMemcpyAsync(host.data(), d_out, sizeof(int) * host.size(), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    size_t total = 0;
    for (int s = 0; s < b; total += g[s].n_out, ++s)
        for (int i = 0; i < g[s].n_out; ++i) out_ids[total + i] = host[(size_t)row0[s] * out_ld + i];
    // scores and n-best stay on the device, sorted stream i's in row i * W and at the traceback's i-th list
    sel.record_transcribe(b, order.data(), n_out, W, true);
    // the cache holds streams of different lengths (and perhaps beams): the incremental API starts over
    reset();
    CUDA_OK(cudaStreamSynchronize(st));
    if (tm) {
        int S4_long = 0;
        for (const StreamGeom &x : g) S4_long = std::max(S4_long, x.S4);
        tm->seq_len = S4_long;
        tm->decode_tokens = n_max;
    }
}

}  // namespace vox
