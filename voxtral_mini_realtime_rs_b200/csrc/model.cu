// model.cu -- GGUF -> HBM loader (with load-time Q4 repack) and the session that runs
// encode_audio / prefill / decode on one CUDA stream.  Graph semantics follow the reference's
// src/gguf/model.rs (cited per function); nothing here is a translation of its Burn code.
#include "model.h"

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
    // RoPEConfig::init (rope.rs:35-64), f32 throughout
    const int half = hd / 2;
    std::vector<float> inv(half), c((size_t)max_seq * half), s((size_t)max_seq * half);
    for (int i = 0; i < half; ++i) inv[i] = 1.0f / powf(theta, (float)(2 * i) / (float)hd);
    for (int p = 0; p < max_seq; ++p)
        for (int i = 0; i < half; ++i) {
            const float f = (float)p * inv[i];
            c[(size_t)p * half + i] = cosf(f);
            s[(size_t)p * half + i] = sinf(f);
        }
    *cos_d = arena.upload(c.data(), c.size());
    *sin_d = arena.upload(s.data(), s.size());
}

}  // namespace

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
static int conv_out(int t) { return (t + 2 - 3) / 2 + 1; }  // conv.rs:47-48

Session *Session::create(Model *m, int max_batch, int max_mel_frames) {
    VOX_CHECK(max_batch >= 1 && max_batch <= 64, VOX_EINVAL, "max_batch %d out of range [1,64]", max_batch);
    VOX_CHECK(max_mel_frames >= 16, VOX_EINVAL, "max_mel_frames %d too small", max_mel_frames);
    CUDA_OK(cudaSetDevice(m->device));
    Session *s = new Session();
    try {
        const vox_model_info &c = m->info;
        s->m = m;
        s->arena.device = m->device;
        s->max_batch = max_batch;
        s->max_mel_frames = max_mel_frames;
        s->T1_max = conv_out(max_mel_frames);
        s->S_max = conv_out(s->T1_max);
        s->S4_max = s->S_max / c.reshape_factor;
        s->M_max = std::max(c.prefix_len, 64);
        VOX_CHECK(s->S_max <= m->enc_rope_len, VOX_EINVAL, "max_mel_frames %d exceeds the encoder RoPE table", max_mel_frames);
        CUDA_OK(cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking));
        for (auto &e : s->ev) CUDA_OK(cudaEventCreate(&e));
        const size_t B = max_batch;
        const int hdq = c.enc_heads * c.enc_head_dim;
        s->mel = s->arena.alloc_n<float>(B * c.n_mels * max_mel_frames);
        s->mel_tm = s->arena.alloc_n<float>(B * c.n_mels * max_mel_frames);
        s->peak_scale = s->arena.alloc_n<float>(B);
        s->h1 = s->arena.alloc_n<float>(B * s->T1_max * c.enc_dim);
        const size_t rows = B * s->S_max;
        s->x_enc = s->arena.alloc_n<float>(rows * c.enc_dim);
        s->h_enc = s->arena.alloc_n<float>(rows * c.enc_dim);
        s->qkv_enc = s->arena.alloc_n<float>(rows * 3 * hdq);
        s->attn_enc = s->arena.alloc_n<float>(rows * hdq);
        s->act_enc = s->arena.alloc_n<float>(rows * c.enc_ffn);
        const size_t rows4 = B * std::max(s->S4_max, 1);
        s->packed = s->arena.alloc_n<float>(rows4 * c.enc_dim * c.reshape_factor);
        s->adapter_h = s->arena.alloc_n<float>(rows4 * c.dec_dim);
        s->audio = s->arena.alloc_n<float>(rows4 * c.dec_dim);
        // decoder
        const int kv_cap = std::max(s->S4_max, s->M_max) + s->M_max;  // room for the incremental API
        s->kv_max_pages = (kv_cap + KV_PAGE - 1) / KV_PAGE;
        s->kv_n_pages = max_batch * s->kv_max_pages;
        s->out_ld = s->kv_max_pages * KV_PAGE;
        const size_t kv_elems = (size_t)c.dec_layers * s->kv_n_pages * c.dec_kv_heads * KV_PAGE * c.dec_head_dim;
        s->kc = s->arena.alloc_n<float>(kv_elems);
        s->vc = s->arena.alloc_n<float>(kv_elems);
        s->page_table_host.resize((size_t)max_batch * s->kv_max_pages);
        for (int b = 0; b < max_batch; ++b)
            for (int pg = 0; pg < s->kv_max_pages; ++pg) s->page_table_host[(size_t)b * s->kv_max_pages + pg] = b * s->kv_max_pages + pg;
        s->d_page_table = s->arena.upload(s->page_table_host.data(), s->page_table_host.size());
        const size_t drows = B * s->M_max;
        const int qkvd = (c.dec_heads + 2 * c.dec_kv_heads) * c.dec_head_dim;
        s->x_dec = s->arena.alloc_n<float>(drows * c.dec_dim);
        s->h_dec = s->arena.alloc_n<float>(drows * c.dec_dim);
        s->qkv_dec = s->arena.alloc_n<float>(drows * qkvd);
        s->attn_dec = s->arena.alloc_n<float>(drows * c.dec_heads * c.dec_head_dim);
        s->act_dec = s->arena.alloc_n<float>(drows * c.dec_ffn);
        s->last_h = s->arena.alloc_n<float>(B * c.dec_dim);
        s->logits = s->arena.alloc_n<float>(B * c.vocab);
        s->ada = s->arena.alloc_n<float>((size_t)c.dec_layers * c.dec_dim);
        s->ffn_gamma_ada = s->arena.alloc_n<float>((size_t)c.dec_layers * c.dec_dim);
        s->t_embed = s->arena.alloc_n<float>(c.dec_dim);
        s->ada_tmp = s->arena.alloc_n<float>(c.t_cond_dim);
        s->d_pos = s->arena.alloc_n<int>(B);      // per row (kernels.h KvView::pos)
        s->d_outpos = s->arena.alloc_n<int>(B);
        s->d_tok = s->arena.alloc_n<int>(B);
        s->d_ids = s->arena.alloc_n<int>(drows);
        s->d_out = s->arena.alloc_n<int>(B * s->out_ld);
        {   // split-tile buffer of the wgmma GEMM: largest (rows, K) pair it is used with
            const int rows_e = max_batch * s->S_max, rows_d = max_batch * s->M_max;
            size_t e = 0;
            for (int K : {c.enc_dim, c.enc_heads * c.enc_head_dim, c.enc_ffn}) e = std::max(e, gemm_tc5_split_elems(rows_e, K / 64 * 64));
            e = std::max(e, gemm_tc5_split_elems(max_batch * std::max(s->S4_max, 1), c.enc_dim * c.reshape_factor / 64 * 64));
            for (int K : {c.dec_dim, c.dec_heads * c.dec_head_dim, c.dec_ffn}) e = std::max(e, gemm_tc5_split_elems(std::max(rows_d, max_batch * std::max(s->S4_max, 1)), K / 64 * 64));
            s->xt_elems = e;
            s->xt_buf = s->arena.alloc(e * 2);
            // split-K scratch of the wgmma GEMM: at most one (slice, tile) partial tile per SM in flight
            s->gemm_work.partial_floats = (size_t)VOX_NUM_SMS * 128 * 128;
            s->gemm_work.partial = s->arena.alloc_n<float>(s->gemm_work.partial_floats);
            s->gemm_work.n_counters = 128;
            s->gemm_work.counters = s->arena.alloc_n<int>(s->gemm_work.n_counters);
            CUDA_OK(cudaMemset(s->gemm_work.counters, 0, sizeof(int) * s->gemm_work.n_counters));
            const char *gv = getenv("VOX_GEMM");
            s->use_gemm_tc = !(gv && std::string(gv) == "simt");
            const char *tv = getenv("VOX_MATVEC");
            s->use_tc = !(tv && std::string(tv) == "simt");
            const char *av = getenv("VOX_ENC_ATTN");
            s->use_enc_attn_tc = !(av && std::string(av) == "simt");
        }
        {   // fused-decode scratch (see TcWork): sized for the largest split-K matvec at max_batch rows
            const int mb = std::min(8, max_batch * 1);
            size_t need = 0;
            auto acc_need = [&](int N, int K) {
                const int n_pairs = (K / 32 + 1) / 2;
                const int S = (n_pairs + 15) / 16;  // worst case: 16 pairs per slice (M > 4)
                need = std::max(need, (size_t)S * 8 * (size_t)((N + 15) / 16) * 16);
            };
            const int qkvd2 = (c.dec_heads + 2 * c.dec_kv_heads) * c.dec_head_dim;
            acc_need(qkvd2, c.dec_dim);
            acc_need(c.dec_dim, c.dec_heads * c.dec_head_dim);
            acc_need(2 * c.dec_ffn, c.dec_dim);
            acc_need(c.dec_dim, c.dec_ffn);
            acc_need(c.vocab, c.dec_dim);
            (void)mb;
            s->tc_partial_floats = need;
            s->tc_partial = s->arena.alloc_n<float>(need);
            s->tc_n_counters = std::max((c.vocab + 15) / 16, (2 * c.dec_ffn + 15) / 16) + 16;
            s->tc_counters = s->arena.alloc_n<int>(s->tc_n_counters);
            CUDA_OK(cudaMemset(s->tc_counters, 0, sizeof(int) * s->tc_n_counters));
            s->ssq_x = s->arena.alloc_n<float>((size_t)((c.dec_dim + 15) / 16) * 8);
            s->am_vals = s->arena.alloc_n<float>((size_t)max_batch * ARGMAX_PARTS);
            s->am_idx = s->arena.alloc_n<int>((size_t)max_batch * ARGMAX_PARTS);
            s->am_cnt = s->arena.alloc_n<int>(max_batch);
            CUDA_OK(cudaMemset(s->am_cnt, 0, sizeof(int) * max_batch));
        }
        {   // persistent decode-step kernel
            const char *mv = getenv("VOX_MEGA");
            s->use_mega = !(mv && mv[0] == '0');
            if (const char *mb = getenv("VOX_MEGA_MIN_B")) s->mega_min_B = atoi(mb);
            s->mega_grid = decode_mega_grid(m->device);
            s->mega_ops_cap = 6 * c.dec_layers + 4;
            s->mega_ops = s->arena.alloc_n<MegaOp>(s->mega_ops_cap);
            s->mega_bar = s->arena.alloc_n<unsigned>(4);
            CUDA_OK(cudaMemset(s->mega_bar, 0, sizeof(unsigned) * 4));
            s->mega_am_vals = s->arena.alloc_n<float>((size_t)s->mega_grid * 8);
            s->mega_am_idx = s->arena.alloc_n<int>((size_t)s->mega_grid * 8);
            s->mega_att_units = std::max(s->mega_grid, 8 * c.dec_kv_heads) + 8 * c.dec_kv_heads;
            s->mega_att_acc = s->arena.alloc_n<float>((size_t)2 * s->mega_att_units * (c.dec_heads / c.dec_kv_heads) * c.dec_head_dim);  // {value, tag}
            s->mega_att_ml = s->arena.alloc_n<float>((size_t)2 * s->mega_att_units * (c.dec_heads / c.dec_kv_heads) * 2);  // {value, tag}
            s->mega_att_flags = s->arena.alloc_n<int>(s->mega_att_units);
            s->mega_epoch = s->arena.alloc_n<int>(1);
            CUDA_OK(cudaMemset(s->mega_att_flags, 0, sizeof(int) * s->mega_att_units));
            // chunk states carry their own validity tag (decode step, layer): never 0
            CUDA_OK(cudaMemset(s->mega_att_acc, 0, sizeof(float) * 2 * s->mega_att_units * (c.dec_heads / c.dec_kv_heads) * c.dec_head_dim));
            CUDA_OK(cudaMemset(s->mega_att_ml, 0, sizeof(float) * 2 * s->mega_att_units * (c.dec_heads / c.dec_kv_heads) * 2));
            CUDA_OK(cudaMemset(s->mega_epoch, 0, sizeof(int)));
            {
                auto blocks = [](int K) { return (size_t)((K / 32 + 1) / 2) * 2; };
                s->mega_xf_blocks = blocks(c.dec_dim);
                s->mega_af_blocks = blocks(c.dec_heads * c.dec_head_dim);
                s->mega_cf_blocks = blocks(c.dec_ffn);
                s->mega_xf_bf = s->arena.alloc_n<uint2>(s->mega_xf_blocks * 16 * 8);
                s->mega_af_bf = s->arena.alloc_n<uint2>(s->mega_af_blocks * 16 * 8);
                s->mega_cf_bf = s->arena.alloc_n<uint2>(s->mega_cf_blocks * 16 * 8);
                s->mega_xf_off = s->arena.alloc_n<float2>(s->mega_xf_blocks * 8);
                s->mega_af_off = s->arena.alloc_n<float2>(s->mega_af_blocks * 8);
                s->mega_cf_off = s->arena.alloc_n<float2>(s->mega_cf_blocks * 8);
            }
            s->mega_trace = s->arena.alloc_n<unsigned long long>((size_t)s->mega_ops_cap * 6);
            CUDA_OK(cudaMemset(s->mega_trace, 0, sizeof(unsigned long long) * s->mega_ops_cap * 6));
            if (const char *ta = getenv("VOX_MEGA_TRACE_ALL")) {
                if (ta[0] == '1') {
                    const size_t n = (size_t)s->mega_grid * s->mega_ops_cap * 4;
                    s->mega_trace_all = s->arena.alloc_n<unsigned long long>(n);
                    CUDA_OK(cudaMemset(s->mega_trace_all, 0, sizeof(unsigned long long) * n));
                    s->mega_trace_w = s->arena.alloc_n<unsigned long long>(16 * 6 * 8);
                    CUDA_OK(cudaMemset(s->mega_trace_w, 0, sizeof(unsigned long long) * 16 * 6 * 8));
                }
            }
        }
        CUDA_OK(cudaMemset(s->d_pos, 0, sizeof(int) * B));
        CUDA_OK(cudaMemset(s->d_outpos, 0, sizeof(int) * B));
        s->set_delay(6.0f);  // CLI default --delay 6 (transcribe.rs:49-51)
    } catch (...) {
        delete s;
        throw;
    }
    return s;
}

Session::~Session() {
    if (step_graph) cudaGraphExecDestroy(step_graph);
    for (auto &e : ev)
        if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
}

void Session::linear_n(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias, const float *res,
                       int epi, const float *gamma, const float *ada, float *tmp) {
    if (M > 8 && use_gemm_tc && gemm_tc5_supported(w, M) && gemm_tc5_split_elems(M, w.K) <= xt_elems) {
        launch_split_tiles(x, M, w.K, gamma, ada, m->norm_eps, xt_buf, st);
        launch_q4_gemm_tc5(w, xt_buf, M, y, ldy, bias, res, epi, &gemm_work, st);
        return;
    }
    if (gamma) {
        launch_rmsnorm(x, gamma, ada, tmp, M, w.K, m->norm_eps, st);
        x = tmp;
    }
    linear(w, x, M, y, ldy, bias, res, epi);
}

void Session::linear(const Q4Weight &w, const float *x, int M, float *y, int ldy, const float *bias,
                     const float *res, int epi) {
    if (M > 8 && use_gemm_tc && gemm_tc5_supported(w, M) && gemm_tc5_split_elems(M, w.K) <= xt_elems) {
        launch_split_tiles(x, M, w.K, nullptr, nullptr, 0.0f, xt_buf, st);
        launch_q4_gemm_tc5(w, xt_buf, M, y, ldy, bias, res, epi, &gemm_work, st);
        return;
    }
    if (M <= 8 && w.qs_tc && use_tc) launch_q4_matvec_tc(w, x, M, y, ldy, bias, res, epi, st);
    else if (M <= 8) launch_q4_matvec(w, x, M, y, ldy, bias, res, epi, st);
    else launch_q4_gemm(w, x, M, y, ldy, bias, res, epi, st);
}

// TimeEmbedding::embed (time_embedding.rs:41-71) + the per-layer ADA scale
// 1 + w2(gelu(w0(t)))  (model.rs:250-255), computed once: t is constant for a session.
void Session::set_delay(float delay) {
    const vox_model_info &c = m->info;
    CUDA_OK(cudaSetDevice(m->device));
    std::vector<float> t(c.dec_dim);
    time_embedding(delay, c.dec_dim, t.data());
    CUDA_OK(cudaMemcpyAsync(t_embed, t.data(), sizeof(float) * c.dec_dim, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
    std::vector<float> ones(c.dec_dim, 1.0f);
    for (int j = 0; j < c.dec_layers; ++j) {
        float *dst = ada + (size_t)j * c.dec_dim;
        CUDA_OK(cudaMemcpyAsync(dst, ones.data(), sizeof(float) * c.dec_dim, cudaMemcpyHostToDevice, st));
        launch_q4_matvec(m->dec[j].ada0, t_embed, 1, ada_tmp, c.t_cond_dim, nullptr, nullptr, EPI_GELU, st);
        // dst = 1 + w2 . gelu(...)   (residual epilogue onto the vector of ones)
        launch_q4_matvec(m->dec[j].ada2, ada_tmp, 1, dst, c.dec_dim, nullptr, dst, EPI_RESIDUAL, st);
        launch_mul_vec(m->dec[j].ffn_norm, dst, ffn_gamma_ada + (size_t)j * c.dec_dim, c.dec_dim, st);
    }
    CUDA_OK(cudaStreamSynchronize(st));
    delay_set = true;
}

// Q4VoxtralModel::encode_audio (model.rs:783-788): conv -> 32 layers -> norm -> reshape x4 -> adapter
void Session::encode(int B, int T) {
    const vox_model_info &c = m->info;
    VOX_CHECK(B >= 1 && B <= max_batch, VOX_EINVAL, "batch %d exceeds session max_batch %d", B, max_batch);
    VOX_CHECK(T >= 1 && T <= max_mel_frames, VOX_EINVAL, "mel frames %d exceed session max_mel_frames %d", T, max_mel_frames);
    const int T1 = conv_out(T), S = conv_out(T1), S4 = S / c.reshape_factor;
    const int d = c.enc_dim, hdq = c.enc_heads * c.enc_head_dim;
    const int rows = B * S;
    // conv1 + GELU as implicit GEMM over the time-major mel [B][T][128] (K = 3*128)
    launch_conv2_gemm(mel_tm, m->conv1_w, m->conv1_b, h1, B, T, T1, c.n_mels, d, st);
    launch_conv2_gemm(h1, m->conv2_w, m->conv2_b, x_enc, B, T1, S, d, d, st);
    if (debug_capture && dbg_conv) CUDA_OK(cudaMemcpyAsync(dbg_conv, x_enc, sizeof(float) * rows * d, cudaMemcpyDeviceToDevice, st));
    const float scale = powf((float)c.enc_head_dim, -0.5f);
    for (int i = 0; i < c.enc_layers; ++i) {
        const EncLayerW &l = m->enc[i];
        linear_n(l.wqkv, x_enc, rows, qkv_enc, 3 * hdq, l.bqkv, nullptr, EPI_NONE, l.attn_norm, nullptr, h_enc);
        launch_rope_inplace(qkv_enc, rows, 3 * hdq, 0, c.enc_heads, hdq, c.enc_heads, c.enc_head_dim, S, 0,
                            m->enc_cos, m->enc_sin, st);
        if (use_enc_attn_tc && enc_attention_tc_supported(c.enc_head_dim, 3 * hdq, 0, hdq, 2 * hdq))
            launch_enc_attention_tc(qkv_enc, attn_enc, B, S, c.enc_heads, c.enc_head_dim, 3 * hdq, 0, hdq, 2 * hdq,
                                    c.enc_window, scale, st);
        else
            launch_enc_attention(qkv_enc, attn_enc, B, S, c.enc_heads, c.enc_head_dim, 3 * hdq, 0, hdq, 2 * hdq,
                                 c.enc_window, scale, st);
        linear(l.wo, attn_enc, rows, x_enc, d, l.bo, x_enc, EPI_RESIDUAL);
        linear_n(l.w13, x_enc, rows, act_enc, c.enc_ffn, nullptr, nullptr, EPI_SILU_MUL, l.ffn_norm, nullptr, h_enc);
        linear(l.w2, act_enc, rows, x_enc, d, l.b2, x_enc, EPI_RESIDUAL);
        if (debug_capture && dbg_layers)
            CUDA_OK(cudaMemcpyAsync(dbg_layers + (size_t)i * rows * d, x_enc, sizeof(float) * rows * d,
                                    cudaMemcpyDeviceToDevice, st));
    }
    launch_rmsnorm(x_enc, m->enc_norm, nullptr, h_enc, rows, d, m->norm_eps, st);
    cur_B = B;
    cur_S = S;
    cur_S4 = S4;
    if (S4 > 0) {
        launch_reshape_rows(h_enc, packed, B, S, S4, d, c.reshape_factor, st);
        linear(m->adapter0, packed, B * S4, adapter_h, c.dec_dim, nullptr, nullptr, EPI_GELU);
        linear(m->adapter2, adapter_h, B * S4, audio, c.dec_dim, nullptr, nullptr, EPI_NONE);
    }
}

// Q4LanguageModel::forward_hidden_with_cache (model.rs:665-677) over x_dec [B*M][D]; positions
// *d_pos + i.  Leaves the final-normed hidden states in h_dec -- or, on the fused decode path, returns
// true and leaves the un-normed stream in x_dec for lm_head_rows().  Does not advance *d_pos.
bool Session::fused_decode(int rows) const { return use_tc && rows <= 8 && m->tok_emb.qs_tc != nullptr; }

TcWork Session::tc_work(bool norm_in, bool ssq_out_) const {
    TcWork w;
    w.partial = tc_partial;
    w.partial_floats = tc_partial_floats;
    w.counters = tc_counters;
    w.n_counters = tc_n_counters;
    if (norm_in) {
        w.ssq_in = ssq_x;
        w.ssq_in_parts = (m->info.dec_dim + 15) / 16;
    }
    if (ssq_out_) w.ssq_out = ssq_x;
    return w;
}

KvView Session::kv_view(int layer) const {
    KvView v;
    v.k = kc + (size_t)layer * kv_layer_stride();
    v.v = vc + (size_t)layer * kv_layer_stride();
    v.page_table = d_page_table;
    v.max_pages = kv_max_pages;
    v.pos = d_pos;
    return v;
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
    const bool fattn = fused && M == 1 && dec_attn_fused_supported(H, Hkv, hd);
    for (int j = 0; j < c.dec_layers; ++j) {
        const DecLayerW &l = m->dec[j];
        const KvView kvl = kv_view(j);
        if (fused) {
            launch_q4_matvec_tc_ex(l.wqkv, x_dec, rows, qkv_dec, qkvd, nullptr, nullptr, EPI_NONE, l.attn_norm, nullptr,
                                   m->norm_eps, &wk_norm, st);
        } else {
            linear_n(l.wqkv, x_dec, rows, qkv_dec, qkvd, nullptr, nullptr, EPI_NONE, l.attn_norm, nullptr, h_dec);
        }
        if (fattn) {
            launch_dec_attn_fused(qkv_dec, B, qkvd, H, Hkv, hd, kvl, c.dec_window, scale, m->dec_cos, m->dec_sin, attn_dec, st);
        } else {
            launch_dec_rope_append(qkv_dec, B, M, qkvd, H, Hkv, hd, kvl, m->dec_cos, m->dec_sin, st);
            launch_dec_attention(qkv_dec, B, M, qkvd, H, Hkv, hd, kvl, c.dec_window, scale, attn_dec, st);
        }
        if (fused)
            launch_q4_matvec_tc_ex(l.wo, attn_dec, rows, x_dec, D, nullptr, x_dec, EPI_RESIDUAL, nullptr, nullptr, 0.f, &wk_res, st);
        else
            linear(l.wo, attn_dec, rows, x_dec, D, nullptr, x_dec, EPI_RESIDUAL);
        if (fused) {
            launch_q4_matvec_tc_ex(l.w13, x_dec, rows, act_dec, c.dec_ffn, nullptr, nullptr, EPI_SILU_MUL, l.ffn_norm,
                                   ada + (size_t)j * D, m->norm_eps, &wk_norm, st);
        } else {
            linear_n(l.w13, x_dec, rows, act_dec, c.dec_ffn, nullptr, nullptr, EPI_SILU_MUL, l.ffn_norm, ada + (size_t)j * D, h_dec);
        }
        if (fused)
            launch_q4_matvec_tc_ex(l.w2, act_dec, rows, x_dec, D, nullptr, x_dec, EPI_RESIDUAL, nullptr, nullptr, 0.f, &wk_res, st);
        else
            linear(l.w2, act_dec, rows, x_dec, D, nullptr, x_dec, EPI_RESIDUAL);
    }
    if (!fused) launch_rmsnorm(x_dec, m->dec_norm, nullptr, h_dec, rows, D, m->norm_eps, st);
    return fused;
}

// lm_head over `rows` decoder rows (model.rs:680-691); `norm_pending`: x_dec still needs the final
// RMSNorm (fused into the matvec), else h_dec already holds the normed hidden states.
void Session::lm_head_rows(int rows, bool norm_pending, float *dst) {
    const vox_model_info &c = m->info;
    if (norm_pending) {
        const TcWork wk = tc_work(true, false);
        launch_q4_matvec_tc_ex(m->tok_emb, x_dec, rows, dst, c.vocab, nullptr, nullptr, EPI_NONE, m->dec_norm, nullptr,
                               m->norm_eps, &wk, st);
    }
    else
        linear(m->tok_emb, h_dec, rows, dst, c.vocab, nullptr, nullptr, EPI_NONE);
}

// Builds (once per batch size) the op table of the persistent decode-step kernel.  Returns false when
// the shapes are outside what decode_mega.cu is instantiated for; the caller then uses per-op launches.
bool Session::mega_prepare(int B) {
    const vox_model_info &c = m->info;
    if (!use_mega || !use_tc || !fused_decode(B) || B < mega_min_B) return false;
    if (!decode_mega_supported(B, c.dec_heads, c.dec_kv_heads, c.dec_head_dim)) return false;
    if (mega_B == B) return mega_n_ops > 0;
    mega_B = B;
    mega_n_ops = 0;
    const int D = c.dec_dim, H = c.dec_heads, Hkv = c.dec_kv_heads, hd = c.dec_head_dim;
    const int qkvd = (H + 2 * Hkv) * hd;
    for (int j = 0; j < c.dec_layers; ++j)
        if (!m->dec[j].wqkv.qs_tc || !m->dec[j].wo.qs_tc || !m->dec[j].w13.qs_tc || !m->dec[j].w2.qs_tc) return false;
    auto pairs = [](int K) { return (K / 32 + 1) / 2; };
    const int max_pairs = std::max(std::max(pairs(D), pairs(H * hd)), pairs(c.dec_ffn));
    mega_plan = decode_mega_plan(B, max_pairs, H, Hkv, hd);
    const size_t layer_stride = kv_layer_stride();
    const int parts = (D + 15) / 16;
    std::vector<MegaOp> ops;
    bool ok = true;
    struct Frag { uint2 *bf; float2 *off; };
    const Frag XF{mega_xf_bf, mega_xf_off}, AF{mega_af_bf, mega_af_off}, CF{mega_cf_bf, mega_cf_off};
    auto matvec = [&](const Q4Weight &w, Frag fin, float *y, int ldy, const float *res, int epi, const float *norm_w,
                      bool ssq_out_, bool track, int unit_tiles, Frag fout, const float *fout_gamma) {
        MegaOp o;
        o.kind = MG_MATVEC;
        o.epi = epi;
        o.qs_tc = w.qs_tc;
        o.d_tc = w.d_tc;
        o.N = w.N;
        o.K = w.K;
        o.n_tiles = (w.N + 15) / 16;
        o.n_pairs = pairs(w.K);
        int S = (o.n_pairs + mega_plan.Ps_cap - 1) / mega_plan.Ps_cap;
        int Ps = (o.n_pairs + S - 1) / S;
        if (S > 1) Ps = std::min(mega_plan.Ps_cap, (Ps + 15) / 16 * 16);
        S = (o.n_pairs + Ps - 1) / Ps;
        o.S = S;
        o.Ps = Ps;
        o.unit_tiles = unit_tiles;
        if (o.n_tiles % unit_tiles != 0) ok = false;
        const int n_units = o.n_tiles / unit_tiles;
        // tile sums kept in shared memory across K slices: 2 tiles per CTA
        if (S > 1 && ((n_units + mega_grid - 1) / mega_grid) * unit_tiles > 2) ok = false;
        o.fin_bf = fin.bf;
        o.fin_off = fin.off;
        o.fout_bf = fout.bf;
        o.fout_off = fout.off;
        o.fout_gamma = fout_gamma;
        o.y = y;
        o.ldy = ldy;
        o.res = res;
        o.gamma = norm_w;  // != nullptr: the input is RMS-normalised (1/rms applied in the epilogue)
        if (norm_w) {
            o.ssq_in = ssq_x;
            o.ssq_in_parts = parts;
        }
        if (ssq_out_) o.ssq_out = ssq_x;
        o.track_argmax = track ? 1 : 0;
        ops.push_back(o);
    };
    const Frag none{nullptr, nullptr};
    {
        MegaOp e;
        e.kind = MG_EMBED;
        ops.push_back(e);
    }
    for (int j = 0; j < c.dec_layers; ++j) {
        const DecLayerW &l = m->dec[j];
        matvec(l.wqkv, XF, qkv_dec, qkvd, nullptr, EPI_NONE, l.attn_norm, false, false, 1, none, nullptr);
        MegaOp a;
        a.kind = MG_ATTN;
        a.kc = kc + (size_t)j * layer_stride;
        a.vc = vc + (size_t)j * layer_stride;
        a.layer = j;
        ops.push_back(a);
        // wo: h += attn . Wo^T; leaves fragments of h x (ffn_norm x ADA) for w13
        matvec(l.wo, AF, x_dec, D, x_dec, EPI_RESIDUAL, nullptr, true, false, 2, XF, ffn_gamma_ada + (size_t)j * D);
        // w13: SwiGLU of the normed stream; leaves fragments of the activation for w2 (no plain copy)
        matvec(l.w13, XF, nullptr, c.dec_ffn, nullptr, EPI_SILU_MUL, l.ffn_norm, false, false, 4, CF, nullptr);
        // w2: h += act . W2^T; leaves fragments of h x (next attention norm | final norm)
        const float *next_norm = j + 1 < c.dec_layers ? m->dec[j + 1].attn_norm : m->dec_norm;
        matvec(l.w2, CF, x_dec, D, x_dec, EPI_RESIDUAL, nullptr, true, false, 2, XF, next_norm);
    }
    matvec(m->tok_emb, XF, logits, c.vocab, nullptr, EPI_NONE, m->dec_norm, false, true, 1, none, nullptr);
    {
        MegaOp f;
        f.kind = MG_ARGMAX;
        ops.push_back(f);
    }
    if (c.dec_ffn % 32 != 0 || (H * hd) % 32 != 0 || c.dec_layers > 63) ok = false;
    // the residual epilogues and the embedding must leave exactly `parts` partial sums of squares
    if ((D + 15) / 16 != parts || D % 32 != 0) ok = false;
    if (!ok || (int)ops.size() > mega_ops_cap) return false;
    // padding tokens (capacity MT > B) and padding blocks must read as zero fragments
    CUDA_OK(cudaMemsetAsync(mega_xf_bf, 0, sizeof(uint2) * mega_xf_blocks * 16 * 8, st));
    CUDA_OK(cudaMemsetAsync(mega_af_bf, 0, sizeof(uint2) * mega_af_blocks * 16 * 8, st));
    CUDA_OK(cudaMemsetAsync(mega_cf_bf, 0, sizeof(uint2) * mega_cf_blocks * 16 * 8, st));
    CUDA_OK(cudaMemsetAsync(mega_xf_off, 0, sizeof(float2) * mega_xf_blocks * 8, st));
    CUDA_OK(cudaMemsetAsync(mega_af_off, 0, sizeof(float2) * mega_af_blocks * 8, st));
    CUDA_OK(cudaMemsetAsync(mega_cf_off, 0, sizeof(float2) * mega_cf_blocks * 8, st));
    mega_ops_host = ops;
    CUDA_OK(cudaMemcpyAsync(mega_ops, mega_ops_host.data(), sizeof(MegaOp) * ops.size(), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
    mega_n_ops = (int)ops.size();
    return true;
}

// One autoregressive step for B streams (model.rs:938-960): embed(prev token) + audio[pos-1],
// 26 layers, lm_head, argmax, device-side feedback; all positions read from device counters.
void Session::decode_step(int B, bool add_audio) {
    const vox_model_info &c = m->info;
    // More than 8 rows: the rows are independent streams, so the step runs as consecutive launches of the persistent
    // kernel over groups of 8 rows (each group streams the weights once; the per-op GEMMs would pad 16-32 rows to a
    // 128-token tile).  The scratch activations are reused by the
    // groups; the per-row state (token, positions, page table, audio row, output row, logits) is addressed from the
    // group's first row.
    const int rows_per_launch = B > 8 ? 8 : B;
    if (mega_prepare(rows_per_launch)) {
        for (int b0 = 0; b0 < B; b0 += 8) decode_step_mega(b0, std::min(8, B - b0), add_audio);
        return;
    }
    launch_embed(m->tok_emb, d_tok, add_audio ? audio : nullptr, cur_S4, B, 1, d_pos, x_dec, fused_decode(B) ? ssq_x : nullptr, st,
                 add_audio ? audio_rows_dev : nullptr);
    const bool pending = decoder_forward(B, 1);
    lm_head_rows(B, pending, logits);
    launch_argmax_multi(logits, B, c.vocab, d_tok, stream_mode ? nullptr : d_out, out_ld, d_outpos, am_vals, am_idx, am_cnt, st);
    launch_advance(d_pos, 1, d_outpos, 1, B, st);
}

// One launch of the persistent kernel for rows [b0, b0 + B) (B <= 8) of the session; mega_prepare() has built the op table.
void Session::decode_step_mega(int b0, int B, bool add_audio) {
    const vox_model_info &c = m->info;
    {
        if (B < mega_B) {
            // a ragged last group on the 8-token instantiation: its padding tokens must read as zero fragments, not as
            // the previous group's rows
            CUDA_OK(cudaMemsetAsync(mega_xf_bf, 0, sizeof(uint2) * mega_xf_blocks * 16 * 8, st));
            CUDA_OK(cudaMemsetAsync(mega_af_bf, 0, sizeof(uint2) * mega_af_blocks * 16 * 8, st));
            CUDA_OK(cudaMemsetAsync(mega_cf_bf, 0, sizeof(uint2) * mega_cf_blocks * 16 * 8, st));
            CUDA_OK(cudaMemsetAsync(mega_xf_off, 0, sizeof(float2) * mega_xf_blocks * 8, st));
            CUDA_OK(cudaMemsetAsync(mega_af_off, 0, sizeof(float2) * mega_af_blocks * 8, st));
            CUDA_OK(cudaMemsetAsync(mega_cf_off, 0, sizeof(float2) * mega_cf_blocks * 8, st));
        }
        MegaParams p;
        p.ops = mega_ops;
        p.n_ops = mega_n_ops;
        p.B = B;
        p.eps = m->norm_eps;
        p.qkv = qkv_dec;
        p.ld_qkv = (c.dec_heads + 2 * c.dec_kv_heads) * c.dec_head_dim;
        p.H = c.dec_heads;
        p.Hkv = c.dec_kv_heads;
        p.hd = c.dec_head_dim;
        p.max_seq = out_ld;
        p.page_table = d_page_table + (size_t)b0 * kv_max_pages;
        p.max_pages = kv_max_pages;
        p.window = c.dec_window;
        p.scale = powf((float)c.dec_head_dim, -0.5f);
        p.cos_t = m->dec_cos;
        p.sin_t = m->dec_sin;
        p.attn_out = attn_dec;
        // key chunks per (stream, kv head): spread the KV walk over idle SMs, but no more than 4 -- the merging CTA waits
        // for the other chunks' states one after the other (an L2 round trip each), and a CTA walks 64 keys per round
        // trip anyway, so more chunks add merge latency without shortening the walk
        p.attn_chunks = std::max(1, std::min(4, std::min(mega_grid, mega_att_units - 8 * c.dec_kv_heads) / (B * c.dec_kv_heads)));
        {
            static const int env_nc = getenv("VOX_MEGA_NC") ? atoi(getenv("VOX_MEGA_NC")) : 0;
            if (env_nc > 0 && env_nc <= p.attn_chunks) p.attn_chunks = env_nc;
        }
        p.att_acc = mega_att_acc;
        p.att_ml = mega_att_ml;
        p.att_flags = mega_att_flags;
        p.d_epoch = mega_epoch;
        p.emb_qs = m->tok_emb.qs;
        p.emb_d = m->tok_emb.d;
        p.D = c.dec_dim;
        p.audio = add_audio && audio ? audio + (size_t)b0 * cur_S4 * c.dec_dim : nullptr;
        p.audio_rows = add_audio && audio_rows_dev ? audio_rows_dev + b0 : nullptr;
        p.audio_seq = cur_S4;
        p.x_dec = x_dec;
        p.ssq_x = ssq_x;
        p.emb_fbf = mega_xf_bf;
        p.emb_foff = mega_xf_off;
        p.emb_gamma = m->dec[0].attn_norm;
        p.att_fbf = mega_af_bf;
        p.att_foff = mega_af_off;
        p.d_pos = d_pos + b0;
        p.d_outpos = d_outpos + b0;
        p.d_tok = d_tok + b0;
        p.d_out = stream_mode ? nullptr : d_out + (size_t)b0 * out_ld;
        p.out_ld = out_ld;
        p.logits_out = logits + (size_t)b0 * c.vocab;
        p.am_vals = mega_am_vals;
        p.am_idx = mega_am_idx;
        p.bar = mega_bar;
        p.nstage = mega_plan.nstage;
        p.scratch_bytes = mega_plan.scratch_bytes;
        p.trace = mega_trace;
        p.trace_all = mega_trace_all;
        p.trace_w = mega_trace_w;
        {
            static const int env_two = getenv("VOX_MEGA_TRACE_W_OP") ? atoi(getenv("VOX_MEGA_TRACE_W_OP")) : -1;
            p.trace_w_op = env_two;
        }
        {
            static const int env_flags = getenv("VOX_MEGA_FLAGS") ? atoi(getenv("VOX_MEGA_FLAGS")) : 0;
            p.flags = env_flags;
        }
        launch_decode_mega(p, mega_plan, mega_grid, st);
    }
}

// Prefill of M positions for B streams (model.rs:894-923 with M = 38; also the incremental vox_prefill).
void Session::prefill(int B, int M, const int *ids_host, bool add_audio) {
    const vox_model_info &c = m->info;
    CUDA_OK(cudaMemcpyAsync(d_ids, ids_host, sizeof(int) * (size_t)B * M, cudaMemcpyHostToDevice, st));
    launch_embed(m->tok_emb, d_ids, add_audio ? (audio_base ? audio_base : audio) : nullptr, audio_base ? S4_max : cur_S4, B, M, d_pos, x_dec,
                 fused_decode(B * M) ? ssq_x : nullptr, st);
    const bool pending = decoder_forward(B, M);
    if (pending) {   // decode-sized prefill (B*M <= 8): final norm still pending in x_dec
        launch_rmsnorm(x_dec, m->dec_norm, nullptr, h_dec, B * M, c.dec_dim, m->norm_eps, st);
    }
    // lm_head on the last row only (the reference computes all M rows and keeps one)
    launch_gather_last(h_dec, last_h, B, M, c.dec_dim, st);
    linear(m->tok_emb, last_h, B, logits, c.vocab, nullptr, nullptr, EPI_NONE);
    launch_argmax(logits, B, c.vocab, d_tok, stream_mode ? nullptr : d_out, out_ld, d_outpos, st);
    launch_advance(d_pos, M, d_outpos, 1, B, st);
}

void Session::reset() {
    CUDA_OK(cudaMemsetAsync(d_pos, 0, sizeof(int) * max_batch, st));
    CUDA_OK(cudaMemsetAsync(d_outpos, 0, sizeof(int) * max_batch, st));
    cache_len = 0;
    // the persistent kernel's attention-chunk states carry the tag epoch * 64 + layer + 1 (int): re-base the device
    // epoch long before that can overflow (2^24 steps ~ 10 hours of continuous decoding) -- and wipe the tagged words, so
    // that no stale state can match a tag of the new numbering
    if (mega_steps_host > (1u << 24)) {
        const vox_model_info &ci = m->info;
        const size_t gq = (size_t)(ci.dec_heads / ci.dec_kv_heads);
        CUDA_OK(cudaMemsetAsync(mega_att_flags, 0, sizeof(int) * mega_att_units, st));
        CUDA_OK(cudaMemsetAsync(mega_att_acc, 0, sizeof(float) * 2 * mega_att_units * gq * ci.dec_head_dim, st));
        CUDA_OK(cudaMemsetAsync(mega_att_ml, 0, sizeof(float) * 2 * mega_att_units * gq * 2, st));
        CUDA_OK(cudaMemsetAsync(mega_epoch, 0, sizeof(int), st));
        mega_steps_host = 0;
    }
}

// Q4VoxtralModel::transcribe_streaming (model.rs:873-963).  Expects the mel in s->mel; records
// ev[1] (after encode) and ev[2] (after decode) on the stream.  Returns tokens per stream.
int Session::transcribe_from_mel(int B, int T, int32_t *out_ids, size_t cap_ids, vox_timings *tm, bool timed_pre) {
    const vox_model_info &c = m->info;
    (void)timed_pre;
    encode(B, T);
    CUDA_OK(cudaEventRecord(ev[2], st));
    const int S4 = cur_S4, P = c.prefix_len;
    int n_out = 0;
    if (S4 >= P) {
        n_out = S4 - P;
        VOX_CHECK(cap_ids >= (size_t)B * n_out, VOX_ECAPACITY, "out_ids capacity %zu < %d x %d", cap_ids, B, n_out);
        reset();
        // prefix = [BOS] + [STREAMING_PAD]*37 (model.rs:883-892)
        std::vector<int> prefix((size_t)B * P, 32);
        for (int b = 0; b < B; ++b) prefix[(size_t)b * P] = 1;
        prefill(B, P, prefix.data(), true);
        CUDA_OK(cudaEventRecord(ev[4], st));
        const int steps = S4 - P - 1;
        if (steps > 0) mega_steps_host += (unsigned)steps;  // upper bound of the device epoch's advance
        if (steps > 0) {
            int done = 0;
            if (use_graph) {
                if (!step_graph || step_graph_B != B || step_graph_S4 != S4) {
                    // first step eagerly (also performs any one-time kernel attribute setup),
                    // then capture one step and replay it
                    decode_step(B);
                    done = 1;
                    if (step_graph) { cudaGraphExecDestroy(step_graph); step_graph = nullptr; }
                    if (steps > 1) {
                        cudaGraph_t graph = nullptr;
                        const uint64_t before = kernel_launch_count();
                        CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
                        try {
                            decode_step(B);
                        } catch (...) {
                            cudaStreamEndCapture(st, &graph);
                            if (graph) cudaGraphDestroy(graph);
                            throw;
                        }
                        CUDA_OK(cudaStreamEndCapture(st, &graph));
                        step_graph_nodes = kernel_launch_count() - before;
                        add_graph_launches(-(int64_t)step_graph_nodes);  // captured, not executed
                        cudaError_t e = cudaGraphInstantiate(&step_graph, graph, 0);
                        cudaGraphDestroy(graph);
                        cuda_check(e, "cudaGraphInstantiate");
                        step_graph_B = B;
                        step_graph_S4 = S4;
                    }
                }
                for (; done < steps; ++done) {
                    CUDA_OK(cudaGraphLaunch(step_graph, st));
                    add_graph_launches((int64_t)step_graph_nodes);
                }
            } else {
                for (; done < steps; ++done) decode_step(B);
            }
        }
    }
    if (S4 < P) CUDA_OK(cudaEventRecord(ev[4], st));
    CUDA_OK(cudaEventRecord(ev[3], st));
    std::vector<int> host((size_t)B * out_ld);
    if (n_out > 0) CUDA_OK(cudaMemcpyAsync(host.data(), d_out, sizeof(int) * host.size(), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b)
        for (int i = 0; i < n_out; ++i) out_ids[(size_t)b * n_out + i] = host[(size_t)b * out_ld + i];
    cache_len = n_out > 0 ? S4 - 1 : 0;
    if (tm) {
        tm->seq_len = S4;
        tm->decode_tokens = n_out;
    }
    return n_out;
}

}  // namespace vox
