// capi.cu -- the extern "C" boundary declared in include/voxtral.h.  Every entry point converts
// exceptions into a status code + thread-local message; nothing here computes on the CPU on
// behalf of the GPU path (no fallback): without a CUDA device the compute calls return VOX_ECUDA.
#include <cuda_profiler_api.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "audio_host.h"
#include "common.h"
#include "gguf.h"
#include "kernels.h"
#include "model.h"
#include "stream.h"
#include "tokenizer.h"

namespace vox {
static thread_local std::string g_last_error;
void set_last_error(const std::string &m) { g_last_error = m; }
}  // namespace vox

using namespace vox;

#define VOX_API_BEGIN try {
#define VOX_API_END                                \
    }                                              \
    catch (const vox::Error &e) {                  \
        vox::set_last_error(e.what());             \
        return e.code;                             \
    }                                              \
    catch (const std::bad_alloc &) {               \
        vox::set_last_error("out of host memory"); \
        return VOX_ENOMEM;                         \
    }                                              \
    catch (const std::exception &e) {              \
        vox::set_last_error(e.what());             \
        return VOX_EINVAL;                         \
    }                                              \
    return VOX_OK;

#define REQUIRE(p) VOX_CHECK((p) != nullptr, VOX_EINVAL, "null argument: " #p)

struct vox_gguf { Gguf *g; };
struct vox_mel {
    int device;
    DeviceArena arena;
    MelTables tables;
    cudaStream_t st = nullptr;
    float *in = nullptr, *out = nullptr;
    size_t in_cap = 0, out_cap = 0;
};
struct vox_q4 {
    int device;
    DeviceArena arena;
    Q4Weight w;
    float *x = nullptr, *y = nullptr, *bias = nullptr;  // scratch for the host-buffer call
    size_t x_cap = 0, y_cap = 0;
    float *norm = nullptr;  // [rows][K] output of the unfused RMSNorm (vox_q4_linear)
    size_t norm_cap = 0;
    TcWork wk;  // split-K scratch of the tensor-core matvec (allocated with the tensor)
    void *xt = nullptr;  // split tiles for the wgmma GEMM (M > 8)
    size_t xt_elems = 0;
    GemmWork gw;  // split-K scratch of the wgmma GEMM (allocated on first use)
};
struct vox_model { Model *m; };
struct vox_session { Session *s; };
struct vox_tokenizer { Tokenizer *t; };
struct vox_stream_pool { StreamPool *p; };

static void require_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    VOX_CHECK(e == cudaSuccess && n > 0, VOX_ECUDA, "no CUDA device available (%s); this library has no CPU fallback",
              cudaGetErrorString(e));
    VOX_CHECK(device >= 0 && device < n, VOX_EINVAL, "device %d out of range (have %d)", device, n);
    CUDA_OK(cudaSetDevice(device));
}

extern "C" {

const char *vox_last_error(void) { return g_last_error.c_str(); }
int32_t vox_version(void) { return 100; }
int32_t vox_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// ---------------------------------------------------------------- GGUF
int32_t vox_gguf_open(const char *path, vox_gguf **out) {
    VOX_API_BEGIN
    REQUIRE(path); REQUIRE(out);
    Gguf *g = Gguf::open_file(path);
    *out = new vox_gguf{g};
    VOX_API_END
}
int32_t vox_gguf_open_shards(const void *const *bufs, const size_t *lens, size_t n, vox_gguf **out) {
    VOX_API_BEGIN
    REQUIRE(bufs); REQUIRE(lens); REQUIRE(out);
    Gguf *g = Gguf::open_shards(bufs, lens, n);
    *out = new vox_gguf{g};
    VOX_API_END
}
int32_t vox_gguf_version(const vox_gguf *g, uint32_t *v) {
    VOX_API_BEGIN
    REQUIRE(g); REQUIRE(v);
    *v = g->g->version();
    VOX_API_END
}
int32_t vox_gguf_tensor_count(const vox_gguf *g, uint64_t *c) {
    VOX_API_BEGIN
    REQUIRE(g); REQUIRE(c);
    *c = g->g->tensor_count();
    VOX_API_END
}
int32_t vox_gguf_tensor_name(const vox_gguf *g, uint64_t i, const char **name) {
    VOX_API_BEGIN
    REQUIRE(g); REQUIRE(name);
    VOX_CHECK(i < g->g->names().size(), VOX_EINVAL, "tensor index %llu out of range", (unsigned long long)i);
    *name = g->g->names()[(size_t)i].c_str();
    VOX_API_END
}
int32_t vox_gguf_tensor_info(const vox_gguf *g, const char *name, uint32_t *dtype, uint32_t *ndim, uint64_t dims[4],
                             uint64_t *nbytes) {
    VOX_API_BEGIN
    REQUIRE(g); REQUIRE(name);
    const GgufTensorInfo *t = g->g->find(name);
    VOX_CHECK(t != nullptr, VOX_ENOTFOUND, "Tensor '%s' not found in GGUF", name);
    if (dtype) *dtype = t->dtype;
    if (ndim) *ndim = (uint32_t)t->dims.size();
    if (dims)
        for (size_t i = 0; i < 4; ++i) dims[i] = i < t->dims.size() ? t->dims[i] : 1;
    if (nbytes) *nbytes = t->byte_size();
    VOX_API_END
}
int32_t vox_gguf_tensor_data(vox_gguf *g, const char *name, void *dst, size_t cap) {
    VOX_API_BEGIN
    REQUIRE(g); REQUIRE(name); REQUIRE(dst);
    const GgufTensorInfo *t = g->g->find(name);
    VOX_CHECK(t != nullptr, VOX_ENOTFOUND, "Tensor '%s' not found in GGUF", name);
    VOX_CHECK(cap >= t->byte_size(), VOX_ECAPACITY, "buffer too small for '%s' (%zu < %llu)", name, cap,
              (unsigned long long)t->byte_size());
    g->g->read_tensor(*t, dst);
    VOX_API_END
}
void vox_gguf_close(vox_gguf *g) {
    if (!g) return;
    delete g->g;
    delete g;
}

// ---------------------------------------------------------------- audio plumbing
int32_t vox_peak_normalize(float *s, size_t n, float target) {
    VOX_API_BEGIN
    if (n) REQUIRE(s);
    peak_normalize(s, n, target);
    VOX_API_END
}
void vox_pad_config_default(vox_pad_config *c) { if (c) pad_config_default(c); }
size_t vox_pad_audio_len(size_t n, const vox_pad_config *cfg) {
    vox_pad_config c;
    if (cfg) c = *cfg; else pad_config_default(&c);
    return pad_audio_len(n, c);
}
int32_t vox_pad_audio(const float *in, size_t n, const vox_pad_config *cfg, float *out, size_t cap, size_t *out_len) {
    VOX_API_BEGIN
    REQUIRE(out);
    if (n) REQUIRE(in);
    vox_pad_config c;
    if (cfg) c = *cfg; else pad_config_default(&c);
    VOX_CHECK(c.frame_rate > 0 && c.sample_rate > 0, VOX_EINVAL, "bad pad config");
    const size_t total = pad_audio_len(n, c);
    VOX_CHECK(cap >= total, VOX_ECAPACITY, "pad_audio: capacity %zu < %zu", cap, total);
    memset(out, 0, sizeof(float) * total);
    if (n) memcpy(out + pad_left(c), in, sizeof(float) * n);
    if (out_len) *out_len = total;
    VOX_API_END
}
int32_t vox_chunk_plan(size_t n, size_t max_mel_frames, size_t overlap, vox_chunk *out, size_t cap, size_t *n_chunks) {
    VOX_API_BEGIN
    REQUIRE(n_chunks);
    std::vector<vox_chunk> v = chunk_plan(n, max_mel_frames, overlap);
    *n_chunks = v.size();
    if (out) {
        VOX_CHECK(cap >= v.size(), VOX_ECAPACITY, "chunk_plan: capacity %zu < %zu", cap, v.size());
        for (size_t i = 0; i < v.size(); ++i) out[i] = v[i];
    }
    VOX_API_END
}
int32_t vox_stream_progress(size_t n_samples, int32_t ended, int32_t reshape_factor, int32_t prefix_len, int64_t out[5]) {
    VOX_API_BEGIN
    REQUIRE(out);
    VOX_CHECK(reshape_factor > 0 && prefix_len > 0, VOX_EINVAL, "stream_progress: reshape_factor %d / prefix_len %d must be positive",
              reshape_factor, prefix_len);
    stream_progress(n_samples, ended != 0, reshape_factor, prefix_len, out);
    VOX_API_END
}
int32_t vox_time_embedding(float t, int32_t dim, float *out) {
    VOX_API_BEGIN
    REQUIRE(out);
    VOX_CHECK(dim > 0 && dim % 2 == 0, VOX_EINVAL, "time_embedding: dim %d must be even", dim);
    time_embedding(t, dim, out);
    VOX_API_END
}

// ---------------------------------------------------------------- mel
int32_t vox_mel_create(int32_t device, vox_mel **out) {
    VOX_API_BEGIN
    REQUIRE(out);
    require_device(device);
    std::unique_ptr<vox_mel> m(new vox_mel());
    m->device = device;
    m->arena.device = device;
    m->tables.build(m->arena);
    CUDA_OK(cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking));
    *out = m.release();
    VOX_API_END
}
size_t vox_mel_num_frames(size_t n) { return mel_num_frames(n); }
int32_t vox_mel_compute_log(vox_mel *mel, const float *samples, size_t n, float *out, size_t cap) {
    VOX_API_BEGIN
    REQUIRE(mel); REQUIRE(out);
    if (n) REQUIRE(samples);
    const size_t frames = mel_num_frames(n);
    VOX_CHECK(cap >= frames * kMelBins, VOX_ECAPACITY, "mel: capacity %zu < %zu", cap, frames * kMelBins);
    if (frames == 0) return VOX_OK;
    CUDA_OK(cudaSetDevice(mel->device));
    if (n > mel->in_cap) {
        mel->in = mel->arena.alloc_n<float>(n);
        mel->in_cap = n;
    }
    if (frames * kMelBins > mel->out_cap) {
        mel->out = mel->arena.alloc_n<float>(frames * kMelBins);
        mel->out_cap = frames * kMelBins;
    }
    CUDA_OK(cudaMemcpyAsync(mel->in, samples, sizeof(float) * n, cudaMemcpyHostToDevice, mel->st));
    launch_mel(mel->in, 1, n, n, mel->tables.window, mel->tables.fb_vals, mel->tables.fb_start, mel->tables.fb_len,
               mel->tables.fb_stride, mel->out, (int)frames, 0, mel->st);
    CUDA_OK(cudaMemcpyAsync(out, mel->out, sizeof(float) * frames * kMelBins, cudaMemcpyDeviceToHost, mel->st));
    CUDA_OK(cudaStreamSynchronize(mel->st));
    VOX_API_END
}
int32_t vox_mel_compute_log_dev(vox_mel *mel, const float *samples_dev, size_t n, float *out_dev, int32_t layout,
                                void *stream) {
    VOX_API_BEGIN
    REQUIRE(mel); REQUIRE(samples_dev); REQUIRE(out_dev);
    VOX_CHECK(layout == 0 || layout == 1, VOX_EINVAL, "mel layout must be 0 or 1");
    CUDA_OK(cudaSetDevice(mel->device));
    const size_t frames = mel_num_frames(n);
    launch_mel(samples_dev, 1, n, n, mel->tables.window, mel->tables.fb_vals, mel->tables.fb_start, mel->tables.fb_len,
               mel->tables.fb_stride, out_dev, (int)frames, layout, stream ? (cudaStream_t)stream : mel->st);
    VOX_API_END
}
int32_t vox_mel_filterbank(const vox_mel *mel, float *out) {
    VOX_API_BEGIN
    REQUIRE(mel); REQUIRE(out);
    memcpy(out, mel->tables.fb_dense.data(), sizeof(float) * kMelBins * kMelFreqs);
    VOX_API_END
}
int32_t vox_mel_window(const vox_mel *mel, float *out) {
    VOX_API_BEGIN
    REQUIRE(mel); REQUIRE(out);
    memcpy(out, mel->tables.window_host.data(), sizeof(float) * kMelNfft);
    VOX_API_END
}
void vox_mel_free(vox_mel *mel) {
    if (!mel) return;
    cudaSetDevice(mel->device);
    if (mel->st) cudaStreamDestroy(mel->st);
    delete mel;
}

// ---------------------------------------------------------------- Q4 operator
int32_t vox_q4_tensor_create(const uint8_t *bytes, size_t nbytes, int64_t n, int64_t k, int32_t device, vox_q4 **out) {
    VOX_API_BEGIN
    REQUIRE(bytes); REQUIRE(out);
    VOX_CHECK(n > 0 && k > 0, VOX_EINVAL, "Q4 tensor shape must be positive");
    VOX_CHECK((n * k) % 32 == 0, VOX_EINVAL, "Q4_0 requires element count divisible by 32, got %lld", (long long)(n * k));
    VOX_CHECK(k % 32 == 0, VOX_EINVAL, "Q4_0 rows must be block aligned: K=%lld is not a multiple of 32", (long long)k);
    const size_t expect = (size_t)(n * k / 32) * 18;
    VOX_CHECK(nbytes == expect, VOX_EINVAL, "Q4_0 byte count mismatch: expected %zu for %lld blocks, got %zu", expect,
              (long long)(n * k / 32), nbytes);
    require_device(device);
    std::unique_ptr<vox_q4> q(new vox_q4());
    q->device = device;
    q->arena.device = device;
    q->w = upload_q4(q->arena, {bytes}, {(int)n}, (int)k, false, true);
    q->wk = q4_matvec_tc_work_size(q->w.N, q->w.K);
    alloc_split_k(q->arena, q->wk);
    *out = q.release();
    VOX_API_END
}
int32_t vox_q4_tensor_shape(const vox_q4 *w, int64_t *n, int64_t *k) {
    VOX_API_BEGIN
    REQUIRE(w);
    if (n) *n = w->w.N;
    if (k) *k = w->w.K;
    VOX_API_END
}
int32_t vox_q4_tensor_dequantize(const vox_q4 *w, float *out) {
    VOX_API_BEGIN
    REQUIRE(w); REQUIRE(out);
    // reads the planes back from HBM (like Q4Tensor::dequantize reads the GPU buffer back) and
    // applies the dequant rule on the host -- diagnostics only
    CUDA_OK(cudaSetDevice(w->device));
    const size_t nb = (size_t)w->w.N * (w->w.K / 32);
    std::vector<uint8_t> qs(nb * 16);
    std::vector<__half> ds(nb);
    CUDA_OK(cudaMemcpy(qs.data(), w->w.qs, qs.size(), cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(ds.data(), w->w.d, ds.size() * sizeof(__half), cudaMemcpyDeviceToHost));
    for (size_t b = 0; b < nb; ++b) {
        const float d = __half2float(ds[b]);
        for (int i = 0; i < 16; ++i) {
            const uint8_t byte = qs[b * 16 + i];
            out[b * 32 + i] = ((float)(byte & 0xF) - 8.0f) * d;
            out[b * 32 + i + 16] = ((float)(byte >> 4) - 8.0f) * d;
        }
    }
    VOX_API_END
}
// kernel choice of the Q4 operator, process-wide and separate from the sessions' (vox_q4_set_matvec_mode)
static Q4Path g_q4_path = {!(getenv("VOX_MATVEC") && std::string(getenv("VOX_MATVEC")) == "simt"), true};
// the handle's scratch for a call over `rows` rows, the wgmma split buffer grown first to what they need
static Q4Scratch q4_scratch(vox_q4 *h, int rows) {
    if (rows > 8) {  // only M > 8 can take the wgmma GEMM
        const size_t need = gemm_tc5_split_elems(rows, h->w.K);
        if (need > h->xt_elems) {
            h->xt = h->arena.alloc(need * 2);
            h->xt_elems = need;
        }
        if (!h->gw.partial) {
            h->gw = gemm_tc5_work_size();
            alloc_split_k(h->arena, h->gw);
        }
    }
    return Q4Scratch{h->xt, h->xt_elems, &h->gw, &h->wk};
}
int32_t vox_q4_set_matvec_mode(int32_t mode) {
    VOX_API_BEGIN
    VOX_CHECK(mode >= 0 && mode <= 3, VOX_EINVAL, "mode bits: 1 = SIMT matvec (M<=8), 2 = SIMT GEMM (M>8)");
    g_q4_path.matvec_tc = (mode & 1) == 0;
    g_q4_path.gemm_tc = (mode & 2) == 0;
    VOX_API_END
}
int32_t vox_q4_matmul(const vox_q4 *w, const float *x_dev, float *y_dev, int32_t b, int32_t m, const float *bias_dev,
                      void *stream) {
    VOX_API_BEGIN
    REQUIRE(w); REQUIRE(x_dev); REQUIRE(y_dev);
    VOX_CHECK(b > 0 && m > 0, VOX_EINVAL, "q4_matmul: B and M must be positive");
    CUDA_OK(cudaSetDevice(w->device));
    launch_q4_linear(w->w, x_dev, b * m, y_dev, w->w.N, bias_dev, nullptr, EPI_NONE, nullptr, 0.0f, nullptr,
                     q4_scratch(const_cast<vox_q4 *>(w), b * m), g_q4_path, (cudaStream_t)stream);
    VOX_API_END
}
int32_t vox_q4_matmul_host(const vox_q4 *wc, const float *x, float *y, int32_t b, int32_t m, const float *bias) {
    VOX_API_BEGIN
    vox_q4 *w = const_cast<vox_q4 *>(wc);
    REQUIRE(w); REQUIRE(x); REQUIRE(y);
    VOX_CHECK(b > 0 && m > 0, VOX_EINVAL, "q4_matmul: B and M must be positive");
    CUDA_OK(cudaSetDevice(w->device));
    const size_t rows = (size_t)b * m, xn = rows * w->w.K, yn = rows * w->w.N;
    if (xn > w->x_cap) { w->x = w->arena.alloc_n<float>(xn); w->x_cap = xn; }
    if (yn > w->y_cap) { w->y = w->arena.alloc_n<float>(yn); w->y_cap = yn; }
    if (bias && !w->bias) w->bias = w->arena.alloc_n<float>(w->w.N);
    CUDA_OK(cudaMemcpyAsync(w->x, x, sizeof(float) * xn, cudaMemcpyHostToDevice, 0));
    if (bias) CUDA_OK(cudaMemcpyAsync(w->bias, bias, sizeof(float) * w->w.N, cudaMemcpyHostToDevice, 0));
    launch_q4_linear(w->w, w->x, (int)rows, w->y, w->w.N, bias ? w->bias : nullptr, nullptr, EPI_NONE, nullptr,
                     0.0f, nullptr, q4_scratch(w, (int)rows), g_q4_path, 0);
    CUDA_OK(cudaMemcpyAsync(y, w->y, sizeof(float) * yn, cudaMemcpyDeviceToHost, 0));
    CUDA_OK(cudaStreamSynchronize(0));
    VOX_API_END
}
static_assert(VOX_EPI_NONE == EPI_NONE && VOX_EPI_RESIDUAL == EPI_RESIDUAL && VOX_EPI_SILU_MUL == EPI_SILU_MUL &&
                  VOX_EPI_GELU == EPI_GELU,
              "the header's epilogue codes are kernels.h Epi");
int32_t vox_q4_linear(const vox_q4 *wc, const float *x_dev, float *y_dev, int32_t rows, int32_t ldy,
                      const float *bias_dev, const float *res_dev, int32_t epi, const float *gamma_dev, float eps,
                      const float *const *ada_dev, int32_t ada_m, const float *ssq_in_dev, float *ssq_out_dev,
                      void *stream) {
    VOX_API_BEGIN
    vox_q4 *w = const_cast<vox_q4 *>(wc);
    REQUIRE(w); REQUIRE(x_dev); REQUIRE(y_dev);
    const int N = w->w.N, K = w->w.K;
    VOX_CHECK(rows >= 1, VOX_EINVAL, "q4_linear: rows=%d must be positive", rows);
    VOX_CHECK(epi >= VOX_EPI_NONE && epi <= VOX_EPI_GELU, VOX_EINVAL, "q4_linear: epilogue %d is not one of 0..3", epi);
    VOX_CHECK((epi == VOX_EPI_RESIDUAL) == (res_dev != nullptr), VOX_EINVAL,
              "q4_linear: a residual epilogue needs res, and res needs the residual epilogue (epi=%d)", epi);
    if (epi == VOX_EPI_SILU_MUL) {
        VOX_CHECK(N % 2 == 0, VOX_EINVAL, "q4_linear: SiLU*up needs (gate, up) row pairs, N=%d is odd", N);
        VOX_CHECK(ldy >= N / 2, VOX_EINVAL, "q4_linear: ldy=%d < N/2=%d", ldy, N / 2);
        VOX_CHECK(!bias_dev, VOX_EINVAL, "q4_linear: SiLU*up takes no bias (no kernel adds one there)");
    } else {
        VOX_CHECK(ldy >= N, VOX_EINVAL, "q4_linear: ldy=%d < N=%d", ldy, N);
    }
    VOX_CHECK(!ada_dev || gamma_dev, VOX_EINVAL, "q4_linear: per-row ADA vectors need a norm (gamma)");
    VOX_CHECK(!ada_dev || ada_m >= 1, VOX_EINVAL, "q4_linear: ada_m=%d must be positive", ada_m);
    VOX_CHECK(!ssq_in_dev || gamma_dev, VOX_EINVAL, "q4_linear: ssq_in feeds the norm and needs gamma");
    VOX_CHECK(!ssq_out_dev || epi == VOX_EPI_RESIDUAL, VOX_EINVAL, "q4_linear: ssq_out is written by a residual epilogue only");
    const bool tc = rows <= 8 && g_q4_path.matvec_tc && w->w.qs_tc;
    VOX_CHECK(!(ssq_in_dev || ssq_out_dev) || tc, VOX_EINVAL,
              "q4_linear: ssq_in / ssq_out need the tensor-core matvec (rows <= 8, matvec mode bit 0 clear), rows=%d",
              rows);
    CUDA_OK(cudaSetDevice(w->device));
    const size_t xn = (size_t)rows * K;
    if (gamma_dev && xn > w->norm_cap) {
        w->norm = w->arena.alloc_n<float>(xn);
        w->norm_cap = xn;
    }
    Q4Scratch sc = q4_scratch(w, rows);
    TcWork wk = w->wk;
    wk.ssq_in = ssq_in_dev;
    wk.ssq_in_parts = ssq_in_dev ? (K + 15) / 16 : 0;
    wk.ssq_out = ssq_out_dev;
    sc.tc = &wk;
    launch_q4_linear(w->w, x_dev, rows, y_dev, ldy, bias_dev, res_dev, epi, gamma_dev, eps, w->norm, sc, g_q4_path,
                     (cudaStream_t)stream, AdaRows{ada_dev, ada_dev ? ada_m : 1, 0});
    VOX_API_END
}
void vox_q4_tensor_free(vox_q4 *w) {
    if (!w) return;
    cudaSetDevice(w->device);
    delete w;
}

int32_t vox_attention(int32_t device, int32_t kernel, const vox_attn_args *a, void *stream) {
    VOX_API_BEGIN
    REQUIRE(a);
    VOX_CHECK(kernel >= VOX_ATTN_ENC_TC && kernel <= VOX_ATTN_STREAM, VOX_EINVAL, "attention: kernel %d is not one of 0..2",
              kernel);
    VOX_CHECK(a->qkv && a->out, VOX_EINVAL, "attention: qkv and out are required");
    VOX_CHECK(a->h >= 1, VOX_EINVAL, "attention: h=%d must be positive", a->h);
    VOX_CHECK(a->window >= 0, VOX_EINVAL, "attention: window=%d is negative", a->window);
    const int hd = a->hd, hq = a->h * a->hd;
    if (kernel == VOX_ATTN_STREAM) {
        VOX_CHECK(hd == 32 || hd == 64 || hd == 128, VOX_EINVAL, "attention: the ring kernel takes hd 32, 64 or 128, not %d", hd);
        VOX_CHECK(a->rows >= 1, VOX_EINVAL, "attention: rows=%d must be positive", a->rows);
        VOX_CHECK(a->row_slot && a->row_pos && a->k_ring && a->v_ring, VOX_EINVAL,
                  "attention: the ring kernel needs row_slot, row_pos, k_ring and v_ring");
        VOX_CHECK(a->ld >= hq, VOX_EINVAL, "attention: ld=%d < h*hd=%d", a->ld, hq);
        VOX_CHECK(a->ring >= 1 && a->window < a->ring, VOX_EINVAL,
                  "attention: window=%d must be below ring=%d (keys older than the ring are overwritten)", a->window, a->ring);
    } else {
        const bool tc = kernel == VOX_ATTN_ENC_TC;
        if (tc)
            VOX_CHECK(hd == 32 || hd == 64, VOX_EINVAL, "attention: K4-TC takes hd 32 or 64, not %d", hd);
        else
            VOX_CHECK(hd == 32 || hd == 64 || hd == 128, VOX_EINVAL, "attention: K4 takes hd 32, 64 or 128, not %d", hd);
        VOX_CHECK(a->b >= 1 && a->s >= 1, VOX_EINVAL, "attention: b=%d and s=%d must be positive", a->b, a->s);
        for (const int off : {a->q_off, a->k_off, a->v_off})
            VOX_CHECK(off >= 0 && off + hq <= a->ld, VOX_EINVAL, "attention: an operand at column %d of h*hd=%d does not fit in ld=%d",
                      off, hq, a->ld);
        VOX_CHECK(!tc || enc_attention_tc_supported(hd, a->ld, a->q_off, a->k_off, a->v_off), VOX_EINVAL,
                  "attention: K4-TC loads float4s: ld=%d and the offsets (%d, %d, %d) must be multiples of 4", a->ld,
                  a->q_off, a->k_off, a->v_off);
        VOX_CHECK(!tc || (reinterpret_cast<uintptr_t>(a->qkv) & 15) == 0, VOX_EINVAL,
                  "attention: K4-TC loads float4s: qkv must be 16-byte aligned");
    }
    require_device(device);
    const cudaStream_t st = (cudaStream_t)stream;
    if (kernel == VOX_ATTN_STREAM)
        launch_stream_attn(a->qkv, a->rows, a->ld, a->h, hd, a->row_slot, a->row_pos, a->k_ring, a->v_ring, a->ring,
                           a->window, a->scale, a->out, st);
    else
        (kernel == VOX_ATTN_ENC_TC ? launch_enc_attention_tc : launch_enc_attention)(
            a->qkv, a->out, a->b, a->s, a->h, hd, a->ld, a->q_off, a->k_off, a->v_off, a->window, a->scale, st, a->seg);
    VOX_API_END
}

int32_t vox_dec_attention(int32_t device, int32_t kernel, const vox_dec_attn_args *a, void *stream) {
    VOX_API_BEGIN
    REQUIRE(a);
    VOX_CHECK(kernel == VOX_DEC_ATTN_FUSED || kernel == VOX_DEC_ATTN_PREFILL, VOX_EINVAL,
              "dec_attention: kernel %d is not one of 0..1", kernel);
    VOX_CHECK(a->kv_dtype == VOX_DTYPE_F32 || a->kv_dtype == VOX_DTYPE_F16 || a->kv_dtype == VOX_DTYPE_KV_Q8, VOX_EINVAL,
              "dec_attention: kv_dtype %d is not f32, f16 or q8", a->kv_dtype);
    VOX_CHECK(a->qkv && a->k_pool && a->v_pool && a->page_table && a->pos && a->cos && a->sin && a->out, VOX_EINVAL,
              "dec_attention: qkv, k_pool, v_pool, page_table, pos, cos, sin and out are required");
    VOX_CHECK(a->b >= 1 && a->m >= 1 && a->h >= 1 && a->hkv >= 1 && a->hd >= 1 && a->max_pages >= 1 && a->rope_rows >= 1,
              VOX_EINVAL, "dec_attention: b=%d, m=%d, h=%d, hkv=%d, hd=%d, max_pages=%d and rope_rows=%d must be positive",
              a->b, a->m, a->h, a->hkv, a->hd, a->max_pages, a->rope_rows);
    VOX_CHECK(a->h % a->hkv == 0, VOX_EINVAL, "dec_attention: h=%d is not a multiple of hkv=%d", a->h, a->hkv);
    VOX_CHECK((int64_t)a->ld >= (int64_t)(a->h + 2 * a->hkv) * a->hd, VOX_EINVAL, "dec_attention: ld=%d < (h + 2 hkv) hd=%d",
              a->ld, (a->h + 2 * a->hkv) * a->hd);
    VOX_CHECK(a->window >= 0, VOX_EINVAL, "dec_attention: window=%d is negative", a->window);
    const bool fused = kernel == VOX_DEC_ATTN_FUSED;
    if (fused) {
        VOX_CHECK(a->m == 1, VOX_EINVAL, "dec_attention: the fused kernel takes m = 1, not %d", a->m);
        VOX_CHECK(dec_attn_fused_supported(a->h, a->hkv, a->hd), VOX_EINVAL,
                  "dec_attention: the fused kernel has no instantiation for h=%d, hkv=%d, hd=%d", a->h, a->hkv, a->hd);
    }
    KvView kv;
    const KvType type = a->kv_dtype == VOX_DTYPE_F16 ? KvType::F16 : (a->kv_dtype == VOX_DTYPE_KV_Q8 ? KvType::Q8 : KvType::F32);
    kv.k = kv_pool(a->k_pool, type);
    kv.v = kv_pool(a->v_pool, type);
    kv.page_table = a->page_table;
    kv.max_pages = a->max_pages;
    kv.ring = a->ring != 0;
    kv.type = type;
    kv.pos = a->pos;
    const RopeView rope{a->cos, a->sin, a->rope_rows};
    require_device(device);
    if (!kv.ring) {
        // the kernels skip a row past the capacity and leave its output as it was
        std::vector<int32_t> pos(a->b);
        CUDA_OK(cudaMemcpy(pos.data(), a->pos, sizeof(int32_t) * a->b, cudaMemcpyDeviceToHost));
        for (int bb = 0; bb < a->b; ++bb)
            VOX_CHECK(pos[bb] >= 0 && (int64_t)pos[bb] + a->m <= std::min(kv.max_seq(), a->rope_rows), VOX_EINVAL,
                      "dec_attention: row %d at pos %d + m=%d runs past the capacity %d or rope_rows %d", bb, pos[bb], a->m,
                      kv.max_seq(), a->rope_rows);
    }
    const cudaStream_t st = (cudaStream_t)stream;
    if (fused) {
        launch_dec_attn_fused(a->qkv, a->b, a->ld, a->h, a->hkv, a->hd, kv, a->window, a->scale, rope, a->out, st);
    } else {
        dec_attention_check(a->m, a->h, a->hkv, a->hd, kv, a->window);
        launch_dec_rope_append(a->qkv, a->b, a->m, a->ld, a->h, a->hkv, a->hd, kv, rope, st);
        launch_dec_attention(a->qkv, a->b, a->m, a->ld, a->h, a->hkv, a->hd, kv, a->window, a->scale, a->out, st);
    }
    VOX_API_END
}

int32_t vox_dev_malloc(int32_t device, size_t bytes, void **p) {
    VOX_API_BEGIN
    REQUIRE(p);
    require_device(device);
    cudaError_t e = cudaMalloc(p, bytes ? bytes : 16);
    VOX_CHECK(e == cudaSuccess, VOX_ENOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    VOX_API_END
}
int32_t vox_dev_free(int32_t device, void *p) {
    VOX_API_BEGIN
    require_device(device);
    CUDA_OK(cudaFree(p));
    VOX_API_END
}
int32_t vox_dev_upload(int32_t device, void *dst, const void *src, size_t bytes) {
    VOX_API_BEGIN
    require_device(device);
    CUDA_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
    VOX_API_END
}
int32_t vox_dev_download(int32_t device, void *dst, const void *src, size_t bytes) {
    VOX_API_BEGIN
    require_device(device);
    CUDA_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    VOX_API_END
}
int32_t vox_dev_sync(int32_t device) {
    VOX_API_BEGIN
    require_device(device);
    CUDA_OK(cudaDeviceSynchronize());
    VOX_API_END
}
int32_t vox_profiler_start(void) {
    VOX_API_BEGIN
    CUDA_OK(cudaProfilerStart());
    VOX_API_END
}
int32_t vox_profiler_stop(void) {
    VOX_API_BEGIN
    CUDA_OK(cudaProfilerStop());
    VOX_API_END
}
int32_t vox_host_alloc_pinned(size_t bytes, void **p) {
    VOX_API_BEGIN
    REQUIRE(p);
    cudaError_t e = cudaHostAlloc(p, bytes ? bytes : 16, cudaHostAllocDefault);
    VOX_CHECK(e == cudaSuccess, VOX_ECUDA, "cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    VOX_API_END
}
int32_t vox_host_free_pinned(void *p) {
    VOX_API_BEGIN
    CUDA_OK(cudaFreeHost(p));
    VOX_API_END
}
int32_t vox_q4_matmul_bench(const vox_q4 *const *ws, int32_t n_w, int32_t m, int32_t iters, int32_t warmup, float *avg_ms) {
    VOX_API_BEGIN
    REQUIRE(ws); REQUIRE(avg_ms);
    VOX_CHECK(n_w > 0 && m > 0 && iters > 0, VOX_EINVAL, "bad bench arguments");
    const vox_q4 *w0 = ws[0];
    CUDA_OK(cudaSetDevice(w0->device));
    DeviceArena arena;
    arena.device = w0->device;
    const int K = w0->w.K, N = w0->w.N;
    std::vector<float> hx((size_t)m * K);
    for (size_t i = 0; i < hx.size(); ++i) hx[i] = sinf((float)i * 0.001f) * 0.1f;  // benches/q4_ops.rs:71-73
    float *x = arena.upload(hx.data(), hx.size());
    float *y = arena.alloc_n<float>((size_t)m * N);
    cudaStream_t st;
    CUDA_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    cudaEvent_t e0, e1;
    CUDA_OK(cudaEventCreate(&e0));
    CUDA_OK(cudaEventCreate(&e1));
    // no scratch: no split-K, and M > 8 takes the SIMT GEMM
    auto run = [&](int i) {
        launch_q4_linear(ws[i % n_w]->w, x, m, y, ws[i % n_w]->w.N, nullptr, nullptr, EPI_NONE, nullptr, 0.0f, nullptr,
                         Q4Scratch{}, g_q4_path, st);
    };
    for (int i = 0; i < warmup; ++i) run(i);
    CUDA_OK(cudaStreamSynchronize(st));
    CUDA_OK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i) run(i);
    CUDA_OK(cudaEventRecord(e1, st));
    CUDA_OK(cudaStreamSynchronize(st));
    float ms = 0;
    CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    *avg_ms = ms / iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaStreamDestroy(st);
    VOX_API_END
}

// ---------------------------------------------------------------- model
int32_t vox_model_load_gguf_handle(vox_gguf *g, int32_t device, vox_model **out) {
    VOX_API_BEGIN
    REQUIRE(g); REQUIRE(out);
    Model *m = Model::load(*g->g, device);
    *out = new vox_model{m};
    VOX_API_END
}
int32_t vox_model_load_gguf(const char *path, int32_t device, vox_model **out) {
    VOX_API_BEGIN
    REQUIRE(path); REQUIRE(out);
    std::unique_ptr<Gguf> g(Gguf::open_file(path));
    Model *m = Model::load(*g, device);
    *out = new vox_model{m};
    VOX_API_END
}
int32_t vox_model_get_info(const vox_model *m, vox_model_info *info) {
    VOX_API_BEGIN
    REQUIRE(m); REQUIRE(info);
    *info = m->m->info;
    VOX_API_END
}
void vox_model_free(vox_model *m) {
    if (!m) return;
    cudaSetDevice(m->m->device);
    delete m->m;
    delete m;
}

// ---------------------------------------------------------------- session
// the element type vox_session_create_ex / vox_stream_pool_create_ex accept
static KvType kv_type_of(int32_t kv_dtype) {
    VOX_CHECK(kv_dtype == VOX_DTYPE_F32 || kv_dtype == VOX_DTYPE_F16 || kv_dtype == VOX_DTYPE_KV_Q8, VOX_EINVAL,
              "kv_dtype %d: VOX_DTYPE_F32, VOX_DTYPE_F16 or VOX_DTYPE_KV_Q8", (int)kv_dtype);
    return kv_dtype == VOX_DTYPE_F16 ? KvType::F16 : (kv_dtype == VOX_DTYPE_KV_Q8 ? KvType::Q8 : KvType::F32);
}
int32_t vox_session_create(vox_model *m, int32_t max_batch, int32_t max_mel_frames, vox_session **out) {
    return vox_session_create_ex(m, max_batch, max_mel_frames, VOX_DTYPE_F32, out);
}
int32_t vox_session_create_ex(vox_model *m, int32_t max_batch, int32_t max_mel_frames, int32_t kv_dtype, vox_session **out) {
    VOX_API_BEGIN
    REQUIRE(m); REQUIRE(out);
    Session *s = Session::create(m->m, max_batch, max_mel_frames, false, kv_type_of(kv_dtype));
    *out = new vox_session{s};
    VOX_API_END
}
int32_t vox_session_device_bytes(const vox_session *s, uint64_t *bytes) {
    VOX_API_BEGIN
    REQUIRE(s); REQUIRE(bytes);
    *bytes = s->s->arena.total;
    VOX_API_END
}
int32_t vox_session_set_delay(vox_session *s, float delay) {
    VOX_API_BEGIN
    REQUIRE(s);
    s->s->set_delay(delay);
    VOX_API_END
}
static void require_any_device();
int32_t vox_session_set_delays(vox_session *s, const float *delays, int32_t b) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(s); REQUIRE(delays);
    s->s->set_delays(delays, b);
    VOX_API_END
}

// the uniform encode of b streams of t frames already in enc.mel_tm (vox_encode_audio, vox_forward_streaming)
static void encode_uniform(Session *s, int b, int t) {
    const std::vector<int> frames(b, t);
    s->enc.encode(*s, b, frames.data());
    s->cur_B = b;
}

int32_t vox_encode_audio(vox_session *sh, const float *mel, int32_t b, int32_t t, float *audio_embeds, size_t cap,
                         int32_t *seq_len) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(mel);
    Session *s = sh->s;
    s->enc.upload_mel(*s, mel, b, t);
    encode_uniform(s, b, t);
    const size_t n = (size_t)b * s->enc.positions * s->m->info.dec_dim;
    if (audio_embeds) {
        VOX_CHECK(cap >= n, VOX_ECAPACITY, "audio_embeds capacity %zu < %zu", cap, n);
        if (n) CUDA_OK(cudaMemcpyAsync(audio_embeds, s->enc.audio, sizeof(float) * n, cudaMemcpyDeviceToHost, s->st));
    }
    CUDA_OK(cudaStreamSynchronize(s->st));
    if (seq_len) *seq_len = s->enc.positions;
    VOX_API_END
}

static void fill_timings(Session *s, vox_timings *tm) {
    if (!tm) return;
    float pre = 0, enc = 0, dec = 0, pf = 0;
    CUDA_OK(cudaEventElapsedTime(&pf, s->ev[2], s->ev[4]));
    tm->prefill_ms = pf;
    CUDA_OK(cudaEventElapsedTime(&pre, s->ev[0], s->ev[1]));
    CUDA_OK(cudaEventElapsedTime(&enc, s->ev[1], s->ev[2]));
    CUDA_OK(cudaEventElapsedTime(&dec, s->ev[2], s->ev[3]));
    tm->preprocess_ms = pre;
    tm->encode_ms = enc;
    tm->decode_ms = dec;
    tm->total_ms = pre + enc + dec;
}

int32_t vox_transcribe_streaming(vox_session *sh, const float *mel, int32_t b, int32_t t, int32_t *out_ids, size_t cap,
                                 int32_t *n_out, vox_timings *tm) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(mel); REQUIRE(out_ids); REQUIRE(n_out);
    Session *s = sh->s;
    s->sel.check_beam_bias();
    CUDA_OK(cudaSetDevice(s->m->device));
    CUDA_OK(cudaEventRecord(s->ev[0], s->st));
    s->enc.upload_mel(*s, mel, b, t);
    CUDA_OK(cudaEventRecord(s->ev[1], s->st));
    *n_out = s->transcribe_from_mel(b, t, out_ids, cap, tm);
    fill_timings(s, tm);
    VOX_API_END
}

// `total`: the getters report the counts over all streams (a ragged call)
static int32_t transcribe_pcm_impl(Session *s, const float *host, const float *dev, int b, size_t n, int normalize,
                                   int32_t *out_ids, size_t cap, int32_t *n_out, vox_timings *tm, bool total = false) {
    s->check_batch(b);
    s->sel.check_beam_bias();
    VOX_CHECK(n >= 1, VOX_EINVAL, "empty audio");
    CUDA_OK(cudaSetDevice(s->m->device));
    vox_pad_config pc;
    pad_config_default(&pc);
    const size_t frames = mel_num_frames(pad_audio_len(n, pc));
    VOX_CHECK(frames >= 1, VOX_EINVAL, "Audio too short to produce mel frames");
    VOX_CHECK(frames <= (size_t)s->enc.max_mel_frames, VOX_EINVAL,
              "audio needs %zu mel frames > session max_mel_frames %d (chunk it: vox_chunk_plan)", frames, s->enc.max_mel_frames);
    const std::vector<size_t> lens(b, n);
    s->enc.prepare_pcm(*s, lens.data(), b, host != nullptr);
    CUDA_OK(cudaEventRecord(s->ev[0], s->st));
    s->enc.pcm_to_mel(*s, host, dev, lens.data(), b, normalize);
    CUDA_OK(cudaEventRecord(s->ev[1], s->st));
    *n_out = s->transcribe_from_mel(b, (int)frames, out_ids, cap, tm, total);
    fill_timings(s, tm);
    return VOX_OK;
}

int32_t vox_transcribe_pcm(vox_session *sh, const float *samples, int32_t b, size_t n, int32_t normalize,
                           int32_t *out_ids, size_t cap, int32_t *n_out, vox_timings *tm) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(samples); REQUIRE(out_ids); REQUIRE(n_out);
    return transcribe_pcm_impl(sh->s, samples, nullptr, b, n, normalize, out_ids, cap, n_out, tm);
    VOX_API_END
}
int32_t vox_transcribe_pcm_ragged(vox_session *sh, const float *samples, const size_t *lens, int32_t b, int32_t normalize,
                                  int32_t *out_ids, size_t cap, int32_t *n_out, vox_timings *tm) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(samples); REQUIRE(lens); REQUIRE(out_ids); REQUIRE(n_out);
    Session *s = sh->s;
    const vox_model_info &c = s->m->info;
    // every argument on the host, before any device work
    s->check_batch(b);
    s->sel.check_rows(b);
    s->sel.check_beam_bias();
    size_t total = 0;
    bool equal = true;
    for (int i = 0; i < b; ++i) {
        VOX_CHECK(lens[i] >= 1, VOX_EINVAL, "stream %d is empty", i);
        const StreamGeom g = stream_geometry(c, lens[i]);
        VOX_CHECK(g.frames >= 1, VOX_EINVAL, "stream %d too short to produce mel frames", i);
        VOX_CHECK(g.frames <= s->enc.max_mel_frames, VOX_EINVAL,
                  "stream %d needs %d mel frames > session max_mel_frames %d (chunk it: vox_chunk_plan)", i, g.frames,
                  s->enc.max_mel_frames);
        total += (size_t)g.n_out;
        equal = equal && lens[i] == lens[0];
    }
    VOX_CHECK(cap >= total, VOX_ECAPACITY, "out_ids capacity %zu < %zu", cap, total);
    if (equal) {   // the batched [b][n] path: its layouts of ids, scores and n-best are the packed ones
        int32_t n = 0;
        const int32_t rc = transcribe_pcm_impl(s, samples, nullptr, b, lens[0], normalize, out_ids, cap, &n, tm, true);
        for (int i = 0; i < b; ++i) n_out[i] = n;
        if (s->sel.beam_w == 1) {   // like a ragged call, leave the decoder cache empty
            s->reset();
            CUDA_OK(cudaStreamSynchronize(s->st));
        }
        return rc;
    }
    s->transcribe_ragged(samples, lens, b, normalize, out_ids, n_out, tm);
    fill_timings(s, tm);
    VOX_API_END
}
int32_t vox_transcribe_pcm_dev(vox_session *sh, const float *samples_dev, int32_t b, size_t n, int32_t *out_ids,
                               size_t cap, int32_t *n_out, vox_timings *tm) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(samples_dev); REQUIRE(out_ids); REQUIRE(n_out);
    return transcribe_pcm_impl(sh->s, nullptr, samples_dev, b, n, 1, out_ids, cap, n_out, tm);
    VOX_API_END
}

int32_t vox_generate_step_with_cache(vox_session *sh, const int32_t *ids, int32_t b, int32_t m, float *logits, size_t cap) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(ids); REQUIRE(logits);
    Session *s = sh->s;
    const vox_model_info &c = s->m->info;
    s->check_batch(b);
    VOX_CHECK(m >= 1 && m <= s->M_max, VOX_EINVAL, "M=%d out of range [1,%d]", m, s->M_max);
    VOX_CHECK(s->cache_len + m <= s->out_ld, VOX_EINVAL, "KV cache full (%d + %d > %d)", s->cache_len, m, s->out_ld);
    s->check_ids(ids, (size_t)b * m);
    const size_t n = (size_t)b * m * c.vocab;
    VOX_CHECK(cap >= n, VOX_ECAPACITY, "logits capacity %zu < %zu", cap, n);
    CUDA_OK(cudaSetDevice(s->m->device));
    if (n > s->logits_all_cap) { s->logits_all = s->arena.alloc_n<float>(n); s->logits_all_cap = n; }
    s->forward_logits(b, m, ids, false, s->logits_all);
    CUDA_OK(cudaMemcpyAsync(logits, s->logits_all, sizeof(float) * n, cudaMemcpyDeviceToHost, s->st));
    CUDA_OK(cudaStreamSynchronize(s->st));
    VOX_API_END
}
// forward_streaming (model.rs:801-814): teacher-forced full pass, inputs = audio_embeds + embed(ids).
int32_t vox_forward_streaming(vox_session *sh, const float *mel, int32_t b, int32_t t, const int32_t *ids, int32_t n_ids,
                              float *logits, size_t cap) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(mel); REQUIRE(ids); REQUIRE(logits);
    Session *s = sh->s;
    const vox_model_info &c = s->m->info;
    s->enc.upload_mel(*s, mel, b, t);
    encode_uniform(s, b, t);
    const int S4 = s->enc.positions;
    VOX_CHECK(n_ids == S4, VOX_EINVAL, "forward_streaming needs one token id per audio position (%d), got %d", S4, n_ids);
    VOX_CHECK(S4 <= s->out_ld, VOX_EINVAL, "sequence %d exceeds the session KV capacity %d", S4, s->out_ld);
    s->check_ids(ids, (size_t)b * n_ids);
    const size_t n = (size_t)b * S4 * c.vocab;
    VOX_CHECK(cap >= n, VOX_ECAPACITY, "logits capacity %zu < %zu", cap, n);
    s->reset();
    const int Mc = s->M_max;
    const size_t chunk_floats = (size_t)b * Mc * c.vocab;
    if (chunk_floats > s->logits_all_cap) { s->logits_all = s->arena.alloc_n<float>(chunk_floats); s->logits_all_cap = chunk_floats; }
    std::vector<int> chunk_ids;
    for (int p0 = 0; p0 < S4; p0 += Mc) {
        const int m = std::min(Mc, S4 - p0);
        chunk_ids.resize((size_t)b * m);
        for (int bb = 0; bb < b; ++bb)
            for (int i = 0; i < m; ++i) chunk_ids[(size_t)bb * m + i] = ids[(size_t)bb * S4 + p0 + i];
        s->forward_logits(b, m, chunk_ids.data(), true, s->logits_all);
        for (int bb = 0; bb < b; ++bb)
            CUDA_OK(cudaMemcpyAsync(logits + ((size_t)bb * S4 + p0) * c.vocab, s->logits_all + (size_t)bb * m * c.vocab,
                                    sizeof(float) * (size_t)m * c.vocab, cudaMemcpyDeviceToHost, s->st));
        CUDA_OK(cudaStreamSynchronize(s->st));  // chunk_ids is reused
    }
    VOX_API_END
}

// Device-side incremental decode (SURVEY 8(b); model.rs:857-867 without the logits round trip): the argmax stays on
// the device and feeds the next step; only b int32 ids cross the bus, and only when the caller asks for them.
int32_t vox_prefill(vox_session *sh, const int32_t *ids, int32_t b, int32_t m, int32_t add_audio, int32_t *next_tok) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(ids);
    Session *s = sh->s;
    s->check_batch(b);
    VOX_CHECK(m >= 1 && m <= s->M_max, VOX_EINVAL, "M=%d out of range [1,%d]", m, s->M_max);
    s->sel.check_greedy("vox_prefill");
    VOX_CHECK(s->cache_len + m <= s->out_ld, VOX_EINVAL, "KV cache full (%d + %d > %d)", s->cache_len, m, s->out_ld);
    if (add_audio)
        VOX_CHECK(b == (int)s->enc.audio_offs.size() && s->cache_len + m <= s->enc.positions, VOX_EINVAL,
                  "add_audio: positions %d..%d need audio embeddings of %d streams (have %d positions for %d streams; call vox_encode_audio first)",
                  s->cache_len, s->cache_len + m, b, s->enc.positions, (int)s->enc.audio_offs.size());
    s->check_ids(ids, (size_t)b * m);
    CUDA_OK(cudaSetDevice(s->m->device));
    s->step_incremental(b, m, ids, add_audio != 0);
    if (next_tok) CUDA_OK(cudaMemcpyAsync(next_tok, s->d_tok, sizeof(int) * b, cudaMemcpyDeviceToHost, s->st));
    CUDA_OK(cudaStreamSynchronize(s->st));   // `ids` is caller memory
    VOX_API_END
}
int32_t vox_decode_step(vox_session *sh, const int32_t *tok, int32_t b, int32_t add_audio, int32_t *next_tok) {
    VOX_API_BEGIN
    REQUIRE(sh);
    Session *s = sh->s;
    s->check_batch(b);
    s->sel.check_greedy("vox_decode_step");
    VOX_CHECK(s->cache_len + 1 <= s->out_ld, VOX_EINVAL, "KV cache full (%d + 1 > %d)", s->cache_len, s->out_ld);
    if (add_audio)
        VOX_CHECK(b == (int)s->enc.audio_offs.size() && s->cache_len < s->enc.positions, VOX_EINVAL,
                  "add_audio: position %d has no audio embedding (%d positions, %d streams encoded)", s->cache_len,
                  s->enc.positions, (int)s->enc.audio_offs.size());
    CUDA_OK(cudaSetDevice(s->m->device));
    if (tok) {
        s->check_ids(tok, b);
        CUDA_OK(cudaMemcpyAsync(s->d_tok, tok, sizeof(int) * b, cudaMemcpyHostToDevice, s->st));
    }
    s->step_incremental(b, 1, nullptr, add_audio != 0);
    if (next_tok) CUDA_OK(cudaMemcpyAsync(next_tok, s->d_tok, sizeof(int) * b, cudaMemcpyDeviceToHost, s->st));
    if (next_tok || tok) CUDA_OK(cudaStreamSynchronize(s->st));
    VOX_API_END
}
static_assert(VOX_MAX_TOP_K == TOPK_MAX, "the score buffers hold VOX_MAX_TOP_K entries per position");
int32_t vox_session_set_top_k(vox_session *s, int32_t k) {
    VOX_API_BEGIN
    REQUIRE(s);
    s->s->sel.set_top_k(k);
    VOX_API_END
}
int32_t vox_session_token_scores(vox_session *sh, int32_t *top_ids, float *top_logprobs, size_t cap, int32_t *b, int32_t *n,
                                 int32_t *k) {
    VOX_API_BEGIN
    REQUIRE(sh);
    Session *s = sh->s;
    s->sel.read_scores(top_ids, top_logprobs, cap, b, n, k, s->st);
    VOX_API_END
}
static_assert(VOX_MAX_BEAM == BEAM_MAX, "the beam kernels handle up to VOX_MAX_BEAM beams per stream");
int32_t vox_session_set_beam(vox_session *s, int32_t width) {
    VOX_API_BEGIN
    REQUIRE(s);
    s->s->sel.set_beam(width);
    VOX_API_END
}
static_assert(VOX_MAX_BIAS_PHRASES == BIAS_MAX_PHRASES && VOX_MAX_BIAS_LEN == BIAS_MAX_LEN &&
                  VOX_FIRST_TEXT_ID == BIAS_FIRST_TEXT_ID,
              "the bias kernel's limits are the header's");
int32_t vox_session_set_bias(vox_session *sh, int32_t stream, const int32_t *ids, const int32_t *lens, const float *boosts,
                             int32_t n_phrases) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(sh);
    sh->s->set_bias(stream, ids, lens, boosts, n_phrases);
    VOX_API_END
}
// vox_session_set_bias_text's expansion: phrase p -> encode(p), then encode(" " + p) unless p starts with White_Space
// (and unless it equals the first form), both at boosts[p], in phrase order.  Checked here, on the host, in full.
struct BiasText {
    std::vector<int32_t> ids, lens;
    std::vector<float> boosts;
};
static BiasText expand_bias_text(const vox_tokenizer *t, const char *const *phrases, const float *boosts, int32_t n) {
    BiasText o;
    VOX_CHECK(n >= 0, VOX_EINVAL, "set_bias_text: %d phrases", n);
    if (n == 0) return o;
    REQUIRE(t); REQUIRE(phrases); REQUIRE(boosts);
    auto add = [&](const std::vector<int32_t> &form, int p) {
        VOX_CHECK(form.size() <= VOX_MAX_BIAS_LEN, VOX_EINVAL, "set_bias_text: phrase %d encodes to %zu ids (at most %d)", p,
                  form.size(), VOX_MAX_BIAS_LEN);
        VOX_CHECK(o.lens.size() < VOX_MAX_BIAS_PHRASES, VOX_EINVAL,
                  "set_bias_text: phrase %d: more than %d id phrases after adding the leading-space forms", p, VOX_MAX_BIAS_PHRASES);
        o.ids.insert(o.ids.end(), form.begin(), form.end());
        o.lens.push_back((int32_t)form.size());
        o.boosts.push_back(boosts[p]);
    };
    for (int p = 0; p < n; ++p) {
        VOX_CHECK(phrases[p] != nullptr, VOX_EINVAL, "set_bias_text: phrase %d is NULL", p);
        const std::string word(phrases[p]);
        VOX_CHECK(!word.empty(), VOX_EINVAL, "set_bias_text: phrase %d is empty", p);
        std::vector<int32_t> bare;
        try {
            bare = t->t->encode(word.data(), word.size());
        } catch (const Error &e) {
            fail(e.code, fmt("set_bias_text: phrase %d: %s", p, e.what()));
        }
        add(bare, p);
        // a phrase that starts with White_Space keeps its one form: " " + p would only lengthen its leading run
        if (Tokenizer::starts_with_white_space(word.data(), word.size())) continue;
        const std::string with_space = " " + word;
        const std::vector<int32_t> spaced = t->t->encode(with_space.data(), with_space.size());
        if (spaced != bare) add(spaced, p);
    }
    return o;
}
int32_t vox_session_set_bias_text(vox_session *sh, int32_t stream, const vox_tokenizer *t, const char *const *phrases,
                                  const float *boosts, int32_t n_phrases) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(sh);
    const BiasText b = expand_bias_text(t, phrases, boosts, n_phrases);
    sh->s->set_bias(stream, b.ids.data(), b.lens.data(), b.boosts.data(), (int)b.lens.size());
    VOX_API_END
}
int32_t vox_session_nbest(vox_session *sh, int32_t *ids, double *scores, size_t cap, int32_t *b, int32_t *w, int32_t *n) {
    VOX_API_BEGIN
    REQUIRE(sh);
    Session *s = sh->s;
    s->sel.read_nbest(ids, scores, cap, b, w, n, s->st);
    VOX_API_END
}
int32_t vox_session_cache_len(const vox_session *s, int32_t *len) {
    VOX_API_BEGIN
    REQUIRE(s); REQUIRE(len);
    *len = s->s->cache_len;
    VOX_API_END
}
int32_t vox_session_reset(vox_session *s) {
    VOX_API_BEGIN
    REQUIRE(s);
    CUDA_OK(cudaSetDevice(s->s->m->device));
    s->s->reset();
    CUDA_OK(cudaStreamSynchronize(s->s->st));
    VOX_API_END
}
int32_t vox_session_debug_read(vox_session *sh, const char *what, float *out, size_t cap, size_t *n_floats) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(what);
    Session *s = sh->s;
    const vox_model_info &c = s->m->info;
    CUDA_OK(cudaSetDevice(s->m->device));
    const std::string w = what;
    const float *src = nullptr;
    size_t n = 0;
    AudioEncoder &e = s->enc;
    const size_t rows = (size_t)e.rows;
    if (w == "capture_on" || w == "capture_off") {
        e.set_capture(*s, w == "capture_on");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "graph_off" || w == "graph_on") {
        s->use_graph = (w == "graph_on");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "enc_attn_simt" || w == "enc_attn_tc") {
        e.use_attn_tc = (w == "enc_attn_tc");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "gemm_simt" || w == "gemm_tc") {
        s->path.gemm_tc = (w == "gemm_tc");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "mega_off" || w == "mega_on" || w == "mega_auto") {
        // mega_on / mega_auto: persistent decode kernel for every batch size (the default policy since round 2: it is no
        // slower than the per-op launches even for a single stream); mega_off: per-op launches
        s->use_mega = (w != "mega_off");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "tc_off" || w == "tc_on") {
        s->path.matvec_tc = (w == "tc_on");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "mega_epoch") {
        // {persistent-kernel launches counted on the host since the last re-base, the device epoch}: equal between calls
        int epoch = 0;
        CUDA_OK(cudaStreamSynchronize(s->st));
        CUDA_OK(cudaMemcpy(&epoch, s->mega.epoch, sizeof(int), cudaMemcpyDeviceToHost));
        const float v[2] = {(float)s->mega.launches, (float)epoch};
        if (n_floats) *n_floats = 2;
        if (out) {
            VOX_CHECK(cap >= 2, VOX_ECAPACITY, "debug_read capacity %zu < 2", cap);
            memcpy(out, v, sizeof(v));
        }
        return VOX_OK;
    } else if (w == "mega_attn") {
        // attention tiling of the last decode step: per persistent launch {rows, token capacity, keys per K/V tile, key
        // chunks per (stream, kv head)}; nothing after a step on the per-op path
        const size_t cnt = s->mega.attn_log.size() * 4;
        if (n_floats) *n_floats = cnt;
        if (out) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            for (size_t i = 0; i < cnt; ++i) out[i] = (float)s->mega.attn_log[i / 4][i % 4];
        }
        return VOX_OK;
    } else if ((w.rfind("kv_k", 0) == 0 || w.rfind("kv_v", 0) == 0) && w.size() > 4) {
        // layer l's cached K or V of rows [0, cur_B) at positions [0, cache length), f32 [row][pos][kv_head][hd]
        const int l = atoi(w.c_str() + 4);
        VOX_CHECK(l >= 0 && l < c.dec_layers && std::to_string(l) == w.substr(4), VOX_EINVAL, "no decoder layer in '%s'", what);
        const int B = s->cur_B;
        std::vector<int> pos(B);
        CUDA_OK(cudaStreamSynchronize(s->st));
        if (B) CUDA_OK(cudaMemcpy(pos.data(), s->d_pos, sizeof(int) * B, cudaMemcpyDeviceToHost));
        const int L = B ? std::min(pos[0], s->kv.capacity()) : 0;
        for (int b = 0; b < B; ++b) VOX_CHECK(pos[b] == pos[0], VOX_EINVAL, "'%s': rows at different positions", what);
        const size_t cnt = (size_t)B * L * c.dec_kv_heads * c.dec_head_dim;
        if (n_floats) *n_floats = cnt;
        if (out && cnt) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            s->kv.read(l, w[3] == 'v', B, L, out);
        }
        return VOX_OK;
    } else if (w == "mega_trace") {
        // phase trace of the last persistent decode step (CTA 0): per op {start, staged, body done,
        // barrier passed, first weights ready | KV walked, last stage consumed} in microseconds since the first stamp; ops 0..mega.n_ops-1
        const size_t cnt = (size_t)s->mega.n_ops * 6;
        if (n_floats) *n_floats = cnt;
        if (out) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            CUDA_OK(cudaStreamSynchronize(s->st));
            std::vector<unsigned long long> t(cnt);
            if (cnt) CUDA_OK(cudaMemcpy(t.data(), s->mega.trace, sizeof(unsigned long long) * cnt, cudaMemcpyDeviceToHost));
            int khz = 0;
            CUDA_OK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, s->m->device));
            for (size_t i = 0; i < cnt; ++i) out[i] = (float)((double)(t[i] - t[0]) / ((double)khz * 1e-3));
        }
        return VOX_OK;
    } else if (w == "mega_trace_all") {
        // [grid][n_ops][4] microseconds relative to each CTA's exit from the first grid barrier (VOX_MEGA_TRACE_ALL=1)
        VOX_CHECK(s->mega.trace_all != nullptr, VOX_ENOTFOUND, "all-CTA trace not enabled (VOX_MEGA_TRACE_ALL=1 at session creation)");
        const size_t per = (size_t)s->mega.n_ops * 4, cnt = per * s->mega.grid;
        if (n_floats) *n_floats = cnt;
        if (out) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            CUDA_OK(cudaStreamSynchronize(s->st));
            std::vector<unsigned long long> t(cnt);
            if (cnt) CUDA_OK(cudaMemcpy(t.data(), s->mega.trace_all, sizeof(unsigned long long) * cnt, cudaMemcpyDeviceToHost));
            int khz = 0;
            CUDA_OK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, s->m->device));
            for (int ctai = 0; ctai < s->mega.grid; ++ctai) {
                const unsigned long long t0 = t[(size_t)ctai * per + 2];
                for (size_t i = 0; i < per; ++i)
                    out[(size_t)ctai * per + i] = (float)((double)((long long)(t[(size_t)ctai * per + i] - t0)) / ((double)khz * 1e-3));
            }
        }
        return VOX_OK;
    } else if (w == "pcm_pad") {
        // each stream's normalised, padded signal of the last PCM call, stream after stream
        const AudioEncoder::FrontEnd &f = e.front;
        VOX_CHECK(!f.padded.empty(), VOX_ENOTFOUND, "'pcm_pad': the last call did not start from PCM");
        size_t cnt = 0;
        for (size_t p : f.padded) cnt += p;
        if (n_floats) *n_floats = cnt;
        if (out) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            CUDA_OK(cudaStreamSynchronize(s->st));
            for (size_t i = 0, o = 0; i < f.padded.size(); o += f.padded[i], ++i)
                CUDA_OK(cudaMemcpy(out + o, e.pcm_pad + f.pad_off[i], sizeof(float) * f.padded[i], cudaMemcpyDeviceToHost));
        }
        return VOX_OK;
    } else if (w == "mel") {
        // PCM call: the time-major mel every stream's frames were packed into; mel call: the caller's [B][128][T]
        const AudioEncoder::FrontEnd &f = e.front;
        VOX_CHECK(!f.frames.empty(), VOX_ENOTFOUND, "'mel': no call has computed or uploaded a mel yet");
        for (int t : f.frames) n += (size_t)t * c.n_mels;
        src = f.padded.empty() ? e.mel : e.mel_tm;
    }
    else if (w == "enc_out") { src = e.h_enc; n = rows * c.enc_dim; }
    else if (w == "audio_embeds") { src = e.audio; n = (size_t)e.audio_n * c.dec_dim; }   // stream after stream
    else if (w == "conv") { src = e.dbg_conv; n = rows * c.enc_dim; }
    else if (w == "logits") { src = s->logits; n = (size_t)s->cur_B * c.vocab; }
    else if (w == "ada") { src = s->ada_sets; n = (size_t)c.dec_layers * c.dec_dim; }   // stream 0's ADA scale
    else if (w.rfind("enc", 0) == 0 && w.size() > 3) {
        const int i = atoi(w.c_str() + 3);
        VOX_CHECK(i >= 0 && i < c.enc_layers && e.dbg_layers, VOX_EINVAL, "no capture for '%s'", what);
        src = e.dbg_layers + (size_t)i * rows * c.enc_dim;
        n = rows * c.enc_dim;
    }
    VOX_CHECK(src != nullptr, VOX_ENOTFOUND, "unknown debug buffer '%s'", what);
    if (n_floats) *n_floats = n;
    if (out) {
        VOX_CHECK(cap >= n, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, n);
        CUDA_OK(cudaStreamSynchronize(s->st));
        if (n) CUDA_OK(cudaMemcpy(out, src, sizeof(float) * n, cudaMemcpyDeviceToHost));
    }
    VOX_API_END
}
int32_t vox_session_launch_count(const vox_session *s, uint64_t *launches) {
    VOX_API_BEGIN
    REQUIRE(s); REQUIRE(launches);
    *launches = kernel_launch_count();
    VOX_API_END
}
void vox_session_free(vox_session *s) {
    if (!s) return;
    cudaSetDevice(s->s->m->device);
    delete s->s;
    delete s;
}

// ---------------------------------------------------------------- streaming sessions
int32_t vox_stream_pool_create(vox_model *m, int32_t max_sessions, float max_seconds, vox_stream_pool **out) {
    return vox_stream_pool_create_ex(m, max_sessions, max_seconds, VOX_DTYPE_F32, out);
}
int32_t vox_stream_pool_create_ex(vox_model *m, int32_t max_sessions, float max_seconds, int32_t kv_dtype,
                                  vox_stream_pool **out) {
    VOX_API_BEGIN
    REQUIRE(m); REQUIRE(out);
    const KvType t = kv_type_of(kv_dtype);
    CUDA_OK(cudaSetDevice(m->m->device));
    *out = new vox_stream_pool{StreamPool::create(m->m, max_sessions, max_seconds, t)};
    VOX_API_END
}
int32_t vox_stream_pool_device_bytes(const vox_stream_pool *p, uint64_t *bytes) {
    VOX_API_BEGIN
    REQUIRE(p); REQUIRE(bytes);
    *bytes = p->p->s->arena.total;
    VOX_API_END
}
int32_t vox_stream_open(vox_stream_pool *p, int32_t *session) {
    VOX_API_BEGIN
    REQUIRE(p); REQUIRE(session);
    *session = p->p->open();
    VOX_API_END
}
int32_t vox_stream_push_pcm(vox_stream_pool *p, int32_t session, const float *samples, size_t n) {
    VOX_API_BEGIN
    REQUIRE(p);
    if (n) REQUIRE(samples);
    p->p->push(session, samples, n);
    VOX_API_END
}
int32_t vox_stream_finish(vox_stream_pool *p, int32_t session) {
    VOX_API_BEGIN
    REQUIRE(p);
    p->p->finish(session);
    VOX_API_END
}
int32_t vox_stream_tick(vox_stream_pool *p, vox_stream_stats *stats) {
    VOX_API_BEGIN
    REQUIRE(p);
    p->p->tick(stats);
    VOX_API_END
}
int32_t vox_stream_poll_ids(vox_stream_pool *p, int32_t session, int32_t *ids, size_t cap, size_t *n, int32_t *done) {
    VOX_API_BEGIN
    REQUIRE(p); REQUIRE(n);
    if (cap) REQUIRE(ids);
    bool d = false;
    *n = p->p->poll(session, ids, nullptr, nullptr, cap, &d);
    if (done) *done = d ? 1 : 0;
    VOX_API_END
}
int32_t vox_stream_pool_set_top_k(vox_stream_pool *p, int32_t k) {
    VOX_API_BEGIN
    REQUIRE(p);
    CUDA_OK(cudaSetDevice(p->p->m->device));
    p->p->set_top_k(k);
    VOX_API_END
}
int32_t vox_stream_poll_scored(vox_stream_pool *p, int32_t session, int32_t *ids, int32_t *top_ids, float *top_logprobs,
                               size_t cap, size_t *n, int32_t *done) {
    VOX_API_BEGIN
    REQUIRE(p); REQUIRE(n);
    VOX_CHECK(p->p->s->sel.top_k > 0, VOX_EINVAL, "no token scores: the pool's top_k is 0 (vox_stream_pool_set_top_k)");
    if (cap) { REQUIRE(ids); REQUIRE(top_ids); REQUIRE(top_logprobs); }
    bool d = false;
    *n = p->p->poll(session, ids, top_ids, top_logprobs, cap, &d);
    if (done) *done = d ? 1 : 0;
    VOX_API_END
}
int32_t vox_stream_audio_embeds(vox_stream_pool *p, int32_t session, float *out, size_t cap, int32_t *n) {
    VOX_API_BEGIN
    REQUIRE(p); REQUIRE(n);
    int cnt = 0;
    const float *src = p->p->audio_embeds(session, &cnt);
    *n = cnt;
    if (out) {
        const size_t need = (size_t)cnt * p->p->m->info.dec_dim;
        VOX_CHECK(cap >= need, VOX_ECAPACITY, "audio_embeds capacity %zu < %zu", cap, need);
        CUDA_OK(cudaSetDevice(p->p->m->device));
        CUDA_OK(cudaStreamSynchronize(p->p->s->st));
        if (need) CUDA_OK(cudaMemcpy(out, src, sizeof(float) * need, cudaMemcpyDeviceToHost));
    }
    VOX_API_END
}
// the device check comes first, as in every compute entry point: without a device no pool can exist
static void require_any_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    VOX_CHECK(e == cudaSuccess && n > 0, VOX_ECUDA, "no CUDA device available (%s); this library has no CPU fallback",
              cudaGetErrorString(e));
}
int32_t vox_stream_audio_embeds_range(vox_stream_pool *p, int32_t session, int64_t first, int64_t n, float *out, size_t cap) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(p);
    const float *src = p->p->audio_embeds_range(session, first, n);
    const size_t need = (size_t)n * p->p->m->info.dec_dim;
    if (need) REQUIRE(out);
    VOX_CHECK(cap >= need, VOX_ECAPACITY, "audio_embeds capacity %zu < %zu", cap, need);
    CUDA_OK(cudaSetDevice(p->p->m->device));
    CUDA_OK(cudaStreamSynchronize(p->p->s->st));
    if (need) CUDA_OK(cudaMemcpy(out, src, sizeof(float) * need, cudaMemcpyDeviceToHost));
    VOX_API_END
}
int32_t vox_stream_mel_range(vox_stream_pool *p, int32_t session, int64_t first, int64_t n, float *out, size_t cap) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(p);
    const float *src = p->p->mel_range(session, first, n);
    const size_t need = (size_t)n * p->p->m->info.n_mels;
    if (need) REQUIRE(out);
    VOX_CHECK(cap >= need, VOX_ECAPACITY, "mel capacity %zu < %zu", cap, need);
    CUDA_OK(cudaSetDevice(p->p->m->device));
    CUDA_OK(cudaStreamSynchronize(p->p->s->st));
    if (need) CUDA_OK(cudaMemcpy(out, src, sizeof(float) * need, cudaMemcpyDeviceToHost));
    VOX_API_END
}
int32_t vox_stream_set_delay(vox_stream_pool *p, int32_t session, float delay_tokens) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(p);
    p->p->set_delay(session, delay_tokens);
    VOX_API_END
}
int32_t vox_stream_set_bias(vox_stream_pool *p, int32_t session, const int32_t *ids, const int32_t *lens, const float *boosts,
                            int32_t n_phrases) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(p);
    p->p->set_bias(session, ids, lens, boosts, n_phrases);
    VOX_API_END
}
int32_t vox_stream_set_bias_text(vox_stream_pool *p, int32_t session, const vox_tokenizer *t, const char *const *phrases,
                                 const float *boosts, int32_t n_phrases) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(p);
    const BiasText b = expand_bias_text(t, phrases, boosts, n_phrases);
    p->p->set_bias(session, b.ids.data(), b.lens.data(), b.boosts.data(), (int)b.lens.size());
    VOX_API_END
}
int32_t vox_stream_session_info(vox_stream_pool *p, int32_t session, struct vox_stream_session_info *out) {
    VOX_API_BEGIN
    require_any_device();
    REQUIRE(p); REQUIRE(out);
    p->p->session_info(session, out);
    VOX_API_END
}
int32_t vox_stream_encode_chunk(vox_stream_pool *p, int32_t session, const float *mel, int32_t t, float *out, size_t cap, int32_t *n) {
    VOX_API_BEGIN
    REQUIRE(p); REQUIRE(mel); REQUIRE(out); REQUIRE(n);
    *n = p->p->encode_chunk(session, mel, t, out, cap);
    VOX_API_END
}
int32_t vox_stream_close(vox_stream_pool *p, int32_t session) {
    VOX_API_BEGIN
    REQUIRE(p);
    p->p->close(session);
    VOX_API_END
}
void vox_stream_pool_free(vox_stream_pool *p) {
    if (!p) return;
    cudaSetDevice(p->p->m->device);
    delete p->p;
    delete p;
}

// ---------------------------------------------------------------- tokenizer
int32_t vox_tokenizer_from_file(const char *path, vox_tokenizer **out) {
    VOX_API_BEGIN
    REQUIRE(path); REQUIRE(out);
    *out = new vox_tokenizer{Tokenizer::from_file(path)};
    VOX_API_END
}
int32_t vox_tokenizer_from_json(const char *json, size_t len, vox_tokenizer **out) {
    VOX_API_BEGIN
    REQUIRE(json); REQUIRE(out);
    *out = new vox_tokenizer{Tokenizer::from_json(json, len)};
    VOX_API_END
}
static void copy_out(const std::string &s, char *buf, size_t cap, size_t *written) {
    if (written) *written = s.size();
    if (buf) {
        VOX_CHECK(cap >= s.size() + 1, VOX_ECAPACITY, "text buffer too small (%zu < %zu)", cap, s.size() + 1);
        memcpy(buf, s.data(), s.size());
        buf[s.size()] = '\0';
    }
}
int32_t vox_tokenizer_decode(const vox_tokenizer *t, const uint32_t *ids, size_t n, char *buf, size_t cap, size_t *written) {
    VOX_API_BEGIN
    REQUIRE(t);
    if (n) REQUIRE(ids);
    copy_out(t->t->decode(ids, n), buf, cap, written);
    VOX_API_END
}
int32_t vox_tokenizer_decode_token(const vox_tokenizer *t, uint32_t id, char *buf, size_t cap, size_t *written, int32_t *found) {
    VOX_API_BEGIN
    REQUIRE(t);
    std::string s;
    const bool ok = t->t->decode_token(id, &s);
    if (found) *found = ok ? 1 : 0;
    copy_out(ok ? s : std::string(), buf, cap, written);
    VOX_API_END
}
int32_t vox_tokenizer_encode(const vox_tokenizer *t, const char *text, size_t len, int32_t *ids, size_t cap, size_t *n) {
    VOX_API_BEGIN
    REQUIRE(t); REQUIRE(n);
    if (len) REQUIRE(text);
    const std::vector<int32_t> out = t->t->encode(text, len);
    *n = out.size();
    if (ids) {
        VOX_CHECK(cap >= out.size(), VOX_ECAPACITY, "id buffer too small (%zu < %zu)", cap, out.size());
        std::copy(out.begin(), out.end(), ids);
    }
    VOX_API_END
}
int32_t vox_tokenizer_vocab_size(const vox_tokenizer *t, size_t *n) {
    VOX_API_BEGIN
    REQUIRE(t); REQUIRE(n);
    *n = t->t->vocab_size();
    VOX_API_END
}
void vox_tokenizer_free(vox_tokenizer *t) {
    if (!t) return;
    delete t->t;
    delete t;
}

}  // extern "C"
