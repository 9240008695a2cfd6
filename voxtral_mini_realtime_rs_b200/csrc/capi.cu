// capi.cu -- the extern "C" boundary declared in include/voxtral.h.  Every entry point converts
// exceptions into a status code + thread-local message; nothing here computes on the CPU on
// behalf of the GPU path (no fallback): without a CUDA device the compute calls return VOX_ECUDA.
#include <cuda_profiler_api.h>
#include <cuda_runtime.h>

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
namespace vox { void set_tc_pdl(bool on); }

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
    {   // split-K scratch: up to ceil(K/64/16) slices x 8 rows x padded N, and one ticket per row tile
        const int n_tiles = (int)((n + 15) / 16), n_pairs = (int)((k / 32 + 1) / 2);
        const size_t S = (size_t)(n_pairs + 15) / 16;
        q->wk.partial_floats = S * 8 * (size_t)n_tiles * 16;
        q->wk.partial = q->arena.alloc_n<float>(q->wk.partial_floats);
        q->wk.n_counters = n_tiles;
        q->wk.counters = q->arena.alloc_n<int>(n_tiles);
        CUDA_OK(cudaMemset(q->wk.counters, 0, sizeof(int) * n_tiles));
    }
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
// 0 = tensor-core-assisted matvec for M <= 8 (default), 1 = SIMT warp-reduce matvec
static int g_matvec_mode = (getenv("VOX_MATVEC") && std::string(getenv("VOX_MATVEC")) == "simt") ? 1 : 0;
static void q4_matmul_dispatch(const Q4Weight &w, const float *x, float *y, int rows, const float *bias, cudaStream_t st,
                               const TcWork *wk = nullptr, vox_q4 *h = nullptr) {
    const bool simt = (g_matvec_mode & 1) != 0;
    if (rows > 8 && h && !(g_matvec_mode & 2) && gemm_tc5_supported(w, rows)) {
        const size_t need = gemm_tc5_split_elems(rows, w.K);
        if (need > h->xt_elems) {
            h->xt = h->arena.alloc(need * 2);
            h->xt_elems = need;
        }
        if (!h->gw.partial) {
            h->gw.partial_floats = (size_t)VOX_NUM_SMS * 128 * 128;
            h->gw.partial = h->arena.alloc_n<float>(h->gw.partial_floats);
            h->gw.n_counters = 128;
            h->gw.counters = h->arena.alloc_n<int>(h->gw.n_counters);
            CUDA_OK(cudaMemset(h->gw.counters, 0, sizeof(int) * h->gw.n_counters));
        }
        launch_split_tiles(x, rows, w.K, nullptr, nullptr, 0.0f, h->xt, st);
        launch_q4_gemm_tc5(w, h->xt, rows, y, w.N, bias, nullptr, EPI_NONE, &h->gw, st);
        return;
    }
    if (rows <= 8 && w.qs_tc && !simt)
        launch_q4_matvec_tc_ex(w, x, rows, y, w.N, bias, nullptr, EPI_NONE, nullptr, nullptr, 0.0f, wk, st);
    else if (rows <= 8) launch_q4_matvec(w, x, rows, y, w.N, bias, nullptr, EPI_NONE, st);
    else launch_q4_gemm(w, x, rows, y, w.N, bias, nullptr, EPI_NONE, st);
}
int32_t vox_q4_set_matvec_mode(int32_t mode) {
    VOX_API_BEGIN
    VOX_CHECK(mode >= 0 && mode <= 3, VOX_EINVAL, "mode bits: 1 = SIMT matvec (M<=8), 2 = SIMT GEMM (M>8)");
    g_matvec_mode = mode;
    VOX_API_END
}
int32_t vox_q4_matmul(const vox_q4 *w, const float *x_dev, float *y_dev, int32_t b, int32_t m, const float *bias_dev,
                      void *stream) {
    VOX_API_BEGIN
    REQUIRE(w); REQUIRE(x_dev); REQUIRE(y_dev);
    VOX_CHECK(b > 0 && m > 0, VOX_EINVAL, "q4_matmul: B and M must be positive");
    CUDA_OK(cudaSetDevice(w->device));
    q4_matmul_dispatch(w->w, x_dev, y_dev, b * m, bias_dev, (cudaStream_t)stream, &w->wk, const_cast<vox_q4 *>(w));
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
    q4_matmul_dispatch(w->w, w->x, w->y, (int)rows, bias ? w->bias : nullptr, 0, &w->wk, w);
    CUDA_OK(cudaMemcpyAsync(y, w->y, sizeof(float) * yn, cudaMemcpyDeviceToHost, 0));
    CUDA_OK(cudaStreamSynchronize(0));
    VOX_API_END
}
void vox_q4_tensor_free(vox_q4 *w) {
    if (!w) return;
    cudaSetDevice(w->device);
    delete w;
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
    for (int i = 0; i < warmup; ++i) q4_matmul_dispatch(ws[i % n_w]->w, x, y, m, nullptr, st);
    CUDA_OK(cudaStreamSynchronize(st));
    CUDA_OK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i) q4_matmul_dispatch(ws[i % n_w]->w, x, y, m, nullptr, st);
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
int32_t vox_session_create(vox_model *m, int32_t max_batch, int32_t max_mel_frames, vox_session **out) {
    VOX_API_BEGIN
    REQUIRE(m); REQUIRE(out);
    Session *s = Session::create(m->m, max_batch, max_mel_frames);
    *out = new vox_session{s};
    VOX_API_END
}
int32_t vox_session_set_delay(vox_session *s, float delay) {
    VOX_API_BEGIN
    REQUIRE(s);
    s->s->set_delay(delay);
    VOX_API_END
}

static void upload_mel(Session *s, const float *mel, int b, int t) {
    const vox_model_info &c = s->m->info;
    VOX_CHECK(b >= 1 && b <= s->max_batch, VOX_EINVAL, "batch %d exceeds session max_batch %d", b, s->max_batch);
    VOX_CHECK(t >= 1 && t <= s->max_mel_frames, VOX_EINVAL, "mel frames %d exceed session max_mel_frames %d", t,
              s->max_mel_frames);
    CUDA_OK(cudaSetDevice(s->m->device));
    CUDA_OK(cudaMemcpyAsync(s->mel, mel, sizeof(float) * (size_t)b * c.n_mels * t, cudaMemcpyHostToDevice, s->st));
    launch_transpose_mel(s->mel, s->mel_tm, b, c.n_mels, t, s->st);
}

int32_t vox_encode_audio(vox_session *sh, const float *mel, int32_t b, int32_t t, float *audio_embeds, size_t cap,
                         int32_t *seq_len) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(mel);
    Session *s = sh->s;
    upload_mel(s, mel, b, t);
    s->encode(b, t);
    const size_t n = (size_t)b * s->cur_S4 * s->m->info.dec_dim;
    if (audio_embeds) {
        VOX_CHECK(cap >= n, VOX_ECAPACITY, "audio_embeds capacity %zu < %zu", cap, n);
        if (n) CUDA_OK(cudaMemcpyAsync(audio_embeds, s->audio, sizeof(float) * n, cudaMemcpyDeviceToHost, s->st));
    }
    CUDA_OK(cudaStreamSynchronize(s->st));
    if (seq_len) *seq_len = s->cur_S4;
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
    CUDA_OK(cudaSetDevice(s->m->device));
    CUDA_OK(cudaEventRecord(s->ev[0], s->st));
    upload_mel(s, mel, b, t);
    CUDA_OK(cudaEventRecord(s->ev[1], s->st));
    *n_out = s->transcribe_from_mel(b, t, out_ids, cap, tm, true);
    fill_timings(s, tm);
    VOX_API_END
}

static int32_t transcribe_pcm_impl(Session *s, const float *host, const float *dev, int b, size_t n, int normalize,
                                   int32_t *out_ids, size_t cap, int32_t *n_out, vox_timings *tm) {
    const vox_model_info &c = s->m->info;
    VOX_CHECK(b >= 1 && b <= s->max_batch, VOX_EINVAL, "batch %d exceeds session max_batch %d", b, s->max_batch);
    VOX_CHECK(n >= 1, VOX_EINVAL, "empty audio");
    CUDA_OK(cudaSetDevice(s->m->device));
    vox_pad_config pc;
    pad_config_default(&pc);
    const size_t padded = pad_audio_len(n, pc), left = pad_left(pc);
    const size_t frames = mel_num_frames(padded);
    VOX_CHECK(frames >= 1, VOX_EINVAL, "Audio too short to produce mel frames");
    VOX_CHECK(frames <= (size_t)s->max_mel_frames, VOX_EINVAL,
              "audio needs %zu mel frames > session max_mel_frames %d (chunk it: vox_chunk_plan)", frames, s->max_mel_frames);
    if ((size_t)b * padded > s->pcm_pad_cap) {
        s->pcm_pad = s->arena.alloc_n<float>((size_t)b * padded);
        s->pcm_pad_cap = (size_t)b * padded;
    }
    CUDA_OK(cudaEventRecord(s->ev[0], s->st));
    const float *src = dev;
    if (host) {
        if ((size_t)b * n > s->pcm_cap) {
            s->pcm = s->arena.alloc_n<float>((size_t)b * n);
            s->pcm_cap = (size_t)b * n;
        }
        CUDA_OK(cudaMemcpyAsync(s->pcm, host, sizeof(float) * (size_t)b * n, cudaMemcpyHostToDevice, s->st));
        src = s->pcm;
    }
    launch_peak_normalize_pad(src, b, n, 0.95f, normalize, s->pcm_pad, padded, left, s->peak_scale, s->st);
    launch_mel(s->pcm_pad, b, padded, padded, s->m->mel.window, s->m->mel.fb_vals, s->m->mel.fb_start, s->m->mel.fb_len,
               s->m->mel.fb_stride, s->mel_tm, (int)frames, 0, s->st);
    CUDA_OK(cudaEventRecord(s->ev[1], s->st));
    (void)c;
    *n_out = s->transcribe_from_mel(b, (int)frames, out_ids, cap, tm, true);
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
    VOX_CHECK(b >= 1 && b <= s->max_batch, VOX_EINVAL, "batch %d exceeds session max_batch %d", b, s->max_batch);
    VOX_CHECK(m >= 1 && m <= s->M_max, VOX_EINVAL, "M=%d out of range [1,%d]", m, s->M_max);
    VOX_CHECK(s->cache_len + m <= s->out_ld, VOX_EINVAL, "KV cache full (%d + %d > %d)", s->cache_len, m, s->out_ld);
    for (int i = 0; i < b * m; ++i)
        VOX_CHECK(ids[i] >= 0 && ids[i] < c.vocab, VOX_EINVAL, "token id %d out of range", ids[i]);
    const size_t n = (size_t)b * m * c.vocab;
    VOX_CHECK(cap >= n, VOX_ECAPACITY, "logits capacity %zu < %zu", cap, n);
    CUDA_OK(cudaSetDevice(s->m->device));
    if (n > s->logits_all_cap) {
        s->logits_all = s->arena.alloc_n<float>(n);
        s->logits_all_cap = n;
    }
    CUDA_OK(cudaMemcpyAsync(s->d_ids, ids, sizeof(int) * (size_t)b * m, cudaMemcpyHostToDevice, s->st));
    launch_embed(s->m->tok_emb, s->d_ids, nullptr, 0, b, m, nullptr, s->x_dec, s->fused_decode(b * m) ? s->ssq_x : nullptr, s->st);
    const bool pending = s->decoder_forward(b, m);
    s->lm_head_rows(b * m, pending, s->logits_all);
    launch_advance(s->d_pos, m, nullptr, 0, b, s->st);
    CUDA_OK(cudaMemcpyAsync(logits, s->logits_all, sizeof(float) * n, cudaMemcpyDeviceToHost, s->st));
    CUDA_OK(cudaStreamSynchronize(s->st));
    s->cache_len += m;
    VOX_API_END
}
// forward_streaming (model.rs:801-814): teacher-forced full pass, inputs = audio_embeds + embed(ids).
int32_t vox_forward_streaming(vox_session *sh, const float *mel, int32_t b, int32_t t, const int32_t *ids, int32_t n_ids,
                              float *logits, size_t cap) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(mel); REQUIRE(ids); REQUIRE(logits);
    Session *s = sh->s;
    const vox_model_info &c = s->m->info;
    upload_mel(s, mel, b, t);
    s->encode(b, t);
    const int S4 = s->cur_S4;
    VOX_CHECK(n_ids == S4, VOX_EINVAL, "forward_streaming needs one token id per audio position (%d), got %d", S4, n_ids);
    VOX_CHECK(S4 <= s->out_ld, VOX_EINVAL, "sequence %d exceeds the session KV capacity %d", S4, s->out_ld);
    for (int i = 0; i < b * n_ids; ++i) VOX_CHECK(ids[i] >= 0 && ids[i] < c.vocab, VOX_EINVAL, "token id %d out of range", ids[i]);
    const size_t n = (size_t)b * S4 * c.vocab;
    VOX_CHECK(cap >= n, VOX_ECAPACITY, "logits capacity %zu < %zu", cap, n);
    s->reset();
    const int Mc = s->M_max;
    const size_t chunk_floats = (size_t)b * Mc * c.vocab;
    if (chunk_floats > s->logits_all_cap) {
        s->logits_all = s->arena.alloc_n<float>(chunk_floats);
        s->logits_all_cap = chunk_floats;
    }
    std::vector<int> chunk_ids;
    for (int p0 = 0; p0 < S4; p0 += Mc) {
        const int m = std::min(Mc, S4 - p0);
        chunk_ids.resize((size_t)b * m);
        for (int bb = 0; bb < b; ++bb)
            for (int i = 0; i < m; ++i) chunk_ids[(size_t)bb * m + i] = ids[(size_t)bb * S4 + p0 + i];
        CUDA_OK(cudaMemcpyAsync(s->d_ids, chunk_ids.data(), sizeof(int) * chunk_ids.size(), cudaMemcpyHostToDevice, s->st));
        launch_embed(s->m->tok_emb, s->d_ids, s->audio, S4, b, m, s->d_pos, s->x_dec, s->fused_decode(b * m) ? s->ssq_x : nullptr, s->st);
        const bool pending = s->decoder_forward(b, m);
        s->lm_head_rows(b * m, pending, s->logits_all);
        launch_advance(s->d_pos, m, nullptr, 0, b, s->st);
        for (int bb = 0; bb < b; ++bb)
            CUDA_OK(cudaMemcpyAsync(logits + ((size_t)bb * S4 + p0) * c.vocab, s->logits_all + (size_t)bb * m * c.vocab,
                                    sizeof(float) * (size_t)m * c.vocab, cudaMemcpyDeviceToHost, s->st));
        CUDA_OK(cudaStreamSynchronize(s->st));  // chunk_ids is reused
    }
    s->cache_len = S4;
    VOX_API_END
}

// Device-side incremental decode (SURVEY 8(b); model.rs:857-867 without the logits round trip): the argmax stays on
// the device and feeds the next step; only b int32 ids cross the bus, and only when the caller asks for them.
int32_t vox_prefill(vox_session *sh, const int32_t *ids, int32_t b, int32_t m, int32_t add_audio, int32_t *next_tok) {
    VOX_API_BEGIN
    REQUIRE(sh); REQUIRE(ids);
    Session *s = sh->s;
    const vox_model_info &c = s->m->info;
    VOX_CHECK(b >= 1 && b <= s->max_batch, VOX_EINVAL, "batch %d exceeds session max_batch %d", b, s->max_batch);
    VOX_CHECK(m >= 1 && m <= s->M_max, VOX_EINVAL, "M=%d out of range [1,%d]", m, s->M_max);
    VOX_CHECK(s->cache_len + m <= s->out_ld, VOX_EINVAL, "KV cache full (%d + %d > %d)", s->cache_len, m, s->out_ld);
    if (add_audio)
        VOX_CHECK(b == s->cur_B && s->cache_len + m <= s->cur_S4, VOX_EINVAL,
                  "add_audio: positions %d..%d need audio embeddings of %d streams (have %d positions for %d streams; call vox_encode_audio first)",
                  s->cache_len, s->cache_len + m, b, s->cur_S4, s->cur_B);
    for (int i = 0; i < b * m; ++i) VOX_CHECK(ids[i] >= 0 && ids[i] < c.vocab, VOX_EINVAL, "token id %d out of range", ids[i]);
    CUDA_OK(cudaSetDevice(s->m->device));
    s->prefill(b, m, ids, add_audio != 0);
    s->cache_len += m;
    if (next_tok) CUDA_OK(cudaMemcpyAsync(next_tok, s->d_tok, sizeof(int) * b, cudaMemcpyDeviceToHost, s->st));
    CUDA_OK(cudaStreamSynchronize(s->st));   // `ids` is caller memory
    VOX_API_END
}
int32_t vox_decode_step(vox_session *sh, const int32_t *tok, int32_t b, int32_t add_audio, int32_t *next_tok) {
    VOX_API_BEGIN
    REQUIRE(sh);
    Session *s = sh->s;
    const vox_model_info &c = s->m->info;
    VOX_CHECK(b >= 1 && b <= s->max_batch, VOX_EINVAL, "batch %d exceeds session max_batch %d", b, s->max_batch);
    VOX_CHECK(s->cache_len + 1 <= s->out_ld, VOX_EINVAL, "KV cache full (%d + 1 > %d)", s->cache_len, s->out_ld);
    if (add_audio)
        VOX_CHECK(b == s->cur_B && s->cache_len < s->cur_S4, VOX_EINVAL,
                  "add_audio: position %d has no audio embedding (%d positions, %d streams encoded)", s->cache_len, s->cur_S4, s->cur_B);
    CUDA_OK(cudaSetDevice(s->m->device));
    if (tok) {
        for (int i = 0; i < b; ++i) VOX_CHECK(tok[i] >= 0 && tok[i] < c.vocab, VOX_EINVAL, "token id %d out of range", tok[i]);
        CUDA_OK(cudaMemcpyAsync(s->d_tok, tok, sizeof(int) * b, cudaMemcpyHostToDevice, s->st));
    }
    s->decode_step(b, add_audio != 0);
    s->mega_steps_host += 1;
    s->cache_len += 1;
    if (next_tok) CUDA_OK(cudaMemcpyAsync(next_tok, s->d_tok, sizeof(int) * b, cudaMemcpyDeviceToHost, s->st));
    if (next_tok || tok) CUDA_OK(cudaStreamSynchronize(s->st));
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
    const size_t rows = (size_t)s->cur_B * s->cur_S;
    if (w == "capture_on") {
        if (!s->dbg_layers) {
            s->dbg_layers = s->arena.alloc_n<float>((size_t)c.enc_layers * s->max_batch * s->S_max * c.enc_dim);
            s->dbg_conv = s->arena.alloc_n<float>((size_t)s->max_batch * s->S_max * c.enc_dim);
        }
        s->debug_capture = true;
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "capture_off") {
        s->debug_capture = false;
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "graph_off") {
        s->use_graph = false;
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "pdl_off" || w == "pdl_on") {
        set_tc_pdl(w == "pdl_on");
        if (s->step_graph) { cudaGraphExecDestroy(s->step_graph); s->step_graph = nullptr; }
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "enc_attn_simt" || w == "enc_attn_tc") {
        s->use_enc_attn_tc = (w == "enc_attn_tc");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "gemm_simt" || w == "gemm_tc") {
        s->use_gemm_tc = (w == "gemm_tc");
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "mega_off" || w == "mega_on" || w == "mega_auto") {
        // mega_on / mega_auto: persistent decode kernel for every batch size (the default policy since round 2: it is no
        // slower than the per-op launches even for a single stream); mega_off: per-op launches
        s->use_mega = (w != "mega_off");
        s->mega_min_B = 1;
        s->mega_B = 0;
        if (s->step_graph) { cudaGraphExecDestroy(s->step_graph); s->step_graph = nullptr; }
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "tc_off" || w == "tc_on") {
        s->use_tc = (w == "tc_on");
        if (s->step_graph) { cudaGraphExecDestroy(s->step_graph); s->step_graph = nullptr; }
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "graph_on") {
        s->use_graph = true;
        if (n_floats) *n_floats = 0;
        return VOX_OK;
    } else if (w == "mega_trace") {
        // phase trace of the last persistent decode step (CTA 0): per op {start, staged, body done,
        // barrier passed, first weights ready | KV walked, last stage consumed} in microseconds since the first stamp; ops 0..mega_n_ops-1
        const size_t cnt = (size_t)s->mega_n_ops * 6;
        if (n_floats) *n_floats = cnt;
        if (out) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            CUDA_OK(cudaStreamSynchronize(s->st));
            std::vector<unsigned long long> t(cnt);
            if (cnt) CUDA_OK(cudaMemcpy(t.data(), s->mega_trace, sizeof(unsigned long long) * cnt, cudaMemcpyDeviceToHost));
            int khz = 0;
            CUDA_OK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, s->m->device));
            for (size_t i = 0; i < cnt; ++i) out[i] = (float)((double)(t[i] - t[0]) / ((double)khz * 1e-3));
        }
        return VOX_OK;
    } else if (w == "mega_trace_w") {
        // [16 warps][6 groups][8] SM cycles relative to the earliest stamp (CTA 0, lm_head phase)
        VOX_CHECK(s->mega_trace_w != nullptr, VOX_ENOTFOUND, "warp trace not enabled (VOX_MEGA_TRACE_ALL=1 at session creation)");
        const size_t cnt = 16 * 6 * 8;
        if (n_floats) *n_floats = cnt;
        if (out) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            CUDA_OK(cudaStreamSynchronize(s->st));
            std::vector<unsigned long long> t(cnt);
            CUDA_OK(cudaMemcpy(t.data(), s->mega_trace_w, sizeof(unsigned long long) * cnt, cudaMemcpyDeviceToHost));
            unsigned long long t0 = ~0ull;
            for (auto v : t) if (v != 0 && v < t0) t0 = v;
            for (size_t i = 0; i < cnt; ++i) out[i] = t[i] ? (float)(t[i] - t0) : -1.0f;
        }
        return VOX_OK;
    } else if (w == "mega_trace_all") {
        // [grid][n_ops][4] microseconds relative to each CTA's exit from the first grid barrier (VOX_MEGA_TRACE_ALL=1)
        VOX_CHECK(s->mega_trace_all != nullptr, VOX_ENOTFOUND, "all-CTA trace not enabled (VOX_MEGA_TRACE_ALL=1 at session creation)");
        const size_t per = (size_t)s->mega_n_ops * 4, cnt = per * s->mega_grid;
        if (n_floats) *n_floats = cnt;
        if (out) {
            VOX_CHECK(cap >= cnt, VOX_ECAPACITY, "debug_read capacity %zu < %zu", cap, cnt);
            CUDA_OK(cudaStreamSynchronize(s->st));
            std::vector<unsigned long long> t(cnt);
            if (cnt) CUDA_OK(cudaMemcpy(t.data(), s->mega_trace_all, sizeof(unsigned long long) * cnt, cudaMemcpyDeviceToHost));
            int khz = 0;
            CUDA_OK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, s->m->device));
            for (int ctai = 0; ctai < s->mega_grid; ++ctai) {
                const unsigned long long t0 = t[(size_t)ctai * per + 2];
                for (size_t i = 0; i < per; ++i)
                    out[(size_t)ctai * per + i] = (float)((double)((long long)(t[(size_t)ctai * per + i] - t0)) / ((double)khz * 1e-3));
            }
        }
        return VOX_OK;
    } else if (w == "enc_out") { src = s->h_enc; n = rows * c.enc_dim; }
    else if (w == "audio_embeds") { src = s->audio; n = (size_t)s->cur_B * s->cur_S4 * c.dec_dim; }
    else if (w == "mel") { src = s->mel; n = 0; /* size unknown here */ }
    else if (w == "conv") { src = s->dbg_conv; n = rows * c.enc_dim; }
    else if (w == "logits") { src = s->logits; n = (size_t)s->cur_B * c.vocab; }
    else if (w == "ada") { src = s->ada; n = (size_t)c.dec_layers * c.dec_dim; }
    else if (w.rfind("enc", 0) == 0 && w.size() > 3) {
        const int i = atoi(w.c_str() + 3);
        VOX_CHECK(i >= 0 && i < c.enc_layers && s->dbg_layers, VOX_EINVAL, "no capture for '%s'", what);
        src = s->dbg_layers + (size_t)i * rows * c.enc_dim;
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
    VOX_API_BEGIN
    REQUIRE(m); REQUIRE(out);
    CUDA_OK(cudaSetDevice(m->m->device));
    *out = new vox_stream_pool{StreamPool::create(m->m, max_sessions, max_seconds)};
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
    *n = p->p->poll(session, ids, cap, &d);
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
