// kv_cache.cu -- host side of the decoder KV cache: pools, page table, page allocation and the debug read.
#include "kv_cache.h"

#include <algorithm>

#include "model.h"

namespace vox {

void DecoderKv::create(DeviceArena &arena, const vox_model_info &c, int rows, int audio, int launch, bool ring_,
                       KvType type) {
    const int cap = std::max(audio, launch) + launch;
    type_ = type;
    ring = ring_;
    layers = c.dec_layers;
    Hkv = c.dec_kv_heads;
    hd = c.dec_head_dim;
    max_pages = ring ? (c.dec_window + launch) / KV_PAGE + 1 : (cap + KV_PAGE - 1) / KV_PAGE;
    n_pages = rows * max_pages;
    const size_t bytes = (size_t)layers * layer_bytes();
    kc = arena.alloc(bytes);
    vc = arena.alloc(bytes);
    identity.resize((size_t)n_pages);
    for (int i = 0; i < n_pages; ++i) identity[i] = i;
    table = arena.upload(identity.data(), identity.size());
    for (int i = n_pages - 1; i >= 0; --i) free_list.push_back(i);
    owned.assign(rows, {});
}

void *DecoderKv::pool(bool v, int layer) const {
    return (char *)(v ? vc : kc) + (size_t)layer * layer_bytes();
}

KvView DecoderKv::view(int layer, const int *pos) const {
    KvView w;
    w.k = kv_pool(pool(false, layer), type_);
    w.v = kv_pool(pool(true, layer), type_);
    w.type = type_;
    w.page_table = table;
    w.max_pages = max_pages;
    w.ring = ring;
    w.pos = pos;
    return w;
}

void DecoderKv::fork(const int *pos, const int *src, int rows, cudaStream_t st) {
    launch_beam_fork(kc, vc, type_, layer_bytes(), layers, table, max_pages, pos, src, rows, Hkv, hd, st);
    forked = true;
}

void DecoderKv::restore_identity(cudaStream_t st) {
    if (!forked) return;
    CUDA_OK(cudaMemcpyAsync(table, identity.data(), sizeof(int) * identity.size(), cudaMemcpyHostToDevice, st));
    forked = false;
}

void DecoderKv::reserve(int stream, int positions) {
    int need = (positions + KV_PAGE - 1) / KV_PAGE;
    if (ring) need = std::min(need, max_pages);  // a full ring: logical page lp reuses slot lp % max_pages
    VOX_CHECK(need <= max_pages, VOX_ECAPACITY, "stream session needs %d decoder positions > capacity %d", positions, capacity());
    std::vector<int> &own = owned[stream];
    while ((int)own.size() < need) {
        VOX_CHECK(!free_list.empty(), VOX_ECAPACITY, "decoder KV page pool exhausted (%d pages)", n_pages);
        own.push_back(free_list.back());
        free_list.pop_back();
    }
}

void DecoderKv::release(int stream) {
    for (int pg : owned[stream]) free_list.push_back(pg);
    owned[stream].clear();
}

void DecoderKv::bind(const std::vector<int> &streams, cudaStream_t st) {
    staged.assign(streams.size() * max_pages, 0);
    for (size_t i = 0; i < streams.size(); ++i) std::copy(owned[streams[i]].begin(), owned[streams[i]].end(), staged.begin() + i * max_pages);
    CUDA_OK(cudaMemcpyAsync(table, staged.data(), sizeof(int) * staged.size(), cudaMemcpyHostToDevice, st));
}

void DecoderKv::read(int layer, bool v, int B, int L, float *out) const {
    VOX_CHECK(!ring, VOX_EINVAL, "'kv_%c%d': not on ring-indexed sessions", v ? 'v' : 'k', layer);
    std::vector<int> pt((size_t)B * max_pages);
    CUDA_OK(cudaMemcpy(pt.data(), table, sizeof(int) * pt.size(), cudaMemcpyDeviceToHost));
    std::vector<unsigned char> bytes(layer_bytes());
    CUDA_OK(cudaMemcpy(bytes.data(), pool(v, layer), bytes.size(), cudaMemcpyDeviceToHost));
    const size_t unit_bytes = kv_unit_bytes(type_, hd);
    size_t o = 0;
    for (int b = 0; b < B; ++b)
        for (int j = 0; j < L; ++j)
            for (int h = 0; h < Hkv; ++h) {
                const unsigned char *unit = bytes.data() + ((size_t)pt[(size_t)b * max_pages + j / KV_PAGE] * Hkv + h) * unit_bytes;
                const int r = j % KV_PAGE;
                if (type_ == KvType::Q8) {
                    const int8_t *q = reinterpret_cast<const int8_t *>(unit) + (size_t)r * hd;
                    const __half *d = reinterpret_cast<const __half *>(unit + (size_t)KV_PAGE * hd) + (size_t)r * (hd / KV_Q8_BLOCK);
                    for (int i = 0; i < hd; ++i, ++o) out[o] = kv_q8_decode_host(q[i], d[i / KV_Q8_BLOCK]);
                } else if (type_ == KvType::F16) {
                    const __half *f16 = reinterpret_cast<const __half *>(unit) + (size_t)r * hd;
                    for (int i = 0; i < hd; ++i, ++o) out[o] = __half2float(f16[i]);
                } else {
                    const float *f32 = reinterpret_cast<const float *>(unit) + (size_t)r * hd;
                    for (int i = 0; i < hd; ++i, ++o) out[o] = f32[i];
                }
            }
}

}  // namespace vox
