// kv_cache.h -- host side of the decoder KV cache (kv_cache.cu); the device format is kernels.h's KvView.
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "common.h"
#include "kernels.h"

namespace vox {

struct DeviceArena;

// A session's decoder KV cache: page pools [layers][n_pages][Hkv] of (page, kv head) units (kernels.h kv_unit_bytes: KV_PAGE
// positions x hd of `type`) for K and V, and a page table
// [rows][max_pages] of physical page ids.  Whole-utterance batches use the identity table (row b owns pages
// b * max_pages ..), which beams fork through; a stream pool gives its streams pages from a free list and binds them to
// the rows of each launch.  The element type is fixed for the cache's lifetime.
struct DecoderKv {
    // pools and table from `arena` (identity table uploaded), for `rows` rows.  Each row holds max(audio, launch) +
    // launch positions (room for the incremental API), where `audio` is the audio positions of a stream and `launch` the
    // positions one launch appends.  ring: each row's pages are a ring just long enough for the decoder window plus
    // `launch` (16 L > dec_window + launch), and positions are unbounded.
    void create(DeviceArena &arena, const vox_model_info &c, int rows, int audio, int launch, bool ring, KvType type);
    int capacity() const { return max_pages * KV_PAGE; }   // positions per row (ring: slots)
    KvType type() const { return type_; }
    // layer `layer` as the attention kernels see it, at the per-row positions `pos` (device [rows])
    KvView view(int layer, const int *pos) const;

    // beams: launch_beam_fork over rows [0, rows) (parent row src[r], positions pos), marking the table forked.  A
    // launch and nothing else, so that it may run under stream capture.
    void fork(const int *pos, const int *src, int rows, cudaStream_t st);
    void restore_identity(cudaStream_t st);   // re-uploads the identity table if a fork has rewritten it

    // stream pools: stream `stream` (a row index) holds pages for `positions` positions (a ring: at most max_pages),
    // taken from the free list, last freed first
    void reserve(int stream, int positions);
    void release(int stream);                 // its pages back to the free list
    int pages(int stream) const { return (int)owned[stream].size(); }
    // table rows [0, streams.size()) := the pages of streams[i], enqueued on st from a host copy that stays alive until
    // the next bind: the caller synchronises st before then
    void bind(const std::vector<int> &streams, cudaStream_t st);

    // debug read of rows [0, B) at positions [0, L): out is f32 [row][pos][kv_head][hd] of the V pools (v) or the K
    // pools.  Synchronous; refuses ring caches.
    void read(int layer, bool v, int B, int L, float *out) const;

  private:
    void *pool(bool v, int layer) const;   // base of one layer's K or V pool
    size_t layer_bytes() const { return (size_t)n_pages * Hkv * kv_unit_bytes(type_, hd); }

    KvType type_ = KvType::F32;
    bool ring = false;
    int layers = 0, Hkv = 0, hd = 0;
    int max_pages = 0, n_pages = 0;        // logical pages per row, physical pages per pool
    void *kc = nullptr, *vc = nullptr;
    int *table = nullptr;                  // device [rows][max_pages]
    std::vector<int> identity;             // host copy of the identity table
    bool forked = false;
    std::vector<int> free_list;            // stream pools: free pages, handed out from the back
    std::vector<std::vector<int>> owned;   // [rows] pages each stream holds, in logical order
    std::vector<int> staged;               // bind's host copy of the table rows
};

}  // namespace vox
