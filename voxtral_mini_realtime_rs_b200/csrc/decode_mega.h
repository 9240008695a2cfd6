// decode_mega.h -- host side of the persistent decode-step kernel (decode_mega.cu).
#pragma once
#include <cuda_runtime.h>

#include <array>
#include <memory>
#include <vector>

namespace vox {

struct Session;

// The kernel's op table, shared-memory plan, scratch, launches and step epoch.  The op format and the scratch layout
// are private to decode_mega.cu.
struct DecodeMega {
    DecodeMega();
    ~DecodeMega();
    // allocates the kernel's state from s.arena, once the session's decoder buffers exist
    void create(Session &s);
    // the op table for a step over R rows, built when the group size changes (a copy and a synchronisation of s.st).
    // Returns the step's launches, one per group of at most 8 rows; 0 when the kernel is not instantiated for the model.
    unsigned prepare(const Session &s, int R);
    // the step over rows [0, R) on s.st, after prepare(s, R)
    void step(const Session &s, int R, bool add_audio);
    void rebase_epoch(cudaStream_t st);   // once the epoch has advanced far (Session::reset)

    // launches executed since the epoch was last re-based: step() counts its own unless `capturing`; a graph replay
    // adds its captured step's launches
    unsigned launches = 0;
    bool capturing = false;
    // per launch of the last step issued or captured (debug "mega_attn"): {rows, token capacity MT, keys per K/V tile,
    // key chunks per (stream, kv head)}; the session empties it after a per-op step
    std::vector<std::array<int, 4>> attn_log;
    // debug reads: the device epoch, SM-clock stamps of CTA 0 [n_ops][6] and of every CTA [grid][n_ops][4] (nullptr
    // unless VOX_MEGA_TRACE_ALL=1 at session creation)
    int grid = 0, n_ops = 0;
    int *epoch = nullptr;
    unsigned long long *trace = nullptr, *trace_all = nullptr;

  private:
    struct State;
    std::unique_ptr<State> state;
};

}  // namespace vox
