// token_select.h -- host side of what happens to a step's logits after its argmax (token_select.cu): token scores (K9),
// beam search (K10), phrase boosting (K11), and the record of where the last call's scores and n-best lists are.  The
// device formats are kernels.h's ScoreWork, BeamWork and BiasLists.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <vector>

#include "kernels.h"

namespace vox {

struct DeviceArena;
struct Session;

// A session's token selection.  Its device state is allocated from the session's arena on first use and kept: the
// score buffers by the first set_top_k(k > 0) or set_beam(W > 1), the beam state and n-best results by the first
// set_beam(W > 1), the phrase lists and the row table by the first non-empty list.
struct TokenSelect {
    // for a session of max_batch rows of out_ld output positions over `vocab` ids, on `device`; allocates nothing
    void create(DeviceArena &arena, int device, int max_batch, int out_ld, int vocab);

    // ---- options and their checks (every argument is checked before anything changes)
    // token confidences: 0 = off (no launch, no memory).  k > 0: every prefill and decode step ends with
    // launch_token_scores over its rows into the score buffers, [max_batch][out_ld][TOPK_MAX] ids / log-probabilities
    void set_top_k(int k);
    // beam search: W beams per stream for the transcribe calls; 1 = greedy (no launch, no memory).  A call over b streams
    // at W > 1 runs b * W rows (kernels.h BeamWork)
    void set_beam(int w);
    // phrase boosting: stream's list (-1: every stream's) := the n phrases of ids / lens / boosts, its history cleared.
    // Returns true when this call allocated the lists and the row table, which the next binding of rows must then fill
    // (bind_rows).  While some stream has a list, every prefill and decode step ends with one launch_bias_select.
    bool set_bias(int stream, const int32_t *ids, const int32_t *lens, const float *boosts, int n, cudaStream_t st);
    void clear_bias_history(int stream, cudaStream_t st);   // -1: every stream's
    bool bias_on() const;
    void check_beam_bias() const;    // a beam transcribe call with a list set is refused
    void check_rows(int b) const;    // b streams of W beam rows each fit the session's rows
    void check_greedy(const char *call) const;   // the incremental calls run at beam width 1 only

    // ---- device work on the session's stream
    // the row table's rows [0, streams.size()) := streams (the stream of each row), when the table exists; enqueued from
    // `streams`, which the caller keeps alive until st has synchronised
    void bind_rows(const std::vector<int> &streams, cudaStream_t st);
    // after the argmax and counter advance of the prefill or decode step over rows [0, B) that just ran: launch_bias_select
    // (while some stream has a list), then launch_token_scores at k = max(top_k, W when W > 1) (when k > 0)
    void after_step(Session &s, int B);
    // the first beam selection, after the prefill of b streams: rank_row[i] is the row holding rank i (b * W of them),
    // every rank at score 0, one live rank per stream
    void beam_begin(Session &s, const std::vector<int> &rank_row, int b);
    // selection + KV fork after a step over the b * W beam rows, with n_live live ranks per stream
    void beam_step(Session &s, int b, int n_live);
    // the n-best lists of streams [0, b) taken in order, stream i with n[i] outputs (non-increasing): one traceback per
    // run of equal counts, stream i's rank-0 ids and token scores into row i * out_stride, its W hypotheses packed after
    // those of stream i - 1, its scores at i * W
    void traceback(Session &s, const int *n, int b, int out_stride);
    void zero_nbest_scores(int s0, int s1, cudaStream_t st);   // streams [s0, s1) have no output: scores 0

    // ---- the results record of the last call
    // an incremental prefill or decode step over rows [0, b): row r's one output at position pos0[r]
    void record_step(int b, const int *pos0);
    // a transcribe call over b streams: its i-th stream order[i] has n_out[order[i]] outputs in row i * row_stride
    // (from position 0), and the i-th n-best list as traceback() packs it.  The counts the getters report are per
    // stream, or the total over the streams (`total`, a ragged call)
    void record_transcribe(int b, const int *order, const int *n_out, int row_stride, bool total);
    // vox_session_token_scores / vox_session_nbest: the counts, and when the arrays are given, the record's entries one
    // stream after the other (synchronous)
    void read_scores(int32_t *top_ids, float *top_lp, size_t cap, int32_t *b, int32_t *n, int32_t *k, cudaStream_t st) const;
    void read_nbest(int32_t *ids, double *scores, size_t cap, int32_t *b, int32_t *w, int32_t *n, cudaStream_t st) const;
    // enqueues the copy of the scores at position 0 of rows [0, n) into [n][top_k] host arrays (a stream pool's step)
    void fetch_rows(int n, int32_t *top_ids, float *top_lp, cudaStream_t st) const;

    int top_k = 0;
    int beam_w = 1;
    std::vector<int> bias_n;   // phrases per stream

  private:
    void alloc_scores();

    DeviceArena *arena = nullptr;
    int device = 0, max_batch = 0, out_ld = 0, vocab = 0;
    int *d_top_ids = nullptr;
    float *d_top_lp = nullptr;
    ScoreWork score_work;
    BeamWork beam;
    int *d_nbest_ids = nullptr;      // every stream's [W][n] ids of the last transcribe, at NbestSpan::ids
    double *d_nbest_scores = nullptr;
    BiasLists bias;
    int *d_row_stream = nullptr;     // [max_batch]
    // Where the results of the last call are, per stream in the caller's order (the buffers outlive reset()).  Token
    // scores, of the last transcribe or incremental call: entries [pos0, pos0 + n) of row `row`, scored with k =
    // scores_k (0: that call ran with scores off).  N-best lists, of the last transcribe: W x n ids at d_nbest_ids + ids,
    // W scores at d_nbest_scores + scores (nbest_w == 0: that transcribe ran greedy).  scores_n / nbest_n are the counts
    // the getters report.
    struct ScoreSpan { int row, pos0, n; };
    struct NbestSpan { size_t ids; int scores, n; };
    std::vector<ScoreSpan> score_spans;
    std::vector<NbestSpan> nbest_spans;
    int scores_k = 0, scores_n = 0, nbest_w = 0, nbest_n = 0;
};

}  // namespace vox
