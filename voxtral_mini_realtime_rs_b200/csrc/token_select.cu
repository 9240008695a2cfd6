// token_select.cu -- host side of token selection: options, lazily allocated device state, the launches after every
// step, beam start-up and traceback, and the results record with its reads.  The only host code that knows the score
// buffers' layout [row][out_ld][TOPK_MAX].
#include "token_select.h"

#include <algorithm>
#include <cmath>

#include "model.h"

namespace vox {

static_assert(BEAM_MAX <= TOPK_MAX, "a beam's candidates are the first W entries of its row's top-k list");

void TokenSelect::create(DeviceArena &arena_, int device_, int max_batch_, int out_ld_, int vocab_) {
    arena = &arena_;
    device = device_;
    max_batch = max_batch_;
    out_ld = out_ld_;
    vocab = vocab_;
    bias_n.assign(max_batch, 0);
}

void TokenSelect::set_top_k(int k) {
    VOX_CHECK(k >= 0 && k <= TOPK_MAX, VOX_EINVAL, "top_k %d out of range [0,%d]", k, TOPK_MAX);
    if (k > 0) alloc_scores();
    top_k = k;
}

void TokenSelect::alloc_scores() {
    if (d_top_ids) return;
    CUDA_OK(cudaSetDevice(device));
    const size_t n = (size_t)max_batch * out_ld * TOPK_MAX, parts = (size_t)max_batch * ARGMAX_PARTS;
    d_top_ids = arena->alloc_n<int>(n);
    d_top_lp = arena->alloc_n<float>(n);
    score_work.m = arena->alloc_n<float>(parts);
    score_work.l = arena->alloc_n<float>(parts);
    score_work.vals = arena->alloc_n<float>(parts * TOPK_MAX);
    score_work.idx = arena->alloc_n<int>(parts * TOPK_MAX);
    score_work.counters = arena->alloc_n<int>(max_batch);
    CUDA_OK(cudaMemset(score_work.counters, 0, sizeof(int) * max_batch));
}

void TokenSelect::set_beam(int w) {
    VOX_CHECK(w >= 1 && w <= BEAM_MAX, VOX_EINVAL, "beam width %d out of range [1,%d]", w, BEAM_MAX);
    if (w > 1 && !beam.rank_row) {
        alloc_scores();
        const size_t rows = max_batch, hist = (size_t)max_batch * out_ld;
        beam.rank_row = arena->alloc_n<int>(rows);
        beam.cum = arena->alloc_n<double>(rows);
        beam.src = arena->alloc_n<int>(rows);
        beam.hist_tok = arena->alloc_n<int>(hist);
        beam.hist_par = arena->alloc_n<int>(hist);
        d_nbest_ids = arena->alloc_n<int>(hist);   // b * W <= max_batch hypotheses of n <= out_ld ids
        d_nbest_scores = arena->alloc_n<double>(rows);
    }
    beam_w = w;
}

bool TokenSelect::set_bias(int stream, const int32_t *ids, const int32_t *lens, const float *boosts, int n, cudaStream_t st) {
    VOX_CHECK(stream >= -1 && stream < max_batch, VOX_EINVAL, "set_bias: stream %d out of range [0,%d) (or -1 for every stream)",
              stream, max_batch);
    VOX_CHECK(n >= 0 && n <= BIAS_MAX_PHRASES, VOX_EINVAL, "set_bias: %d phrases out of range [0,%d]", n, BIAS_MAX_PHRASES);
    VOX_CHECK(n == 0 || (ids && lens && boosts), VOX_EINVAL, "set_bias: NULL ids, lens or boosts with %d phrases", n);
    // phrase p is ids[off_p .. off_p + lens[p]), padded to BIAS_MAX_LEN ids in the device layout
    std::vector<int> packed((size_t)n * BIAS_MAX_LEN, 0), hist(BIAS_HIST + 1, 0);
    for (int p = 0, off = 0; p < n; off += lens[p], ++p) {
        VOX_CHECK(lens[p] >= 1 && lens[p] <= BIAS_MAX_LEN, VOX_EINVAL, "set_bias: phrase %d has %d ids (1..%d)", p, lens[p],
                  BIAS_MAX_LEN);
        VOX_CHECK(std::isfinite(boosts[p]) && boosts[p] > 0.0f, VOX_EINVAL, "set_bias: boost %g of phrase %d must be finite and > 0",
                  boosts[p], p);
        for (int j = 0; j < lens[p]; ++j) {
            const int t = ids[off + j];
            VOX_CHECK(t >= BIAS_FIRST_TEXT_ID && t < vocab, VOX_EINVAL, "set_bias: id %d of phrase %d outside [%d,%d)", t, p,
                      BIAS_FIRST_TEXT_ID, vocab);
            packed[(size_t)p * BIAS_MAX_LEN + j] = t;
        }
    }
    if (n == 0 && !bias.ids) return false;   // nothing was ever set: nothing to clear
    CUDA_OK(cudaSetDevice(device));
    const bool allocated = !bias.ids;
    if (allocated) {
        const size_t S = max_batch;
        bias.ids = arena->alloc_n<int>(S * BIAS_MAX_PHRASES * BIAS_MAX_LEN);
        bias.lens = arena->alloc_n<int>(S * BIAS_MAX_PHRASES);
        bias.boosts = arena->alloc_n<float>(S * BIAS_MAX_PHRASES);
        bias.n_phrases = arena->alloc_n<int>(S);
        bias.hist = arena->alloc_n<int>(S * (BIAS_HIST + 1));
        d_row_stream = arena->alloc_n<int>(S);
        CUDA_OK(cudaMemsetAsync(bias.n_phrases, 0, sizeof(int) * S, st));
        CUDA_OK(cudaMemsetAsync(bias.hist, 0, sizeof(int) * S * (BIAS_HIST + 1), st));
    }
    for (int s = stream < 0 ? 0 : stream; s < (stream < 0 ? max_batch : stream + 1); ++s) {
        const size_t p0 = (size_t)s * BIAS_MAX_PHRASES;
        if (n > 0) {
            CUDA_OK(cudaMemcpyAsync(bias.ids + p0 * BIAS_MAX_LEN, packed.data(), sizeof(int) * packed.size(), cudaMemcpyHostToDevice, st));
            CUDA_OK(cudaMemcpyAsync(bias.lens + p0, lens, sizeof(int) * n, cudaMemcpyHostToDevice, st));
            CUDA_OK(cudaMemcpyAsync(bias.boosts + p0, boosts, sizeof(float) * n, cudaMemcpyHostToDevice, st));
        }
        CUDA_OK(cudaMemcpyAsync(bias.n_phrases + s, &n, sizeof(int), cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaMemcpyAsync(bias.hist + (size_t)s * (BIAS_HIST + 1), hist.data(), sizeof(int) * hist.size(),
                                cudaMemcpyHostToDevice, st));
        bias_n[s] = n;
    }
    CUDA_OK(cudaStreamSynchronize(st));   // the staging vectors and the caller's buffers
    return allocated;
}

void TokenSelect::clear_bias_history(int stream, cudaStream_t st) {
    if (!bias.hist) return;
    const size_t per = BIAS_HIST + 1;
    if (stream < 0) CUDA_OK(cudaMemsetAsync(bias.hist, 0, sizeof(int) * max_batch * per, st));
    else CUDA_OK(cudaMemsetAsync(bias.hist + (size_t)stream * per, 0, sizeof(int) * per, st));
}

bool TokenSelect::bias_on() const { return std::any_of(bias_n.begin(), bias_n.end(), [](int n) { return n > 0; }); }

void TokenSelect::check_beam_bias() const {
    VOX_CHECK(beam_w == 1 || !bias_on(), VOX_EINVAL, "beam search (width %d) does not take phrase boosting: clear the bias lists",
              beam_w);
}

void TokenSelect::check_rows(int b) const {
    VOX_CHECK(beam_w == 1 || b * beam_w <= max_batch, VOX_EINVAL, "beam width %d x %d streams exceeds session max_batch %d",
              beam_w, b, max_batch);
}

void TokenSelect::check_greedy(const char *call) const {
    VOX_CHECK(beam_w == 1, VOX_EINVAL, "%s runs greedy only: the session's beam width is %d", call, beam_w);
}

void TokenSelect::bind_rows(const std::vector<int> &streams, cudaStream_t st) {
    if (d_row_stream)
        CUDA_OK(cudaMemcpyAsync(d_row_stream, streams.data(), sizeof(int) * streams.size(), cudaMemcpyHostToDevice, st));
}

// row b's scores land at its output position d_outpos[b] - 1
void TokenSelect::after_step(Session &s, int B) {
    if (bias_on()) launch_bias_select(s.logits, B, vocab, d_row_stream, bias, s.d_tok, s.d_out, out_ld, s.d_outpos, s.st);
    // at W > 1 every step belongs to a beam call (the incremental calls refuse to run), whose selection reads W candidates
    const int k = std::max(top_k, beam_w > 1 ? beam_w : 0);
    if (k > 0) launch_token_scores(s.logits, B, vocab, k, s.d_outpos, out_ld, d_top_ids, d_top_lp, score_work, s.st);
}

void TokenSelect::beam_begin(Session &s, const std::vector<int> &rank_row, int b) {
    CUDA_OK(cudaMemcpyAsync(beam.rank_row, rank_row.data(), sizeof(int) * rank_row.size(), cudaMemcpyHostToDevice, s.st));
    CUDA_OK(cudaMemsetAsync(beam.cum, 0, sizeof(double) * rank_row.size(), s.st));
    CUDA_OK(cudaStreamSynchronize(s.st));   // rank_row is the caller's
    beam_step(s, b, 1);
}

void TokenSelect::beam_step(Session &s, int b, int n_live) {
    launch_beam_select(d_top_ids, d_top_lp, s.d_outpos, out_ld, b, beam_w, n_live, beam, s.d_tok, s.st);
    s.kv.fork(s.d_pos, beam.src, b * beam_w, s.st);
}

void TokenSelect::traceback(Session &s, const int *n, int b, int out_stride) {
    const int W = beam_w;
    for (int i0 = 0, off = 0; i0 < b;) {
        int i1 = i0;
        while (i1 < b && n[i1] == n[i0]) ++i1;
        launch_beam_traceback(beam, i1 - i0, W, n[i0], out_ld, d_nbest_ids + off, d_nbest_scores, s.d_out,
                              top_k > 0 ? d_top_ids : nullptr, d_top_lp, s.st, i0, out_stride);
        off += (i1 - i0) * W * n[i0];
        i0 = i1;
    }
}

void TokenSelect::zero_nbest_scores(int s0, int s1, cudaStream_t st) {
    CUDA_OK(cudaMemsetAsync(d_nbest_scores + s0 * beam_w, 0, sizeof(double) * (s1 - s0) * beam_w, st));
}

void TokenSelect::record_step(int b, const int *pos0) {
    scores_k = top_k;
    scores_n = 1;
    score_spans.resize(b);
    for (int r = 0; r < b; ++r) score_spans[r] = {r, pos0[r], 1};
}

void TokenSelect::record_transcribe(int b, const int *order, const int *n_out, int row_stride, bool total) {
    const int W = beam_w;
    scores_k = top_k;
    nbest_w = W > 1 ? W : 0;
    score_spans.resize(b);
    nbest_spans.resize(b);
    int sum = 0;
    for (size_t i = 0, off = 0; i < (size_t)b; off += (size_t)W * n_out[order[i]], ++i) {
        const int s = order[i];
        score_spans[s] = {(int)i * row_stride, 0, n_out[s]};
        nbest_spans[s] = {off, (int)i * W, n_out[s]};
        sum += n_out[s];
    }
    scores_n = nbest_n = total ? sum : n_out[order[0]];
}

void TokenSelect::read_scores(int32_t *top_ids, float *top_lp, size_t cap, int32_t *b, int32_t *n, int32_t *k,
                              cudaStream_t st) const {
    const int K = scores_k;
    VOX_CHECK(K > 0, VOX_EINVAL, "no token scores: the last transcribe, prefill or decode step ran with top_k 0 (vox_session_set_top_k)");
    if (b) *b = (int32_t)score_spans.size();
    if (n) *n = scores_n;
    if (k) *k = K;
    if (!top_ids && !top_lp) return;
    VOX_CHECK(top_ids != nullptr, VOX_EINVAL, "null argument: top_ids");
    VOX_CHECK(top_lp != nullptr, VOX_EINVAL, "null argument: top_logprobs");
    size_t need = 0;
    for (const ScoreSpan &r : score_spans) need += (size_t)r.n * K;
    VOX_CHECK(cap >= need, VOX_ECAPACITY, "token scores capacity %zu < %zu", cap, need);
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaStreamSynchronize(st));
    // one stream after the other: entries [pos0, pos0 + n) of its row, the first K of each
    const size_t pitch = sizeof(int32_t) * TOPK_MAX;
    size_t dst = 0;
    for (const ScoreSpan &r : score_spans) {
        if (r.n == 0) continue;
        const size_t at = ((size_t)r.row * out_ld + r.pos0) * TOPK_MAX;
        CUDA_OK(cudaMemcpy2D(top_ids + dst, sizeof(int32_t) * K, d_top_ids + at, pitch, sizeof(int32_t) * K, r.n,
                             cudaMemcpyDeviceToHost));
        CUDA_OK(cudaMemcpy2D(top_lp + dst, sizeof(float) * K, d_top_lp + at, pitch, sizeof(float) * K, r.n,
                             cudaMemcpyDeviceToHost));
        dst += (size_t)r.n * K;
    }
}

void TokenSelect::read_nbest(int32_t *ids, double *scores, size_t cap, int32_t *b, int32_t *w, int32_t *n, cudaStream_t st) const {
    const int W = nbest_w;
    VOX_CHECK(W > 0, VOX_EINVAL, "no n-best list: the last transcribe ran at beam width 1 (vox_session_set_beam)");
    if (b) *b = (int32_t)nbest_spans.size();
    if (w) *w = W;
    if (n) *n = nbest_n;
    if (!ids && !scores) return;
    VOX_CHECK(ids != nullptr, VOX_EINVAL, "null argument: ids");
    VOX_CHECK(scores != nullptr, VOX_EINVAL, "null argument: scores");
    size_t need = 0;
    for (const NbestSpan &r : nbest_spans) need += (size_t)W * r.n;
    VOX_CHECK(cap >= need, VOX_ECAPACITY, "n-best capacity %zu < %zu", cap, need);
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaStreamSynchronize(st));
    // one stream after the other: its W hypotheses of n ids each, and its W scores
    for (const NbestSpan &r : nbest_spans) {
        if (r.n > 0) CUDA_OK(cudaMemcpy(ids, d_nbest_ids + r.ids, sizeof(int32_t) * W * r.n, cudaMemcpyDeviceToHost));
        CUDA_OK(cudaMemcpy(scores, d_nbest_scores + r.scores, sizeof(double) * W, cudaMemcpyDeviceToHost));
        ids += (size_t)W * r.n;
        scores += W;
    }
}

void TokenSelect::fetch_rows(int n, int32_t *top_ids, float *top_lp, cudaStream_t st) const {
    const int k = top_k;
    if (k == 0) return;
    const size_t row = (size_t)out_ld * TOPK_MAX;
    CUDA_OK(cudaMemcpy2DAsync(top_ids, sizeof(int32_t) * k, d_top_ids, sizeof(int32_t) * row, sizeof(int32_t) * k, n,
                              cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpy2DAsync(top_lp, sizeof(float) * k, d_top_lp, sizeof(float) * row, sizeof(float) * k, n,
                              cudaMemcpyDeviceToHost, st));
}

}  // namespace vox
