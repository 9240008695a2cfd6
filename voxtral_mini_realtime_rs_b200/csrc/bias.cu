// bias.cu -- phrase boosting after the decode step's argmax (kernels.h launch_bias_select).
// Every boost is positive, so the argmax of the boosted logits is either the greedy id a or an id the list offers: an
// unboosted u has logit(u) <= logit(a), and a < u on equality.  The kernel compares a with the offered ids only and never
// sweeps the vocabulary.
#include "kernels.h"

#include <climits>
#include <cmath>

#include "common.h"

namespace vox {

void tc_count_launch(const char *name);   // kernels.cu: launch count + launch error check

constexpr int BIAS_THREADS = 256;
static_assert(BIAS_THREADS >= BIAS_HIST, "one thread per history entry stages the history");

// the greedy argmax's order: the larger value, the lower id on equal values
__device__ __forceinline__ void bias_combine(float &bv, int &bx, float ov, int ox) {
    if (ov > bv || (ov == bv && ox < bx)) { bv = ov; bx = ox; }
}

// One CTA per row.  Thread i takes phrases i, i + BIAS_THREADS, ...; for each j <= min(len - 1, |h|) whose prefix
// phrase[0..j) equals the last j ids of the history it proposes (fl32(logit[phrase[j]] + boost), phrase[j]).
__global__ void __launch_bounds__(BIAS_THREADS)
bias_select_kernel(const float *__restrict__ logits, int V, const int *__restrict__ row_stream, BiasLists bl, int *tok,
                   int *out_ids, int out_ld, const int *__restrict__ out_pos) {
    __shared__ int s_hist[BIAS_HIST];
    __shared__ float s_v[BIAS_THREADS / 32];
    __shared__ int s_i[BIAS_THREADS / 32];
    const int r = blockIdx.x, s = row_stream[r];
    const int n = bl.n_phrases[s];
    if (n == 0) return;
    int *hist = bl.hist + (size_t)s * (BIAS_HIST + 1);
    const int hn = hist[BIAS_HIST];
    if (threadIdx.x < hn) s_hist[threadIdx.x] = hist[threadIdx.x];
    __syncthreads();
    const float *row = logits + (size_t)r * V;
    float best = -INFINITY;
    int bi = INT_MAX;
    if (threadIdx.x == 0) {   // the greedy id at its own value (a NaN row ranks like -inf, as in the argmax)
        bi = tok[r];
        const float la = row[bi];
        best = isnan(la) ? -INFINITY : la;
    }
    for (int i = threadIdx.x; i < n; i += BIAS_THREADS) {
        const size_t p = (size_t)s * BIAS_MAX_PHRASES + i;
        const int *ph = bl.ids + p * BIAS_MAX_LEN;
        const int jmax = min(bl.lens[p] - 1, hn);
        const float beta = bl.boosts[p];
        for (int j = 0; j <= jmax; ++j) {
            bool match = true;
            for (int q = 0; q < j && match; ++q) match = s_hist[hn - j + q] == ph[q];
            if (match) {
                const int t = ph[j];
                bias_combine(best, bi, __fadd_rn(row[t], beta), t);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        bias_combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { s_v[warp] = best; s_i[warp] = bi; }
    __syncthreads();
    if (warp != 0) return;
    best = lane < BIAS_THREADS / 32 ? s_v[lane] : -INFINITY;
    bi = lane < BIAS_THREADS / 32 ? s_i[lane] : INT_MAX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        bias_combine(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
    if (lane != 0) return;
    tok[r] = bi;
    out_ids[(size_t)r * out_ld + out_pos[r] - 1] = bi;
    if (bi >= BIAS_FIRST_TEXT_ID) {   // keep the last BIAS_HIST text ids
        if (hn < BIAS_HIST) {
            hist[hn] = bi;
            hist[BIAS_HIST] = hn + 1;
        } else {
            for (int q = 1; q < BIAS_HIST; ++q) hist[q - 1] = s_hist[q];
            hist[BIAS_HIST - 1] = bi;
        }
    }
}

void launch_bias_select(const float *logits, int B, int V, const int *row_stream, const BiasLists &lists, int *tok, int *out_ids,
                        int out_ld, const int *out_pos, cudaStream_t st) {
    bias_select_kernel<<<B, BIAS_THREADS, 0, st>>>(logits, V, row_stream, lists, tok, out_ids, out_ld, out_pos);
    tc_count_launch("bias_select");
}

}  // namespace vox
