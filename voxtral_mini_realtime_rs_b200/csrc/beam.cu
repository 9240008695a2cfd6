// beam.cu -- beam search around the decode step (kernels.h launch_beam_select / launch_beam_fork /
// launch_beam_traceback).  The beams of a stream are rows of the batched step; the selection runs on the token-score
// kernel's per-row top-k, and a beam that changes rows takes its parent's KV history through the page table.
#include "kernels.h"

#include <cmath>

#include "common.h"

namespace vox {

void tc_count_launch(const char *name);   // kernels.cu: launch count + launch error check

// One CTA per stream.  Candidate t = j * W + i is the i-th entry of the top-k list of the row holding live rank j.
__global__ void __launch_bounds__(BEAM_MAX * BEAM_MAX)
beam_select_kernel(const int *__restrict__ top_ids, const float *__restrict__ top_lp, const int *__restrict__ out_pos,
                   int out_ld, int W, int n_live, BeamWork w, int *tok) {
    __shared__ double s_score[BEAM_MAX * BEAM_MAX], s_cum[BEAM_MAX];
    __shared__ int s_id[BEAM_MAX * BEAM_MAX];
    __shared__ int s_old_row[BEAM_MAX], s_par[BEAM_MAX], s_tok[BEAM_MAX], s_row[BEAM_MAX];
    const int s = blockIdx.x, t = threadIdx.x, nc = n_live * W;
    if (t < W) s_old_row[t] = w.rank_row[s * W + t];
    __syncthreads();
    if (t < nc) {
        const int j = t / W, q = s_old_row[j];
        const size_t at = ((size_t)q * out_ld + out_pos[q] - 1) * TOPK_MAX + t % W;
        const int id = top_ids[at];
        const float lp = top_lp[at];
        s_id[t] = id;
        // no id (fewer than W finite logits) or no finite log-probability: ranks after every real candidate
        s_score[t] = id < 0 || !(lp > -INFINITY) ? -INFINITY : w.cum[s * W + j] + (double)lp;
    }
    __syncthreads();
    if (t < nc) {
        // rank of t = candidates ordered before it: higher score, then lower parent rank, then lower id (-1 as unsigned
        // sorts last); the slot index makes the order total
        const double v = s_score[t];
        const int j = t / W;
        const unsigned id = (unsigned)s_id[t];
        int r = 0;
        for (int u = 0; u < nc; ++u) {
            const double x = s_score[u];
            const int ju = u / W;
            const unsigned iu = (unsigned)s_id[u];
            r += x > v || (x == v && (ju < j || (ju == j && (iu < id || (iu == id && u < t)))));
        }
        if (r < W) {
            s_par[r] = j;
            s_tok[r] = s_id[t] < 0 ? 0 : s_id[t];   // (an id-less pick still feeds an in-range embedding row)
            s_cum[r] = v;
        }
    }
    __syncthreads();
    if (t == 0) {
        // the first child of each surviving parent stays in the parent's row; the other children take the rows of the
        // ranks without children, in rank order.  So no row that is a fork source is overwritten by this fork.
        unsigned has = 0;
        for (int r = 0; r < W; ++r) {
            const int j = s_par[r];
            s_row[r] = (has >> j) & 1u ? -1 : s_old_row[j];
            has |= 1u << j;
        }
        int f = 0;
        for (int r = 0; r < W; ++r)
            if (s_row[r] < 0) {
                while ((has >> f) & 1u) ++f;
                s_row[r] = s_old_row[f++];
            }
    }
    __syncthreads();
    if (t < W) {
        const int R = s_row[t], q = s_old_row[s_par[t]];
        const size_t at = (size_t)R * out_ld + out_pos[R] - 1;
        w.rank_row[s * W + t] = R;
        w.cum[s * W + t] = s_cum[t];
        w.src[R] = q;
        w.hist_tok[at] = s_tok[t];
        w.hist_par[at] = q;
        tok[R] = s_tok[t];
    }
}

void launch_beam_select(const int *top_ids, const float *top_lp, const int *out_pos, int out_ld, int b, int W, int n_live,
                        const BeamWork &w, int *tok, cudaStream_t st) {
    beam_select_kernel<<<b, BEAM_MAX * BEAM_MAX, 0, st>>>(top_ids, top_lp, out_pos, out_ld, W, n_live, w, tok);
    tc_count_launch("beam_select");
}

// grid (rows, layers): a row whose beam came from another row q takes q's page-table entries of the full pages and a
// copy of the filled part of q's current page into its own current page.  Full pages are never written again (a row
// writes only its own page at the current logical index, which only grows), so sharing them is safe.
template <typename KV>
__global__ void __launch_bounds__(256)
beam_fork_kernel(KV *kc, KV *vc, size_t layer_stride, int *page_table, int max_pages, const int *__restrict__ pos,
                 const int *__restrict__ src, int Hkv, int hd) {
    const int row = blockIdx.x, layer = blockIdx.y, q = src[row];
    if (q == row) return;
    const int p = pos[row], c = p / KV_PAGE, rem = p % KV_PAGE;
    int *dst_pt = page_table + (size_t)row * max_pages;
    const int *src_pt = page_table + (size_t)q * max_pages;
    const int own = dst_pt[c], from = src_pt[c];   // entries >= c are not written by this launch
    if (layer == 0)
        for (int lp = threadIdx.x; lp < c; lp += blockDim.x) dst_pt[lp] = src_pt[lp];
    if (rem == 0) return;
    if constexpr (kv_type_of<KV>() == KvType::Q8) {
        // a (page, kv head) unit of layer_stride-byte layers: values [KV_PAGE][hd], then scales [KV_PAGE][hd / 16] f16;
        // positions [0, rem) are the first rem rows of each plane (values in 16-byte chunks, scales in 4-byte words)
        const size_t ub = kv_unit_bytes(KvType::Q8, hd);
        const int n16 = rem * hd / 16, n4 = rem * (hd / KV_Q8_BLOCK) / 2;
        for (int kv = 0; kv < 2; ++kv) {
            KV *base = (kv ? vc : kc) + (size_t)layer * layer_stride;
            for (int h = 0; h < Hkv; ++h) {
                const KV *s = base + ((size_t)from * Hkv + h) * ub;
                KV *d = base + ((size_t)own * Hkv + h) * ub;
                for (int i = threadIdx.x; i < n16; i += blockDim.x) reinterpret_cast<uint4 *>(d)[i] = reinterpret_cast<const uint4 *>(s)[i];
                for (int i = threadIdx.x; i < n4; i += blockDim.x)
                    reinterpret_cast<uint32_t *>(d + (size_t)KV_PAGE * hd)[i] = reinterpret_cast<const uint32_t *>(s + (size_t)KV_PAGE * hd)[i];
            }
        }
        return;
    }
    const int n4 = rem * hd / (16 / (int)sizeof(KV));   // 16-byte chunks: positions [0, rem) of one kv head are contiguous in a page
    for (int kv = 0; kv < 2; ++kv) {
        KV *base = (kv ? vc : kc) + (size_t)layer * layer_stride;
        for (int h = 0; h < Hkv; ++h) {
            const float4 *s4 = reinterpret_cast<const float4 *>(base + ((size_t)from * Hkv + h) * KV_PAGE * hd);
            float4 *d4 = reinterpret_cast<float4 *>(base + ((size_t)own * Hkv + h) * KV_PAGE * hd);
            for (int i = threadIdx.x; i < n4; i += blockDim.x) d4[i] = s4[i];
        }
    }
}

void launch_beam_fork(void *kc, void *vc, KvType type, size_t layer_bytes, int layers, int *page_table, int max_pages,
                      const int *pos, const int *src, int rows, int Hkv, int hd, cudaStream_t st) {
    if (type == KvType::Q8)
        beam_fork_kernel<int8_t><<<dim3(rows, layers), 256, 0, st>>>((int8_t *)kc, (int8_t *)vc, layer_bytes, page_table,
                                                                     max_pages, pos, src, Hkv, hd);
    else if (type == KvType::F16)
        beam_fork_kernel<__half><<<dim3(rows, layers), 256, 0, st>>>((__half *)kc, (__half *)vc, layer_bytes / 2, page_table,
                                                                     max_pages, pos, src, Hkv, hd);
    else
        beam_fork_kernel<float><<<dim3(rows, layers), 256, 0, st>>>((float *)kc, (float *)vc, layer_bytes / 4, page_table,
                                                                    max_pages, pos, src, Hkv, hd);
    tc_count_launch("beam_fork");
}

// One CTA per stream, lane r walks rank r's parent rows from the last position back to the first.  Lane 0 also writes
// the rank-0 ids into the stream's output row and gathers the scores of the distributions its tokens were chosen from
// into the stream's own score row (position i is read from another row at position i only, before the walk moves on
// to lower positions, so the gather runs in place).
__global__ void __launch_bounds__(32)
beam_traceback_kernel(BeamWork w, int W, int n, int out_ld, int *ids, double *scores, int *out, int *top_ids, float *top_lp,
                      int s0, int out_stride) {
    const int s = s0 + blockIdx.x, r = threadIdx.x;
    if (r >= W) return;
    int R = w.rank_row[s * W + r];
    int *dst = ids + ((size_t)blockIdx.x * W + r) * n;
    for (int i = n - 1; i >= 0; --i) {
        const size_t at = (size_t)R * out_ld + i;
        const int tk = w.hist_tok[at], q = w.hist_par[at];
        dst[i] = tk;
        if (r == 0) {
            const size_t o = (size_t)s * out_stride * out_ld + i;
            out[o] = tk;
            if (top_ids)
                for (int j = 0; j < TOPK_MAX; ++j) {
                    top_ids[o * TOPK_MAX + j] = top_ids[((size_t)q * out_ld + i) * TOPK_MAX + j];
                    top_lp[o * TOPK_MAX + j] = top_lp[((size_t)q * out_ld + i) * TOPK_MAX + j];
                }
        }
        R = q;
    }
    scores[s * W + r] = w.cum[s * W + r];
}

void launch_beam_traceback(const BeamWork &w, int b, int W, int n, int out_ld, int *ids, double *scores, int *out,
                           int *top_ids, float *top_lp, cudaStream_t st, int s0, int out_stride) {
    if (b <= 0) return;
    beam_traceback_kernel<<<b, 32, 0, st>>>(w, W, n, out_ld, ids, scores, out, top_ids, top_lp, s0, out_stride);
    tc_count_launch("beam_traceback");
}

}  // namespace vox
