// decode_mega.h -- op table of the persistent decode-step kernel (decode_mega.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "kernels.h"

namespace vox {

enum MegaKind : int {
    MG_EMBED = 0,   // x_dec[b] = audio of row b at pos[b] + dequant(E[tok[b]])  (+ sums of squares for the first norm)
    MG_MATVEC = 1,  // y = epi(norm?(x) . W^T), weights streamed through the CTA's TMA ring
    MG_ATTN = 2,    // GQA attention of one layer over its KV cache (key chunks combined by the last chunk's CTA)
    MG_ARGMAX = 3,  // combine the per-CTA lm_head candidates, write the token, advance the counters
};

// One grid-wide phase.  A grid barrier separates consecutive phases.
struct MegaOp {
    int kind = 0, epi = 0;
    // MG_MATVEC
    const uint4 *qs_tc = nullptr;
    const uint2 *d_tc = nullptr;
    int N = 0, K = 0, n_tiles = 0, n_pairs = 0;
    int S = 1, Ps = 0;  // CTA-private K slices: the activation fragments of one slice fit the scratch region
    // activation fragments (tensor-core B operands + per-block offsets, see decode_mega.cu) of the input,
    // written by the phase that produced the activations; bulk-copied into shared memory, never re-derived
    const uint2 *fin_bf = nullptr;    // [K/32 (+pad)][2][2*MT][4]
    const float2 *fin_off = nullptr;  // [K/32 (+pad)][MT]
    // fragments of this op's OUTPUT for the next matvec (nullptr: plain output only): one 32-value block per
    // unit of `unit_tiles` consecutive tiles (2: plain rows, 4: SiLU pairs), scaled by fout_gamma if set (or per row:
    // fout_ada_layer)
    uint2 *fout_bf = nullptr;
    float2 *fout_off = nullptr;
    const float *fout_gamma = nullptr;
    int unit_tiles = 1;
    float *y = nullptr;               // plain output (nullptr: fragments only)
    int ldy = 0;
    const float *bias = nullptr, *res = nullptr;
    const float *gamma = nullptr;   // fused RMSNorm weight (x ADA scale where the layer has one)
    const float *ssq_in = nullptr;  // [ssq_in_parts][B]
    int ssq_in_parts = 0;
    float *ssq_out = nullptr;       // [n_tiles][B]
    int track_argmax = 0;
    // MG_ATTN, and the layer's qkv MG_MATVEC, whose epilogue applies RoPE to the q and k rows and appends k and v
    KvPool kc, vc;   // this layer's KV page pools [n_pages][Hkv][KV_PAGE][hd] of MegaPlan::kv_bytes elements (kernels.h)
    int layer = 0;
    // MG_MATVEC whose output fragments take layer j's ffn_norm x ADA scale (wo): j, else -1.  Token b's fragments are
    // scaled by MegaParams::ffn_ada_rows[b] + j * D (fout_gamma is unset).
    int fout_ada_layer = -1;
};

struct MegaParams {
    const MegaOp *ops = nullptr;
    int n_ops = 0;
    int B = 0;  // streams (= token rows of every matvec)
    float eps = 0.f;
    // attention
    float *qkv = nullptr;
    int ld_qkv = 0, H = 0, Hkv = 0, hd = 0, max_seq = 0, window = 0;  // max_seq = max_pages * KV_PAGE
    const int *page_table = nullptr;  // [B][max_pages] physical KV pages of each batch row
    int max_pages = 0;
    float scale = 0.f;
    const float *cos_t = nullptr, *sin_t = nullptr;
    float *attn_out = nullptr;
    int attn_chunks = 1;          // key chunks per (stream, kv head): spreads the KV walk over the grid
    // chunk states as 8-byte words {value, tag}, tag = epoch * 64 + layer + 1 (unique per decode step and layer, never 0):
    float *att_acc = nullptr;     // [B*Hkv*chunks][G][hd][2] unnormalised weighted V per chunk
    float *att_ml = nullptr;      // [B*Hkv*chunks][G][2][2]  running max, sum of exp
    int *d_epoch = nullptr;       // decode steps executed by this session (never reset)
    // embedding (row-major planes of the tied table)
    const uint4 *emb_qs = nullptr;
    const __half *emb_d = nullptr;
    int D = 0;
    // audio embeddings (nullptr: none); row b's position p at audio + audio_off[b] + p * D (kernels.h launch_embed)
    const float *audio = nullptr;
    const int64_t *audio_off = nullptr;
    float *x_dec = nullptr, *ssq_x = nullptr;
    uint2 *emb_fbf = nullptr;         // fragments of the embedded row (x first layer's attn_norm) for layer 0
    float2 *emb_foff = nullptr;
    const float *emb_gamma = nullptr;
    uint2 *att_fbf = nullptr;         // fragments of the attention output (input of wo)
    float2 *att_foff = nullptr;
    // device-side step state; d_pos / d_outpos are PER ROW ([B]): sessions of different ages share a step
    int *d_pos = nullptr, *d_outpos = nullptr, *d_tok = nullptr, *d_out = nullptr;
    int out_ld = 0;
    // per-CTA argmax candidates [grid][8]
    float *am_vals = nullptr;
    int *am_idx = nullptr;
    // grid barrier: [0] arrivals, [1] finished CTAs, [2] watchdog code
    unsigned *bar = nullptr;
    // shared-memory plan
    int nstage = 0, scratch_bytes = 0;
    // optional phase trace of CTA 0: 6 SM-clock stamps per op (start, staged, body done, barrier passed,
    // first weights ready | KV walked, last weight stage consumed)
    unsigned long long *trace = nullptr;
    // optional all-CTA trace [grid][n_ops][4]: op start, body done, barrier passed, first weights ready / KV walk
    // start (SM clocks; the host aligns the CTAs on their exit from the first grid barrier)
    unsigned long long *trace_all = nullptr;
    float *logits_out = nullptr;  // != nullptr: where the lm_head op writes its rows (row groups of a larger batch)
    // sessions of an unbounded stream pool: page_table rows are rings of max_pages slots, positions are uncapped and
    // RoPE row of position pos is pos % rope_rows of cos_t / sin_t (kernels.h KvView, RopeView)
    int ring = 0;
    int rope_rows = 0;
    // [B]: each row's [L][D] ffn_norm x ADA set (the rows' streams may be at different transcription delays)
    const float *const *ffn_ada_rows = nullptr;
};

struct MegaPlan {
    int MT = 0;             // token capacity of the instantiation (1, 2, 4, 8)
    int Ps_cap = 0;         // pairs per K slice that fit the scratch region
    int scratch_bytes = 0;
    int nstage = 0;
    int attn_tile = 0;      // keys per K/V tile of the attention phase (what the scratch region holds)
    int kv_bytes = 4;       // KV cache element: 4 (f32) or 2 (f16); selects the kernel instantiation
    size_t smem_bytes = 0;
};

// Shapes the persistent kernel is instantiated for.
bool decode_mega_supported(int B, int H, int Hkv, int hd);
// Shared-memory plan for B streams given the largest K (in block pairs) of any matvec of the step and the KV cache's
// element size in bytes (4: f32, 2: f16).
MegaPlan decode_mega_plan(int B, int max_pairs, int H, int Hkv, int hd, int kv_bytes);
int decode_mega_grid(int device);
void launch_decode_mega(const MegaParams &p, const MegaPlan &plan, int grid, cudaStream_t st);

}  // namespace vox
