// decode_mega.cu -- one autoregressive decode step for B <= 8 streams as ONE persistent kernel
// (reference src/gguf/model.rs:938-960 generate_step: embed(prev token) + audio[pos], 26 decoder
// layers forward_with_cache (model.rs:125-197, 250-255, 665-677), tied lm_head (680-691), argmax).
//
// Why: as separate launches the step is 134 dependent kernels whose weight streams each last only a
// few microseconds: launch gaps, per-kernel activation staging and CTA-wide barriers dominate.  Here one CTA per SM lives for the whole step:
//
//   * 20 warps in three roles: 16 consumer warps (the weight stream's arithmetic, attention, embedding), and one
//     warpgroup of helpers: the producer warp and 3 epilogue warps.  The launch gives every thread 96 registers;
//     setmaxnreg moves the helpers' surplus to the consumers (64 / 104).  Spills are poison here: 227 KB of the SM's 256 KB
//     are shared memory, there is no L1 left to catch local-memory traffic, every reload is an L2 round trip.
//   * The producer thread walks the step's entire weight schedule (every matvec of every layer, in order) and streams
//     this CTA's share through a ring of TMA bulk-copy stages (16 block pairs = 9 KB per tile, full/empty mbarriers).  It
//     never waits for activations, so the HBM stream runs ahead across op boundaries: while the consumers sit in a grid
//     barrier or stage the next op's activations, the ring (90-180 KB) keeps filling.
//   * a phase (op) = embed | matvec | attention | argmax; consecutive phases are separated by a grid barrier (one atomic
//     arrival per CTA, acquire spin by one thread).
//   * matvec arithmetic is matvec_tc.cu's: Q4 nibbles enter mma.sync.m16n8k16 as f16 subnormals, activations as per-block
//     power-of-two scaled f16 hi+mid pieces, the block scale d applied to the f32 block sum (shader.wgsl:96-127
//     re-associated).  A CTA owns whole 16-row tiles (tile = cta, cta+grid, ...): the 16 consumer warps take one block pair
//     each of every stage; their partial sums of a tile group go to shared memory (double-buffered) and are handed to the
//     epilogue warps through named arrive/wait barriers -- the consumers go straight on to the next group's stream.  The
//     epilogue warps add the 16 partials in fixed tree order and run the epilogue (bias / residual + sums of squares for the
//     next fused RMSNorm / SiLU*up / running argmax / activation fragments of the next matvec) => no atomics, no split-K
//     scratch, bitwise deterministic.  When the activation fragments of all of K do not fit shared memory (M > 2 and
//     K > 3072) the CTA walks K in private slices and keeps tile sums in shared memory.
//   * attention: RoPE + KV append + GQA as in decode_attn.cu, one CTA per (stream, kv head, key chunk); the chunks' softmax
//     states travel as 8-byte {value, (step, layer) tag} words that the merging CTA polls directly.
//
// All activations written by other CTAs are read with ld.global.cg (L1 is not coherent).
// Every spin loop has a watchdog that traps instead of hanging the GPU.
#include <cuda_fp16.h>

#include <cfloat>
#include <cstdlib>

#include "common.h"
#include "decode_mega.h"
#include "kernels.h"

namespace vox {

void tc_count_launch(const char *name);

namespace {

inline void cuda_check_mg(cudaError_t e, const char *what) {
    if (e != cudaSuccess) fail(VOX_ECUDA, fmt("CUDA error: %s: %s", what, cudaGetErrorString(e)));
}

constexpr int MG_CWARPS = 16;                    // consumer warps
constexpr int MG_CTHREADS = MG_CWARPS * 32;
// + the helpers' warpgroup: warp 16 is the producer, warps 17-19 run the matvec epilogues; the warpgroup hands a third of
// its registers to the consumers (setmaxnreg works on whole warpgroups of 4 warps).  The register file is allocated in
// units of 4 warps anyway: 17 warps cost as many registers as 20.
constexpr int MG_THREADS = MG_CTHREADS + 128;
constexpr int MG_REGS_CONSUMER = 104;            // 16 x 32 x (104 - 96) = 4096 registers moved ...
constexpr int MG_REGS_PRODUCER = 64;             // ... from the producer / epilogue warpgroup: 4 x 32 x (96 - 64) = 4096
constexpr int MG_EWARPS = 3;                     // epilogue warps (17..19)
constexpr int MG_ETHREADS = MG_EWARPS * 32;
constexpr int MG_ATHREADS = MG_CTHREADS + MG_ETHREADS;  // consumers + epilogue warps (the producer joins no barrier)
// named barriers: 1 consumers (512), 2 epilogue warps (96), 3 consumers + epilogue warps (phase ends), 4/5 partial sums of
// the group in red[0/1] complete (consumers arrive, epilogue warps wait), 6/7 red[0/1] read (the other way round)
constexpr int MG_BAR_FULL = 4, MG_BAR_FREE = 6;
constexpr int MG_CHUNK = 16;                     // block pairs per ring stage (one per consumer warp)
constexpr int MG_SLOT_Q = MG_CHUNK * 512;        // nibble bytes of one tile's part of a stage; its scales follow
constexpr int MG_SLOT_BYTES = MG_CHUNK * 576;    // a stage holds NT such slots (NT tiles advance together)
constexpr int MG_MAX_STAGES = 24;
constexpr int MG_ACC_TILES = 2;                  // tiles per CTA whose sums may persist across K slices
constexpr int MG_SMEM_MAX = 227 * 1024;
constexpr int MG_SCRATCH_CAP = 104448;           // 48 pairs at 8 tokens
constexpr long long MG_SPIN_CYCLES = 4000000000ll;  // ~2 s: watchdog

// tiles a CTA advances together (independent accumulation chains per warp, shared activation fragments)
__host__ __device__ constexpr int mg_nt(int MT) { return MT <= 2 ? 4 : 2; }
// epilogue outputs waiting to become fragments: up to two 32-value blocks x MT tokens per tile group
__host__ __device__ constexpr int mg_vals(int MT) { return (MT <= 2 ? 2 : 1) * 32 * MT; }
static_assert(mg_vals(1) >= 2 * mg_nt(1) * 1 && mg_vals(2) >= 2 * mg_nt(2) * 2 && mg_vals(4) >= 2 * mg_nt(4) * 4 &&
                  mg_vals(8) >= 2 * mg_nt(8) * 8,
              "vals also holds the lm_head phase's per-slot argmax candidates");
// barriers + rinv + rpart[4][8] + stgc[4] + red[2][16 warps][NT*16*MT] + acc_tile[MG_ACC_TILES][16*MT] + vals
__host__ __device__ constexpr int mg_misc_bytes(int MT) {
    return ((592 + 2048 * mg_nt(MT) * MT + 64 * MG_ACC_TILES * MT + 4 * mg_vals(MT) + 256) + 127) & ~127;  // + s_op
}
__host__ __device__ constexpr int mg_pair_bytes(int MT) { return 272 * MT; }  // fragments + offsets of one block pair

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __noinline__ void mg_die(unsigned *flag, unsigned code) {
    atomicExch(flag, code);
    __threadfence_system();
    __trap();
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity, unsigned *flag, unsigned code) {
    if (mbar_try(bar, parity)) return;
    const long long t0 = clock64();
    unsigned n = 0;
    while (!mbar_try(bar, parity)) {
        if ((++n & 0x3FFFu) == 0 && clock64() - t0 > MG_SPIN_CYCLES) mg_die(flag, code);
    }
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned *p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// A float published together with its validity tag in ONE 8-byte word (single-copy atomic): the reader polls the word
// itself -- no flag, no fence, no second round trip.
__device__ __forceinline__ void st_tagged(float2 *p, const float v, const int tag) {
    asm volatile("st.relaxed.gpu.global.v2.f32 [%0], {%1, %2};\n" ::"l"(p), "f"(v), "f"(__int_as_float(tag)) : "memory");
}
__device__ __forceinline__ float2 ld_tagged(const float2 *p) {
    float2 v;
    asm volatile("ld.relaxed.gpu.global.v2.f32 {%0, %1}, [%2];\n" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_add(unsigned *p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void prefetch_l1(const void *p) { asm volatile("prefetch.global.L1 [%0];\n" ::"l"(p)); }
// L2 prefetch of a byte range (16-byte multiple)
__device__ __forceinline__ void bulk_prefetch_l2(const void *p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;\n" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
        : "memory");
}
// barrier among the 512 consumer threads (the producer warp never joins)
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, 512;\n" ::: "memory"); }
// barrier among the epilogue warps
__device__ __forceinline__ void ebar() { asm volatile("bar.sync 2, %0;\n" ::"n"(MG_ETHREADS) : "memory"); }
// consumers + epilogue warps
__device__ __forceinline__ void abar() { asm volatile("bar.sync 3, %0;\n" ::"n"(MG_ATHREADS) : "memory"); }
// producer/consumer hand-off on barrier `id` (MG_ATHREADS participants: one side arrives, the other waits)
// (`publish`: the arriving thread's shared-memory stores must be visible to the waiting side.  Not __threadfence_block():
// that compiles to MEMBAR.SC, which on the epilogue warps waited for their outstanding GLOBAL stores -- an L2 round trip per
// tile group.)
__device__ __forceinline__ void hbar_arrive(const int id, const bool publish) {
    if (publish) asm volatile("fence.acq_rel.cta;\n" ::: "memory");
    asm volatile("bar.arrive %0, %1;\n" ::"r"(id), "n"(MG_ATHREADS) : "memory");
}
__device__ __forceinline__ void hbar_sync(const int id) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "n"(MG_ATHREADS) : "memory"); }

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t a0, const uint32_t a1, const uint32_t a2,
                                         const uint32_t a3, const uint32_t b0, const uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}
// The CTA's tile list of a matvec: units of UT consecutive tiles dealt round-robin to the CTAs
// (UT = 1: plain interleaving).  n_tiles % UT == 0 (host-checked).
__device__ __forceinline__ int mg_tile_count(const int n_tiles, const int UT, const int cta, const int nctas) {
    const int n_units = n_tiles / UT;
    return cta < n_units ? ((n_units - cta + nctas - 1) / nctas) * UT : 0;
}
__device__ __forceinline__ int mg_tile_of(const int i, const int UT, const int cta, const int nctas) {
    return (cta + (i / UT) * nctas) * UT + (i % UT);
}
// exp for the decoder attention's softmax: ex2.approx(x * log2 e) (2 instructions; the full-range expf is ~25 and
// made a one-key-per-warp KV walk cost 3.3 us).  Relative error <= ~|x| * 2^-23: far below the 1e-3 parity bound,
// and the reference's own softmax runs WGSL exp on the GPU.
__device__ __forceinline__ float fast_exp(const float x) { return __expf(x); }
__device__ __forceinline__ void amax_combine(float &bv, int &bx, const float ov, const int ox) {
    if (ov > bv || (ov == bv && ox < bx)) { bv = ov; bx = ox; }
}

// Fused RMSNorm: `gamma` is the norm weight, for the FFN norm pre-multiplied by the session's ADA scale
// (1 + w2.gelu(w0.t), constant per session; Session::set_delay).  The per-token factor 1/rms is a scalar
// of the whole row, so it is applied to the finished dot product in the epilogue
// (y = rinv * sum w*(x*gamma)) instead of to every activation: the staging pass then does not wait
// for the row statistics.
__device__ __forceinline__ float4 mul4(const float4 a, const float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }

// Activation fragments of one 32-element block for one token (same encoding as matvec_tc.cu tc_stage):
//   bf_blk  : uint2  [2 (nibble half j)][2*MT cols][4 t]   B fragments {b0,b1} of lane (g = col, t);
//             column 2*m = f16 hi piece of token m, 2*m+1 = mid piece            (MT <= 4)
//             uint2  [2 (piece: hi, mid)][32 lanes = (token m, t)][2 (nibble half j)]   (MT == 8: the columns of
//             the MMA are the 8 tokens; hi and mid pieces are chained into one accumulator)
//   off_blk : float2 [MT]   { -8 * sum_{k in block} x , 2^24 / block scale }
// One work item = (token m, t): elements 4t..4t+3 (l) and 16+4t..16+4t+3 (h) of the block, already
// multiplied by the consumer's norm weight.  The four t-items of a block must sit in four adjacent
// lanes (t = lane & 3) and all 32 lanes must call (inactive ones with act = false): block sum and
// block max are 2-step shuffles.
template <int MT>
__device__ __forceinline__ void frag_build(const float4 l, const float4 h, const bool act, const int t, const int m,
                                           uint2 *__restrict__ bf_blk, float2 *__restrict__ off_blk) {
    float bs = ((l.x + l.y) + (l.z + l.w)) + ((h.x + h.y) + (h.z + h.w));
    float bm = fmaxf(fmaxf(fmaxf(fabsf(l.x), fabsf(l.y)), fmaxf(fabsf(l.z), fabsf(l.w))),
                     fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fmaxf(fabsf(h.z), fabsf(h.w))));
    bs += __shfl_xor_sync(0xffffffffu, bs, 1);
    bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 1));
    bs += __shfl_xor_sync(0xffffffffu, bs, 2);
    bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, 2));
    if (!act) return;
    int e = (int)((__float_as_uint(bm) >> 23) & 0xFF) - 127;
    if (!(bm > 0.0f) || bm > 3.0e38f) e = 7;  // all-zero (or non-finite) block: scale 1
    e = e < -100 ? -100 : (e > 100 ? 100 : e);
    const float s = __uint_as_float((uint32_t)(7 - e + 127) << 23);     // block max -> [2^7, 2^8)
    const float inv = __uint_as_float((uint32_t)(17 + e + 127) << 23);  // 2^24 / s
    const float ev[8] = {l.x * s, l.y * s, l.z * s, l.w * s,
                         h.x * s * 0.0625f, h.y * s * 0.0625f, h.z * s * 0.0625f, h.w * s * 0.0625f};
    float hh[8], md[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        hh[q] = __half2float(__float2half_rn(ev[q]));
        md[q] = ev[q] - hh[q];
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int o = 4 * j;
        uint2 fh, fm;
        fh.x = pack_h2(hh[o + 0], hh[o + 2]);
        fh.y = pack_h2(hh[o + 1], hh[o + 3]);
        fm.x = pack_h2(md[o + 0], md[o + 2]);
        fm.y = pack_h2(md[o + 1], md[o + 3]);
        if constexpr (MT == 8) {
            // token-column layout: [piece p][lane = m*4+t][j] -- a consumer lane (g = token, t) fetches its hi pieces of
            // both nibble halves with one 128-bit load and its mid pieces with another (no bank conflicts)
            bf_blk[((0 * 32 + m * 4 + t) * 2) + j] = fh;
            bf_blk[((1 * 32 + m * 4 + t) * 2) + j] = fm;
        } else {
            uint2 *dst = bf_blk + (size_t)j * (2 * MT) * 4;
            dst[(2 * m + 0) * 4 + t] = fh;
            dst[(2 * m + 1) * 4 + t] = fm;
        }
    }
    if (t == 0) off_blk[m] = make_float2(-8.0f * bs, inv);
}

// One block pair (64 k) of NTV tiles against the activation fragments: the arithmetic of matvec_tc.cu.  The nibbles of
// the two blocks enter m16n8k16 as f16 subnormals (low nibbles n * 2^-24, high nibbles n * 2^-20, whose activation
// pieces are pre-scaled by 1/16); the f32 block sum is scaled by 2^24 / (block scale), offset by -8 * sum(x) and
// multiplied by the row's f16 scale d.
//   MT <= 4: MMA columns = (token, piece) pairs; hi and mid land in neighbouring columns and are added in f32.
//   MT == 8: MMA columns = the 8 tokens; the hi and mid pieces of both nibble halves are chained into ONE accumulator
//            (4 MMAs per block and tile, 2 FFMA per output): each lane finishes rows g, g+8 x tokens 2t, 2t+1.
template <int MT, int NT, int NTV>
__device__ __forceinline__ void mg_pair(const unsigned char *__restrict__ sb, const uint32_t slot_q, const uint32_t slot_d,
                                        const uint2 *__restrict__ bfp, const float2 *__restrict__ ofp, const int g, const int t,
                                        const int lane, float (&acc)[NT][2 * ((MT + 3) / 4)], uint64_t *release) {
    constexpr int CG = (MT + 3) / 4;
    uint4 wq[NTV];
    uint2 wd[NTV];
#pragma unroll
    for (int u = 0; u < NTV; ++u) {
        wq[u] = *reinterpret_cast<const uint4 *>(sb + (size_t)u * MG_SLOT_BYTES + slot_q);
        wd[u] = *reinterpret_cast<const uint2 *>(sb + (size_t)u * MG_SLOT_BYTES + slot_d);
    }
    // the warp's share of the stage is in registers: hand the stage back to the producer BEFORE the arithmetic (the ring
    // is only a few stages deep at 8 tokens -- the refill latency, not the MMAs, then sets the pace)
    if (release != nullptr) {
        __syncwarp();
        if (lane == 0) mbar_arrive(release);
    }
#pragma unroll
    for (int bb = 0; bb < 2; ++bb) {
        if constexpr (MT == 8) {
            const uint4 *bq = reinterpret_cast<const uint4 *>(bfp + (size_t)bb * (16 * MT));
            const uint4 fh = bq[lane], fm = bq[32 + lane];  // {b0,b1} of the low-nibble half, {b0,b1} of the high-nibble half
            const float4 o = *reinterpret_cast<const float4 *>(ofp + bb * MT + 2 * t);  // {off, inv} of tokens 2t, 2t+1
            // the tiles' accumulation chains are interleaved MMA by MMA: a chained m16n8k16 waits ~33 cycles for its
            // predecessor, the asm statements keep their source order, and one chain after the other left the warp idle
            // for most of that latency
            uint32_t al[NTV][4], ah[NTV][4];
            float cc[NTV][4];
#pragma unroll
            for (int u = 0; u < NTV; ++u) {
                const uint32_t wg = bb ? wq[u].z : wq[u].x, wg8 = bb ? wq[u].w : wq[u].y;
                const uint32_t sg = wg >> 8, sg8 = wg8 >> 8;
                al[u][0] = wg & 0x000F000Fu; al[u][1] = wg8 & 0x000F000Fu; al[u][2] = sg & 0x000F000Fu; al[u][3] = sg8 & 0x000F000Fu;
                ah[u][0] = wg & 0x00F000F0u; ah[u][1] = wg8 & 0x00F000F0u; ah[u][2] = sg & 0x00F000F0u; ah[u][3] = sg8 & 0x00F000F0u;
                cc[u][0] = cc[u][1] = cc[u][2] = cc[u][3] = 0.f;
            }
#pragma unroll
            for (int u = 0; u < NTV; ++u) mma16816(cc[u], al[u][0], al[u][1], al[u][2], al[u][3], fh.x, fh.y);
#pragma unroll
            for (int u = 0; u < NTV; ++u) mma16816(cc[u], ah[u][0], ah[u][1], ah[u][2], ah[u][3], fh.z, fh.w);
#pragma unroll
            for (int u = 0; u < NTV; ++u) mma16816(cc[u], al[u][0], al[u][1], al[u][2], al[u][3], fm.x, fm.y);
#pragma unroll
            for (int u = 0; u < NTV; ++u) mma16816(cc[u], ah[u][0], ah[u][1], ah[u][2], ah[u][3], fm.z, fm.w);
#pragma unroll
            for (int u = 0; u < NTV; ++u) {
                const uint32_t dw = bb ? wd[u].y : wd[u].x;
                const float2 d = __half22float2(*reinterpret_cast<const __half2 *>(&dw));
                acc[u][0] = fmaf(d.x, fmaf(cc[u][0], o.y, o.x), acc[u][0]);
                acc[u][1] = fmaf(d.x, fmaf(cc[u][1], o.w, o.z), acc[u][1]);
                acc[u][2] = fmaf(d.y, fmaf(cc[u][2], o.y, o.x), acc[u][2]);
                acc[u][3] = fmaf(d.y, fmaf(cc[u][3], o.w, o.z), acc[u][3]);
            }
        } else {
            const uint2 *bfb = bfp + (size_t)(bb * 2) * (2 * MT) * 4;
            uint2 blo[CG], bhi[CG];
            float2 of[CG];
#pragma unroll
            for (int c = 0; c < CG; ++c) {
                const int col = c * 8 + g;
                blo[c] = make_uint2(0u, 0u);
                bhi[c] = blo[c];
                if (col < 2 * MT) {
                    blo[c] = bfb[col * 4 + t];
                    bhi[c] = bfb[(2 * MT + col) * 4 + t];
                }
                const int tok = c * 4 + t;
                of[c] = tok < MT ? ofp[bb * MT + tok] : make_float2(0.0f, 0.0f);
            }
#pragma unroll
            for (int u = 0; u < NTV; ++u) {
                const uint32_t wg = bb ? wq[u].z : wq[u].x, wg8 = bb ? wq[u].w : wq[u].y;
                const uint32_t dw = bb ? wd[u].y : wd[u].x;
                const float2 d = __half22float2(*reinterpret_cast<const __half2 *>(&dw));
                const uint32_t sg = wg >> 8, sg8 = wg8 >> 8;
#pragma unroll
                for (int c = 0; c < CG; ++c) {
                    float cc[4] = {0.f, 0.f, 0.f, 0.f};
                    mma16816(cc, wg & 0x000F000Fu, wg8 & 0x000F000Fu, sg & 0x000F000Fu, sg8 & 0x000F000Fu, blo[c].x, blo[c].y);
                    mma16816(cc, wg & 0x00F000F0u, wg8 & 0x00F000F0u, sg & 0x00F000F0u, sg8 & 0x00F000F0u, bhi[c].x, bhi[c].y);
                    acc[u][2 * c] = fmaf(d.x, fmaf(cc[0] + cc[1], of[c].y, of[c].x), acc[u][2 * c]);
                    acc[u][2 * c + 1] = fmaf(d.y, fmaf(cc[2] + cc[3], of[c].y, of[c].x), acc[u][2 * c + 1]);
                }
            }
        }
    }
}

template <int MT, int G, int DPL>
__global__ void __launch_bounds__(MG_THREADS, 1) decode_mega_kernel(const MegaParams p) {
    constexpr int CG = (MT + 3) / 4;
    constexpr int HD = DPL * 32;
    static_assert(G * HD <= MG_CTHREADS, "one attention output per consumer thread");
    constexpr int NT = mg_nt(MT);
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem);
    uint64_t *empty = full + MG_MAX_STAGES;
    float *rinv = reinterpret_cast<float *>(empty + MG_MAX_STAGES + 2);  // [8]
    float *rpart = rinv + 8;                                          // [4 warps][8 tokens] partial sums of squares
    uint64_t *stgc = reinterpret_cast<uint64_t *>(rpart + 32);        // [4] activation fragments of K chunk c landed in scratch
    float *red = reinterpret_cast<float *>(stgc + 4);                 // [2][MG_CWARPS][NT*16*MT]
    float *acc_tile = red + 2 * MG_CWARPS * NT * 16 * MT;             // [MG_ACC_TILES][16*MT]
    float *vals = acc_tile + MG_ACC_TILES * 16 * MT;                  // [1 or 2 blocks][32][MT]
    MegaOp *s_op = reinterpret_cast<MegaOp *>(vals + mg_vals(MT));  // the current op's descriptor for the epilogue warps
    static_assert(sizeof(MegaOp) <= 256 && sizeof(MegaOp) % 4 == 0, "s_op");
    uint64_t *stg = empty + MG_MAX_STAGES;                            // activation fragments landed in scratch
    unsigned char *scratch = smem + mg_misc_bytes(MT);
    unsigned char *ring = scratch + p.scratch_bytes;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int cta = blockIdx.x, nctas = gridDim.x;
    const int B = p.B, nstage = p.nstage;
    unsigned *wd_flag = p.bar + 2;

    if (tid == 0) {
        for (int i = 0; i < nstage; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], MG_CWARPS);
        }
        mbar_init(stg, 1);
        for (int c = 0; c < 4; ++c) mbar_init(&stgc[c], 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    // Register split (the launch gives every thread 96: 640 threads x 96 = 61440 of the SM's 65536).  The kernel keeps the
    // operand fragments of the weight loop, the epilogue's prefetched operands and the op parameters live at once; at 96
    // registers that spills, and with 227 KB of the SM's 256 KB configured as shared memory there is next to no L1 left to
    // catch local-memory traffic: every spill reload is an L2 round trip.  The producer needs few registers, the three filler warps none.
    // =========================== producer: the step's whole weight schedule ===========================
    if (warp >= MG_CWARPS) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(MG_REGS_PRODUCER));
        if (warp == MG_CWARPS && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            bool wrapped = false;
            // weights are read once per step: evict-first keeps the KV cache, the activations and the norm
            // vectors resident in L2 under the 1.9 GB/step weight stream
            const uint64_t pol = policy_evict_first();
            const int flags = p.flags;
            for (int oi = 0; oi < p.n_ops; ++oi) {
                const MegaOp &op = p.ops[oi];
                // pull what the consumers touch first in the NEXT phase into L2 now
                if (oi + 1 < p.n_ops) {
                    const MegaOp &nx = p.ops[oi + 1];
                    if (nx.kind == MG_MATVEC && (oi % nctas) == cta && !(flags & 4)) {
                        if (nx.fout_gamma) bulk_prefetch_l2(nx.fout_gamma, (uint32_t)nx.N * 4u);
                    }
                }
                if (op.kind != MG_MATVEC) continue;
                const int n_tiles = op.n_tiles, n_pairs = op.n_pairs, S = op.S, Ps = op.Ps, UT = op.unit_tiles;
                const uint4 *qs = op.qs_tc;
                const uint2 *ds = op.d_tc;
                const int ntl = mg_tile_count(n_tiles, UT, cta, nctas);
                for (int s = 0; s < S; ++s) {
                    const int pb = s * Ps;
                    const int np = min(Ps, n_pairs - pb);
                    for (int it = 0; it < ntl; it += NT) {
                        const int nt = min(NT, ntl - it);
                        for (int c0 = 0; c0 < np; c0 += MG_CHUNK) {
                            const int nb = min(MG_CHUNK, np - c0);
                            if (wrapped) mbar_wait(&empty[stage], phase ^ 1u, wd_flag, 0x100u + (unsigned)oi);
                            unsigned char *dst = ring + (size_t)stage * (NT * MG_SLOT_BYTES);
                            mbar_expect_tx(&full[stage], (uint32_t)(nt * nb) * 576u);
                            for (int u = 0; u < nt; ++u) {
                                const size_t pair0 = (size_t)mg_tile_of(it + u, UT, cta, nctas) * n_pairs + pb + c0;
                                if (flags & 1) {
                                    bulk_g2s(dst + (size_t)u * MG_SLOT_BYTES, qs + pair0 * 32, (uint32_t)nb * 512u, &full[stage]);
                                    bulk_g2s(dst + (size_t)u * MG_SLOT_BYTES + MG_SLOT_Q, ds + pair0 * 8, (uint32_t)nb * 64u, &full[stage]);
                                } else {
                                    bulk_g2s_hint(dst + (size_t)u * MG_SLOT_BYTES, qs + pair0 * 32, (uint32_t)nb * 512u, &full[stage], pol);
                                    bulk_g2s_hint(dst + (size_t)u * MG_SLOT_BYTES + MG_SLOT_Q, ds + pair0 * 8, (uint32_t)nb * 64u, &full[stage], pol);
                                }
                            }
                            if (++stage == nstage) {
                                stage = 0;
                                phase ^= 1u;
                                wrapped = true;
                            }
                        }
                    }
                }
            }
        } else if (warp > MG_CWARPS) {
            // =========================== epilogue warps ===========================
            // The 16 consumer warps leave their partial sums of a tile group in red[par] and go straight on to the next
            // group's weight stream; the epilogue warps add the 16 partials per output in fixed (tree) order and run the
            // epilogue (norm / bias / residual / SiLU*up / running argmax / fragments for the next matvec).
            // These warps share the SM's issue slots with 16 busy consumer warps (they get ~1/5 of a sub-partition), so the
            // role is written for instruction count: thread e owns FOUR consecutive rows of one (tile slot, token) --
            // outputs rt = 4e .. 4e+3 of the group, (slot, token, row) = (rt / 16MT, (rt % 16MT) / 16, rt % 16) -- i.e. one
            // 128-bit load per partial, one 128-bit residual load and one 128-bit store; a first version with one output per
            // thread and three passes (~1070 instructions per group and warp) could not keep up with the consumers.
            constexpr int NOUT = NT * 16 * MT;
            constexpr int NQ = NOUT / 4;                      // active epilogue threads (64 at 8 tokens)
            static_assert(NQ <= MG_ETHREADS && NOUT % 4 == 0, "one quad of rows per epilogue thread");
            const int e = tid - (MG_CTHREADS + 32);
            const bool qact = e < NQ;
            const int q_slot = (4 * e) / (16 * MT), q_tok = ((4 * e) % (16 * MT)) >> 4, q_r0 = (4 * e) & 15;
            int par = 0;
            float best_v = -INFINITY;
            int best_i = 0x7fffffff;
            for (int oi = 0; oi < p.n_ops; ++oi) {
                const MegaOp &op = p.ops[oi];
                if (op.kind == MG_MATVEC) {
                    const int n_tiles = op.n_tiles, S = op.S, N = op.N;
                    const int epi = op.epi, ldy = op.ldy, track = op.track_argmax, UT = op.unit_tiles;
                    const int ush = UT == 4 ? 2 : (UT == 2 ? 1 : 0);   // unit_tiles is 1, 2 or 4 (host-checked)
                    const bool has_norm = op.gamma != nullptr;
                    // The descriptor's pointers are needed a few times per group: they live in shared memory (an LDS at the
                    // point of use), not in registers -- this role runs on 64 registers, and spills are expensive here.
                    {
                        const uint32_t *src = reinterpret_cast<const uint32_t *>(&op);
                        uint32_t *dst = reinterpret_cast<uint32_t *>(s_op);
                        if (e < (int)(sizeof(MegaOp) / 4)) dst[e] = src[e];
                        ebar();
                    }
                    const volatile MegaOp *const vop = s_op;
                    // (run by the last epilogue thread, which has nothing to do until the first tile group arrives: on the
                    // consumers' thread 0 the dependent loads of positions and page table delayed the fragment copies of the
                    // qkv phase by ~1.3 us)
                    if (e == MG_ETHREADS - 1 && oi + 1 < p.n_ops && !(p.flags & 2)) {
                        // the next phase is this layer's attention: pull this CTA's chunk of the KV cache into L2 now, so the
                        // walk does not wait on DRAM behind the weight stream
                        const MegaOp &nx = p.ops[oi + 1];
                        if (nx.kind == MG_ATTN) {
                            const int NC = p.attn_chunks;
                            for (int unit = cta; unit < B * p.Hkv * NC; unit += nctas) {
                                const int ch = unit % NC, bk = unit / NC;
                                const int b = bk / p.Hkv, kvh = bk - b * p.Hkv;
                                const int pos = p.d_pos[b];
                                if (pos >= p.max_seq) continue;
                                const int j_lo = pos - p.window > 0 ? pos - p.window : 0;
                                const int per = (pos - j_lo + NC) / NC;
                                const int j0 = j_lo + ch * per, j1 = min(pos, j0 + per);  // row `pos` is not written yet
                                for (int pg = j0 / KV_PAGE; pg * KV_PAGE < j1; ++pg) {     // pages are the contiguous unit
                                    const int ka = max(j0, pg * KV_PAGE), ke = min(j1, (pg + 1) * KV_PAGE);
                                    const size_t off = (((size_t)p.page_table[(size_t)b * p.max_pages + pg] * p.Hkv + kvh) * KV_PAGE + (ka - pg * KV_PAGE)) * HD;
                                    bulk_prefetch_l2(nx.kc + off, (uint32_t)(ke - ka) * HD * 4u);
                                    bulk_prefetch_l2(nx.vc + off, (uint32_t)(ke - ka) * HD * 4u);
                                }
                            }
                        }
                    }
#define yout ((track && p.logits_out) ? p.logits_out : vop->y)
#define bias (vop->bias)
#define resid (vop->res)
#define ssq_out (vop->ssq_out)
#define fout_bf (vop->fout_bf)
#define fout_off (vop->fout_off)
#define fout_gamma (vop->fout_gamma)
                    const int ntl = mg_tile_count(n_tiles, UT, cta, nctas);
                    const bool vec_ok = ((ldy | N) & 3) == 0;   // 128-bit residual loads / output stores are aligned
                    // fragment builders: thread e = (block within the group, token, t)
                    const int bi = e / (4 * MT), bm_ = (e % (4 * MT)) >> 2, bt = e & 3;
                    for (int s = 0; s < S && ntl > 0; ++s) {
                        const bool last = s + 1 == S;
                        for (int it = 0; it < ntl; it += NT) {
                            const int nt = min(NT, ntl - it);
                            const int li = it + q_slot;                                   // index in the CTA's tile list
                            const int r_tile = ((cta + (li >> ush) * nctas) << ush) + (li & (UT - 1));
                            const int r_row = r_tile * 16 + q_r0;
                            const bool r_valid = qact && q_slot < nt;
                            const bool live = r_valid && q_tok < B;
                            // the epilogue's residual operand and the builder's norm weight: L2 round trips, started while
                            // the consumers are still streaming the group
                            float4 res4 = make_float4(0.f, 0.f, 0.f, 0.f);
                            const bool quad_in = r_row + 3 < N;   // (else: a ragged last tile, handled row by row)
                            if (epi == EPI_RESIDUAL && last && live) {
                                const float *rsrc = resid + (size_t)q_tok * ldy + r_row;
                                if (vec_ok && quad_in) {
                                    res4 = __ldcg(reinterpret_cast<const float4 *>(rsrc));
                                } else {
                                    if (r_row + 0 < N) res4.x = __ldcg(rsrc + 0);
                                    if (r_row + 1 < N) res4.y = __ldcg(rsrc + 1);
                                    if (r_row + 2 < N) res4.z = __ldcg(rsrc + 2);
                                    if (r_row + 3 < N) res4.w = __ldcg(rsrc + 3);
                                }
                            }
                            const int f_nblk = UT <= NT ? nt / UT : (((it + NT) % UT == 0) ? 1 : 0);
                            const int f_lb = UT <= NT ? it + bi * UT : it + NT - UT;  // list index of the block's first tile
                            const int f_blk = cta + (f_lb >> ush) * nctas;            // unit index = block index
                            const bool bact = fout_bf != nullptr && last && bi < f_nblk && bm_ < B;
                            float4 fg_lo = make_float4(1.f, 1.f, 1.f, 1.f), fg_hi = fg_lo;
                            if (bact && fout_gamma) {
                                const float4 *gq4 = reinterpret_cast<const float4 *>(fout_gamma + (size_t)f_blk * 32);
                                fg_lo = gq4[bt];
                                fg_hi = gq4[4 + bt];
                            }
                            hbar_sync(MG_BAR_FULL + par);   // the 16 warps' partial sums of this group are in red[par]
                            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (r_valid) {
                                // fixed-shape tree over the 16 warps' partials (((0+1)+(2+3))+((4+5)+(6+7)))+(...), four loads at a time
                                const float4 *rp = reinterpret_cast<const float4 *>(red + (size_t)par * MG_CWARPS * NOUT) + e;
                                auto add4 = [](const float4 a, const float4 c) { return make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w); };
                                float4 oct[2];
#pragma unroll
                                for (int o = 0; o < 2; ++o) {
                                    float4 quad[2];
#pragma unroll
                                    for (int qd = 0; qd < 2; ++qd) {
                                        const int w0 = o * 8 + qd * 4;
                                        const float4 p0 = rp[(w0 + 0) * (NOUT / 4)], p1 = rp[(w0 + 1) * (NOUT / 4)];
                                        const float4 p2 = rp[(w0 + 2) * (NOUT / 4)], p3 = rp[(w0 + 3) * (NOUT / 4)];
                                        quad[qd] = add4(add4(p0, p1), add4(p2, p3));
                                    }
                                    oct[o] = add4(quad[0], quad[1]);
                                }
                                v = add4(oct[0], oct[1]);
                                if (S > 1) {
                                    float4 *at = reinterpret_cast<float4 *>(acc_tile + (size_t)li * 16 * MT) + (e % (4 * MT));
                                    if (s > 0) v = add4(v, *at);
                                    if (!last) *at = v;
                                }
                            }
                            if (last) {
                                if (has_norm && live) {
                                    const float ri = rinv[q_tok];
                                    v.x *= ri; v.y *= ri; v.z *= ri; v.w *= ri;
                                }
                                const int be = UT <= NT ? q_slot / UT : 0;        // block within this group
                                const int ti = li & (UT - 1);                     // tile within its unit
                                if (fout_bf) ebar();  // the previous group's builders are done with vals
                                if (epi == EPI_SILU_MUL) {
                                    // rows (2i, 2i+1) = (gate, up) of output i: both pairs of this quad are in this thread
                                    if (live && r_row + 3 < N) {
                                        const float f0 = (v.x / (1.0f + expf(-v.x))) * v.y, f1 = (v.z / (1.0f + expf(-v.z))) * v.w;
                                        if (yout) {
                                            yout[(size_t)q_tok * ldy + (r_row >> 1)] = f0;
                                            yout[(size_t)q_tok * ldy + (r_row >> 1) + 1] = f1;
                                        }
                                        if (fout_bf) {
                                            float *vd = vals + (size_t)(be * 32 + ti * 8 + (q_r0 >> 1)) * MT + q_tok;
                                            vd[0] = f0;
                                            vd[MT] = f1;
                                        }
                                    }
                                } else {
                                    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
                                    if (live && r_row < N) {
                                        out = v;
                                        if (!quad_in) {   // rows beyond N contribute nothing (statistics, fragments, argmax)
                                            if (r_row + 1 >= N) out.y = 0.0f;
                                            if (r_row + 2 >= N) out.z = 0.0f;
                                            out.w = 0.0f;
                                        }
                                        if (bias) {
                                            out.x += bias[r_row];
                                            if (r_row + 1 < N) out.y += bias[r_row + 1];
                                            if (r_row + 2 < N) out.z += bias[r_row + 2];
                                            if (r_row + 3 < N) out.w += bias[r_row + 3];
                                        }
                                        if (epi == EPI_RESIDUAL) { out.x += res4.x; out.y += res4.y; out.z += res4.z; out.w += res4.w; }
                                        if (epi == EPI_GELU) {
                                            out.x = 0.5f * out.x * (1.0f + erff(out.x * 0.70710678118654752440f));
                                            out.y = 0.5f * out.y * (1.0f + erff(out.y * 0.70710678118654752440f));
                                            out.z = 0.5f * out.z * (1.0f + erff(out.z * 0.70710678118654752440f));
                                            out.w = 0.5f * out.w * (1.0f + erff(out.w * 0.70710678118654752440f));
                                        }
                                        if (yout) {
                                            float *yd = yout + (size_t)q_tok * ldy + r_row;
                                            if (vec_ok && quad_in) {
                                                *reinterpret_cast<float4 *>(yd) = out;
                                            } else {
                                                yd[0] = out.x;
                                                if (r_row + 1 < N) yd[1] = out.y;
                                                if (r_row + 2 < N) yd[2] = out.z;
                                                if (r_row + 3 < N) yd[3] = out.w;
                                            }
                                        }
                                        if (track) {   // ascending rows: the lowest index wins ties
                                            amax_combine(best_v, best_i, out.x, r_row);
                                            if (r_row + 1 < N) amax_combine(best_v, best_i, out.y, r_row + 1);
                                            if (r_row + 2 < N) amax_combine(best_v, best_i, out.z, r_row + 2);
                                            if (r_row + 3 < N) amax_combine(best_v, best_i, out.w, r_row + 3);
                                        }
                                        if (fout_bf) {
                                            float *vd = vals + (size_t)(be * 32 + ti * 16 + q_r0) * MT + q_tok;
                                            vd[0] = out.x;
                                            vd[MT] = out.y;
                                            vd[2 * MT] = out.z;
                                            vd[3 * MT] = out.w;
                                        }
                                    }
                                    if (ssq_out) {   // sum of squares of the tile's 16 rows: 4 in this thread, 4 lanes per tile
                                        float sq = (out.x * out.x + out.y * out.y) + (out.z * out.z + out.w * out.w);
                                        sq += __shfl_xor_sync(0xffffffffu, sq, 2);
                                        sq += __shfl_xor_sync(0xffffffffu, sq, 1);
                                        if (live && q_r0 == 0) ssq_out[(size_t)r_tile * 8 + q_tok] = sq;   // [part][8 tokens]
                                    }
                                }
                                if (fout_bf) {
                                    // ---- this group's outputs become the next matvec's activation fragments:
                                    // a unit of UT consecutive tiles = one 32-value block per token
                                    ebar();
                                    if (e < ((2 * 4 * MT + 31) / 32) * 32) {  // warp-uniform: the warps holding builder lanes
                                        float4 l = make_float4(0.f, 0.f, 0.f, 0.f), h = l;
                                        if (bact) {
                                            const float *vb = vals + (size_t)(bi * 32) * MT + bm_;
                                            l = make_float4(vb[(4 * bt + 0) * MT], vb[(4 * bt + 1) * MT], vb[(4 * bt + 2) * MT], vb[(4 * bt + 3) * MT]);
                                            h = make_float4(vb[(16 + 4 * bt + 0) * MT], vb[(16 + 4 * bt + 1) * MT], vb[(16 + 4 * bt + 2) * MT],
                                                            vb[(16 + 4 * bt + 3) * MT]);
                                            l = mul4(l, fg_lo);
                                            h = mul4(h, fg_hi);
                                        }
                                        frag_build<MT>(l, h, bact, bt, bm_, fout_bf + (size_t)f_blk * (16 * MT), fout_off + (size_t)f_blk * MT);
                                    }
                                }
                            }
                            // red[par] has been read (the partials were consumed by the sums above; the stores that depend
                            // on them have been issued): the consumers may overwrite it two groups from now
                            hbar_arrive(MG_BAR_FREE + par, false);
                            par ^= 1;
                        }
                    }
                    if (fout_bf) asm volatile("fence.proxy.async;\n" ::: "memory");  // fragments are read by bulk copies next phase
                    if (track) {
                        // this CTA's best candidate per stream (lowest index wins ties: order independent):
                        // first the 4 quads (16 rows) of a (slot, token) group, then the NT slots through shared memory
                        float *cv = vals;   // idle in this op (only fragment-producing ops use it): [NT][MT] values, then indices
                        int *ci = reinterpret_cast<int *>(vals + NT * MT);
#pragma unroll
                        for (int o = 2; o > 0; o >>= 1) {
                            const float ov = __shfl_xor_sync(0xffffffffu, best_v, o);
                            const int ox = __shfl_xor_sync(0xffffffffu, best_i, o);
                            amax_combine(best_v, best_i, ov, ox);
                        }
                        if (qact && (e & 3) == 0) {
                            cv[e >> 2] = best_v;     // = slot * MT + token
                            ci[e >> 2] = best_i;
                        }
                        best_v = -INFINITY;
                        best_i = 0x7fffffff;
                        ebar();
                        if (e < B) {
                            float bv = -INFINITY;
                            int bx = 0x7fffffff;
#pragma unroll
                            for (int u = 0; u < NT; ++u) amax_combine(bv, bx, cv[u * MT + e], ci[u * MT + e]);
                            p.am_vals[(size_t)cta * 8 + e] = bv;
                            p.am_idx[(size_t)cta * 8 + e] = bx;
                        }
                    }
#undef yout
#undef bias
#undef resid
#undef ssq_out
#undef fout_bf
#undef fout_off
#undef fout_gamma
                }
                // phase end: (1) everything this CTA wrote is ordered before thread 0's arrival at the grid barrier,
                // (2) the next phase starts for all roles once thread 0 has seen every CTA arrive
                if (oi + 1 < p.n_ops) {
                    abar();
                    abar();
                }
            }
        }
        return;
    }

    // =========================== consumers ===========================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(MG_REGS_CONSUMER));
    const int epoch = *p.d_epoch;  // decode steps run by this session so far (attention chunk flags)
    int stage = 0;
    uint32_t phase = 0, stg_phase = 0;
    const bool early_release = !(p.flags & 32);  // flag 32: experiment -- release a stage after the arithmetic
    int par = 0, group_ctr = 0;
    unsigned bar_target = 0;

    for (int oi = 0; oi < p.n_ops; ++oi) {
        const MegaOp &op = p.ops[oi];
        const int kind = op.kind;
        const bool tracing = p.trace != nullptr && cta == 0 && tid == 0;
        const bool tr_all = p.trace_all != nullptr && tid == 0;
        unsigned long long *const ta = tr_all ? p.trace_all + ((size_t)cta * p.n_ops + oi) * 4 : nullptr;
        if (tr_all) ta[0] = ta[3] = (unsigned long long)clock64();
        if (tracing) {
            const unsigned long long now = (unsigned long long)clock64();
            p.trace[oi * 6 + 0] = now;
            p.trace[oi * 6 + 1] = now;
            p.trace[oi * 6 + 4] = now;
            p.trace[oi * 6 + 5] = now;
        }
        if (tid == 0 && oi + 1 < p.n_ops) {  // next phase's descriptor -> L1 (off its critical path)
            prefetch_l1(&p.ops[oi + 1]);
            prefetch_l1(reinterpret_cast<const unsigned char *>(&p.ops[oi + 1]) + 128);
        }
        if (kind == MG_MATVEC) {
            const int n_tiles = op.n_tiles, n_pairs = op.n_pairs, S = op.S, Ps = op.Ps, K = op.K;
            const int UT = op.unit_tiles;
            const bool has_norm = op.gamma != nullptr;
            const int ntl = mg_tile_count(n_tiles, UT, cta, nctas);
            float2 *off2 = reinterpret_cast<float2 *>(scratch);             // [2*Ps][MT]
            uint2 *bf = reinterpret_cast<uint2 *>(off2 + (size_t)Ps * 2 * MT);  // [2*Ps][2][2*MT][4]
            if (ntl > 0) {
                for (int s = 0; s < S; ++s) {
                    const int pb = s * Ps;
                    const int np = min(Ps, n_pairs - pb);
                    // The fragments land in up to 4 K chunks (whole ring stages of 16 pairs), each with its own barrier: the
                    // first tile group starts on chunk 0 while the rest of the copy is still in flight (the copy is L2-bandwidth
                    // bound: all 132 CTAs fetch the same 70-104 KB).
                    const int CP = 16 * ((((np + 15) >> 4) + 3) >> 2);  // pairs per chunk
                    cbar();  // every warp is done with the previous contents of scratch (and has seen all its chunks)
                    if (tid == 0) {
                        // the input's fragments were written (generic proxy, other SMs) before the grid barrier
                        asm volatile("fence.proxy.async;\n" ::: "memory");
                        const uint32_t ob = (uint32_t)(2 * np * MT) * 8u;
                        const unsigned char *src = reinterpret_cast<const unsigned char *>(op.fin_bf + (size_t)(2 * pb) * (16 * MT));
                        unsigned char *dstb = reinterpret_cast<unsigned char *>(bf);
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const int p0 = min(np, c * CP), p1 = min(np, (c + 1) * CP);
                            const uint32_t o = (uint32_t)p0 * (256u * MT), cb = (uint32_t)(p1 - p0) * (256u * MT);
                            mbar_expect_tx(&stgc[c], cb + (c == 0 ? ob : 0u));   // an empty chunk completes at once
                            if (c == 0) bulk_g2s(off2, op.fin_off + (size_t)(2 * pb) * MT, ob, &stgc[0]);
                            if (cb) bulk_g2s(dstb + o, src + o, cb, &stgc[c]);
                        }
                    }
                    const uint32_t stg_par = stg_phase;
                    stg_phase ^= 1u;
                    // row statistics of the fused RMSNorm (first used by the epilogue).  The partial sums live as
                    // [part][8 tokens]: warps 1..4 read them with coalesced loads (lane % 8 = token).  (One warp per token reading
                    // its column cost 2048 sector requests per CTA for the same 6 KB, by all 132 CTAs at once: the normed phases'
                    // staging was ~1 us longer than the others'.)
                    if (s == 0 && has_norm && warp >= 1 && warp <= 4) {
                        const int total = op.ssq_in_parts * 8;
                        float pr[12];
#pragma unroll
                        for (int q = 0; q < 12; ++q) {
                            const int f = (warp - 1) * 32 + lane + 128 * q;
                            pr[q] = f < total ? __ldcg(op.ssq_in + f) : 0.0f;
                        }
                        float ss = 0.0f;
#pragma unroll
                        for (int q = 0; q < 12; ++q) ss += pr[q];
                        for (int f = (warp - 1) * 32 + lane + 128 * 12; f < total; f += 128) ss += __ldcg(op.ssq_in + f);
                        ss += __shfl_xor_sync(0xffffffffu, ss, 8);
                        ss += __shfl_xor_sync(0xffffffffu, ss, 16);
                        if (lane < 8) rpart[(warp - 1) * 8 + lane] = ss;
                    }
                    cbar();  // the warps' partial sums are visible
                    // 1/rms per token: read by the epilogue warps behind the first tile group's hand-off barrier
                    if (s == 0 && has_norm && tid < B)
                        rinv[tid] = 1.0f / sqrtf((((rpart[tid] + rpart[8 + tid]) + (rpart[16 + tid] + rpart[24 + tid]))) / (float)K + p.eps);
                    if (tracing && s == 0) p.trace[oi * 6 + 1] = (unsigned long long)clock64();
                    // the CTA's tiles NT at a time: every warp carries NT independent accumulation chains that
                    // share one read of the activation fragments
                    for (int it = 0; it < ntl; it += NT) {
                        const int nt = min(NT, ntl - it);
#ifdef VOX_MEGA_WARP_TRACE
                        // warp-level trace of the lm_head phase's first groups (CTA 0; debug "mega_trace_w")
                        unsigned long long *tw = nullptr;
                        if (p.trace_w != nullptr && cta == 0 && lane == 0 && oi == p.n_ops - 2 && s == 0 && it / NT < 6)
                            tw = p.trace_w + ((size_t)warp * 6 + it / NT) * 8;
                        if (tw) tw[0] = (unsigned long long)clock64();
#else
                        constexpr unsigned long long *tw = nullptr;   // compile with -DVOX_MEGA_WARP_TRACE to record
#endif
                        float acc[NT][2 * CG];
#pragma unroll
                        for (int u = 0; u < NT; ++u)
#pragma unroll
                            for (int c = 0; c < 2 * CG; ++c) acc[u][c] = 0.0f;
                        // ---- the weight loop: one block pair per warp per ring stage, for the group's nt tiles.
                        // Guard-free bodies (nt is warp-uniform: one instantiation per count; a warp without a pair in
                        // a ragged last chunk only recycles the stage).
                        {
                            const uint32_t slot_q = (uint32_t)warp * 512u + (uint32_t)lane * 16u;
                            const uint32_t slot_d = (uint32_t)MG_SLOT_Q + (uint32_t)warp * 64u + (uint32_t)g * 8u;
                            int next_chunk_c0 = it == 0 ? 0 : 0x7fffffff, chunk = 0;   // first pass over the slice: wait per chunk
                            for (int c0 = 0; c0 < np; c0 += MG_CHUNK) {
                                if (c0 == next_chunk_c0) {   // the fragments of this K chunk must have landed
                                    mbar_wait(&stgc[chunk], stg_par, wd_flag, 0x500u + (unsigned)oi);
                                    ++chunk;
                                    next_chunk_c0 += CP;
                                }
                                mbar_wait(&full[stage], phase, wd_flag, 0x200u + (unsigned)oi);
                                if (tracing && s == 0 && it == 0 && c0 == 0) p.trace[oi * 6 + 4] = (unsigned long long)clock64();
                                if (tr_all && s == 0 && it == 0 && c0 == 0) ta[3] = (unsigned long long)clock64();
                                if (tw && c0 / MG_CHUNK < 3) tw[1 + c0 / MG_CHUNK] = (unsigned long long)clock64();
                                const int pp = c0 + warp;  // pair index inside the slice
                                if (pp < np && !(p.flags & 16)) {   // flag 16: experiment -- consume the ring without the arithmetic
                                    const unsigned char *sb = ring + (size_t)stage * (NT * MG_SLOT_BYTES);
                                    const uint2 *bfp = bf + (size_t)pp * (2 * 16 * MT);
                                    const float2 *ofp = off2 + (size_t)pp * (2 * MT);
                                    uint64_t *rel = early_release ? &empty[stage] : nullptr;
                                    if (nt == NT) mg_pair<MT, NT, NT>(sb, slot_q, slot_d, bfp, ofp, g, t, lane, acc, rel);
                                    else if (NT > 1 && nt == 1) mg_pair<MT, NT, 1>(sb, slot_q, slot_d, bfp, ofp, g, t, lane, acc, rel);
                                    else if (NT > 2 && nt == 2) mg_pair<MT, NT, 2>(sb, slot_q, slot_d, bfp, ofp, g, t, lane, acc, rel);
                                    else if (NT > 3 && nt == 3) mg_pair<MT, NT, 3>(sb, slot_q, slot_d, bfp, ofp, g, t, lane, acc, rel);
                                    if (!early_release) {
                                        __syncwarp();
                                        if (lane == 0) mbar_arrive(&empty[stage]);
                                    }
                                } else {
                                    __syncwarp();
                                    if (lane == 0) mbar_arrive(&empty[stage]);
                                }
                                if (++stage == nstage) {
                                    stage = 0;
                                    phase ^= 1u;
                                }
                            }
                        }
                        if (tracing && s + 1 == S && it + NT >= ntl) p.trace[oi * 6 + 5] = (unsigned long long)clock64();
                        if (tw) tw[4] = (unsigned long long)clock64();
                        // ---- the 16 warps' partial sums of these tiles meet in shared memory: red[par] is handed to the epilogue
                        // warps (they read it, run the epilogue, and give it back two groups later); this warp goes straight on
                        // to the next group's weight stream
                        if (group_ctr >= 2) hbar_sync(MG_BAR_FREE + par);   // the buffer's previous contents have been read
                        float *rw = red + (size_t)(par * MG_CWARPS + warp) * (NT * 16 * MT);
#pragma unroll
                        for (int u = 0; u < NT; ++u) {
                            if (u < nt) {
                                if constexpr (MT == 8) {  // lane (g, t): rows g, g+8 x tokens 2t, 2t+1
                                    rw[(u * MT + 2 * t) * 16 + g] = acc[u][0];
                                    rw[(u * MT + 2 * t + 1) * 16 + g] = acc[u][1];
                                    rw[(u * MT + 2 * t) * 16 + g + 8] = acc[u][2];
                                    rw[(u * MT + 2 * t + 1) * 16 + g + 8] = acc[u][3];
                                } else {
#pragma unroll
                                    for (int c = 0; c < CG; ++c) {
                                        const int tok = c * 4 + t;
                                        if (tok < MT) {
                                            rw[(u * MT + tok) * 16 + g] = acc[u][2 * c];
                                            rw[(u * MT + tok) * 16 + g + 8] = acc[u][2 * c + 1];
                                        }
                                    }
                                }
                            }
                        }
                        hbar_arrive(MG_BAR_FULL + par, true);
                        if (tw) tw[5] = (unsigned long long)clock64();
                        ++group_ctr;
                        if (tw) tw[6] = (unsigned long long)clock64();
                        par ^= 1;
                    }
                }
            }
        } else if (kind == MG_ATTN) {
            // unit = (stream, kv head, key chunk): the 4 query heads of a GQA group share one pass over their
            // chunk of K and V; the chunks' softmax states are combined by the last chunk's CTA (tagged words, below).  (With
            // one CTA per (stream, kv head), a few CTAs walk all keys -- issue-bound -- while the other SMs wait.)
            float *qs = reinterpret_cast<float *>(scratch);       // [G][HD]
            float *kvs = qs + G * HD;                              // [2][HD]
            float *red_m = kvs + 2 * HD;                           // [MG_CWARPS][G]
            float *red_l = red_m + MG_CWARPS * G;                  // [MG_CWARPS][G]
            float *red_acc = red_l + MG_CWARPS * G;                // [MG_CWARPS][G][HD]
            const int H = p.H, Hkv = p.Hkv, max_seq = p.max_seq, NC = p.attn_chunks;
            KvView kvw;
            kvw.k = op.kc;
            kvw.v = op.vc;
            kvw.page_table = p.page_table;
            kvw.max_pages = p.max_pages;
            for (int unit = cta; unit < B * Hkv * NC; unit += nctas) {
                const int ch = unit % NC, bk = unit / NC;
                const int b = bk / Hkv, kvh = bk - b * Hkv;
                const int pos = p.d_pos[b];              // per row: sessions of different ages share the step
                if (pos >= max_seq) continue;
                const int j_lo = pos - p.window > 0 ? pos - p.window : 0;
                const int per = (pos - j_lo + NC) / NC;  // ceil((pos - j_lo + 1) / NC) keys per chunk
                const int j0 = j_lo + ch * per, j1 = min(pos + 1, j0 + per);  // keys [j0, j1)
                const bool has_new = j0 <= pos && pos < j1;                    // this chunk holds the new row
                const float *row = p.qkv + (size_t)b * p.ld_qkv;
                cbar();  // scratch free (previous unit / previous op)
                // q (G heads) and k through RoPE on the way in (rope.rs:103-141: interleaved pairs), v as is
                constexpr int half = HD / 2;
                for (int i = tid; i < (G + 1) * half; i += MG_CTHREADS) {
                    const int h = i / half, pi = i - h * half;
                    const float *src = (h < G) ? row + (size_t)(kvh * G + h) * HD + 2 * pi : row + (size_t)H * HD + kvh * HD + 2 * pi;
                    const float2 xv = __ldcg(reinterpret_cast<const float2 *>(src));
                    const float c = p.cos_t[(size_t)pos * half + pi], sn = p.sin_t[(size_t)pos * half + pi];
                    float *dst = (h < G) ? &qs[h * HD + 2 * pi] : &kvs[2 * pi];
                    dst[0] = xv.x * c - xv.y * sn;
                    dst[1] = xv.x * sn + xv.y * c;
                }
                for (int i = tid; i < HD; i += MG_CTHREADS) kvs[HD + i] = __ldcg(row + (size_t)(H + Hkv) * HD + kvh * HD + i);
                cbar();
                if (tracing) p.trace[oi * 6 + 1] = (unsigned long long)clock64();
                if (tr_all) ta[3] = (unsigned long long)clock64();
                if (has_new) {
                    const size_t at = kv_index(kvw, b, Hkv, kvh, pos, HD);
                    for (int i = tid; i < HD; i += MG_CTHREADS) {
                        kvw.k[at + i] = kvs[i];
                        kvw.v[at + i] = kvs[HD + i];
                    }
                }
                float q[G][DPL];
#pragma unroll
                for (int h = 0; h < G; ++h)
#pragma unroll
                    for (int i = 0; i < DPL; ++i) q[h][i] = qs[h * HD + lane * DPL + i];
                float m_run[G], l_run[G], acc[G][DPL];
#pragma unroll
                for (int h = 0; h < G; ++h) {
                    m_run[h] = -INFINITY;
                    l_run[h] = 0.0f;
#pragma unroll
                    for (int i = 0; i < DPL; ++i) acc[h][i] = 0.0f;
                }
                constexpr int KU = 4;  // keys in flight per warp; one softmax rescale per KU keys
                for (int jb = j0 + warp; jb < j1; jb += KU * MG_CWARPS) {
                    float kk[KU][DPL], vv[KU][DPL];
#pragma unroll
                    for (int u = 0; u < KU; ++u) {
                        const int j = jb + u * MG_CWARPS;
                        if (j < j1 && j != pos) {
                            const size_t at = kv_index(kvw, b, Hkv, kvh, j, HD) + lane * DPL;
                            const float *kr = kvw.k + at;
                            const float *vr = kvw.v + at;
                            if constexpr (DPL == 4) {
                                const float4 k4 = *reinterpret_cast<const float4 *>(kr);
                                const float4 v4 = *reinterpret_cast<const float4 *>(vr);
                                kk[u][0] = k4.x; kk[u][1] = k4.y; kk[u][2] = k4.z; kk[u][3] = k4.w;
                                vv[u][0] = v4.x; vv[u][1] = v4.y; vv[u][2] = v4.z; vv[u][3] = v4.w;
                            } else {
#pragma unroll
                                for (int i = 0; i < DPL; ++i) {
                                    kk[u][i] = kr[i];
                                    vv[u][i] = vr[i];
                                }
                            }
                        } else {  // j == pos: the row appended above, still in shared memory (j >= j1: unused)
#pragma unroll
                            for (int i = 0; i < DPL; ++i) {
                                kk[u][i] = kvs[lane * DPL + i];
                                vv[u][i] = kvs[HD + lane * DPL + i];
                            }
                        }
                    }
                    float sc[KU][G];
#pragma unroll
                    for (int u = 0; u < KU; ++u)
#pragma unroll
                        for (int h = 0; h < G; ++h) {
                            float d = 0.0f;
#pragma unroll
                            for (int i = 0; i < DPL; ++i) d = fmaf(q[h][i], kk[u][i], d);
                            sc[u][h] = d;
                        }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
                        for (int u = 0; u < KU; ++u)
#pragma unroll
                            for (int h = 0; h < G; ++h) sc[u][h] += __shfl_xor_sync(0xffffffffu, sc[u][h], o);
#pragma unroll
                    for (int h = 0; h < G; ++h) {
                        float m_new = m_run[h];
#pragma unroll
                        for (int u = 0; u < KU; ++u) {
                            sc[u][h] = (jb + u * MG_CWARPS < j1) ? sc[u][h] * p.scale : -INFINITY;
                            m_new = fmaxf(m_new, sc[u][h]);
                        }
                        const float alpha = fast_exp(m_run[h] - m_new);  // exp(-inf) = 0 on the first batch
                        float pe[KU], ps = 0.0f;
#pragma unroll
                        for (int u = 0; u < KU; ++u) {
                            pe[u] = fast_exp(sc[u][h] - m_new);  // masked keys: exp(-inf) = 0
                            ps += pe[u];
                        }
                        l_run[h] = l_run[h] * alpha + ps;
                        m_run[h] = m_new;
#pragma unroll
                        for (int i = 0; i < DPL; ++i) {
                            float a = acc[h][i] * alpha;
#pragma unroll
                            for (int u = 0; u < KU; ++u) a = fmaf(pe[u], vv[u][i], a);
                            acc[h][i] = a;
                        }
                    }
                }
                if (tracing) p.trace[oi * 6 + 4] = (unsigned long long)clock64();
#pragma unroll
                for (int h = 0; h < G; ++h) {
                    if (lane == 0) {
                        red_m[warp * G + h] = m_run[h];
                        red_l[warp * G + h] = l_run[h];
                    }
#pragma unroll
                    for (int i = 0; i < DPL; ++i) red_acc[((size_t)warp * G + h) * HD + lane * DPL + i] = acc[h][i];
                }
                cbar();
                // ---- combine the warps; with several key chunks per (stream, kv head) the last chunk's CTA also
                // combines the chunks (pairwise release/acquire flags: no grid-wide phase for the merge)
                const int u0 = bk * NC;
                const int target = epoch * 64 + op.layer + 1;  // unique per (decode step, layer), never 0
                float2 *const acc2 = reinterpret_cast<float2 *>(p.att_acc);   // [unit][G][hd] {value, tag}
                float2 *const ml2 = reinterpret_cast<float2 *>(p.att_ml);     // [unit][G][2]  {value, tag}
                float o_final = 0.0f;                           // thread i < G*HD: output (head i / HD, dim i % HD)
                for (int i = tid; i < G * HD; i += MG_CTHREADS) {
                    const int h = i / HD, d = i - h * HD;
                    float mx = -INFINITY;
#pragma unroll
                    for (int w = 0; w < MG_CWARPS; ++w) mx = fmaxf(mx, red_m[w * G + h]);
                    float num = 0.0f, den = 0.0f;
#pragma unroll
                    for (int w = 0; w < MG_CWARPS; ++w) {
                        const float mw = red_m[w * G + h];
                        const float f = (mw == -INFINITY) ? 0.0f : fast_exp(mw - mx);
                        num = fmaf(red_acc[((size_t)w * G + h) * HD + d], f, num);
                        den = fmaf(red_l[w * G + h], f, den);
                    }
                    if (NC == 1) {
                        o_final = num / den;
                    } else if (ch != NC - 1) {
                        // publish this chunk's state; every word carries the (step, layer) tag, so the merging CTA polls the
                        // words themselves: no CTA barrier, fence and flag on this side, no flag wait + reload on the other
                        st_tagged(acc2 + ((size_t)unit * G + h) * HD + d, num, target);
                        if (d == 0) {
                            st_tagged(ml2 + ((size_t)unit * G + h) * 2 + 0, mx, target);
                            st_tagged(ml2 + ((size_t)unit * G + h) * 2 + 1, den, target);
                        }
                    } else {
                        // the last chunk's CTA combines the chunks: its own state from registers, the others' as they arrive
                        // (online rescaling, ascending chunk order: a few registers whatever the chunk count)
                        float m_all = mx, nsum = num, dsum = den;
                        const long long t0 = clock64();
                        for (int c = 0; c < NC - 1; ++c) {
                            const float2 *pa = acc2 + ((size_t)(u0 + c) * G + h) * HD + d;
                            const float2 *pm = ml2 + ((size_t)(u0 + c) * G + h) * 2;
                            float2 va = ld_tagged(pa), vm = ld_tagged(pm), vl = ld_tagged(pm + 1);
                            unsigned n = 0;
                            while (__float_as_int(va.y) != target || __float_as_int(vm.y) != target || __float_as_int(vl.y) != target) {
                                if ((++n & 0x3FFu) == 0 && clock64() - t0 > MG_SPIN_CYCLES) mg_die(wd_flag, 0x600u + (unsigned)oi);
                                if (__float_as_int(va.y) != target) va = ld_tagged(pa);
                                if (__float_as_int(vm.y) != target) vm = ld_tagged(pm);
                                if (__float_as_int(vl.y) != target) vl = ld_tagged(pm + 1);
                            }
                            const float m_new = fmaxf(m_all, vm.x);
                            const float fo = (m_all == -INFINITY) ? 0.0f : fast_exp(m_all - m_new);
                            const float fc = (vm.x == -INFINITY) ? 0.0f : fast_exp(vm.x - m_new);
                            nsum = fmaf(va.x, fc, nsum * fo);
                            dsum = fmaf(vl.x, fc, dsum * fo);
                            m_all = m_new;
                        }
                        o_final = nsum / dsum;
                    }
                }
                if (NC > 1 && ch != NC - 1) continue;  // only the last chunk's CTA produces the output
                // ---- attention output + its fragments for wo: a warp holds 32 consecutive dims of one head = one block
                if (tid < ((G * HD + 31) / 32) * 32) {
                    const bool oact = tid < G * HD;
                    const int h = tid / HD, d = tid - h * HD;
                    if (oact) p.attn_out[(size_t)b * (H * HD) + (size_t)(kvh * G + h) * HD + d] = o_final;
                    const int bt = lane & 3;
                    float4 l, hq;
                    l.x = __shfl_sync(0xffffffffu, o_final, 4 * bt + 0);
                    l.y = __shfl_sync(0xffffffffu, o_final, 4 * bt + 1);
                    l.z = __shfl_sync(0xffffffffu, o_final, 4 * bt + 2);
                    l.w = __shfl_sync(0xffffffffu, o_final, 4 * bt + 3);
                    hq.x = __shfl_sync(0xffffffffu, o_final, 16 + 4 * bt + 0);
                    hq.y = __shfl_sync(0xffffffffu, o_final, 16 + 4 * bt + 1);
                    hq.z = __shfl_sync(0xffffffffu, o_final, 16 + 4 * bt + 2);
                    hq.w = __shfl_sync(0xffffffffu, o_final, 16 + 4 * bt + 3);
                    const int blk = ((kvh * G) * HD + (tid - lane)) >> 5;  // block of wo's K = H*HD input
                    frag_build<MT>(l, hq, oact && lane < 4, bt, b, p.att_fbf + (size_t)blk * (16 * MT), p.att_foff + (size_t)blk * MT);
                }
            }
            asm volatile("fence.proxy.async;\n" ::: "memory");
        } else if (kind == MG_EMBED) {
            // x_dec[b] = audio[b][pos] + dequant(E[tok[b]])   (model.rs:584-618, 938-946)
            const int D = p.D, bpr = D >> 5, n = bpr * 16;
            float *xr = reinterpret_cast<float *>(scratch);  // the embedded row, for the fragment builders
            for (int b = cta; b < B; b += nctas) {
                cbar();
                const int id = p.d_tok[b];
                const float *arow = p.audio_rows ? p.audio_rows[b]
                                                 : (p.audio ? p.audio + ((size_t)b * p.audio_seq + p.d_pos[b]) * D : nullptr);
                for (int base = 0; base < n; base += MG_CTHREADS) {
                    const int i = base + tid;
                    const bool act = i < n;
                    const int blk = i >> 4, j = i & 15;
                    float lo = 0.0f, hi = 0.0f;
                    if (act) {
                        const uint8_t byte = reinterpret_cast<const uint8_t *>(p.emb_qs + (size_t)id * bpr + blk)[j];
                        const float dd = __half2float(p.emb_d[(size_t)id * bpr + blk]);
                        const int k = blk * 32 + j;
                        lo = ((float)(byte & 0xF) - 8.0f) * dd;
                        hi = ((float)(byte >> 4) - 8.0f) * dd;
                        if (arow) {
                            lo = arow[k] + lo;
                            hi = arow[k + 16] + hi;
                        }
                        p.x_dec[(size_t)b * D + k] = lo;
                        p.x_dec[(size_t)b * D + k + 16] = hi;
                        xr[k] = lo;
                        xr[k + 16] = hi;
                    }
                    float sl = lo * lo, sh = hi * hi;
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) {
                        sl += __shfl_xor_sync(0xffffffffu, sl, o);
                        sh += __shfl_xor_sync(0xffffffffu, sh, o);
                    }
                    if (act && j == 0) {
                        p.ssq_x[(size_t)(2 * blk) * 8 + b] = sl;
                        p.ssq_x[(size_t)(2 * blk + 1) * 8 + b] = sh;
                    }
                }
                cbar();
                // fragments of (row x first layer's attention-norm weight) for layer 0's wqkv
                for (int base = 0; base < bpr * 4; base += MG_CTHREADS) {
                    const int i = base + tid;
                    const bool act = i < bpr * 4;
                    const int blk = act ? i >> 2 : 0, bt = i & 3;
                    float4 l = make_float4(0.f, 0.f, 0.f, 0.f), h = l;
                    if (act) {
                        l = *reinterpret_cast<const float4 *>(xr + blk * 32 + 4 * bt);
                        h = *reinterpret_cast<const float4 *>(xr + blk * 32 + 16 + 4 * bt);
                        if (p.emb_gamma) {
                            l = mul4(l, *reinterpret_cast<const float4 *>(p.emb_gamma + blk * 32 + 4 * bt));
                            h = mul4(h, *reinterpret_cast<const float4 *>(p.emb_gamma + blk * 32 + 16 + 4 * bt));
                        }
                    }
                    frag_build<MT>(l, h, act, bt, b, p.emb_fbf + (size_t)blk * (16 * MT), p.emb_foff + (size_t)blk * MT);
                }
            }
            asm volatile("fence.proxy.async;\n" ::: "memory");
        } else {  // MG_ARGMAX
            if (cta == 0) {
                if (warp < B) {
                    float bv = -INFINITY;
                    int bx = 0x7fffffff;
                    for (int c = lane; c < nctas; c += 32)
                        amax_combine(bv, bx, __ldcg(p.am_vals + (size_t)c * 8 + warp), __ldcg(p.am_idx + (size_t)c * 8 + warp));
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                        const int ox = __shfl_xor_sync(0xffffffffu, bx, o);
                        amax_combine(bv, bx, ov, ox);
                    }
                    if (lane == 0) {
                        if (bx == 0x7fffffff) bx = 0;
                        p.d_tok[warp] = bx;
                        const int outpos = p.d_outpos[warp];
                        if (p.d_out) p.d_out[(size_t)warp * p.out_ld + outpos] = bx;
                        p.d_pos[warp] += 1;       // every other CTA read the positions before the preceding barriers
                        p.d_outpos[warp] = outpos + 1;
                    }
                }
                if (tid == 0) *p.d_epoch = epoch + 1;
            }
        }
        if (tracing) p.trace[oi * 6 + 2] = (unsigned long long)clock64();
        if (tr_all) ta[1] = ta[2] = (unsigned long long)clock64();
        // ---- grid barrier between phases
        if (oi + 1 < p.n_ops) {
            abar();   // consumers + epilogue warps: every store of this phase precedes thread 0's arrival
            if (tid == 0) {
                // release: ordered after every consumer thread's stores by the barrier above (cumulativity);
                // acquire: the spin load; the barrier below extends it to the CTA
                red_release_add(&p.bar[0], 1u);
                bar_target += (unsigned)nctas;
                const long long t0 = clock64();
                unsigned n = 0;
                // relaxed polls (an acquire load would invalidate L1 on every iteration), one acquire fence at the end
                while (ld_relaxed_u32(&p.bar[0]) < bar_target) {
                    if ((++n & 0x3FFu) == 0 && clock64() - t0 > MG_SPIN_CYCLES) mg_die(wd_flag, 0x300u + (unsigned)oi);
                }
                asm volatile("fence.acq_rel.gpu;\n" ::: "memory");
            }
            abar();
            if (tracing) p.trace[oi * 6 + 3] = (unsigned long long)clock64();
            if (tr_all) ta[2] = (unsigned long long)clock64();
        }
    }
    // the last CTA to finish re-arms the barrier for the next launch
    if (tid == 0) {
        __threadfence();
        const unsigned old = atomicAdd(&p.bar[1], 1u);
        if (old == (unsigned)nctas - 1u) {
            p.bar[0] = 0u;
            p.bar[1] = 0u;
            __threadfence();
        }
    }
}

template <int MT, int G, int DPL>
void launch_t(const MegaParams &p, const MegaPlan &plan, int grid, cudaStream_t st) {
    static SmemAttr smem_attr;
    cuda_check_mg(ensure_dyn_smem(decode_mega_kernel<MT, G, DPL>, MG_SMEM_MAX, smem_attr), "cudaFuncSetAttribute(decode_mega)");
    // cooperative launch: the runtime refuses the launch (instead of the grid barrier hanging) if the
    // `grid` CTAs cannot all be resident at once
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(MG_THREADS);
    cfg.dynamicSmemBytes = plan.smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cuda_check_mg(cudaLaunchKernelEx(&cfg, decode_mega_kernel<MT, G, DPL>, p), "decode_mega launch");
    tc_count_launch("decode_mega");
}

template <int MT>
void launch_m(const MegaParams &p, const MegaPlan &plan, int grid, cudaStream_t st) {
    const int G = p.H / p.Hkv;
    if (G == 4 && p.hd == 128) launch_t<MT, 4, 4>(p, plan, grid, st);
    else if (G == 2 && p.hd == 32) launch_t<MT, 2, 1>(p, plan, grid, st);
    else fail(VOX_EINVAL, "decode_mega: unsupported attention shape");
}

}  // namespace

bool decode_mega_supported(int B, int H, int Hkv, int hd) {
    if (B < 1 || B > 8 || Hkv <= 0 || H % Hkv != 0) return false;
    const int G = H / Hkv;
    return (G == 4 && hd == 128) || (G == 2 && hd == 32);
}

MegaPlan decode_mega_plan(int B, int max_pairs, int H, int Hkv, int hd) {
    MegaPlan pl;
    pl.MT = B <= 1 ? 1 : (B <= 2 ? 2 : (B <= 4 ? 4 : 8));
    const int G = H / Hkv;
    const int attn_bytes = ((G + 2) * hd + 2 * MG_CWARPS * G + MG_CWARPS * G * hd) * (int)sizeof(float);
    const int per_pair = mg_pair_bytes(pl.MT);
    int cap_pairs = MG_SCRATCH_CAP / per_pair;
    if (cap_pairs >= MG_CHUNK) cap_pairs = cap_pairs / MG_CHUNK * MG_CHUNK;
    pl.Ps_cap = max_pairs < cap_pairs ? max_pairs : cap_pairs;
    if (pl.Ps_cap < 1) pl.Ps_cap = 1;
    int scratch = pl.Ps_cap * per_pair;
    if (scratch < attn_bytes) scratch = attn_bytes;
    pl.scratch_bytes = (scratch + 127) & ~127;
    const int left = MG_SMEM_MAX - mg_misc_bytes(pl.MT) - pl.scratch_bytes;
    const int stage_bytes = mg_nt(pl.MT) * MG_SLOT_BYTES;
    int ns = left / stage_bytes;
    pl.nstage = ns > MG_MAX_STAGES ? MG_MAX_STAGES : ns;
    VOX_CHECK(pl.nstage >= 2, VOX_EINVAL, "decode_mega: no room for the weight ring (%d stages)", pl.nstage);
    pl.smem_bytes = (size_t)mg_misc_bytes(pl.MT) + pl.scratch_bytes + (size_t)pl.nstage * stage_bytes;
    return pl;
}

int decode_mega_grid(int device) {
    int sms = 0;
    cuda_check_mg(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device), "cudaDeviceGetAttribute(SM count)");
    return sms;
}

void launch_decode_mega(const MegaParams &p, const MegaPlan &plan, int grid, cudaStream_t st) {
    VOX_CHECK(p.nstage == plan.nstage && p.scratch_bytes == plan.scratch_bytes, VOX_EINVAL, "decode_mega: plan mismatch");
    switch (plan.MT) {
        case 1: launch_m<1>(p, plan, grid, st); break;
        case 2: launch_m<2>(p, plan, grid, st); break;
        case 4: launch_m<4>(p, plan, grid, st); break;
        case 8: launch_m<8>(p, plan, grid, st); break;
        default: fail(VOX_EINVAL, "decode_mega: bad token capacity");
    }
}

}  // namespace vox
