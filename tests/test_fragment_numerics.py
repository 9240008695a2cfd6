"""Numerical model (numpy) of the tensor-core Q4 matvec arithmetic used by matvec_tc.cu / decode_mega.cu:

    y = sum_blocks d_b * ( (sum_k n_k * hi_k + sum_k n_k * mid_k) * 2^24/s_b  -  8 * sum_k x_k )

with n = nibbles as the f16 subnormals n * 2^-24, x scaled per 32-block by the power of two s_b that puts the block
maximum in [2^7, 2^8) and split into two f16 pieces hi = f16(x s), mid = f16(x s - hi), f32 accumulation.  This does
not run the CUDA code (the GPU parity tests do); it pins the ALGORITHM's accuracy claim against an f64 reference,
including adversarial activations: the error is f32 rounding relative to  sum_b d_b * sum_k (n_k + 8) |x_k|  (the
magnitude of the two re-associated terms  sum n x  and  8 sum x), independent of the dynamic range across blocks.
That is the same scale as the strict-order f32 loop's error (sum |w||x|) except for weights whose nibble is exactly 8
(w = 0) sitting on an activation outlier: there the strict loop adds an exact 0 and this scheme a rounding residue of
~ 8 d |x| 2^-24 -- the same absolute error every other row already has."""
import numpy as np

from oracle import q4 as oq4

F32 = np.float32


def tc_matvec_model(x: np.ndarray, raw: np.ndarray, n: int, k: int) -> np.ndarray:
    blocks = raw.reshape(n, k // 32, 18)
    d = blocks[:, :, :2].copy().view(np.float16).astype(F32)[:, :, 0]          # [n, kb]
    qs = blocks[:, :, 2:]
    nib = np.concatenate([(qs & 0x0F), (qs >> 4)], axis=2).astype(F32)         # [n, kb, 32] element order
    xb = x.reshape(k // 32, 32).astype(F32)
    bm = np.abs(xb).max(axis=1)
    e = np.where(bm > 0, np.floor(np.log2(np.where(bm > 0, bm, 1.0))), 7).astype(np.int32)
    e = np.clip(e, -100, 100)
    s = np.ldexp(F32(1.0), (7 - e)).astype(F32)                                 # block max -> [2^7, 2^8)
    inv = np.ldexp(F32(1.0), (17 + e)).astype(F32)                              # 2^24 / s
    ev = (xb * s[:, None]).astype(F32)
    ev[:, 16:] = (ev[:, 16:] * F32(0.0625)).astype(F32)                         # high nibbles enter as 16 n 2^-24
    hi = ev.astype(np.float16).astype(F32)
    mid = (ev - hi).astype(np.float16).astype(F32)
    a = nib.copy()
    a[:, :, :16] *= F32(2.0 ** -24)
    a[:, :, 16:] *= F32(16.0 * 2.0 ** -24)
    # tensor-core block sums: exact products, f32 accumulation (order is irrelevant at this magnitude)
    cc = (a * hi[None]).astype(F32).sum(axis=2, dtype=F32) + (a * mid[None]).astype(F32).sum(axis=2, dtype=F32)
    off = (F32(-8.0) * xb.sum(axis=1, dtype=F32)).astype(F32)
    per_block = (d * (cc * inv[None] + off[None]).astype(F32)).astype(F32)
    return per_block.sum(axis=1, dtype=F32)


def pack_q4(d: np.ndarray, q: np.ndarray) -> np.ndarray:
    """Q4_0 bytes of f16 scales d [N, K/32] and nibbles q [N, K] (element i low, i + 16 high nibble of byte i)."""
    n, kb = d.shape
    qb = q.reshape(n, kb, 32).astype(np.uint8)
    raw = np.empty((n, kb, 18), np.uint8)
    raw[:, :, :2] = d.astype(np.float16).reshape(n, kb, 1).view(np.uint8)
    raw[:, :, 2:] = qb[:, :, :16] | (qb[:, :, 16:] << 4)
    return raw.reshape(-1)


def gemm_split_weights(raw: np.ndarray, n: int, k: int):
    """The wgmma GEMM's weight pieces: (q-8)*d' as f16 hi + the f16 residual lo, d' = f16(d * 2^8).  Exact inside the
    kernel's |d| < 32 domain."""
    blocks = raw.reshape(n, k // 32, 18)
    d = blocks[:, :, :2].copy().view(np.float16)[:, :, 0]
    qs = blocks[:, :, 2:]
    n8 = np.concatenate([(qs & 0x0F), (qs >> 4)], axis=2).reshape(n, k).astype(np.float64) - 8.0
    d2 = np.repeat((d.astype(np.float32) * 256).astype(np.float16), 32, 1).astype(np.float64)
    hi = (n8 * d2).astype(np.float16)                                  # HMUL2: RN_f16(n8 * d')
    lo = (n8 * d2 - hi.astype(np.float64)).astype(np.float16)          # HFMA2: the residual
    return n8 * d2, hi, lo


def gemm_split_model(x: np.ndarray, raw: np.ndarray, n: int, k: int) -> np.ndarray:
    """numpy model of the wgmma GEMM (csrc/gemm_tc5.cu): x [M, K] times the per-token power of two that puts the row
    maximum (x 1.0001) in [2^7, 2^8) (exponent clamped to +-100, all-zero rows scale 1) as f16 hi + mid; products
    w_hi x_h + w_hi x_m + w_lo x_h in f64 (the MMA accumulates in f32).  Returns [M, N] in f64."""
    _, hi, lo = gemm_split_weights(raw, n, k)
    x64 = np.asarray(x, np.float32).astype(np.float64)
    mx = np.abs(x64).max(1) * 1.0001
    e0 = np.where(mx > 0, np.frexp(mx)[1] - 1, 7)                      # floor(log2(mx))
    e = np.clip(e0, -100, 100)
    sc = np.ldexp(1.0, 7 - e)[:, None]
    xs = x64 * sc
    xh = xs.astype(np.float16)
    xm = (xs - xh.astype(np.float64)).astype(np.float16)
    assert np.all(np.isfinite(xh.astype(np.float64))) and np.all((np.abs(xs).max(1) < 256.0) | (e != e0))
    h, l = hi.astype(np.float64), lo.astype(np.float64)
    return (xh.astype(np.float64) @ h.T + xm.astype(np.float64) @ h.T + xh.astype(np.float64) @ l.T) / sc / 256.0


def _case(x, n=64, seed=0):
    k = x.size
    rng = np.random.default_rng(seed)
    raw = np.empty((n * k // 32, 18), np.uint8)
    raw[:, :2] = rng.uniform(0.002, 0.02, n * k // 32).astype(np.float16).view(np.uint8).reshape(-1, 2)
    raw[:, 2:] = rng.integers(0, 256, (n * k // 32, 16), dtype=np.uint8)
    raw = raw.reshape(-1)
    w = oq4.dequantize_q4_0(raw).reshape(n, k).astype(np.float64)
    exact = w @ x.astype(np.float64)
    # error scale of the re-associated form: sum_b d_b * sum_k (n_k + 8) |x_k|  (>= sum |w||x|)
    blocks = raw.reshape(n, k // 32, 18)
    dd = np.repeat(blocks[:, :, :2].copy().view(np.float16).astype(np.float64)[:, :, 0], 32, axis=1)
    scale = (np.abs(w) + 16.0 * dd) @ np.abs(x.astype(np.float64))
    model = tc_matvec_model(x.astype(F32), raw, n, k).astype(np.float64)
    ref32 = oq4.q4_matmul_c(x.astype(F32)[None], raw, n, k)[0].astype(np.float64)
    return np.abs(model - exact) / scale, np.abs(ref32 - exact) / scale


def test_accuracy_is_f32_grade_for_gaussian_activations():
    rng = np.random.default_rng(1)
    em, er = _case(rng.standard_normal(3072).astype(F32))
    assert em.max() < 4e-7 and em.max() < 4 * er.max() + 1e-7


def test_accuracy_independent_of_dynamic_range_across_blocks():
    rng = np.random.default_rng(2)
    x = rng.standard_normal(3072).astype(F32)
    x[:1024] *= F32(1e4)
    x[1024:2048] *= F32(1e-5)
    em, er = _case(x, seed=3)
    assert em.max() < 4e-7 and em.max() < 4 * er.max() + 1e-7


def test_outlier_inside_a_block_and_zero_blocks():
    rng = np.random.default_rng(4)
    x = (rng.standard_normal(3072) * 1e-3).astype(F32)
    x[5] = F32(300.0)          # one huge value: its block's small entries keep >= 22 bits relative to the block max
    x[64:128] = 0.0            # all-zero blocks: scale 1, contributes exactly nothing
    x[200] = F32(-0.0)
    em, er = _case(x, seed=5)
    assert em.max() < 4e-7 and em.max() < 4 * er.max() + 1e-7


def test_tiny_and_huge_magnitudes():
    rng = np.random.default_rng(6)
    for mag in (1e-30, 1e-12, 1e12, 1e28):
        em, _ = _case((rng.standard_normal(1024) * mag).astype(F32), seed=7)
        assert em.max() < 4e-7, mag


def test_gemm_f16_two_by_two_split_three_products():
    """numpy model of the wgmma GEMM's operand split (csrc/gemm_tc5.cu): weights (q-8)*d*2^8 as f16 hi + the
    exact f16 residual, activations * 2^s_t as f16 hi + mid, products w_hi x_h + w_hi x_m + w_lo x_h in f64 (the MMA
    accumulates in f32).  Error relative to sum |w||x| stays at the f32 rounding level even with outlier activations and
    tiny / large block scales -- i.e. 3 MMAs per k-step carry f32-grade accuracy (round 1 spent 5 on bf16 pieces)."""
    rng = np.random.default_rng(0)
    K, N, M = 5120, 48, 12
    for dscale in (1e-4, 1e-2, 3.0):
        d = (rng.uniform(0.5, 1.5, (N, K // 32)) * dscale).astype(np.float16)
        q = rng.integers(0, 16, (N, K))
        n8 = (q - 8).astype(np.float64)
        w = n8 * np.repeat(d.astype(np.float64), 32, 1)
        x = (rng.standard_normal((M, K)) * rng.uniform(0.01, 30, (M, 1))).astype(np.float32)
        x[:, ::97] *= 50.0
        raw = pack_q4(d, q)
        wd, hi, lo = gemm_split_weights(raw, N, K)
        assert np.all(np.isfinite(hi.astype(np.float64)))
        if dscale >= 1e-2:                                                 # normal range: the split is exact
            assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), wd)
        got = gemm_split_model(x, raw, N, K)
        exact = x.astype(np.float64) @ w.T
        den = np.abs(x.astype(np.float64)) @ np.abs(w).T
        err = float((np.abs(got - exact) / den).max())
        assert err < 2.0 ** -22, (dscale, err)
