"""CPU side of the Q4_0 format-edge tests (tests/test_q4_format_edges_gpu.py runs the CUDA kernels on the same inputs).

  * the sign-flipped twin: real Q4_0 files carry negative block scales (ggml's quantiser sets d = max / -8 with `max`
    the signed element of largest magnitude, so every block whose largest weight is positive gets d < 0), while every
    synthetic scale is positive.  sign_flipped_twin rewrites a seeded half of the blocks whose nibbles are all in 1..15
    as (-d, 16 - n): the same weights, since (n - 8) * d = ((16 - n) - 8) * (-d) exactly (a weight of 0 keeps its value
    and changes the sign of its zero);
  * the f64 reference can see a lost sign: the twin with those blocks' sign bits cleared again is far outside the
    decode logit bound;
  * the wgmma GEMM's exact domain: an emulation of its weight dequantisation (nibble -> f32, Veltkamp split, f16 bit
    patterns by shifts and masks) over every finite f16 scale and every nibble is exact if and only if |d| < 32;
  * the GPU bound comes from the algorithms: the numpy models of the tensor-core matvec and of the wgmma GEMM
    (tests/test_fragment_numerics.py) stay below a quarter of it on every weight / activation set the GPU test uses.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle import q4 as oq4
from oracle.gguf_synth import Q4_0_T, GgufFile, nbytes_of
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes
from test_fragment_numerics import gemm_split_model, pack_q4, tc_matvec_model

TWIN_SEED = 11

# ------------------------------------------------------------------------------------------- the sign-flipped twin


def sign_flipped_twin(data: bytes, seed: int, keep_sign: bool = True) -> bytes:
    """`data` with a seeded half of the Q4_0 blocks whose nibbles are all in 1..15 rewritten as (-d, 16 - n).
    keep_sign=False writes (d, 16 - n) instead: the same blocks with the sign lost.  Aliased tensors share a payload,
    which is rewritten once."""
    g = GgufFile(data)
    out = bytearray(data)
    rng = np.random.default_rng(seed)
    done = set()
    for dt, shape, off in g.tensors.values():
        if dt != Q4_0_T or off in done:
            continue
        done.add(off)
        a = g.data_off + off
        blk = np.frombuffer(data, np.uint8, nbytes_of(dt, shape), a).reshape(-1, 18).copy()
        lo, hi = blk[:, 2:] & 0x0F, blk[:, 2:] >> 4
        flip = np.all(lo != 0, 1) & np.all(hi != 0, 1) & (rng.random(len(blk)) < 0.5)
        if keep_sign:
            blk[flip, 1] ^= 0x80                      # f16 sign bit (little-endian high byte)
        blk[flip, 2:] = (16 - lo[flip]) | ((16 - hi[flip]) << 4)
        out[a:a + blk.size] = blk.tobytes()
    return bytes(out)


def q4_payload_mask(g: GgufFile, size: int) -> np.ndarray:
    mask = np.zeros(size, bool)
    for dt, shape, off in g.tensors.values():
        if dt == Q4_0_T:
            mask[g.data_off + off:g.data_off + off + nbytes_of(dt, shape)] = True
    return mask


@pytest.fixture(scope="module")
def geometry_twin():
    data = geometry_model_bytes(40)
    return data, sign_flipped_twin(data, TWIN_SEED)


def test_twin_dequantises_to_the_same_weights(geometry_twin):
    data, twin = geometry_twin
    g, gt = GgufFile(data), GgufFile(twin)
    assert g.tensors == gt.tensors
    for name, (dt, _, _) in g.tensors.items():
        if dt == Q4_0_T:
            a, b = oq4.dequantize_q4_0(g.raw(name)), oq4.dequantize_q4_0(gt.raw(name))
            assert np.array_equal(a, b), name                 # equal values (+0 and -0 compare equal)


def test_twin_flips_a_quarter_of_every_q4_tensor(geometry_twin):
    data, twin = geometry_twin
    g, gt = GgufFile(data), GgufFile(twin)
    seen = {"encoder": 0, "adapter": 0, "ada": 0, "decoder": 0, "tok_emb": 0}
    for name, (dt, _, _) in g.tensors.items():
        if dt != Q4_0_T:
            continue
        d0 = g.raw(name).reshape(-1, 18)[:, :2].copy().view(np.float16)[:, 0]
        d1 = gt.raw(name).reshape(-1, 18)[:, :2].copy().view(np.float16)[:, 0]
        assert np.all(d0 > 0), name                            # the synthetic scales are all positive
        frac = float(np.mean(d1 < 0))
        assert frac >= 0.25, (name, frac)
        assert np.array_equal(np.abs(d0), np.abs(d1)), name
        kind = ("encoder" if "whisper_encoder" in name else "adapter" if "audio_language_projection" in name else
                "tok_emb" if "tok_embeddings" in name else "ada" if "ada_rms_norm" in name else "decoder")
        seen[kind] += 1
    assert all(seen.values()), seen
    # nothing but Q4 payloads changed: header, norms, biases, conv weights and padding are byte-identical
    a, b = np.frombuffer(data, np.uint8), np.frombuffer(twin, np.uint8)
    mask = q4_payload_mask(g, a.size)
    assert np.array_equal(a[~mask], b[~mask])
    assert np.mean(a[mask] != b[mask]) > 0.2


def test_lost_sign_exceeds_logit_bound(geometry_twin):
    """A kernel that dropped the sign of d would compute the twin with its flipped blocks at (+d, 16 - n).  That model's
    f64 logits differ from the original's by more than 20x the decode test's bound at every position, so the GPU tests
    on the twin would see such a defect."""
    data, _ = geometry_twin
    lost = sign_flipped_twin(data, TWIN_SEED, keep_sign=False)
    o64 = OracleModel(data, dtype=torch.float64)
    o64_lost = OracleModel(lost, dtype=torch.float64)
    mel = omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(6.0, 1234)))
    emb = OracleModel(data).encode_audio(mel)
    ids = np.random.default_rng(1).integers(0, o64.cfg.vocab, emb.shape[0])
    ids[:PREFIX_LEN] = [1] + [32] * (PREFIX_LEN - 1)
    t_embed = omel.time_embedding(6.0, o64.cfg.dec_dim)
    ref = o64.forward_streaming(None, ids.tolist(), t_embed, audio_embeds=emb).numpy()
    other = o64_lost.forward_streaming(None, ids.tolist(), t_embed, audio_embeds=emb).numpy()
    bound = LOGIT_REL_BOUND * np.maximum(1.0, np.abs(ref).max(-1))
    ratio = np.abs(other - ref).max(-1) / bound
    print(f"\n[lost sign] {ratio.size} positions: min max|dlogit| = {ratio.min():.0f}x the bound")
    assert ratio.min() > 20, (int(np.argmin(ratio)), ratio.min())


# ------------------------------------------------------------------------- the wgmma GEMM's weight dequantisation


def k3_weight_split(d16: np.ndarray, n: np.ndarray) -> np.ndarray:
    """gemm_tc5_kernel's dequantisation of nibble n with block scale d16 (f16), step by step in f32 (no FMA
    contraction, denormals kept), returning w_hi + w_lo as the f16 pieces the MMAs read, in f64 (value * 2^8)."""
    F = np.float32
    dd = (d16.astype(F) * F(256.0)).astype(F) * F(2.0 ** -112)
    nf = (np.uint32(0x4B000000) | n.astype(np.uint32)).view(F)
    w = ((nf - F(8388616.0)).astype(F) * dd).astype(F)
    c = (w * F(8193.0)).astype(F)
    hi = (c - (c - w).astype(F)).astype(F)
    lo = (w - hi).astype(F)

    def pack(v):   # g5_pack_f16x2, one lane
        b = v.view(np.uint32)
        return (((b >> np.uint32(13)) & np.uint32(0x7FFF)) | ((b >> np.uint32(16)) & np.uint32(0x8000))).astype(
            np.uint16).view(np.float16)

    return pack(hi).astype(np.float64) + pack(lo).astype(np.float64)


def test_k3_split_is_exact_iff_scale_below_32():
    bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    d = bits.view(np.float16)
    d = d[np.isfinite(d)]
    assert d.size == 63488
    nib = np.arange(16, dtype=np.uint32)
    with np.errstate(all="ignore"):
        got = k3_weight_split(d[:, None], nib[None, :])
        want = (nib[None, :].astype(np.float64) - 8.0) * d[:, None].astype(np.float64) * 256.0
    exact = np.all(got == want, axis=1)
    small = np.abs(d.astype(np.float64)) < 32.0
    wrong = d[~exact].astype(np.float64)
    print(f"\n[K3 split] {int(exact.sum())} of {d.size} finite f16 scales exact; smallest inexact |d| = "
          f"{np.abs(wrong).min():g}; d=32 nibble 0 -> {got[d == 32][0, 0]}, d=64 nibble 0 -> {got[d == 64][0, 0]}")
    assert np.array_equal(exact, small)
    assert d.view(np.uint16)[small].max() & 0x7FFF == 0x4FFF        # the test upload_q4 applies: (bits & 0x7FFF) < 0x5000
    assert np.array_equal(small, (d.view(np.uint16) & 0x7FFF) < 0x5000)


# ----------------------------------------------------------------------- weight and activation sets, and the bound

WEIGHT_SETS = ("signed", "f16_subnormal", "zero_blocks", "nibbles_0_15",
               "d8", "d31.98", "d32", "d64", "d1000", "d65504")
ACT_SETS = ("gauss", "outlier_1e4", "blocks_1e5", "zeros", "neg_zero", "f32_subnormal", "rows_1e-30", "rows_1e30")


def large_d(wset: str) -> bool:
    return wset.startswith("d") and float(wset[1:]) >= 8


def pairs():
    """(weight set, activation set) pairs whose products stay below 1e37: large scales skip the 1e30 rows."""
    return [(w, a) for w in WEIGHT_SETS for a in ACT_SETS if not (large_d(w) and a == "rows_1e30")]


def make_weights(wset: str, n: int, k: int, seed: int) -> np.ndarray:
    """Q4_0 bytes of an N x K weight: random nibbles 0..15, scales of random sign."""
    rng = np.random.default_rng(seed)
    kb = k // 32
    q = rng.integers(0, 16, (n, k))
    q[::7, :32] = 0                                              # a whole block of nibble 0 (-8 d) in every 7th row
    mag = rng.uniform(0.002, 0.02, (n, kb))
    if wset == "f16_subnormal":
        mag = rng.integers(1, 1024, (n, kb)) * 2.0 ** -24        # f16 subnormals, down to 2^-24
        mag[:, ::5] = 2.0 ** -24
    elif wset == "zero_blocks":
        mag[rng.random((n, kb)) < 0.3] = 0.0                      # +0 and -0 scales (random sign below)
    elif wset == "nibbles_0_15":
        pick = rng.random((n, k)) < 0.8
        q[pick] = np.where(rng.random(int(pick.sum())) < 0.5, 0, 15)
    elif wset.startswith("d") and wset != "d":
        mag[:] = float(wset[1:])
    d = (mag * np.where(rng.random((n, kb)) < 0.5, -1.0, 1.0)).astype(np.float16)
    return pack_q4(d, q)


def make_acts(aset: str, m: int, k: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((m, k)) * rng.uniform(0.1, 3.0, (m, 1))
    xb = x.reshape(m, k // 32, 32)
    if aset == "outlier_1e4":
        x[np.arange(m), rng.integers(0, k, m)] = 1e4 * np.where(rng.random(m) < 0.5, -1, 1)
    elif aset == "blocks_1e5":
        xb[:, 0::3] *= 1e5
        xb[:, 1::3] *= 1e-5
    elif aset == "zeros":
        xb[:, 1::3] = 0.0
        x[1::4] = 0.0
    elif aset == "neg_zero":
        x[:, ::7] = -0.0
        xb[:, -1] = -0.0
    elif aset == "f32_subnormal":
        sub = rng.integers(1, 1 << 23, (m, k)).astype(np.float64) * 2.0 ** -149 * np.where(rng.random((m, k)) < .5, -1, 1)
        x[:, ::3] = sub[:, ::3]
        xb[:, 1] = sub.reshape(m, k // 32, 32)[:, 1]            # one whole block of subnormals
    elif aset == "rows_1e-30":
        x[(np.arange(m) % 3) != 2] *= 1e-30
    elif aset == "rows_1e30":
        x[(np.arange(m) % 3) != 2] *= 1e30
    return x.astype(np.float32)


def scales_of(raw: np.ndarray, n: int, k: int) -> np.ndarray:
    return np.repeat(raw.reshape(n, k // 32, 18)[:, :, :2].copy().view(np.float16)[:, :, 0].astype(np.float64), 32, 1)


def largest_term(x64: np.ndarray, wd: np.ndarray, top: int = 4) -> np.ndarray:
    """[M, N] upper bound of max_k wd[n, k] |x[m, k]|: exact over each row's `top` largest |x|, and the next |x| times
    max_k wd for the rest."""
    ax = np.abs(x64)
    order = np.argsort(ax, axis=1)
    out = np.empty((ax.shape[0], wd.shape[0]))
    wmax = wd.max(1)
    for m in range(ax.shape[0]):
        idx = order[m, -top:]
        rest = ax[m, order[m, -top - 1]] if ax.shape[1] > top else 0.0
        out[m] = np.maximum((wd[:, idx] * ax[m, idx]).max(1), rest * wmax)
    return out


def f64_and_bound(raw: np.ndarray, n: int, k: int, x: np.ndarray, bias=None):
    """(y64, bound): the f64 product (+ bias) and the per-output bound
        2^-20 * sum_k (|w_k| + 16 |d_b|) |x_k|  +  2^-15 * max_k (|w_k| + 16 |d_b|) |x_k|  +  |bias| * 2^-23.
    The first term is the error scale of the re-associated matvec form, whose terms n |x| |d| and 8 |x| |d| are at most
    16 |d| |x|.  The second is the floor of accumulation when one term dominates the row (an activation outlier): from
    the step that adds it on, the running sum is that term, so later roundings are relative to it rather than to the
    spread sum.  On the tensor cores an MMA aligns its 16 products to the largest and truncates, up to 2^-23 of it per
    product; a 32-block of the matvec takes four MMAs (two k-groups, x_hi and x_mid): 2^6 * 2^-23 = 2^-17.  The factor
    4 above that covers the f32 additions of the chain that follow (block sums, k-steps, split-K slices), which round
    at 2^-24 of the same term.  It does not grow with K: what grows with K is the spread sum, in the first term."""
    w = oq4.dequantize_q4_0(raw).reshape(n, k).astype(np.float64)
    x64 = x.astype(np.float64)
    y = x64 @ w.T
    wd = np.abs(w) + 16.0 * np.abs(scales_of(raw, n, k))
    bound = 2.0 ** -20 * (np.abs(x64) @ wd.T) + 2.0 ** -15 * largest_term(x64, wd)
    if bias is not None:
        y = y + bias.astype(np.float64)
        bound = bound + np.abs(bias.astype(np.float64)) * 2.0 ** -23
    return y, bound


@pytest.mark.parametrize("wset,aset", pairs())
def test_algorithm_models_within_a_quarter_of_the_bound(wset, aset):
    """The matvec model (every row, K = 4192: 131 blocks) and, inside the GEMM's |d| < 32 domain, the GEMM model
    (K = 4160) against the f64 product: worst |model - y64| / bound < 1/4."""
    n, m = 24, 6
    worst = {}
    k = 4192
    raw = make_weights(wset, n, k, 1)
    x = make_acts(aset, m, k, 2)
    y64, bound = f64_and_bound(raw, n, k, x)
    assert np.all(np.abs(y64) < 1e37)
    with np.errstate(all="ignore"):
        tc = np.stack([tc_matvec_model(x[i], raw, n, k).astype(np.float64) for i in range(m)])
    worst["matvec"] = float((np.abs(tc - y64) / np.maximum(bound, 1e-300)).max())
    if not (large_d(wset) and float(wset[1:]) >= 32):
        k = 4160
        raw = make_weights(wset, n, k, 3)
        x = make_acts(aset, m, k, 4)
        y64, bound = f64_and_bound(raw, n, k, x)
        g = gemm_split_model(x, raw, n, k)
        worst["gemm"] = float((np.abs(g - y64) / np.maximum(bound, 1e-300)).max())
    print(f"\n[model / bound] {wset:>13s} x {aset:<13s} " + "  ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    assert max(worst.values()) < 0.25, worst
