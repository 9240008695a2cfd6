"""CPU pins of the 8-bit decoder KV cache (vox_session_create_ex(..., VOX_DTYPE_KV_Q8)) that tests/test_kv_q8_gpu.py
relies on.

  * The storage rule, pinned with numpy: each block of 16 head dims x[0..16) stores d = f16_rn(min(a / 127, 65504))
    with a = max |x_i|, and q_i = clamp(rint(x_i / d), -127, 127) (0 when d == 0); a block with a NaN stores d = NaN,
    q = 0.  Decoded: (float)d * q_i.  Ties of x / d, clamping, zero and underflowing blocks, subnormal scales, +-inf and
    NaN are covered.
  * KvQ8Oracle: OracleModel whose decoder attention reads K (after RoPE) and V through that rule -- the function a q8
    session computes.  Unlike f16 the rule is not elementwise: one ulp on a block's largest element can move d and so
    every q of the block.  The encoder's attention is untouched.
  * KV8_LOGIT_REL_BOUND, derived on the decoder-geometry model at windows 8192 (positions 37..52, where the GPU test's
    first steps are) and 383 (positions 450..465) the way KV16_LOGIT_REL_BOUND was: the GPU computes K and V in f32,
    not in f64, so some q (and some d) round the other way.  Emulated by perturbing K and V by 64 f32 ulps before the
    rule; that moves the logits by less than half the bound, and the f32 path's own error against f64
    (LOGIT_REL_BOUND = 1e-4) takes the rest.
  * The read-path mistakes the GPU test is meant to catch -- a neighbouring block's scale, the scale plane off by one
    position, int8 read as uint8, K read for V, a key tile shifted by half a tile, the last key dropped -- move the
    logits past the bound.
  * The f32-KV and f16-KV references differ from the q8 reference by more than the bound at the first steps, so a
    session that ignored the option (or stored f16) would fail the GPU test there.
"""
import numpy as np
import pytest
import torch

from oracle.model import OracleModel
from test_kv_half_ref import PROBE_ROWS, PROBES, KvHalfOracle, _probe_logits, geometry_inputs  # noqa: F401  (fixture)

# per decode step of a q8 session: max |GPU logit - q8-KV f64 logit| <= KV8_LOGIT_REL_BOUND * max(1, max |ref|)
KV8_LOGIT_REL_BOUND = 8e-4
BLOCK = 16
F16_MAX = 65504.0


def kv8_quant(x: np.ndarray):
    """The rule on f32 values x [..., hd]: (q int8 [..., hd], d float16 [..., hd / 16]), bitwise as the kernels store."""
    x = np.asarray(x, np.float32)
    b = x.reshape(*x.shape[:-1], x.shape[-1] // BLOCK, BLOCK)
    nan = np.isnan(b).any(-1)
    a = np.abs(b).max(-1)
    d = np.minimum(a / np.float32(127), np.float32(F16_MAX)).astype(np.float16)
    d[nan] = np.float16(np.nan)
    df = d.astype(np.float32)[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.rint(b / df)
    q = np.clip(r, -127, 127)
    q[~(df[..., 0] > 0)] = 0
    return q.astype(np.int8).reshape(x.shape), d


def kv8_decode(q: np.ndarray, d: np.ndarray) -> np.ndarray:
    """Decoded f32 values: (float)d * q, block by block."""
    qb = q.reshape(*q.shape[:-1], q.shape[-1] // BLOCK, BLOCK).astype(np.float32)
    return (d.astype(np.float32)[..., None] * qb).reshape(q.shape)


def kv8(x: np.ndarray) -> np.ndarray:
    """What a q8 cache returns for K or V computed as x (any float dtype; the rule takes it as f32), as float64."""
    return kv8_decode(*kv8_quant(np.asarray(x, np.float64).astype(np.float32))).astype(np.float64)


class KvQ8Oracle(KvHalfOracle):
    """OracleModel whose decoder attention reads kv8(K after RoPE) and kv8(V).  Applying the rule where attention reads
    the cache equals applying it where the cache is written (the rule is per position and idempotent).  `perturb`
    moves K and V by that relative amount, with a fixed random sign pattern, before the rule; `mistake` names a
    read-path error: the f16 oracle's (k_for_v, half_tile, dropped_tail) or one of the 8-bit format's below."""

    def _round(self, t):
        x = t.numpy().astype(np.float64)
        if self.perturb:
            sign = np.random.default_rng(x.shape[0]).choice([-1.0, 1.0], x.shape)
            x = x * (1.0 + self.perturb * sign)
        q, d = kv8_quant(x.astype(np.float32))
        m = self.mistake
        if m == "neighbour_scale":      # block i decoded with block i ^ 1's scale
            nb = d.shape[-1]
            d = d[..., np.arange(nb) ^ 1]
        elif m == "scale_row_shift":    # the scale plane read one position off
            d = np.roll(d, 1, 0)
        elif m == "uint8":              # the stored bytes read as unsigned
            q = q.view(np.uint8)
        return torch.from_numpy(kv8_decode(q, d).astype(np.float64)).to(t.dtype)


def test_storage_rule_rounds_half_to_even_and_decodes_exactly():
    # a = 127: d = 1, so q = rint(x) with ties to even
    x = np.zeros(BLOCK, np.float32)
    x[:7] = [127.0, 2.5, 3.5, -2.5, -3.5, 0.5, -0.5]
    q, d = kv8_quant(x)
    assert d[0] == np.float16(1.0)
    assert q[:7].tolist() == [127, 2, 4, -2, -4, 0, 0]
    # random blocks: |q| <= 127 (never -128), the decoded value within d / 2 of x, and the product exact in f32
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((4000, 128)) * np.exp(rng.uniform(-12, 12, (4000, 1)))).astype(np.float32)
    q, d = kv8_quant(x)
    assert q.min() >= -127 and q.max() <= 127
    dec = kv8_decode(q, d)
    dd = np.repeat(d.astype(np.float64), BLOCK, -1)
    assert np.array_equal(dec.astype(np.float64), dd * q.astype(np.float64))
    # with a normal d (relative rounding <= 2^-11, so a / d < 127.07) nothing clamps: each value within d / 2, and the
    # block's largest element stores +-127.  (Subnormal scales: test_storage_rule_clamps_when_the_scale_rounds_down.)
    normal = dd >= 2.0 ** -14
    assert normal.mean() > 0.5
    assert np.all((np.abs(dec.astype(np.float64) - x) <= dd / 2 * (1 + 1e-6))[normal])
    qmax = np.abs(q.reshape(4000, 8, BLOCK).astype(np.int32)).max(-1)
    assert np.all(qmax[d.astype(np.float64) >= 2.0 ** -14] == 127)


def test_storage_rule_clamps_when_the_scale_rounds_down():
    # d subnormal: a / 127 = 64.3 f16 subnormal ulps rounds down to 64, so a / d = 127.59 and rint gives 128 -> 127
    a = np.float32(127 * 64.3 * 2.0 ** -24)
    x = np.zeros(BLOCK, np.float32)
    x[0], x[1] = a, -a
    q, d = kv8_quant(x)
    assert d[0] == np.float16(64 * 2.0 ** -24) and float(d[0]) < float(a / np.float32(127))
    assert np.rint(a / np.float32(d[0])) == 128
    assert q[0] == 127 and q[1] == -127


def test_storage_rule_zero_underflow_inf_and_nan_blocks():
    z = np.zeros(BLOCK, np.float32)
    q, d = kv8_quant(z)
    assert d[0] == 0 and not q.any()
    tiny = np.full(BLOCK, 1e-10, np.float32)     # a / 127 underflows f16: d = 0, every q = 0, decodes to 0
    q, d = kv8_quant(tiny)
    assert d[0] == 0 and not q.any() and not kv8_decode(q, d).any()
    sub = np.linspace(-3e-4, 3e-4, BLOCK).astype(np.float32)   # d subnormal (< 2^-14): a coarser scale, still decoded
    q, d = kv8_quant(sub)
    assert 0 < float(d[0]) < 2.0 ** -14 and np.abs(q).max() >= 124
    assert np.abs(kv8_decode(q, d) - sub).max() <= float(d[0])
    big = np.linspace(-1.0, 1.0, BLOCK).astype(np.float32)
    big[3], big[7] = np.inf, -np.inf                           # d = 65504; inf / d clamps
    q, d = kv8_quant(big)
    assert d[0] == np.float16(F16_MAX) and q[3] == 127 and q[7] == -127 and q[0] == 0
    huge = np.full(BLOCK, 3e38, np.float32)                    # a / 127 past the f16 range: d = 65504
    q, d = kv8_quant(huge)
    assert d[0] == np.float16(F16_MAX) and np.all(q == 127)
    nan = np.arange(2 * BLOCK, dtype=np.float32)
    nan[BLOCK + 5] = np.nan                                    # only the second block is NaN
    q, d = kv8_quant(nan)
    assert np.isnan(d[1]) and not q[BLOCK:].any() and np.isnan(kv8_decode(q, d)[BLOCK:]).all()
    assert np.isfinite(kv8_decode(q, d)[:BLOCK]).all()


@pytest.mark.parametrize("window", sorted(PROBES))
def test_kv8_bound_covers_rounding_flips_and_not_read_mistakes(geometry_inputs, window):  # noqa: F811
    data, x, ada = geometry_inputs
    p0 = PROBES[window]

    def logits(cls=KvQ8Oracle, **kw):
        o = cls(data, dtype=torch.float64, **kw)
        o.cfg.dec_window = window
        return _probe_logits(o, x, ada, p0)

    ref = logits()
    bound = KV8_LOGIT_REL_BOUND * np.maximum(1.0, np.abs(ref).max(-1))
    ratios = {}
    # f32-versus-f64 differences of K and V before the rule flip some q and d
    ratios["perturb"] = (np.abs(logits(perturb=64 * 2.0 ** -24) - ref).max(-1) / bound).max()
    assert ratios["perturb"] < 0.5, ratios
    for m in ("neighbour_scale", "scale_row_shift", "uint8", "k_for_v", "half_tile", "dropped_tail"):
        ratios[m] = (np.abs(logits(mistake=m) - ref).max(-1) / bound).max()
        assert ratios[m] > 5, (window, m, ratios[m])
    # a session that ignored kv_dtype, or stored f16
    if window == 8192:
        o32 = OracleModel(data, dtype=torch.float64)
        o32.cfg.dec_window = window
        ratios["f32_kv"] = (np.abs(_probe_logits(o32, x, ada, p0) - ref).max(-1) / bound).max()
        ratios["f16_kv"] = (np.abs(logits(KvHalfOracle) - ref).max(-1) / bound).max()
        assert ratios["f32_kv"] > 1 and ratios["f16_kv"] > 1, ratios
    print(f"\n[kv8] window {window}, positions {p0}..{p0 + PROBE_ROWS - 1}: largest logit change as a multiple of "
          "the bound: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))

