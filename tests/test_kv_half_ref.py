"""CPU pins of the f16 decoder KV cache (vox_session_create_ex(..., VOX_DTYPE_F16)) that tests/test_kv_half_gpu.py
relies on.

  * The storage rule, pinned with numpy: inside the f16 range a value stores as np.float16 (round to nearest even),
    past it the value is clamped to +-65504 first (never +-inf), NaN stays NaN.
  * KvHalfOracle: OracleModel whose decoder attention reads K (after RoPE) and V rounded by that rule -- the function
    an f16 session computes.  The encoder's attention is untouched.
  * KV16_LOGIT_REL_BOUND, derived on the decoder-geometry model at windows 8192 (positions 37..52, where the GPU test's
    first steps are) and 383 (positions 450..465): the GPU computes K and V in f32 through the Q4 kernels, not in f64, so
    some values round to the neighbouring f16 value.  Emulated by perturbing K and V by 64 f32 ulps (3.8e-6, about what
    the GPU's first steps show) before the rounding, that moves the logits by less than half the bound; the f32 path's
    own error against f64 (LOGIT_REL_BOUND = 1e-4, at most 2.5e-5 measured) takes the rest.
  * The read-path mistakes the GPU test is meant to catch -- a key tile shifted by half a tile, the last key dropped,
    K read in place of V, the two halves of an f16 pair swapped when widening -- move the logits past the bound.
  * The f16-KV reference differs from the f32-KV reference by more than the bound at the first steps, so a session that
    ignored the option would fail the GPU test there.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import geometry_model_bytes

# per decode step of an f16 session: max |GPU logit - f16-KV f64 logit| <= KV16_LOGIT_REL_BOUND * max(1, max |ref|)
KV16_LOGIT_REL_BOUND = 1.5e-4
F16_MAX = 65504.0
PROBE_ROWS = 16
PROBES = {8192: PREFIX_LEN - 1, 383: 450}   # the prefill's last row on; a 90 s utterance gives ~590 positions


def kv16(x: np.ndarray) -> np.ndarray:
    """The stored value of x (any float dtype) as float64: clamp to [-65504, 65504], then round to nearest even."""
    x = np.asarray(x, np.float64)
    return np.clip(x, -F16_MAX, F16_MAX).astype(np.float16).astype(np.float64)   # np.clip keeps NaN


def kv16_from_f32(x: np.ndarray) -> np.ndarray:
    """The same rule applied to f32 values, as the kernels apply it (bitwise: float16 bits)."""
    x = np.asarray(x, np.float32)
    return np.clip(x, np.float32(-F16_MAX), np.float32(F16_MAX)).astype(np.float16)


class KvHalfOracle(OracleModel):
    """OracleModel whose decoder caches hold kv16(K after RoPE) and kv16(V).  Rounding where attention reads the cache
    equals rounding where it is stored: the rule is elementwise and idempotent.  `perturb` (relative size) moves K and V
    by that much, with a fixed random sign pattern, before the rounding; `mistake` names a read-path error."""

    def __init__(self, *a, perturb=0.0, mistake=None, **kw):
        super().__init__(*a, **kw)
        self.perturb, self.mistake, self._decoding = perturb, mistake, False

    def decoder_forward_with_cache(self, *a, **kw):
        self._decoding = True
        try:
            return super().decoder_forward_with_cache(*a, **kw)
        finally:
            self._decoding = False

    def decoder_forward_batched(self, *a, **kw):
        self._decoding = True
        try:
            return super().decoder_forward_batched(*a, **kw)
        finally:
            self._decoding = False

    def _round(self, t):
        x = t.numpy().astype(np.float64)
        if self.perturb:
            sign = np.random.default_rng(x.shape[0]).choice([-1.0, 1.0], x.shape)
            x = x * (1.0 + self.perturb * sign)
        return torch.from_numpy(kv16(x)).to(t.dtype)

    def _attention(self, q, k, v, scale, q_offset, window, causal=True):
        if not self._decoding:
            return super()._attention(q, k, v, scale, q_offset, window, causal)
        k, v = self._round(k), self._round(v)
        m = self.mistake
        if m == "k_for_v":
            v = k
        elif m == "dropped_tail":   # the newest key of every row's window is never read
            out = [super(KvHalfOracle, self)._attention(q[i:i + 1], k[:q_offset + i], v[:q_offset + i], scale,
                                                        q_offset + i, window, causal) for i in range(q.shape[0])]
            return torch.cat(out)
        elif m == "half_tile":      # the keys of the window read 16 positions late (half a 32-key tile)
            k, v = torch.roll(k, 16, 0), torch.roll(v, 16, 0)
        elif m == "pair_swap":      # elements (2i, 2i+1) of every row swapped when widening an f16 pair
            hd = k.shape[-1]
            k = k.reshape(*k.shape[:-1], hd // 2, 2).flip(-1).reshape(k.shape)
            v = v.reshape(*v.shape[:-1], hd // 2, 2).flip(-1).reshape(v.shape)
        return super()._attention(q, k, v, scale, q_offset, window, causal)


def test_storage_rule_inside_range_is_float16_round_to_nearest_even():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(100000) * np.exp(rng.uniform(-20, 11, 100000))).astype(np.float32)
    x = x[np.abs(x) < F16_MAX]
    assert np.array_equal(kv16_from_f32(x), x.astype(np.float16))
    # ties go to even: 1 + 2^-11 lies halfway between 1 and 1 + 2^-10
    assert kv16_from_f32(np.float32(1 + 2.0 ** -11)) == np.float16(1.0)
    assert kv16_from_f32(np.float32(1 + 3 * 2.0 ** -11)) == np.float16(1 + 2.0 ** -9)
    # f16 subnormals and underflow to signed zero
    assert kv16_from_f32(np.float32(2.0 ** -24)) == np.float16(2.0 ** -24)
    assert np.signbit(kv16_from_f32(np.float32(-2.0 ** -30)))


def test_storage_rule_clamps_at_the_edges_and_keeps_nan():
    edge = np.array([65504.0, 65519.0, 65520.0, 1e6, 3e38, np.inf], np.float32)
    assert np.all(kv16_from_f32(edge) == np.float16(F16_MAX))
    assert np.all(kv16_from_f32(-edge) == np.float16(-F16_MAX))
    with np.errstate(over="ignore"):
        assert np.isinf(edge[2:].astype(np.float16)).all()      # what a plain conversion would have stored
    assert np.isnan(kv16_from_f32(np.float32(np.nan)))
    assert np.isnan(kv16(np.nan)) and kv16(1e300) == F16_MAX


@pytest.fixture(scope="module")
def geometry_inputs():
    """The decoder-geometry model's weights, the f32 oracle's audio embeddings of a 90 s utterance and random teacher
    tokens as f64 decoder inputs, and the ADA scales."""
    data = geometry_model_bytes(8192)
    mel = omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(90.0, 4321)))
    emb = OracleModel(data).encode_audio(mel)
    o = KvHalfOracle(data, dtype=torch.float64)
    ids = np.random.default_rng(2).integers(0, o.cfg.vocab, emb.shape[0])
    ids[:PREFIX_LEN] = [1] + [32] * (PREFIX_LEN - 1)
    x = torch.as_tensor(emb).to(torch.float64) + o.embed_tokens(ids.tolist())
    return data, x, o.ada_scales(omel.time_embedding(6.0, o.cfg.dec_dim))


def _probe_logits(o, x, ada, p0):
    """Logits of rows [p0, p0 + PROBE_ROWS) after the rows before them."""
    cache = o.new_cache()
    o.decoder_forward_with_cache(x[:p0], ada, cache)
    return o.lm_head(o.decoder_forward_with_cache(x[p0:p0 + PROBE_ROWS], ada, cache)).numpy()


@pytest.mark.parametrize("window", sorted(PROBES))
def test_kv16_bound_covers_rounding_flips_and_not_read_mistakes(geometry_inputs, window):
    data, x, ada = geometry_inputs
    p0 = PROBES[window]

    def logits(**kw):
        o = KvHalfOracle(data, dtype=torch.float64, **kw)
        o.cfg.dec_window = window
        return _probe_logits(o, x, ada, p0)

    ref = logits()
    bound = KV16_LOGIT_REL_BOUND * np.maximum(1.0, np.abs(ref).max(-1))
    ratios = {}
    # f32-versus-f64 differences of K and V before the rounding flip f16 roundings
    ratios["perturb"] = (np.abs(logits(perturb=64 * 2.0 ** -24) - ref).max(-1) / bound).max()
    assert ratios["perturb"] < 0.5, ratios
    for m in ("half_tile", "dropped_tail", "k_for_v", "pair_swap"):
        ratios[m] = (np.abs(logits(mistake=m) - ref).max(-1) / bound).max()
        assert ratios[m] > 5, (window, m, ratios[m])
    # the f32-KV reference: a session that ignored kv_dtype
    o32 = OracleModel(data, dtype=torch.float64)
    o32.cfg.dec_window = window
    ratios["f32_kv"] = (np.abs(_probe_logits(o32, x, ada, p0) - ref).max(-1) / bound).max()
    if window == 8192:
        assert ratios["f32_kv"] > 1, ratios
    print(f"\n[kv16] window {window}, positions {p0}..{p0 + PROBE_ROWS - 1}: largest logit change as a multiple of "
          "the bound: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
