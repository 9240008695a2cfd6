"""CPU pins of the float64 decoder reference that tests/test_decode_geometry_gpu.py compares the CUDA decode step with.

  * f64 vs f32 oracle on the tiny model: the two agree to f32 rounding noise (and the f64 mode really computes in f64);
  * sensitivity: on the decoder-geometry model (synth.decoder_geometry_config), at every position where the sliding
    window bites, the reference at window W differs from the reference at W - 1 and at W + 1 by far more than the
    GPU test's logit bound -- so an off-by-one in a kernel's window start cannot hide inside that bound.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from voxtral_mini_realtime_rs_b200 import synth

# per decode step: max |GPU logit - f64 logit| <= LOGIT_REL_BOUND * max(1, max |f64 logit|)
LOGIT_REL_BOUND = 1e-4
GEOMETRY_SEED = 5


def geometry_model_bytes(dec_window: int) -> bytes:
    """The decoder-geometry GGUF (in memory, ~190 MB) with the given decoder sliding window; same weights for every
    window."""
    return synth.build_aliased_gguf_bytes(synth.decoder_geometry_config(dec_window), seed=GEOMETRY_SEED)


def rel_err(got, ref) -> np.ndarray:
    """Per row: max |got - ref| / max(1, max |ref|)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return np.abs(got - ref).max(-1) / np.maximum(1.0, np.abs(ref).max(-1))


def test_f64_oracle_matches_f32_oracle_on_tiny_model(tiny_gguf, tiny_oracle):
    o64 = OracleModel(tiny_gguf, dtype=torch.float64)
    mel = omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(4.0, 9)))
    emb = tiny_oracle.encode_audio(mel)
    ids = np.random.default_rng(0).integers(0, tiny_oracle.cfg.vocab, emb.shape[0])
    ids[0] = 1
    t_embed = omel.time_embedding(6.0, tiny_oracle.cfg.dec_dim)
    l32 = tiny_oracle.forward_streaming(None, ids.tolist(), t_embed, audio_embeds=emb)
    l64 = o64.forward_streaming(None, ids.tolist(), t_embed, audio_embeds=emb)
    assert l32.dtype == torch.float32 and l64.dtype == torch.float64
    err = rel_err(l32.numpy(), l64.numpy())
    print(f"\n[f64 oracle] tiny model, {err.size} positions: max rel |f32 - f64| = {err.max():.2e}")
    assert err.max() < 1e-5                  # f32 rounding noise on logits of O(1)
    assert err.max() > 0                     # the f64 mode is a different arithmetic, not the f32 one
    # greedy decoding agrees too (the tiny model's smallest top-2 margin is far above that noise)
    info = {}
    assert o64.transcribe_streaming(mel, t_embed, audio_embeds=emb, info=info) == \
        tiny_oracle.transcribe_streaming(mel, t_embed, audio_embeds=emb)
    assert min(info["margins"]) > 100 * err.max()


@pytest.fixture(scope="module")
def geometry_ref():
    """f64 oracle of the decoder-geometry model, the f32 oracle's audio embeddings of a 6 s utterance (84 positions)
    and random teacher tokens."""
    data = geometry_model_bytes(40)
    o64 = OracleModel(data, dtype=torch.float64)
    mel = omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(6.0, 1234)))
    emb = OracleModel(data).encode_audio(mel)
    ids = np.random.default_rng(1).integers(0, o64.cfg.vocab, emb.shape[0])
    ids[:PREFIX_LEN] = [1] + [32] * (PREFIX_LEN - 1)
    return o64, emb, ids.tolist(), omel.time_embedding(6.0, o64.cfg.dec_dim)


@pytest.mark.parametrize("window", [40, 8])
def test_window_off_by_one_exceeds_logit_bound(geometry_ref, window):
    """Position p attends to keys [p - window, p].  ref(W) and ref(W +- 1) must be equal before the window bites and
    differ per row by > 20x the GPU bound at every decode position where it does (p >= W for W - 1, p >= W + 1 for
    W + 1; decode positions are p >= 38).  In the prefix (BOS + 37 pad tokens over the silent left padding of the audio)
    the inputs of neighbouring positions are nearly identical, so dropping one of them barely moves the result there."""
    o64, emb, ids, t_embed = geometry_ref
    saved = o64.cfg.dec_window
    try:
        logits = {}
        for w in (window - 1, window, window + 1):
            o64.cfg.dec_window = w
            logits[w] = o64.forward_streaming(None, ids, t_embed, audio_embeds=emb).numpy()
    finally:
        o64.cfg.dec_window = saved
    ref = logits[window]
    bound = LOGIT_REL_BOUND * np.maximum(1.0, np.abs(ref).max(-1))
    for other, first in ((window - 1, window), (window + 1, window + 1)):
        d = np.abs(logits[other] - ref).max(-1)
        assert np.all(d[:first] == 0), (other, np.nonzero(d[:first])[0])
        lo = max(first, PREFIX_LEN)
        ratio = d[lo:] / bound[lo:]
        print(f"\n[window sensitivity] ref({window}) vs ref({other}): positions {lo}..{len(d) - 1}, "
              f"min max|dlogit| = {d[lo:].min():.3e} = {ratio.min():.0f}x the bound")
        assert ratio.min() > 20, (other, int(np.argmin(ratio)) + lo, ratio.min())
