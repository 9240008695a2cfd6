"""CPU pins of the float64 encoder reference that tests/test_encoder_geometry_gpu.py compares the CUDA encoder with, and
the bounds that test imports.

  * the f64 encoder really is f64: OracleModel(dtype=float64) and the f32 oracle agree to f32 rounding noise at every
    stage (conv stem, each layer, final norm, adapter) on the tiny model and on the encoder-geometry model
    (synth.encoder_geometry_config), and every f64 stage's output is float64;
  * the per-layer bound is sensitive to the window: on the encoder-geometry model, one layer at window W +- 1 differs
    from the same layer at W by > 10x ENC_LAYER_REL_BOUND at every position where the window bites, for W = 750 (the
    production window) and W = 64 -- an off-by-one key in a kernel's mask cannot hide inside the bound;
  * the per-layer bounds catch a lost low f16 piece: the tensor-core attention and the wgmma GEMM's operand split carry
    every f32 operand as two f16 pieces (hi + lo).  Keeping only hi -- Q, K, V and the softmax probabilities rounded to
    one f16 piece (against ENC_LAYER_REL_BOUND, the bound of the paths that check the attention kernels with the SIMT
    GEMM), or separately the normed operand of the Q/K/V and w1/w3 GEMMs (against WGMMA_LAYER_REL_BOUND) -- moves one
    layer's output by > PIECE_SEPARATION x that bound (see the note below the bounds).

Errors are reported as max |got - ref| / max(1, max |ref|) over the whole compared tensor.
"""
import functools
import struct

import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.gguf_synth import GgufFile
from oracle.model import OracleModel
from voxtral_mini_realtime_rs_b200 import synth

# Bounds: >= 3x the largest error measured on an H100 80GB HBM3 (700 W) over every stage x path x window of
# tests/test_encoder_geometry_gpu.py (largest measured in brackets).  Stages fed the GPU's own input to them:
ENC_LAYER_REL_BOUND = 1.2e-5   # conv stem, final norm, and a layer whose linears run the SIMT GEMM, with either attention
                               # kernel [conv 2.9e-6, layer 3.5e-6]
WGMMA_LAYER_REL_BOUND = 7.5e-5 # a layer whose linears run the wgmma GEMM [2.45e-5; 9.3e-6 with 5 K slices at S = 250]
ADAPTER_REL_BOUND = 1.3e-5     # adapter, fed the GPU's own encoder output [4.3e-6]
EMBED_REL_BOUND = 3.5e-5       # audio embeddings end to end from the mel [1.1e-5 full size; 5.3e-6 at 2 layers]
SEPARATION = 10                # the window pins exceed ENC_LAYER_REL_BOUND by at least this factor
# The one-f16-piece pins do not reach SEPARATION at layer level: losing the low piece of Q/K/V/P moves layer 1 by
# 5.2e-5 = 4.3x ENC_LAYER_REL_BOUND, and losing the low piece of the normed GEMM operand moves a layer by >= 1.85e-4 =
# 2.5x WGMMA_LAYER_REL_BOUND.  The attention's four pieces are pinned at operator level instead, each at >= 59x its
# per-output bound (tests/test_attention_ref.py, test_planted_mistake_exceeds_the_bound; tests/test_attention_gpu.py
# holds the kernels to that bound).  The wgmma GEMM's per-layer error is ~7x the SIMT GEMM's and shrinks when K is
# split into slices, which points at its f32 accumulation over long K.  At layer level these pins hold at:
PIECE_SEPARATION = 2

GEOMETRY_SEED = 5
WINDOWS = (750, 64, 1)
LEFT_PAD_FRAMES = 76 * 1280 // 160 // 4     # encoder frames of the left padding (pad_audio): identical, silent inputs


def rel_err(got, ref) -> float:
    """max |got - ref| / max(1, max |ref|) over the whole array."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(got - ref).max() / max(1.0, float(np.abs(ref).max())))


@functools.lru_cache(maxsize=1)
def _geometry_bytes_750() -> bytes:
    return synth.build_aliased_gguf_bytes(synth.encoder_geometry_config(750), seed=GEOMETRY_SEED)


@functools.lru_cache(maxsize=None)
def encoder_geometry_bytes(enc_window: int) -> bytes:
    """The encoder-geometry GGUF (in memory, ~260 MB) with the given encoder sliding window.  The tensor bytes do not
    depend on the window: they are generated once, and only the header's u32 window value is rewritten."""
    base = _geometry_bytes_750()
    key = b"voxtral.enc.sliding_window"
    tag = struct.pack("<Q", len(key)) + key + struct.pack("<I", 4)
    at = base.find(tag)
    assert at > 0 and base.find(tag, at + 1) < 0
    at += len(tag)
    data = base[:at] + struct.pack("<I", enc_window) + base[at + 4:]
    assert GgufFile(data).config().enc_window == enc_window
    return data


def geometry_mel(seconds: float, seed: int) -> np.ndarray:
    return omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(seconds, seed)))


def _stages(o, mel):
    cap = {}
    emb = o.encode_audio(mel, cap)
    cap["audio_embeds"] = emb
    return cap


@pytest.mark.parametrize("model", ["tiny", "geometry"])
def test_f64_encoder_matches_f32_encoder(tiny_gguf, model):
    src = tiny_gguf if model == "tiny" else encoder_geometry_bytes(750)
    o32, o64 = OracleModel(src), OracleModel(src, dtype=torch.float64)
    mel = geometry_mel(12.0, 3)
    s32, s64 = _stages(o32, mel), _stages(o64, mel)
    assert list(s32) == ["conv"] + [f"enc{i}" for i in range(o32.cfg.enc_layers)] + ["enc_out", "audio_embeds"]
    for k in s32:
        err = rel_err(s32[k].numpy(), s64[k].numpy())
        print(f"\n[f64 encoder] {model:8s} {k:12s} max rel |f32 - f64| = {err:.2e}")
        assert s32[k].dtype == torch.float32 and s64[k].dtype == torch.float64, k
        assert 0 < err < 1e-5, (k, err)          # f32 rounding noise; and a different arithmetic from the f32 one
    # the stage functions the GPU tests feed with the GPU's own inputs, and the cached (chunked) encoder
    assert o64.conv_stem(mel).dtype == o64.adapter(s64["enc_out"]).dtype == torch.float64
    assert torch.equal(o64.adapter(s64["enc_out"]), s64["audio_embeds"])
    c32, c64 = o32.new_encoder_cache(), o64.new_encoder_cache()
    for a, b in ((0, 400), (400, mel.shape[2])):
        e32, e64 = o32.encode_audio_with_cache(mel[:, :, a:b], c32), o64.encode_audio_with_cache(mel[:, :, a:b], c64)
        assert e64.dtype == torch.float64 and 0 < rel_err(e32.numpy(), e64.numpy()) < 1e-5


@pytest.fixture(scope="module")
def geometry_f64():
    """f64 oracle of the encoder-geometry model and the conv stem of 30 s of audio: 37.4 s of padded mel, 936 encoder
    frames, so the window of 750 bites from frame 750 on."""
    o = OracleModel(encoder_geometry_bytes(750), dtype=torch.float64)
    return o, o.conv_stem(geometry_mel(30.0, 77))


@pytest.mark.parametrize("window", [750, 64])
def test_window_off_by_one_exceeds_layer_bound(geometry_f64, window):
    """Query p attends to keys [p - window, p].  Stage by stage (layer i fed the window-W reference of layer i - 1), the
    layer at W - 1 and W + 1 equals the layer at W before the window bites (p < W, p < W + 1) and differs from it by
    > SEPARATION x the bound at every later position whose window reaches the audio (p >= LEFT_PAD_FRAMES: over the
    silent left padding every key holds the same vector, so dropping one of them changes nothing)."""
    o, x = geometry_f64
    saved = o.cfg.enc_window
    try:
        for i in range(o.cfg.enc_layers):
            out = {}
            for w in (window - 1, window, window + 1):
                o.cfg.enc_window = w
                out[w] = o.encoder_layer(x, i).numpy()
            ref = out[window]
            scale = max(1.0, float(np.abs(ref).max()))
            for other, first in ((window - 1, window), (window + 1, window + 1)):
                d = np.abs(out[other] - ref).max(-1)
                assert np.all(d[:first] == 0), (i, other, np.nonzero(d[:first])[0])
                lo = max(first, LEFT_PAD_FRAMES)
                ratio = d[lo:] / (ENC_LAYER_REL_BOUND * scale)
                print(f"\n[window sensitivity] layer {i} ref({window}) vs ref({other}): positions {lo}..{len(d) - 1}, "
                      f"min max|d| / max(1, max|ref|) = {d[lo:].min() / scale:.2e} = {ratio.min():.0f}x the bound")
                assert len(ratio) >= 150 and ratio.min() > SEPARATION, (i, other, int(np.argmin(ratio)) + lo, ratio.min())
            x = torch.from_numpy(ref)
    finally:
        o.cfg.enc_window = saved


def f16_piece(t: torch.Tensor) -> torch.Tensor:
    """The hi piece alone: t rounded to f16 (values here are far inside f16's normal range)."""
    return t.to(torch.float16).to(t.dtype)


class _OnePieceAttention(OracleModel):
    """Attention with Q, K, V and the softmax probabilities rounded to one f16 piece."""

    def _attention(self, q, k, v, scale, q_offset, window, causal=True):
        sq, h, hd = q.shape
        qh, kh, vh = (f16_piece(t).permute(1, 0, 2) for t in (q, k, v))
        s = torch.matmul(qh, kh.transpose(1, 2)) * scale
        i = torch.arange(sq)[:, None] + q_offset
        j = torch.arange(k.shape[0])[None, :]
        s = s.masked_fill(((j > i) | ((i - j).abs() > window))[None], float("-inf"))
        p = torch.exp(s - s.amax(-1, keepdim=True))
        out = torch.matmul(f16_piece(p), vh) / p.sum(-1, keepdim=True)
        return out.permute(1, 0, 2).reshape(sq, h * hd)


class _OnePieceNormedOperand(OracleModel):
    """The RMSNorm output feeding the Q/K/V and w1/w3 GEMMs rounded to one f16 piece."""

    def linear(self, x, wname, bname=None):
        if ".whisper_encoder." in wname and wname.endswith(("wq.weight", "wk.weight", "wv.weight", "w1.weight", "w3.weight")):
            x = f16_piece(x)
        return super().linear(x, wname, bname)


@pytest.mark.parametrize("window", WINDOWS)
def test_lost_low_f16_piece_exceeds_layer_bound(geometry_f64, window):
    o, x = geometry_f64
    data = encoder_geometry_bytes(window)
    ref_m = OracleModel(data, dtype=torch.float64)
    for name, cls, bound in (("attention", _OnePieceAttention, ENC_LAYER_REL_BOUND),
                             ("normed operand", _OnePieceNormedOperand, WGMMA_LAYER_REL_BOUND)):
        m = cls(data, dtype=torch.float64)
        xi = x
        for i in range(ref_m.cfg.enc_layers):
            ref = ref_m.encoder_layer(xi, i)
            err = rel_err(m.encoder_layer(xi, i).numpy(), ref.numpy())
            print(f"\n[one f16 piece] window {window:3d} {name:14s} layer {i}: max rel = {err:.2e} = "
                  f"{err / bound:.1f}x the bound")
            assert err > PIECE_SEPARATION * bound, (name, i, err)
            xi = ref
