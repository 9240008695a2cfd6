"""Reference for a SUFFIX of a long stream: the streaming oracle's arithmetic (oracle/streaming.py, oracle/model.py)
started at absolute padded sample s0 (a multiple of 2560 = one decoder position) with empty caches and ABSOLUTE
positions, the decoder teacher-forced along given ids.

Why it is exact: both attentions are sliding-window and the front end is local, so past a warm-up -- the conv / mel
receptive field plus enc_layers x enc_window encoder frames, and dec_layers x dec_window decoder positions -- nothing
the suffix is missing can reach its outputs.  This is how a CPU reference follows a session far past the model's RoPE
tables: the tables are rebuilt longer with oracle.model.rope_tables' own formula (rows inside the model's tables are
bitwise the same) and shifted so that relative cache offsets land on absolute rows.

Everything after the (f32) mel runs in the model's dtype: with OracleModel(dtype=torch.float64) this is a float64
reference for a suffix of an unbounded session.  Used by tests.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import mel as omel
from oracle.model import ENC, PREFIX_LEN, rope_tables
from oracle.streaming import StreamingOracle

SAMPLES_PER_POS = 2560


def extended_rope(head_dim: int, rows: int, theta: float):
    return rope_tables(head_dim, rows, theta)


class _Frames:
    """Absolute-index view of frames [f0, f0 + len(frames)); frames before f0 (not computed) read as zeros."""

    def __init__(self, frames, f0, dim):
        self.frames, self.f0, self.zero = frames, f0, torch.zeros(dim)

    def __getitem__(self, i):
        return self.frames[i - self.f0] if i >= self.f0 else self.zero


def _mel(signal: np.ndarray, s0: int, f0: int, f1: int) -> list:
    """Log-mel frames [f0, f1) of the padded signal whose samples [s0, s0 + len(signal)) are given (earlier ones read
    as zero) -- StreamingOracle._mel_frames' f32 operations, all frames at once."""
    ms = omel.MelSpectrogram()
    idx = np.arange(f0, f1)[:, None] * omel.HOP - omel.N_FFT // 2 + np.arange(omel.N_FFT)[None, :] - s0
    ok = (idx >= 0) & (idx < signal.size)
    win = np.where(ok, signal[np.clip(idx, 0, signal.size - 1)], omel.F32(0)).astype(omel.F32)
    frame = (win * ms.window).astype(omel.F32)
    spec = np.fft.rfft(frame, axis=1)
    p = (spec.real.astype(omel.F32) ** 2 + spec.imag.astype(omel.F32) ** 2).astype(omel.F32)
    acc = np.zeros((p.shape[0], omel.N_MELS), omel.F32)
    for j in range(p.shape[1]):
        acc += (ms.mel_basis[None, :, j] * p[:, j:j + 1]).astype(omel.F32)
    lm = np.log10(np.maximum(acc, omel.F32(1e-10))).astype(omel.F32)
    lm = np.maximum(lm, omel.F32(omel.LOG_MEL_MAX - omel.F32(8.0)))
    return list(((lm + omel.F32(4.0)) / omel.F32(4.0)).astype(omel.F32))


def suffix_reference(model, t_embed: np.ndarray, padded: np.ndarray, s0: int, ids: list, n_pos: int | None = None):
    """`padded`: the session's padded signal known so far (left padding included), `s0` a multiple of 2560.
    Returns (p0, audio embeddings [p0, ...) as [n, dec_dim], {position p: (argmax, top-2 margin)}) where position
    p >= max(p0, 38) consumes audio embedding p and ids[p - 38] and its argmax is compared with ids[p - 37]
    (ids[0] is the prefill's).  Positions up to n_pos (default: every one whose audio and input id exist)."""
    c = model.cfg
    assert s0 % SAMPLES_PER_POS == 0
    p0 = s0 // SAMPLES_PER_POS
    f0 = s0 // omel.HOP
    n = padded.size
    f1 = (n - omel.N_FFT // 2) // omel.HOP + 1                      # frame i final once samples < 160 i + 200 known
    mel = _mel(np.asarray(padded[s0:], omel.F32), s0, f0, f1)                       # f32, as the product computes it
    w1, b1 = model.param(f"{ENC}.conv_layers.0.conv.weight"), model.param(f"{ENC}.conv_layers.0.conv.bias")
    w2, b2 = model.param(f"{ENC}.conv_layers.1.conv.weight"), model.param(f"{ENC}.conv_layers.1.conv.bias")
    big = 1 << 60
    t0, t1 = f0 // 2, (f1 - 2) // 2 + 1                              # conv1 output t needs mel 2t+1
    mv = _Frames(mel, f0, c.n_mels)
    c1 = [StreamingOracle._conv_at(None, mv, t, big, w1, b1) for t in range(t0, t1)]
    e0, e1 = t0 // 2, (t1 - 2) // 2 + 1
    cv = _Frames(c1, t0, c.enc_dim)
    x = torch.stack([StreamingOracle._conv_at(None, cv, t, big, w2, b2) for t in range(e0, e1)])
    saved = (model.enc_cos, model.enc_sin, model.dec_cos, model.dec_sin)
    try:
        model.enc_cos, model.enc_sin = (t.to(model.dtype) for t in extended_rope(c.enc_head_dim, e1 + 1, c.rope_theta))
        cache = [{"k": None, "v": None, "base": e0, "evict": True} for _ in range(c.enc_layers)]
        for i in range(c.enc_layers):
            x = model.encoder_layer_with_cache(x, i, cache[i])
        emb = model.adapter(model.encoder_norm(x))                    # audio embeddings p0 .. p0 + n_emb - 1
        n_emb = emb.shape[0]
        # decoder: positions p0 .. (teacher-forced), RoPE rows shifted so that cache offset 0 is position p0
        last = min(p0 + n_emb - 1, PREFIX_LEN + len(ids) - 2)
        if n_pos is not None:
            last = min(last, n_pos - 1)
        first = max(p0, PREFIX_LEN)
        out = {}
        if last >= first:
            cos, sin = extended_rope(c.dec_head_dim, last + 1, c.rope_theta)
            model.dec_cos, model.dec_sin = cos[first:], sin[first:]
            xs = emb[first - p0:last + 1 - p0] + model.embed_tokens(ids[first - PREFIX_LEN:last + 1 - PREFIX_LEN])
            h = model.decoder_forward_with_cache(xs, model.ada_scales(t_embed), model.new_cache())
            logits = model.lm_head(h)
            top = torch.topk(logits, 2, dim=1)
            for r, p in enumerate(range(first, last + 1)):
                out[p] = (int(top.indices[r, 0]), float(top.values[r, 0] - top.values[r, 1]))
    finally:
        model.enc_cos, model.enc_sin, model.dec_cos, model.dec_sin = saved
    return p0, emb.numpy(), out


def enc_warmup_positions(cfg) -> int:
    """Decoder positions (4 encoder frames each) before a suffix's audio embeddings are exact: the encoder layers'
    reach plus the conv / mel receptive field, rounded up."""
    return (cfg.enc_layers * cfg.enc_window + 8) // cfg.reshape_factor + 2


def dec_warmup_positions(cfg) -> int:
    return enc_warmup_positions(cfg) + cfg.dec_layers * cfg.dec_window + 1
