"""Incremental ("true streaming") restatement of the whole-utterance path -- test infrastructure for the
streaming-session row of SURVEY 8(f)-1 (see oracle/__init__.py; nothing in the product imports this).

`Q4VoxtralModel::transcribe_streaming` (reference src/gguf/model.rs:873-963) consumes a complete mel
spectrogram.  This module feeds the same arithmetic sample by sample and emits every token as soon as its
inputs are final, which pins down WHAT STATE a streaming session has to carry and HOW MUCH LOOKAHEAD each
stage needs for the ids to equal the offline ones:

  stage (reference)                          output i is final once ...                      carried state
  mel frame (mel.rs:185-244; hop 160, n_fft 400, centre) samples < 160 i + 200 are known        last 240 samples
  conv1 k3 s2 p1 (conv.rs:78-83)              mel frame 2 i + 1 is known (or the stream ended)  last mel frame(s)
  conv2 k3 s2 p1                              conv1 frame 2 i + 1 is known (or ended)           last conv1 frame(s)
  encoder layer, causal, window 750           immediately (KV cache, model.rs:125-174, 437-452) K/V per layer
  adapter, 4-frame stack (adapter.rs:108-122) encoder frames 4 i .. 4 i + 3 are known           up to 3 frames
  decoder position p (model.rs:906-960)       audio embedding p - 1 is known (prefill: 0..37)   K/V per layer

so audio embedding p needs samples up to 2560 p + 2600: one decoder position per 160 ms of audio with
162.5 ms of lookahead.  The reflect padding of the STFT never sees non-zero samples because pad_audio
(pad.rs:89-103) surrounds the utterance with >= 21 760 zeros; peak normalisation (io.rs:59-68) needs the
whole utterance and stays with the caller.

Everything is computed with the same torch/numpy f32 operations as oracle/model.py on windows of the
stream; per-window convolutions may differ from the whole-utterance convolution in the last bit (GEMM
blocking), which the tests bound.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import mel as omel
from .model import ADAPTER, BOS_TOKEN, ENC, PREFIX_LEN, STREAMING_PAD, rms_norm


class StreamingOracle:
    def __init__(self, model, t_embed: np.ndarray, pad_cfg: omel.PadConfig | None = None):
        self.m = model
        self.cfg = model.cfg
        self.pad_cfg = pad_cfg or omel.PadConfig()
        self.ada = model.ada_scales(t_embed)
        self.melspec = omel.MelSpectrogram()
        self.samples = np.zeros(0, omel.F32)     # padded signal so far (left pad + audio [+ right pad])
        self.n_audio = 0
        self.mel = []                            # final log-mel frames, each [128]
        self.c1 = []                             # final conv1 frames, each [d]
        self.c2_count = 0                        # conv2 (= encoder input) frames produced
        self.enc_cache = model.new_encoder_cache()
        self.enc_out = []                        # final encoder output frames (after the final norm), each [d]
        self.audio_embeds = []                   # adapter outputs, each [dec_dim]
        self.dec_cache = model.new_cache()
        self.last_tok = None
        self.pos = 0                             # decoder positions consumed
        self.ids = []                            # emitted ids (positions >= PREFIX_LEN)
        self.ended = False
        self._push(np.zeros(self.pad_cfg.left_pad_samples(), omel.F32))

    # ------------------------------------------------------------------ public API
    def feed(self, samples: np.ndarray) -> list[int]:
        """Append (already peak-normalised) 16 kHz samples; returns the ids that became final."""
        assert not self.ended
        s = np.asarray(samples, omel.F32).reshape(-1)
        self.n_audio += s.size
        return self._push(s)

    def finish(self) -> list[int]:
        """End of the utterance: right padding per pad_audio (pad.rs:89-103), then flush every stage."""
        assert not self.ended
        total = self.pad_cfg.left_pad_samples() + self.n_audio
        out = self._push(np.zeros(self.pad_cfg.right_pad_samples(total), omel.F32), ended=True)
        return out

    # ------------------------------------------------------------------ stages
    def _push(self, s: np.ndarray, ended: bool = False) -> list[int]:
        self.samples = np.concatenate([self.samples, s])
        self.ended = ended
        n_before = len(self.ids)
        self._mel_frames()
        self._conv_frames()
        self._adapter_and_decode()
        return self.ids[n_before:]

    def _mel_frames(self):
        n = self.samples.size
        total = omel.num_frames(n) if self.ended else None
        i = len(self.mel)
        while True:
            if total is not None:
                if i >= total:
                    break
            elif omel.HOP * i + omel.N_FFT // 2 > n:   # needs samples [160 i - 200, 160 i + 200)
                break
            lo, hi = omel.HOP * i - omel.N_FFT // 2, omel.HOP * i + omel.N_FFT // 2
            win = np.zeros(omel.N_FFT, omel.F32)
            a, b = max(lo, 0), min(hi, n)
            if b > a:
                win[a - lo:b - lo] = self.samples[a:b]   # outside [0, n): reflect of zeros = zeros (see header)
            frame = (win * self.melspec.window).astype(omel.F32)
            spec = np.fft.rfft(frame[None, :], axis=1)
            p = (spec.real.astype(omel.F32) ** 2 + spec.imag.astype(omel.F32) ** 2).astype(omel.F32)
            acc = np.zeros((1, omel.N_MELS), omel.F32)
            for j in range(p.shape[1]):
                acc += (self.melspec.mel_basis[None, :, j] * p[:, j:j + 1]).astype(omel.F32)
            lm = np.log10(np.maximum(acc, omel.F32(1e-10))).astype(omel.F32)
            lm = np.maximum(lm, omel.F32(omel.LOG_MEL_MAX - omel.F32(8.0)))
            self.mel.append(((lm + omel.F32(4.0)) / omel.F32(4.0)).astype(omel.F32)[0])
            i += 1

    @staticmethod
    def _conv_out(t: int) -> int:
        return (t + 2 - 3) // 2 + 1 if t > 0 else 0

    def _conv_at(self, frames: list, t: int, total_in: int, w, b) -> torch.Tensor:
        """k3 s2 p1 convolution output t from input frames 2t-1 .. 2t+1 (zeros outside [0, total_in)), in w's dtype."""
        cols = []
        for idx in (2 * t - 1, 2 * t, 2 * t + 1):
            if 0 <= idx < total_in:
                cols.append(torch.as_tensor(frames[idx]).to(w.dtype))
            else:
                cols.append(torch.zeros(w.shape[1], dtype=w.dtype))
        x = torch.stack(cols, 1)[None]                       # [1, C_in, 3]
        return F.gelu(F.conv1d(x, w, b))[0, :, 0]            # [C_out]

    def _conv_frames(self):
        m = self.m
        w1, b1 = m.f32(f"{ENC}.conv_layers.0.conv.weight"), m.f32(f"{ENC}.conv_layers.0.conv.bias")
        w2, b2 = m.f32(f"{ENC}.conv_layers.1.conv.weight"), m.f32(f"{ENC}.conv_layers.1.conv.bias")
        t_mel = len(self.mel)
        # conv1: output t final when mel frame 2t+1 exists, or (stream ended) for every t < conv_out(T)
        if self.ended:
            lim1 = self._conv_out(t_mel)
        else:  # largest final t has 2t + 1 <= t_mel - 1
            lim1 = (t_mel - 2) // 2 + 1 if t_mel >= 2 else 0
        total_mel = t_mel if self.ended else 1 << 60
        while len(self.c1) < lim1:
            self.c1.append(self._conv_at(self.mel, len(self.c1), total_mel, w1, b1))
        t1 = len(self.c1)
        if self.ended:
            lim2 = self._conv_out(t1)
        else:
            lim2 = max(0, (t1 - 2) // 2 + 1) if t1 >= 2 else 0
        total_c1 = t1 if self.ended else 1 << 60
        new = []
        while self.c2_count + len(new) < lim2:
            new.append(self._conv_at(self.c1, self.c2_count + len(new), total_c1, w2, b2))
        if new:
            x = torch.stack(new)                              # [n_new, d] encoder input frames
            self.c2_count += len(new)
            for i in range(self.cfg.enc_layers):
                x = m.encoder_layer_with_cache(x, i, self.enc_cache[i])
            x = rms_norm(x, m.f32(f"{ENC}.transformer.norm.weight"), self.cfg.norm_eps)
            self.enc_out.extend(list(x))

    def _adapter_and_decode(self):
        m, c = self.m, self.cfg
        rf = c.reshape_factor
        while (len(self.audio_embeds) + 1) * rf <= len(self.enc_out):
            s = len(self.audio_embeds)
            x = torch.cat(self.enc_out[s * rf:(s + 1) * rf])[None]   # [1, d*rf]
            x = F.gelu(m.linear(x, f"{ADAPTER}.0.weight"))
            self.audio_embeds.append(m.linear(x, f"{ADAPTER}.2.weight")[0])
        n_emb = len(self.audio_embeds)
        # prefill once the 38 prefix positions have their audio (model.rs:883-923)
        if self.pos == 0 and n_emb >= PREFIX_LEN:
            prefix = [BOS_TOKEN] + [STREAMING_PAD] * (PREFIX_LEN - 1)
            x = torch.stack(self.audio_embeds[:PREFIX_LEN]) + m.embed_tokens(prefix)
            h = m.decoder_forward_with_cache(x, self.ada, self.dec_cache)
            self.last_tok = int(torch.argmax(m.lm_head(h[-1:])[0]).item())
            self.ids.append(self.last_tok)
            self.pos = PREFIX_LEN + 1
        # one step per further audio embedding: position p consumes audio[p-1] + embed(tok[p-1]) (model.rs:938-960)
        # (the offline loop stops at position S - 1: the last audio embedding is never consumed, model.rs:938)
        last_pos = n_emb - 1 if self.ended else n_emb
        while self.pos >= PREFIX_LEN + 1 and self.pos <= last_pos:
            x = self.audio_embeds[self.pos - 1][None] + m.embed_tokens([self.last_tok])
            h = m.decoder_forward_with_cache(x, self.ada, self.dec_cache)
            self.last_tok = int(torch.argmax(m.lm_head(h)[0]).item())
            self.ids.append(self.last_tok)
            self.pos += 1
