"""Q4 Voxtral model oracle -- CPU f32 restatement (test infrastructure, see oracle/__init__.py).

Follows, function by function:
  src/gguf/model.rs          Q4Attention 77-198, Q4FeedForward 220-224, Q4AdaRmsNorm 250-255,
                             Q4EncoderLayer 287-297, Q4DecoderLayer 370-387, Q4AudioEncoder 425-434,
                             Q4LanguageModel 566-691, Q4Adapter 745-749,
                             Q4VoxtralModel::encode_audio 783-788, transcribe_streaming 873-963
  src/models/layers/         rope.rs 35-141, masking.rs 9-107, rms_norm.rs 42-47 (burn RmsNorm:
                             x / sqrt(mean(x^2)+eps) * gamma), conv.rs 78-83, kv_cache.rs 116-142
  src/models/adapter.rs      reshape_encoder_output 108-122
  src/gguf/loader.rs         which tensors carry biases (226-250), RoPE table sizes/theta (196,284)
Cross-checked against the torch scripts scripts/generate_padded_reference.py:95-187 and
scripts/compare_full_forward.py:278-361 (same graph).

Third-party arithmetic (Burn 0.20 matmul/softmax/conv/gelu/silu/argmax; absent crate) is
replaced by torch-CPU f32 ops with the same definitions (erf-GELU, x*sigmoid(x), exp(x-max)/sum);
the reference's `.npy` layer fixtures are absent => **parity unpinned for those ops' rounding**;
argmax tie-break is defined here as lowest index.  Q4 linears use oracle/q4_ref.c (shader
accumulation order) for M<=8 and dequantise + torch.mm for larger M (same maths, f32).
"""
from __future__ import annotations

import math
import numpy as np
import torch
import torch.nn.functional as F

from . import q4
from .gguf_synth import GgufFile, VoxtralConfig, ENC, ADAPTER, TOK_EMB, FINAL_NORM

PREFIX_LEN = 38
BOS_TOKEN = 1
STREAMING_PAD = 32


def rope_tables(head_dim: int, max_seq: int, theta: float = 1e6):
    """rope.rs:35-64."""
    half = head_dim // 2
    inv = np.array([np.float32(1.0) / np.power(np.float32(theta), np.float32(2 * i) / np.float32(head_dim))
                    for i in range(half)], dtype=np.float32)
    pos = np.arange(max_seq, dtype=np.float32)
    fr = (pos[:, None] * inv[None, :]).astype(np.float32)
    return torch.from_numpy(np.cos(fr).astype(np.float32)), torch.from_numpy(np.sin(fr).astype(np.float32))


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, offset: int) -> torch.Tensor:
    """rope.rs:103-141.  x [S, H, hd] interleaved pairs; cos/sin in x's dtype."""
    s, h, hd = x.shape
    xp = x.reshape(s, h, hd // 2, 2)
    xr, xi = xp[..., 0], xp[..., 1]
    c = cos[offset:offset + s][:, None, :]
    sn = sin[offset:offset + s][:, None, :]
    out_r = xr * c - xi * sn
    out_i = xr * sn + xi * c
    return torch.stack([out_r, out_i], dim=-1).reshape(s, h, hd)


def rms_norm(x: torch.Tensor, gamma: torch.Tensor, eps: float) -> torch.Tensor:
    rms = torch.sqrt(torch.mean(x * x, dim=-1, keepdim=True) + eps)
    return (x / rms) * gamma


class OracleModel:
    """`dtype=torch.float64` runs the whole model in float64 -- a high-precision reference for the f32 GPU path.  The
    encoder side: the conv stem on the f32 mel cast, with erf-GELU; every RMSNorm, Q4 linear, RoPE, attention and
    softmax of the layers (with and without KV caches); the final norm, the x4 reshape and the adapter.  The decoder
    side: embed_tokens, ada_scales, every linear, RMSNorm, RoPE, attention and softmax, lm_head.  The Q4 weights
    dequantise exactly to f32 and are cast per call (the f32 dequantisations are cached, never f64 copies); the f32
    conv weights, biases and norm gammas are cast; the RoPE tables are the f32 tables cast, as the product uses f32
    tables too.  The default float32 mode is unchanged."""

    def __init__(self, gguf, threads: int = 0, exact_order_max_m: int = 8, dtype: torch.dtype = torch.float32):
        self.g = gguf if isinstance(gguf, GgufFile) else GgufFile(gguf)
        self.cfg: VoxtralConfig = self.g.config()
        self.threads = threads
        self.exact_order_max_m = exact_order_max_m
        assert dtype in (torch.float32, torch.float64), dtype
        self.dtype = dtype
        c = self.cfg
        self.enc_cos, self.enc_sin = rope_tables(c.enc_head_dim, 4096, c.rope_theta)
        self.enc_cos, self.enc_sin = self.enc_cos.to(dtype), self.enc_sin.to(dtype)
        self.dec_cos, self.dec_sin = rope_tables(c.dec_head_dim, 16384, c.rope_theta)
        self.dec_cos, self.dec_sin = self.dec_cos.to(dtype), self.dec_sin.to(dtype)
        self._f32 = {}
        self._deq = {}
        self.cache_dequant = dtype == torch.float64

    # ---- primitives -------------------------------------------------------
    def f32(self, name) -> torch.Tensor:
        if name not in self._f32:
            self._f32[name] = torch.from_numpy(self.g.f32(name))
        return self._f32[name]

    def param(self, name) -> torch.Tensor:
        """f32 tensor `name` in the model's dtype."""
        return self.f32(name).to(self.dtype)

    def has(self, name) -> bool:
        return self.g.info(name) is not None

    def linear(self, x: torch.Tensor, wname: str, bname: str | None = None) -> torch.Tensor:
        """Q4Linear::forward (linear.rs:34-40): q4_matmul then + bias."""
        dt, (n, k), _ = self.g.info(wname)
        assert dt == 2, f"Expected Q4_0 for '{wname}'"
        lead = x.shape[:-1]
        x2 = x.reshape(-1, k).contiguous()
        m = x2.shape[0]
        raw = self.g.raw(wname)
        if m <= self.exact_order_max_m and self.dtype == torch.float32:
            y = torch.from_numpy(q4.q4_matmul_c(x2.numpy(), raw, n, k, threads=self.threads))
        else:
            if wname in self._deq:
                w = self._deq[wname]
            else:
                w = torch.from_numpy(q4.dequantize_c(raw)).reshape(n, k)
                if self.cache_dequant:
                    self._deq[wname] = w
            y = x2.to(self.dtype) @ w.to(self.dtype).t()
        if bname is not None and self.has(bname):
            y = y + self.param(bname)
        return y.reshape(*lead, n)

    # ---- encoder ----------------------------------------------------------
    def conv_downsample(self, mel) -> torch.Tensor:
        """conv.rs:78-83; mel [1,128,T] (f32, numpy or torch) -> [1, d, T/4] in the model's dtype."""
        mel = torch.as_tensor(np.ascontiguousarray(mel, np.float32)).to(self.dtype)
        x = F.conv1d(mel, self.param(f"{ENC}.conv_layers.0.conv.weight"),
                     self.param(f"{ENC}.conv_layers.0.conv.bias"), stride=2, padding=1)
        x = F.gelu(x)
        x = F.conv1d(x, self.param(f"{ENC}.conv_layers.1.conv.weight"),
                     self.param(f"{ENC}.conv_layers.1.conv.bias"), stride=2, padding=1)
        return F.gelu(x)

    def conv_stem(self, mel) -> torch.Tensor:
        """The encoder's input frames: mel [1,128,T] -> [S, d]."""
        return self.conv_downsample(mel)[0].transpose(0, 1).contiguous()

    def encoder_norm(self, x: torch.Tensor) -> torch.Tensor:
        """The encoder's final RMSNorm."""
        return rms_norm(x, self.param(f"{ENC}.transformer.norm.weight"), self.cfg.norm_eps)

    def adapter(self, enc_out: torch.Tensor) -> torch.Tensor:
        """Reshape x4 (adapter.rs:108-122; a trailing partial group is dropped) + Q4Adapter (model.rs:745-749):
        enc_out [S, d] -> audio_embeds [S/4, dec_dim]."""
        rf = self.cfg.reshape_factor
        s4 = enc_out.shape[0] // rf
        x = enc_out[: s4 * rf].reshape(s4, self.cfg.enc_dim * rf)
        x = F.gelu(self.linear(x, f"{ADAPTER}.0.weight"))
        return self.linear(x, f"{ADAPTER}.2.weight")

    def _attention(self, q, k, v, scale, q_offset, window, causal=True):
        """q [Sq,H,hd], k/v [Skv,Hkv,hd] -> [Sq, H*hd]; masks per masking.rs:9-107."""
        sq, h, hd = q.shape
        skv, hkv, _ = k.shape
        rep = h // hkv
        qh = q.permute(1, 0, 2)                                  # [H,Sq,hd]
        kh = k.permute(1, 0, 2).repeat_interleave(rep, dim=0)    # expand_kv, model.rs:177-197
        vh = v.permute(1, 0, 2).repeat_interleave(rep, dim=0)
        scores = torch.matmul(qh, kh.transpose(1, 2)) * scale    # [H,Sq,Skv]
        i = torch.arange(sq)[:, None] + q_offset
        j = torch.arange(skv)[None, :]
        mask = torch.zeros(sq, skv, dtype=scores.dtype)
        if causal:
            mask = mask.masked_fill(j > i, float("-inf"))
        if window is not None:
            mask = mask.masked_fill((i - j).abs() > window, float("-inf"))
        scores = scores + mask[None]
        attn = torch.softmax(scores, dim=-1)
        out = torch.matmul(attn, vh)                             # [H,Sq,hd]
        return out.permute(1, 0, 2).reshape(sq, h * hd)

    def encoder_attention_block(self, h: torch.Tensor, i: int) -> torch.Tensor:
        """Q4Attention::forward (model.rs:77-122) on already-normed input h [S, d]: q/k/v (+biases), RoPE,
        masked softmax attention, wo (+bias).  No residual."""
        c = self.cfg
        p = f"{ENC}.transformer.layers.{i}"
        s = h.shape[0]
        q = self.linear(h, f"{p}.attention.wq.weight", f"{p}.attention.wq.bias").reshape(s, c.enc_heads, c.enc_head_dim)
        k = self.linear(h, f"{p}.attention.wk.weight").reshape(s, c.enc_heads, c.enc_head_dim)
        v = self.linear(h, f"{p}.attention.wv.weight", f"{p}.attention.wv.bias").reshape(s, c.enc_heads, c.enc_head_dim)
        q = apply_rope(q, self.enc_cos, self.enc_sin, 0)
        k = apply_rope(k, self.enc_cos, self.enc_sin, 0)
        a = self._attention(q, k, v, float(np.float32(c.enc_head_dim) ** np.float32(-0.5)), 0, c.enc_window)
        return self.linear(a, f"{p}.attention.wo.weight", f"{p}.attention.wo.bias")

    def swiglu(self, h: torch.Tensor, prefix: str, bias: bool = False) -> torch.Tensor:
        """Q4FeedForward::forward (model.rs:220-224): w2(silu(w1 h) * w3 h)."""
        gate = F.silu(self.linear(h, f"{prefix}.feed_forward.w1.weight"))
        up = self.linear(h, f"{prefix}.feed_forward.w3.weight")
        return self.linear(gate * up, f"{prefix}.feed_forward.w2.weight", f"{prefix}.feed_forward.w2.bias" if bias else None)

    def encoder_layer(self, x: torch.Tensor, i: int) -> torch.Tensor:
        c = self.cfg
        p = f"{ENC}.transformer.layers.{i}"
        s = x.shape[0]
        h = rms_norm(x, self.param(f"{p}.attention_norm.weight"), c.norm_eps)
        q = self.linear(h, f"{p}.attention.wq.weight", f"{p}.attention.wq.bias")
        k = self.linear(h, f"{p}.attention.wk.weight")
        v = self.linear(h, f"{p}.attention.wv.weight", f"{p}.attention.wv.bias")
        q = q.reshape(s, c.enc_heads, c.enc_head_dim)
        k = k.reshape(s, c.enc_heads, c.enc_head_dim)
        v = v.reshape(s, c.enc_heads, c.enc_head_dim)
        q = apply_rope(q, self.enc_cos, self.enc_sin, 0)
        k = apply_rope(k, self.enc_cos, self.enc_sin, 0)
        a = self._attention(q, k, v, float(np.float32(c.enc_head_dim) ** np.float32(-0.5)), 0, c.enc_window)
        x = self.linear(a, f"{p}.attention.wo.weight", f"{p}.attention.wo.bias") + x
        h = rms_norm(x, self.param(f"{p}.ffn_norm.weight"), c.norm_eps)
        gate = F.silu(self.linear(h, f"{p}.feed_forward.w1.weight"))
        up = self.linear(h, f"{p}.feed_forward.w3.weight")
        return self.linear(gate * up, f"{p}.feed_forward.w2.weight", f"{p}.feed_forward.w2.bias") + x

    def encoder_forward(self, mel: np.ndarray, capture: dict | None = None) -> torch.Tensor:
        """Q4AudioEncoder::forward (model.rs:425-434): mel [1,128,T] -> [S, enc_dim]."""
        x = self.conv_stem(mel)
        if capture is not None:
            capture["conv"] = x.clone()
        for i in range(self.cfg.enc_layers):
            x = self.encoder_layer(x, i)
            if capture is not None:
                capture[f"enc{i}"] = x.clone()
        return self.encoder_norm(x)

    def encode_audio(self, mel: np.ndarray, capture: dict | None = None) -> torch.Tensor:
        """model.rs:783-788 -> audio_embeds [S/4, dec_dim]."""
        x = self.encoder_forward(mel, capture)
        if capture is not None:
            capture["enc_out"] = x.clone()
        return self.adapter(x)

    # ---- encoder with KV cache (incremental API; SURVEY 8(f)-1: not yet behind the C ABI) -------------
    def new_encoder_cache(self, evict: bool = False):
        """Q4AudioEncoder::create_cache (model.rs:460-462): one dynamic KVCache per encoder layer.
        `evict`: drop keys that no future query can see (older than the sliding window) while keeping ABSOLUTE
        positions for RoPE and the masks -- the bounded-memory form a long-running streaming session needs.
        (Upstream's KVCache::apply_sliding_window, kv_cache.rs:176-203, is unused and would re-base positions.)"""
        return [{"k": None, "v": None, "base": 0, "evict": evict} for _ in range(self.cfg.enc_layers)]

    def encoder_layer_with_cache(self, x: torch.Tensor, i: int, cache: dict) -> torch.Tensor:
        """Q4EncoderLayer::forward_with_cache (model.rs:300-315) over Q4Attention::forward_with_cache
        (model.rs:125-174): RoPE offset = cached length, K/V appended (kv_cache.rs:70-142), causal and
        sliding-window masks with offset (masking.rs:50-107)."""
        c = self.cfg
        p = f"{ENC}.transformer.layers.{i}"
        s = x.shape[0]
        base = cache.get("base", 0)                                   # absolute position of the first cached key
        offset = base + (0 if cache["k"] is None else cache["k"].shape[0])
        if cache.get("evict") and cache["k"] is not None and c.enc_window is not None:
            drop = min(max(offset - c.enc_window - base, 0), cache["k"].shape[0])   # keys older than offset - window
            if drop > 0:
                cache["k"], cache["v"] = cache["k"][drop:], cache["v"][drop:]
                base += drop
                cache["base"] = base
        h = rms_norm(x, self.param(f"{p}.attention_norm.weight"), c.norm_eps)
        q = self.linear(h, f"{p}.attention.wq.weight", f"{p}.attention.wq.bias").reshape(s, c.enc_heads, c.enc_head_dim)
        k = self.linear(h, f"{p}.attention.wk.weight").reshape(s, c.enc_heads, c.enc_head_dim)
        v = self.linear(h, f"{p}.attention.wv.weight", f"{p}.attention.wv.bias").reshape(s, c.enc_heads, c.enc_head_dim)
        q = apply_rope(q, self.enc_cos, self.enc_sin, offset)
        k = apply_rope(k, self.enc_cos, self.enc_sin, offset)
        cache["k"] = k if cache["k"] is None else torch.cat([cache["k"], k], 0)
        cache["v"] = v if cache["v"] is None else torch.cat([cache["v"], v], 0)
        a = self._attention(q, cache["k"], cache["v"], float(np.float32(c.enc_head_dim) ** np.float32(-0.5)),
                            offset - base, c.enc_window)   # masks only depend on position differences
        x = self.linear(a, f"{p}.attention.wo.weight", f"{p}.attention.wo.bias") + x
        h = rms_norm(x, self.param(f"{p}.ffn_norm.weight"), c.norm_eps)
        gate = F.silu(self.linear(h, f"{p}.feed_forward.w1.weight"))
        up = self.linear(h, f"{p}.feed_forward.w3.weight")
        return self.linear(gate * up, f"{p}.feed_forward.w2.weight", f"{p}.feed_forward.w2.bias") + x

    def encoder_forward_with_cache(self, mel: np.ndarray, enc_cache: list) -> torch.Tensor:
        """Q4AudioEncoder::forward_with_cache (model.rs:437-452): the conv stem runs on the chunk alone
        (zero padding at the chunk edges, no carried state -- as upstream), the layers extend the caches."""
        x = self.conv_stem(mel)
        for i in range(self.cfg.enc_layers):
            x = self.encoder_layer_with_cache(x, i, enc_cache[i])
        return self.encoder_norm(x)

    def encode_audio_with_cache(self, mel: np.ndarray, enc_cache: list) -> torch.Tensor:
        """Q4VoxtralModel::encode_audio_with_cache (model.rs:790-799)."""
        return self.adapter(self.encoder_forward_with_cache(mel, enc_cache))

    # ---- decoder ----------------------------------------------------------
    def ada_scales(self, t_embed: np.ndarray):
        """Q4AdaRmsNorm (model.rs:250-255): 1 + w2(gelu(w0(t))) per layer (t constant)."""
        t = torch.from_numpy(np.ascontiguousarray(t_embed, np.float32)).reshape(1, -1).to(self.dtype)
        out = []
        for j in range(self.cfg.dec_layers):
            s = self.linear(t, f"layers.{j}.ada_rms_norm_t_cond.0.weight")
            s = self.linear(F.gelu(s), f"layers.{j}.ada_rms_norm_t_cond.2.weight")
            out.append((s + 1.0)[0])
        return out

    def embed_tokens(self, ids) -> torch.Tensor:
        """embed_from_q4_bytes (model.rs:584-618)."""
        dt, (v, d), _ = self.g.info(TOK_EMB)
        raw = self.g.raw(TOK_EMB).reshape(v, d // 32 * 18)
        rows = [torch.from_numpy(q4.dequantize_q4_0(raw[int(i)])) for i in ids]
        return torch.stack(rows).to(self.dtype)

    def new_cache(self):
        return [dict(k=None, v=None) for _ in range(self.cfg.dec_layers)]

    def decoder_forward_with_cache(self, x: torch.Tensor, ada, cache, capture=None) -> torch.Tensor:
        """forward_hidden_with_cache (model.rs:665-677); x [M, D]."""
        c = self.cfg
        m = x.shape[0]
        scale = float(np.float32(c.dec_head_dim) ** np.float32(-0.5))
        for j in range(c.dec_layers):
            p = f"layers.{j}"
            off = 0 if cache[j]["k"] is None else cache[j]["k"].shape[0]
            h = rms_norm(x, self.param(f"{p}.attention_norm.weight"), c.norm_eps)
            q = self.linear(h, f"{p}.attention.wq.weight").reshape(m, c.dec_heads, c.dec_head_dim)
            k = self.linear(h, f"{p}.attention.wk.weight").reshape(m, c.dec_kv_heads, c.dec_head_dim)
            v = self.linear(h, f"{p}.attention.wv.weight").reshape(m, c.dec_kv_heads, c.dec_head_dim)
            q = apply_rope(q, self.dec_cos, self.dec_sin, off)
            k = apply_rope(k, self.dec_cos, self.dec_sin, off)
            if off == 0:
                cache[j]["k"], cache[j]["v"] = k, v
            else:
                cache[j]["k"] = torch.cat([cache[j]["k"], k])
                cache[j]["v"] = torch.cat([cache[j]["v"], v])
            a = self._attention(q, cache[j]["k"], cache[j]["v"], scale, off, c.dec_window)
            x = self.linear(a, f"{p}.attention.wo.weight") + x
            h = rms_norm(x, self.param(f"{p}.ffn_norm.weight"), c.norm_eps)
            h = h * ada[j]
            gate = F.silu(self.linear(h, f"{p}.feed_forward.w1.weight"))
            up = self.linear(h, f"{p}.feed_forward.w3.weight")
            x = self.linear(gate * up, f"{p}.feed_forward.w2.weight") + x
            if capture is not None:
                capture[f"dec{j}"] = x.clone()
        return rms_norm(x, self.param(FINAL_NORM), c.norm_eps)

    def decoder_forward_batched(self, x: torch.Tensor, ada, caches, rows_per_stream: int = 1) -> torch.Tensor:
        """forward_hidden_with_cache (model.rs:665-677) for B independent streams in ONE weight sweep: x
        [B*rows_per_stream, D] (stream-major), caches = one LayerCaches per stream.  Every linear sees all rows at once
        (the weights are read once for the whole batch, as the GPU path does); attention stays per stream.  Same
        arithmetic per row as decoder_forward_with_cache -- used by bench.py's CPU arm so that the CPU baseline runs the
        SAME batched workload as the GPU arm."""
        c = self.cfg
        m = rows_per_stream
        nb = x.shape[0] // m
        scale = float(np.float32(c.dec_head_dim) ** np.float32(-0.5))
        for j in range(c.dec_layers):
            p = f"layers.{j}"
            h = rms_norm(x, self.param(f"{p}.attention_norm.weight"), c.norm_eps)
            q = self.linear(h, f"{p}.attention.wq.weight")
            k = self.linear(h, f"{p}.attention.wk.weight")
            v = self.linear(h, f"{p}.attention.wv.weight")
            outs = []
            for b in range(nb):
                cache = caches[b]
                off = 0 if cache[j]["k"] is None else cache[j]["k"].shape[0]
                sl = slice(b * m, (b + 1) * m)
                qb = apply_rope(q[sl].reshape(m, c.dec_heads, c.dec_head_dim), self.dec_cos, self.dec_sin, off)
                kb = apply_rope(k[sl].reshape(m, c.dec_kv_heads, c.dec_head_dim), self.dec_cos, self.dec_sin, off)
                vb = v[sl].reshape(m, c.dec_kv_heads, c.dec_head_dim)
                cache[j]["k"] = kb if off == 0 else torch.cat([cache[j]["k"], kb])
                cache[j]["v"] = vb if off == 0 else torch.cat([cache[j]["v"], vb])
                outs.append(self._attention(qb, cache[j]["k"], cache[j]["v"], scale, off, c.dec_window))
            x = self.linear(torch.cat(outs), f"{p}.attention.wo.weight") + x
            h = rms_norm(x, self.param(f"{p}.ffn_norm.weight"), c.norm_eps) * ada[j]
            gate = F.silu(self.linear(h, f"{p}.feed_forward.w1.weight"))
            up = self.linear(h, f"{p}.feed_forward.w3.weight")
            x = self.linear(gate * up, f"{p}.feed_forward.w2.weight") + x
        return rms_norm(x, self.param(FINAL_NORM), c.norm_eps)

    def lm_head(self, h: torch.Tensor) -> torch.Tensor:
        """model.rs:680-691 (tied embeddings)."""
        return self.linear(h, TOK_EMB)

    def forward_streaming(self, mel: np.ndarray, token_ids, t_embed: np.ndarray, audio_embeds=None,
                          return_hidden: bool = False):
        """Q4VoxtralModel::forward_streaming (model.rs:801-814): logits [S, V] for a full teacher-forced pass,
        inputs = audio_embeds + embed(token_ids), no cache carried in.  This is the graph the reference's
        scripts/compare_full_forward.py:262-361 evaluates (token_ids = [32]*S)."""
        audio = self.encode_audio(mel) if audio_embeds is None else audio_embeds
        ids = list(token_ids)
        assert len(ids) == audio.shape[0]
        x = torch.as_tensor(audio).to(self.dtype) + self.embed_tokens(ids)
        hidden = self.decoder_forward_with_cache(x, self.ada_scales(t_embed), self.new_cache())
        logits = self.lm_head(hidden)
        return (logits, hidden) if return_hidden else logits

    def transcribe_streaming(self, mel: np.ndarray, t_embed: np.ndarray, audio_embeds=None,
                             info: dict | None = None):
        """model.rs:873-963 -> list[int] of length seq_len-38 ([] if seq_len<38).
        `info` (optional) receives top-2 logit margins per emitted token."""
        audio = self.encode_audio(mel) if audio_embeds is None else audio_embeds
        seq_len = audio.shape[0]
        if seq_len < PREFIX_LEN:
            return []
        ada = self.ada_scales(t_embed)
        prefix = [BOS_TOKEN] + [STREAMING_PAD] * (PREFIX_LEN - 1)
        x = audio[:PREFIX_LEN] + self.embed_tokens(prefix)
        cache = self.new_cache()
        hidden = self.decoder_forward_with_cache(x, ada, cache)
        margins = []
        seconds = []

        def pick(hrow):
            logits = self.lm_head(hrow.reshape(1, -1))[0]
            top2 = torch.topk(logits, 2)
            margins.append(float(top2.values[0] - top2.values[1]))
            seconds.append(int(top2.indices[1]))
            return int(torch.argmax(logits))          # lowest index on ties

        generated = prefix + [pick(hidden[PREFIX_LEN - 1])]
        for pos in range(PREFIX_LEN + 1, seq_len):
            tok = generated[pos - 1]
            x = audio[pos - 1:pos] + self.embed_tokens([tok])
            hidden = self.decoder_forward_with_cache(x, ada, cache)
            generated.append(pick(hidden[0]))
        if info is not None:
            info["margins"] = margins
            info["second"] = seconds
            info["audio_embeds"] = audio
        return generated[PREFIX_LEN:]
