"""Synthetic inputs for tests and benchmarks (no real weights / audio exist offline, SURVEY F3).

  * a GGUF v3 *writer* producing files with the exact tensor names, shapes and dtypes the reference's
    loader expects (src/gguf/loader.rs:215-383, names src/models/weights.rs:219-230,294-390; layout
    src/gguf/reader.rs:105-188: dims stored reversed, 32-byte aligned data section) filled with
    deterministic random Q4_0 blocks / f32 vectors;
  * in-memory builders shaped like the reference's test helpers (src/gguf/tests.rs:90-168);
  * synthetic 16 kHz signals (benches/audio.rs:13-18 sine, a noise+chirp, a speech-like mix).

This is data generation only -- no model arithmetic lives here.  Model dims are hard-coded in the
reference (config.rs:441-486) and it skips all metadata KVs; tiny test models carry optional
`voxtral.*` u32 KVs so the same loader can run them (the reference would skip those keys).
"""
from __future__ import annotations

import io
import math
import os
import struct
import zlib
from dataclasses import dataclass, replace

import numpy as np

GGUF_MAGIC = 0x46554747
ALIGN = 32
F32_T, F16_T, Q4_0_T = 0, 1, 2
SAMPLE_RATE = 16000

ENC = "mm_streams_embeddings.embedding_module.whisper_encoder"
ADAPTER = "mm_streams_embeddings.embedding_module.audio_language_projection"
TOK_EMB = "mm_streams_embeddings.embedding_module.tok_embeddings.weight"
FINAL_NORM = "norm.weight"
ATTN_OUT_GAIN = float(os.environ.get("VOX_SYNTH_ATTN_GAIN", "0.25"))


@dataclass
class VoxtralConfig:
    # encoder (config.rs:441-460)
    n_mels: int = 128
    enc_dim: int = 1280
    enc_layers: int = 32
    enc_heads: int = 32
    enc_head_dim: int = 64
    enc_ffn: int = 5120
    enc_window: int = 750
    # decoder (config.rs:462-486)
    dec_dim: int = 3072
    dec_layers: int = 26
    dec_heads: int = 32
    dec_kv_heads: int = 8
    dec_head_dim: int = 128
    dec_ffn: int = 9216
    dec_window: int = 8192
    vocab: int = 131072
    t_cond_dim: int = 32
    reshape_factor: int = 4
    rope_theta: float = 1_000_000.0
    norm_eps: float = 1e-5

    @staticmethod
    def tiny() -> "VoxtralConfig":
        """Small config with the same structure (non-square projections, GQA 2:1, sliding window
        small enough to bite)."""
        return VoxtralConfig(enc_dim=64, enc_layers=2, enc_heads=4, enc_head_dim=32, enc_ffn=128,
                             enc_window=20, dec_dim=96, dec_layers=2, dec_heads=4, dec_kv_heads=2,
                             dec_head_dim=32, dec_ffn=160, dec_window=8192, vocab=512)

    def kv_items(self):
        return [
            ("voxtral.enc.n_layers", self.enc_layers), ("voxtral.enc.n_heads", self.enc_heads),
            ("voxtral.enc.head_dim", self.enc_head_dim), ("voxtral.enc.sliding_window", self.enc_window),
            ("voxtral.dec.n_layers", self.dec_layers), ("voxtral.dec.n_heads", self.dec_heads),
            ("voxtral.dec.n_kv_heads", self.dec_kv_heads), ("voxtral.dec.head_dim", self.dec_head_dim),
            ("voxtral.dec.sliding_window", self.dec_window),
            ("voxtral.reshape_factor", self.reshape_factor),
        ]


def tensor_manifest(cfg: VoxtralConfig):
    """[(name, dtype_code, torch_shape)] in file order (SURVEY Appendix A)."""
    out = []
    d, hd = cfg.enc_dim, cfg.enc_heads * cfg.enc_head_dim
    out += [(f"{ENC}.conv_layers.0.conv.weight", F32_T, (d, cfg.n_mels, 3)),
            (f"{ENC}.conv_layers.0.conv.bias", F32_T, (d,)),
            (f"{ENC}.conv_layers.1.conv.weight", F32_T, (d, d, 3)),
            (f"{ENC}.conv_layers.1.conv.bias", F32_T, (d,))]
    for i in range(cfg.enc_layers):
        p = f"{ENC}.transformer.layers.{i}"
        out += [(f"{p}.attention_norm.weight", F32_T, (d,)),
                (f"{p}.attention.wq.weight", Q4_0_T, (hd, d)), (f"{p}.attention.wq.bias", F32_T, (hd,)),
                (f"{p}.attention.wk.weight", Q4_0_T, (hd, d)),
                (f"{p}.attention.wv.weight", Q4_0_T, (hd, d)), (f"{p}.attention.wv.bias", F32_T, (hd,)),
                (f"{p}.attention.wo.weight", Q4_0_T, (d, hd)), (f"{p}.attention.wo.bias", F32_T, (d,)),
                (f"{p}.ffn_norm.weight", F32_T, (d,)),
                (f"{p}.feed_forward.w1.weight", Q4_0_T, (cfg.enc_ffn, d)),
                (f"{p}.feed_forward.w2.weight", Q4_0_T, (d, cfg.enc_ffn)),
                (f"{p}.feed_forward.w2.bias", F32_T, (d,)),
                (f"{p}.feed_forward.w3.weight", Q4_0_T, (cfg.enc_ffn, d))]
    out += [(f"{ENC}.transformer.norm.weight", F32_T, (d,))]
    D = cfg.dec_dim
    out += [(f"{ADAPTER}.0.weight", Q4_0_T, (D, d * cfg.reshape_factor)),
            (f"{ADAPTER}.2.weight", Q4_0_T, (D, D)),
            (TOK_EMB, Q4_0_T, (cfg.vocab, D))]
    qd, kvd = cfg.dec_heads * cfg.dec_head_dim, cfg.dec_kv_heads * cfg.dec_head_dim
    for j in range(cfg.dec_layers):
        p = f"layers.{j}"
        out += [(f"{p}.ada_rms_norm_t_cond.0.weight", Q4_0_T, (cfg.t_cond_dim, D)),
                (f"{p}.ada_rms_norm_t_cond.2.weight", Q4_0_T, (D, cfg.t_cond_dim)),
                (f"{p}.attention_norm.weight", F32_T, (D,)),
                (f"{p}.attention.wq.weight", Q4_0_T, (qd, D)),
                (f"{p}.attention.wk.weight", Q4_0_T, (kvd, D)),
                (f"{p}.attention.wv.weight", Q4_0_T, (kvd, D)),
                (f"{p}.attention.wo.weight", Q4_0_T, (D, qd)),
                (f"{p}.ffn_norm.weight", F32_T, (D,)),
                (f"{p}.feed_forward.w1.weight", Q4_0_T, (cfg.dec_ffn, D)),
                (f"{p}.feed_forward.w2.weight", Q4_0_T, (D, cfg.dec_ffn)),
                (f"{p}.feed_forward.w3.weight", Q4_0_T, (cfg.dec_ffn, D))]
    out += [(FINAL_NORM, F32_T, (D,))]
    return out


def nbytes_of(dtype: int, shape) -> int:
    n = int(np.prod(shape))
    return {F32_T: n * 4, F16_T: n * 2, Q4_0_T: n // 32 * 18}[dtype]


def _rng(seed: int, name: str) -> np.random.Generator:
    return np.random.Generator(np.random.PCG64([seed, zlib.crc32(name.encode())]))


def random_q4_blocks(rng: np.random.Generator, n_elements: int, std: float) -> np.ndarray:
    """Random Q4_0 payload whose dequantised values have std ~= `std`: nibbles uniform in 1..15
    (q-8 symmetric in -7..7) with ~1/64 forced to 0 (= -8*d, which the reference's test quantiser
    never emits but the dequant rule must accept), f16 scales d = std/4.3 * U(0.5,1.5)."""
    nb = n_elements // 32
    out = np.empty((nb, 18), np.uint8)
    d = (std / 4.3 * rng.uniform(0.5, 1.5, nb)).astype(np.float16)
    out[:, 0:2] = d.view(np.uint8).reshape(nb, 2)
    a = rng.integers(0, 225, size=(nb, 16), dtype=np.uint8)   # 225 = 15^2: two independent base-15 digits
    lo = (a % 15 + 1).astype(np.uint8)
    hi = (a // 15 + 1).astype(np.uint8)
    z = rng.integers(0, 256, size=(nb, 16), dtype=np.uint8)
    # forced nibble 0 (-8) on 4/256 of the entries, balanced by nibble 15 (+7) on 5/256 so that the
    # weights stay zero-mean (mean(q-8) = 3/256): a coherent negative mean would otherwise be
    # amplified through the residual stack (K*mean vs sqrt(K)*std) and collapse every position
    # onto the all-ones direction.
    lo[z < 4] = 0
    lo[(z >= 4) & (z < 9)] = 15
    hi[(z >= 9) & (z < 13)] = 0
    hi[(z >= 13) & (z < 18)] = 15
    out[:, 2:] = lo | (hi << 4)
    return out.reshape(-1)


def synth_tensor_bytes(name: str, dtype: int, shape, seed: int, audio_gain: float = 2.0) -> np.ndarray:
    """Deterministic synthetic payload (uint8 array) for one tensor.  Linear weights are
    variance-preserving (std 1/sqrt(K)); the last adapter layer is scaled so that audio and text
    embeddings have comparable magnitude (token feedback then matters for the greedy sequence)."""
    rng = _rng(seed, name)
    n = int(np.prod(shape))
    if dtype == Q4_0_T:
        k = int(shape[-1])
        s = 1.0 / math.sqrt(k)
        if name == f"{ADAPTER}.2.weight":
            s = audio_gain / k
        elif name.endswith("attention.wo.weight"):
            # softmax attention averages values over positions; at gain 1 a random deep stack
            # rank-collapses (every position converges to the same vector).  A small output
            # projection keeps the per-position signal alive so the greedy tokens depend on the audio.
            s *= ATTN_OUT_GAIN
        return random_q4_blocks(rng, n, s)
    if name.endswith("norm.weight"):
        v = 1.0 + 0.01 * rng.standard_normal(n)
    elif name.endswith(".bias"):
        v = 0.01 * rng.standard_normal(n)
    else:  # conv weights [out, in, 3]
        v = (1.5 / math.sqrt(shape[1] * shape[2])) * rng.standard_normal(n)
    if dtype == F16_T:
        return v.astype(np.float16).view(np.uint8)
    return v.astype(np.float32).view(np.uint8)


def _w_str(b, s: str):
    e = s.encode()
    b.write(struct.pack("<Q", len(e)))
    b.write(e)


def header_bytes(tensors, kvs, version=3) -> bytes:
    """tensors: [(name, dtype, torch_shape, offset)]"""
    b = io.BytesIO()
    b.write(struct.pack("<IIQQ", GGUF_MAGIC, version, len(tensors), len(kvs)))
    for key, val in kvs:
        _w_str(b, key)
        if isinstance(val, str):
            b.write(struct.pack("<I", 8))
            _w_str(b, val)
        elif isinstance(val, float):
            b.write(struct.pack("<If", 6, val))
        else:
            b.write(struct.pack("<II", 4, int(val)))
    for name, dtype, shape, off in tensors:
        _w_str(b, name)
        b.write(struct.pack("<I", len(shape)))
        for dim in reversed(shape):  # GGUF order = reversed torch order (loader.rs:497-499)
            b.write(struct.pack("<Q", int(dim)))
        b.write(struct.pack("<IQ", dtype, off))
    b.write(b"\0" * ((-b.tell()) % ALIGN))
    return b.getvalue()


def build_gguf_bytes(tensors, kvs=(("general.architecture", "voxtral"),), version=3) -> bytes:
    """In-memory GGUF like tests.rs:90-168.  tensors: [(name, dtype, torch_shape, uint8 data)].
    Offsets are cumulative without inter-tensor padding, as in the reference's builders."""
    metas, off = [], 0
    for name, dtype, shape, data in tensors:
        metas.append((name, dtype, shape, off))
        off += len(data)
    out = io.BytesIO()
    out.write(header_bytes(metas, list(kvs), version))
    for _, _, _, data in tensors:
        out.write(bytes(data))
    return out.getvalue()


def write_synthetic_gguf(path: str, cfg: VoxtralConfig, seed: int = 42, f16_norms: bool = False,
                         audio_gain: float = 2.0) -> dict:
    """Stream a synthetic Voxtral GGUF to `path` (tensor data 32-byte aligned, like llama.cpp-produced
    files).  Returns {"bytes": total, "q4_bytes": ..., "tensors": ...}."""
    man = tensor_manifest(cfg)
    if f16_norms:
        man = [(n, F16_T if (dt == F32_T and n.endswith("norm.weight")) else dt, sh) for n, dt, sh in man]
    metas, off, q4b = [], 0, 0
    for name, dtype, shape in man:
        off = (off + ALIGN - 1) // ALIGN * ALIGN
        metas.append((name, dtype, shape, off))
        nb = nbytes_of(dtype, shape)
        off += nb
        if dtype == Q4_0_T:
            q4b += nb
    kvs = [("general.architecture", "voxtral")] + cfg.kv_items()
    hdr = header_bytes(metas, kvs)
    tmp = f"{path}.tmp{os.getpid()}"
    with open(tmp, "wb") as f:
        f.write(hdr)
        base = f.tell()
        for name, dtype, shape, o in metas:
            cur = f.tell() - base
            if cur < o:
                f.write(b"\0" * (o - cur))
            f.write(synth_tensor_bytes(name, dtype, shape, seed, audio_gain).tobytes())
        total = f.tell()
    os.replace(tmp, path)
    return {"bytes": total, "q4_bytes": q4b, "tensors": len(metas)}


def refshape_config() -> VoxtralConfig:
    """Every dimension the reference's torch scripts hard-code (scripts/generate_padded_reference.py:95-187,
    compare_full_forward.py:278-361: 1280 / 32x64 / 32 layers, 3072 / 32:8x128 / 26 layers) with small FFNs and
    vocabulary -- the model tests/golden/make_reference_fixtures.py runs the reference Python on."""
    return VoxtralConfig(enc_ffn=512, dec_ffn=512, vocab=4096)


def decoder_geometry_config(dec_window: int = 8192) -> VoxtralConfig:
    """The production decoder layer (3072, 32:8 x 128 heads, FFN 9216) at 2 layers, a 32768-token vocabulary and the
    tiny encoder: every decoder matvec, attention shape and persistent-kernel plan (K slices, 2048 lm_head tiles) is the
    full model's, at a size a CPU reference can follow step by step.  `dec_window` makes the decoder's sliding window
    small enough to bite within a few seconds of audio."""
    t = VoxtralConfig.tiny()
    return VoxtralConfig(enc_dim=t.enc_dim, enc_layers=t.enc_layers, enc_heads=t.enc_heads, enc_head_dim=t.enc_head_dim,
                         enc_ffn=t.enc_ffn, enc_window=t.enc_window, dec_layers=2, dec_window=dec_window, vocab=32768)


def encoder_geometry_config(enc_window: int = 750) -> VoxtralConfig:
    """The production encoder layer (1280, 32 x 64 heads, FFN 5120) at 2 layers, the production adapter (5120 -> 3072 ->
    3072) and decoder_geometry_config's decoder (3072, 32:8 x 128 heads, FFN 9216, 2 layers, vocabulary 32768): every
    encoder GEMM, matvec, attention shape and K/V ring of the full model at a size a CPU reference can follow layer by
    layer.  `enc_window` (production 750) sets where the encoder's sliding window bites."""
    return replace(decoder_geometry_config(), enc_dim=1280, enc_layers=2, enc_heads=32, enc_head_dim=64, enc_ffn=5120,
                   enc_window=enc_window)


def tiny_window_config(dec_window: int = 48) -> VoxtralConfig:
    """The tiny model with a decoder window short enough that a reference started part-way into a long stream (empty
    caches, absolute positions) equals the whole stream's after dec_layers x dec_window positions."""
    return replace(VoxtralConfig.tiny(), dec_window=dec_window)


def build_aliased_gguf_bytes(cfg: VoxtralConfig, seed: int, unique: int = 2) -> bytes:
    """In-memory GGUF whose layers i >= `unique` alias the bytes of layer i % unique (several names, one offset
    in the tensor index -- legal GGUF), so a full-depth model costs `unique` layers of bytes and of generation
    time.  Deterministic; data 32-byte aligned."""
    def canon(name):
        for pre in (f"{ENC}.transformer.layers.", "layers."):
            if name.startswith(pre):
                idx, rest = name[len(pre):].split(".", 1)
                return f"{pre}{int(idx) % unique}.{rest}"
        return name

    metas, blobs, offs, off = [], [], {}, 0
    for name, dt, shape in tensor_manifest(cfg):
        c = canon(name)
        if c not in offs:
            off = (off + ALIGN - 1) // ALIGN * ALIGN
            data = synth_tensor_bytes(c, dt, shape, seed).tobytes()
            offs[c] = off
            blobs.append((off, data))
            off += len(data)
        metas.append((name, dt, shape, offs[c]))
    hdr = header_bytes(metas, [("general.architecture", "voxtral")] + cfg.kv_items())
    out = bytearray(hdr)
    for o, data in blobs:
        out.extend(b"\0" * (len(hdr) + o - len(out)))
        out.extend(data)
    return bytes(out)


# ------------------------------------------------------------------------------ signals
def sine_16k(seconds: float, freq: float = 440.0, amp: float = 0.5) -> np.ndarray:
    """benches/audio.rs:13-18."""
    n = int(seconds * SAMPLE_RATE)
    i = np.arange(n, dtype=np.float64)
    return (amp * np.sin(2.0 * math.pi * freq * i / SAMPLE_RATE)).astype(np.float32)


def noise_chirp(seconds: float, seed: int = 1234) -> np.ndarray:
    """Seeded N(0,1)*0.1 noise + linear chirp 100->4000 Hz (SURVEY 8d config 3)."""
    n = int(seconds * SAMPLE_RATE)
    rng = np.random.Generator(np.random.PCG64(seed))
    t = np.arange(n, dtype=np.float64) / SAMPLE_RATE
    f0, f1 = 100.0, 4000.0
    phase = 2.0 * math.pi * (f0 * t + 0.5 * (f1 - f0) * t * t / max(seconds, 1e-9))
    return (0.1 * rng.standard_normal(n) + 0.5 * np.sin(phase)).astype(np.float32)


def speechlike(seconds: float, seed: int = 1234) -> np.ndarray:
    """Synthetic 'speech-like' signal: 40-200 ms segments, each a mix of three random sinusoids
    (80-5000 Hz) with a random envelope, ~15% silent gaps, plus a noise floor -- a mel spectrogram
    that changes every few frames."""
    n = int(seconds * SAMPLE_RATE)
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.zeros(n, np.float64)
    pos = 0
    while pos < n:
        seg = int(rng.uniform(0.04, 0.2) * SAMPLE_RATE)
        end = min(n, pos + seg)
        if rng.random() > 0.15:
            t = np.arange(end - pos) / SAMPLE_RATE
            amp = rng.uniform(0.05, 0.6)
            sig = np.zeros(end - pos)
            for _ in range(3):
                f = math.exp(rng.uniform(math.log(80.0), math.log(5000.0)))
                sig += rng.uniform(0.2, 1.0) * np.sin(2 * math.pi * f * t + rng.uniform(0, 2 * math.pi))
            env = np.hanning(end - pos) ** 0.25
            out[pos:end] = amp * sig * env / 3.0
        pos = end
    out += 0.003 * rng.standard_normal(n)
    return out.astype(np.float32)
