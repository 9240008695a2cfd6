"""ctypes binding of libvoxtral_b200.so, shaped like the reference crate's API (see __init__).

Error behaviour mirrors the reference: loader/IO problems surface as exceptions with the
reference's message texts where it has them (``anyhow`` contexts in reader.rs / loader.rs);
shape panics (op.rs:92-100) become ``VoxtralError`` instead of process aborts.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_NAME = "libvoxtral_b200.so"


class VoxtralError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"[vox {code}] {msg}")
        self.code = code
        self.msg = msg


def lib_path() -> str:
    # VOX_LIB_PATH: load another build of the same library (A/B runs of two kernel versions on one GPU box)
    return os.environ.get("VOX_LIB_PATH") or os.path.join(_HERE, _LIB_NAME)


_lib = None


class _PadConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_uint32), ("n_left_pad_tokens", C.c_uint32), ("frame_rate", C.c_float),
                ("extra_right_pad_tokens", C.c_uint32)]


class _Chunk(C.Structure):
    _fields_ = [("start_sample", C.c_size_t), ("end_sample", C.c_size_t), ("index", C.c_size_t),
                ("is_last", C.c_int32)]


class _ModelInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mels", "enc_dim", "enc_layers", "enc_heads", "enc_head_dim", "enc_ffn", "enc_window",
        "dec_dim", "dec_layers", "dec_heads", "dec_kv_heads", "dec_head_dim", "dec_ffn", "dec_window",
        "vocab", "t_cond_dim", "reshape_factor", "prefix_len")] + [
        ("q4_bytes", C.c_uint64), ("device_bytes", C.c_uint64), ("decode_step_bytes", C.c_uint64)]


class _Timings(C.Structure):
    _fields_ = [("preprocess_ms", C.c_float), ("encode_ms", C.c_float), ("decode_ms", C.c_float),
                ("total_ms", C.c_float), ("prefill_ms", C.c_float), ("decode_tokens", C.c_int32), ("seq_len", C.c_int32)]


@dataclass
class Timings:
    preprocess_ms: float = 0.0
    encode_ms: float = 0.0
    decode_ms: float = 0.0
    total_ms: float = 0.0
    prefill_ms: float = 0.0
    decode_tokens: int = 0
    seq_len: int = 0


# name -> (restype, argtypes); every declaration in include/voxtral.h appears here
_P = C.c_void_p
_SIGS = {
    "vox_last_error": (C.c_char_p, []),
    "vox_version": (C.c_int32, []),
    "vox_device_count": (C.c_int32, []),
    "vox_gguf_open": (C.c_int32, [C.c_char_p, C.POINTER(_P)]),
    "vox_gguf_open_shards": (C.c_int32, [C.POINTER(_P), C.POINTER(C.c_size_t), C.c_size_t, C.POINTER(_P)]),
    "vox_gguf_version": (C.c_int32, [_P, C.POINTER(C.c_uint32)]),
    "vox_gguf_tensor_count": (C.c_int32, [_P, C.POINTER(C.c_uint64)]),
    "vox_gguf_tensor_name": (C.c_int32, [_P, C.c_uint64, C.POINTER(C.c_char_p)]),
    "vox_gguf_tensor_info": (C.c_int32, [_P, C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                         C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "vox_gguf_tensor_data": (C.c_int32, [_P, C.c_char_p, _P, C.c_size_t]),
    "vox_gguf_close": (None, [_P]),
    "vox_peak_normalize": (C.c_int32, [_P, C.c_size_t, C.c_float]),
    "vox_pad_config_default": (None, [C.POINTER(_PadConfig)]),
    "vox_pad_audio_len": (C.c_size_t, [C.c_size_t, C.POINTER(_PadConfig)]),
    "vox_pad_audio": (C.c_int32, [_P, C.c_size_t, C.POINTER(_PadConfig), _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "vox_stream_progress": (C.c_int32, [C.c_size_t, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]),
    "vox_chunk_plan": (C.c_int32, [C.c_size_t, C.c_size_t, C.c_size_t, C.POINTER(_Chunk), C.c_size_t,
                                   C.POINTER(C.c_size_t)]),
    "vox_time_embedding": (C.c_int32, [C.c_float, C.c_int32, _P]),
    "vox_mel_create": (C.c_int32, [C.c_int32, C.POINTER(_P)]),
    "vox_mel_num_frames": (C.c_size_t, [C.c_size_t]),
    "vox_mel_compute_log": (C.c_int32, [_P, _P, C.c_size_t, _P, C.c_size_t]),
    "vox_mel_compute_log_dev": (C.c_int32, [_P, _P, C.c_size_t, _P, C.c_int32, _P]),
    "vox_mel_filterbank": (C.c_int32, [_P, _P]),
    "vox_mel_window": (C.c_int32, [_P, _P]),
    "vox_mel_free": (None, [_P]),
    "vox_q4_tensor_create": (C.c_int32, [_P, C.c_size_t, C.c_int64, C.c_int64, C.c_int32, C.POINTER(_P)]),
    "vox_q4_tensor_shape": (C.c_int32, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "vox_q4_tensor_dequantize": (C.c_int32, [_P, _P]),
    "vox_q4_matmul": (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P]),
    "vox_q4_matmul_host": (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P]),
    "vox_q4_linear": (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, C.c_float, _P,
                                  C.c_int32, _P, _P, _P]),
    "vox_q4_tensor_free": (None, [_P]),
    "vox_attention": (C.c_int32, [C.c_int32, C.c_int32, _P, _P]),
    "vox_dec_attention": (C.c_int32, [C.c_int32, C.c_int32, _P, _P]),
    "vox_q4_set_matvec_mode": (C.c_int32, [C.c_int32]),
    "vox_dev_malloc": (C.c_int32, [C.c_int32, C.c_size_t, C.POINTER(_P)]),
    "vox_dev_free": (C.c_int32, [C.c_int32, _P]),
    "vox_dev_upload": (C.c_int32, [C.c_int32, _P, _P, C.c_size_t]),
    "vox_dev_download": (C.c_int32, [C.c_int32, _P, _P, C.c_size_t]),
    "vox_dev_sync": (C.c_int32, [C.c_int32]),
    "vox_profiler_start": (C.c_int32, []),
    "vox_profiler_stop": (C.c_int32, []),
    "vox_host_alloc_pinned": (C.c_int32, [C.c_size_t, C.POINTER(_P)]),
    "vox_host_free_pinned": (C.c_int32, [_P]),
    "vox_q4_matmul_bench": (C.c_int32, [C.POINTER(_P), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.POINTER(C.c_float)]),
    "vox_model_load_gguf": (C.c_int32, [C.c_char_p, C.c_int32, C.POINTER(_P)]),
    "vox_model_load_gguf_handle": (C.c_int32, [_P, C.c_int32, C.POINTER(_P)]),
    "vox_model_get_info": (C.c_int32, [_P, C.POINTER(_ModelInfo)]),
    "vox_model_free": (None, [_P]),
    "vox_session_create": (C.c_int32, [_P, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "vox_session_create_ex": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "vox_session_device_bytes": (C.c_int32, [_P, C.POINTER(C.c_uint64)]),
    "vox_session_set_delay": (C.c_int32, [_P, C.c_float]),
    "vox_session_set_delays": (C.c_int32, [_P, _P, C.c_int32]),
    "vox_encode_audio": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_int32)]),
    "vox_transcribe_streaming": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_int32),
                                             C.POINTER(_Timings)]),
    "vox_transcribe_pcm": (C.c_int32, [_P, _P, C.c_int32, C.c_size_t, C.c_int32, _P, C.c_size_t,
                                       C.POINTER(C.c_int32), C.POINTER(_Timings)]),
    "vox_transcribe_pcm_ragged": (C.c_int32, [_P, _P, _P, C.c_int32, C.c_int32, _P, C.c_size_t, _P,
                                              C.POINTER(_Timings)]),
    "vox_transcribe_pcm_dev": (C.c_int32, [_P, _P, C.c_int32, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_int32),
                                           C.POINTER(_Timings)]),
    "vox_generate_step_with_cache": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, C.c_size_t]),
    "vox_forward_streaming": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P, C.c_int32, _P, C.c_size_t]),
    "vox_prefill": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    "vox_decode_step": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, _P]),
    "vox_session_set_top_k": (C.c_int32, [_P, C.c_int32]),
    "vox_session_token_scores": (C.c_int32, [_P, _P, _P, C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                             C.POINTER(C.c_int32)]),
    "vox_session_set_beam": (C.c_int32, [_P, C.c_int32]),
    "vox_session_nbest": (C.c_int32, [_P, _P, _P, C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                      C.POINTER(C.c_int32)]),
    "vox_session_set_bias": (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32]),
    "vox_session_set_bias_text": (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32]),
    "vox_session_cache_len": (C.c_int32, [_P, C.POINTER(C.c_int32)]),
    "vox_session_reset": (C.c_int32, [_P]),
    "vox_session_debug_read": (C.c_int32, [_P, C.c_char_p, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "vox_session_launch_count": (C.c_int32, [_P, C.POINTER(C.c_uint64)]),
    "vox_session_free": (None, [_P]),
    "vox_stream_pool_create": (C.c_int32, [_P, C.c_int32, C.c_float, C.POINTER(_P)]),
    "vox_stream_pool_create_ex": (C.c_int32, [_P, C.c_int32, C.c_float, C.c_int32, C.POINTER(_P)]),
    "vox_stream_pool_device_bytes": (C.c_int32, [_P, C.POINTER(C.c_uint64)]),
    "vox_stream_open": (C.c_int32, [_P, C.POINTER(C.c_int32)]),
    "vox_stream_set_delay": (C.c_int32, [_P, C.c_int32, C.c_float]),
    "vox_stream_set_bias": (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32]),
    "vox_stream_set_bias_text": (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_int32]),
    "vox_stream_push_pcm": (C.c_int32, [_P, C.c_int32, _P, C.c_size_t]),
    "vox_stream_finish": (C.c_int32, [_P, C.c_int32]),
    "vox_stream_tick": (C.c_int32, [_P, _P]),
    "vox_stream_poll_ids": (C.c_int32, [_P, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int32)]),
    "vox_stream_pool_set_top_k": (C.c_int32, [_P, C.c_int32]),
    "vox_stream_poll_scored": (C.c_int32, [_P, C.c_int32, _P, _P, _P, C.c_size_t, C.POINTER(C.c_size_t),
                                           C.POINTER(C.c_int32)]),
    "vox_stream_audio_embeds": (C.c_int32, [_P, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_int32)]),
    "vox_stream_audio_embeds_range": (C.c_int32, [_P, C.c_int32, C.c_int64, C.c_int64, _P, C.c_size_t]),
    "vox_stream_mel_range": (C.c_int32, [_P, C.c_int32, C.c_int64, C.c_int64, _P, C.c_size_t]),
    "vox_stream_session_info": (C.c_int32, [_P, C.c_int32, _P]),
    "vox_stream_encode_chunk": (C.c_int32, [_P, C.c_int32, _P, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_int32)]),
    "vox_stream_close": (C.c_int32, [_P, C.c_int32]),
    "vox_stream_pool_free": (None, [_P]),
    "vox_tokenizer_from_file": (C.c_int32, [C.c_char_p, C.POINTER(_P)]),
    "vox_tokenizer_from_json": (C.c_int32, [C.c_char_p, C.c_size_t, C.POINTER(_P)]),
    "vox_tokenizer_decode": (C.c_int32, [_P, _P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "vox_tokenizer_decode_token": (C.c_int32, [_P, C.c_uint32, _P, C.c_size_t, C.POINTER(C.c_size_t),
                                               C.POINTER(C.c_int32)]),
    "vox_tokenizer_vocab_size": (C.c_int32, [_P, C.POINTER(C.c_size_t)]),
    "vox_tokenizer_encode": (C.c_int32, [_P, C.c_char_p, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "vox_tokenizer_free": (None, [_P]),
}


def lib():
    """Load libvoxtral_b200.so (fails loudly if it was not built: there is no fallback)."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.exists(path):
            raise VoxtralError(-1, f"{path} not found -- run `python -m voxtral_mini_realtime_rs_b200.build` "
                                   "(or __graft_entry__.build()); there is no CPU/PyTorch fallback")
        l = C.CDLL(path)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def _check(code: int):
    if code != 0:
        raise VoxtralError(code, lib().vox_last_error().decode("utf-8", "replace"))


def device_count() -> int:
    return int(lib().vox_device_count())


def _bias_args(phrases, boost):
    """(ids, lens, boosts, n) of vox_session_set_bias for a list of id phrases and one boost or one per phrase."""
    phrases = [[int(t) for t in p] for p in phrases]
    n = len(phrases)
    boosts = np.broadcast_to(np.asarray(boost, np.float32), (n,)).copy()
    lens = np.array([len(p) for p in phrases], np.int32)
    ids = np.array([t for p in phrases for t in p], np.int32)
    keep = [ids, lens, boosts]
    ptr = (lambda a: _ptr(a) if a.size else None)
    return keep, ptr(ids), ptr(lens), ptr(boosts), n


def _bias_text_args(phrases, boost):
    """(keep, phrases, boosts, n) of vox_session_set_bias_text for a list of words and one boost or one per word."""
    words = [p.encode("utf-8") if isinstance(p, str) else bytes(p) for p in phrases]
    if any(b"\0" in w for w in words):
        raise ValueError("a phrase contains a NUL character")
    n = len(words)
    arr = (C.c_char_p * max(n, 1))(*words)
    boosts = np.broadcast_to(np.asarray(boost, np.float32), (n,)).copy()
    return (arr, boosts), (C.cast(arr, _P) if n else None), (_ptr(boosts) if n else None), n


def _tok_handle(tokenizer):
    return None if tokenizer is None else tokenizer._h


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------ GGUF
class GgufReader:
    """GgufReader (reader.rs:88-223).  `open(path)`, `from_bytes(b)`, `from_shards([b0,b1,..])`."""

    def __init__(self, handle, keep=None):
        self._h = handle
        self._keep = keep

    @staticmethod
    def open(path: str) -> "GgufReader":
        h = _P()
        _check(lib().vox_gguf_open(os.fsencode(path), C.byref(h)))
        return GgufReader(h)

    @staticmethod
    def from_shards(shards) -> "GgufReader":
        bufs = [np.frombuffer(s, dtype=np.uint8) for s in shards]
        n = len(bufs)
        ptrs = (_P * n)(*[b.ctypes.data for b in bufs])
        lens = (C.c_size_t * n)(*[b.size for b in bufs])
        h = _P()
        _check(lib().vox_gguf_open_shards(ptrs, lens, n, C.byref(h)))
        return GgufReader(h, keep=(bufs, shards))

    @staticmethod
    def from_bytes(data) -> "GgufReader":
        return GgufReader.from_shards([data])

    def version(self) -> int:
        v = C.c_uint32()
        _check(lib().vox_gguf_version(self._h, C.byref(v)))
        return v.value

    def tensor_count(self) -> int:
        v = C.c_uint64()
        _check(lib().vox_gguf_tensor_count(self._h, C.byref(v)))
        return v.value

    def tensor_names(self):
        out = []
        for i in range(self.tensor_count()):
            s = C.c_char_p()
            _check(lib().vox_gguf_tensor_name(self._h, i, C.byref(s)))
            out.append(s.value.decode())
        return out

    def tensor_info(self, name: str):
        """-> dict(shape=<GGUF-order dims>, dtype=<code>, nbytes=...) or None (reader.rs:201)."""
        dt, nd, nb = C.c_uint32(), C.c_uint32(), C.c_uint64()
        dims = (C.c_uint64 * 4)()
        code = lib().vox_gguf_tensor_info(self._h, name.encode(), C.byref(dt), C.byref(nd), dims, C.byref(nb))
        if code == 3:
            return None
        _check(code)
        return dict(shape=tuple(dims[i] for i in range(nd.value)), dtype=dt.value, nbytes=nb.value)

    def tensor_data(self, name: str) -> np.ndarray:
        info = self.tensor_info(name)
        if info is None:
            raise VoxtralError(3, f"Tensor '{name}' not found in GGUF")
        buf = np.empty(info["nbytes"], np.uint8)
        _check(lib().vox_gguf_tensor_data(self._h, name.encode(), _ptr(buf), buf.size))
        return buf

    def close(self):
        if self._h:
            lib().vox_gguf_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------ audio plumbing
def peak_normalize(samples, target_peak: float = 0.95) -> np.ndarray:
    """AudioBuffer::peak_normalize (io.rs:59-68); returns a new array."""
    s = _f32(samples).copy()
    _check(lib().vox_peak_normalize(_ptr(s), s.size, target_peak))
    return s


peak_normalize_samples = peak_normalize


class PadConfig:
    """PadConfig (pad.rs:20-46)."""

    def __init__(self, sample_rate=16000, n_left_pad_tokens=76, frame_rate=12.5, extra_right_pad_tokens=17):
        self.c = _PadConfig(sample_rate, n_left_pad_tokens, frame_rate, extra_right_pad_tokens)

    @staticmethod
    def voxtral() -> "PadConfig":
        return PadConfig()

    def samples_per_token(self) -> int:
        return int(np.float32(self.c.sample_rate) / np.float32(self.c.frame_rate))

    def left_pad_samples(self) -> int:
        return self.c.n_left_pad_tokens * self.samples_per_token()


def pad_audio(samples, config: PadConfig | None = None) -> np.ndarray:
    """pad_audio (pad.rs:89-103)."""
    s = _f32(samples)
    cfg = C.byref(config.c) if config else None
    n = lib().vox_pad_audio_len(s.size, cfg)
    out = np.empty(n, np.float32)
    ln = C.c_size_t()
    _check(lib().vox_pad_audio(_ptr(s), s.size, cfg, _ptr(out), out.size, C.byref(ln)))
    return out[:ln.value]


def chunk_audio(n_samples: int, max_mel_frames: int = 1500, overlap_frames: int = 0):
    """chunk_audio (chunk.rs:159-161) as a plan: [(start, end, index, is_last)]."""
    cnt = C.c_size_t()
    _check(lib().vox_chunk_plan(n_samples, max_mel_frames, overlap_frames, None, 0, C.byref(cnt)))
    arr = (_Chunk * max(cnt.value, 1))()
    _check(lib().vox_chunk_plan(n_samples, max_mel_frames, overlap_frames, arr, cnt.value, C.byref(cnt)))
    return [(arr[i].start_sample, arr[i].end_sample, arr[i].index, bool(arr[i].is_last)) for i in range(cnt.value)]


def stream_progress(n_samples: int, ended: bool = False, reshape_factor: int = 4, prefix_len: int = 38):
    """Final outputs per stage once `n_samples` padded samples are known: (mel frames, conv1 frames, encoder
    frames, audio embeddings, emit-able token ids) -- the bookkeeping of a streaming session (SURVEY 8(f)-1)."""
    out = (C.c_int64 * 5)()
    _check(lib().vox_stream_progress(n_samples, 1 if ended else 0, reshape_factor, prefix_len, out))
    return tuple(int(v) for v in out)


def needs_chunking(n_samples: int, max_mel_frames: int = 1500) -> bool:
    return n_samples > max_mel_frames * 160


def stream_n_out(n_samples: int, reshape_factor: int = 4, prefix_len: int = 38) -> int:
    """Token ids a transcribe call emits for one stream of n_samples: pad_audio length -> mel frames -> two
    stride-2 convolutions (k3 p1) -> / reshape_factor -> minus the prefix (0 when shorter)."""
    return frames_n_out(lib().vox_mel_num_frames(lib().vox_pad_audio_len(n_samples, None)), reshape_factor, prefix_len)


def frames_n_out(mel_frames: int, reshape_factor: int = 4, prefix_len: int = 38) -> int:
    """Token ids a transcribe call emits for mel_frames frames (see stream_n_out)."""
    t = mel_frames
    for _ in range(2):
        t = (t + 2 - 3) // 2 + 1
    return max(0, t // reshape_factor - prefix_len)


def join_chunk_texts(tokenizer, chunk_ids) -> str:
    """The reference CLI's join of independently transcribed chunks (transcribe.rs:256-275): per chunk keep the ids
    >= 1000 (text tokens), decode, trim; drop empty texts; join with one space."""
    texts = []
    for ids in chunk_ids:
        text = tokenizer.decode([int(i) for i in ids if int(i) >= 1000]).strip()
        if text:
            texts.append(text)
    return " ".join(texts)


class TimeEmbedding:
    """TimeEmbedding (time_embedding.rs:12-71)."""

    def __init__(self, dim: int):
        self.dim = dim

    def embed(self, t: float) -> np.ndarray:
        out = np.empty(self.dim, np.float32)
        _check(lib().vox_time_embedding(t, self.dim, _ptr(out)))
        return out.reshape(1, 1, self.dim)


# ------------------------------------------------------------------------------ mel
class MelSpectrogram:
    """MelSpectrogram::voxtral() (mel.rs:73-182) on the GPU."""

    def __init__(self, device: int = 0):
        self._h = _P()
        self.device = device
        _check(lib().vox_mel_create(device, C.byref(self._h)))

    @staticmethod
    def voxtral(device: int = 0) -> "MelSpectrogram":
        return MelSpectrogram(device)

    @staticmethod
    def num_frames(num_samples: int) -> int:
        return int(lib().vox_mel_num_frames(num_samples))

    def compute_log(self, samples) -> np.ndarray:
        """-> float32 [n_frames, 128] (mel.rs:128-165)."""
        s = _f32(samples)
        fr = self.num_frames(s.size)
        out = np.empty((fr, 128), np.float32)
        _check(lib().vox_mel_compute_log(self._h, _ptr(s), s.size, _ptr(out), out.size))
        return out

    def mel_basis(self) -> np.ndarray:
        out = np.empty((128, 201), np.float32)
        _check(lib().vox_mel_filterbank(self._h, _ptr(out)))
        return out

    def window(self) -> np.ndarray:
        out = np.empty(400, np.float32)
        _check(lib().vox_mel_window(self._h, _ptr(out)))
        return out

    def __del__(self):
        try:
            if self._h:
                lib().vox_mel_free(self._h)
                self._h = None
        except Exception:
            pass


# ------------------------------------------------------------------------------ Q4 operator
class DeviceBuffer:
    """Raw device allocation for driving the *_dev entry points without torch."""

    def __init__(self, nbytes: int, device: int = 0):
        self.device, self.nbytes = device, nbytes
        self.ptr = _P()
        _check(lib().vox_dev_malloc(device, nbytes, C.byref(self.ptr)))

    @staticmethod
    def from_numpy(a: np.ndarray, device: int = 0) -> "DeviceBuffer":
        a = np.ascontiguousarray(a)
        b = DeviceBuffer(a.nbytes, device)
        _check(lib().vox_dev_upload(device, b.ptr, _ptr(a), a.nbytes))
        return b

    def to_numpy(self, dtype, shape) -> np.ndarray:
        out = np.empty(shape, dtype)
        _check(lib().vox_dev_download(self.device, _ptr(out), self.ptr, out.nbytes))
        return out

    def free(self):
        if self.ptr:
            lib().vox_dev_free(self.device, self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PinnedArray:
    """float32/int32 numpy view over page-locked host memory (cudaHostAlloc)."""

    def __init__(self, shape, dtype=np.float32):
        self.nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self.ptr = _P()
        _check(lib().vox_host_alloc_pinned(max(self.nbytes, 16), C.byref(self.ptr)))
        buf = (C.c_char * max(self.nbytes, 16)).from_address(self.ptr.value)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def free(self):
        if self.ptr:
            self.array = None
            lib().vox_host_free_pinned(self.ptr)
            self.ptr = None


class Q4Tensor:
    """Q4Tensor (tensor.rs:16-113): raw Q4_0 blocks -> HBM (repacked at upload)."""

    def __init__(self, handle, shape, device):
        self._h, self._shape, self.device = handle, tuple(shape), device

    @staticmethod
    def from_q4_bytes(raw_bytes, shape, device: int = 0) -> "Q4Tensor":
        raw = np.ascontiguousarray(np.frombuffer(raw_bytes, dtype=np.uint8) if not isinstance(raw_bytes, np.ndarray)
                                   else raw_bytes.astype(np.uint8, copy=False))
        n, k = int(shape[0]), int(shape[1])
        h = _P()
        _check(lib().vox_q4_tensor_create(_ptr(raw), raw.size, n, k, device, C.byref(h)))
        return Q4Tensor(h, (n, k), device)

    def shape(self):
        return self._shape

    def num_blocks(self) -> int:
        return self._shape[0] * self._shape[1] // 32

    def dequantize(self) -> np.ndarray:
        out = np.empty(self._shape, np.float32)
        _check(lib().vox_q4_tensor_dequantize(self._h, _ptr(out)))
        return out

    def __del__(self):
        try:
            if self._h:
                lib().vox_q4_tensor_free(self._h)
                self._h = None
        except Exception:
            pass


def q4_matmul(x, weights: Q4Tensor, bias=None) -> np.ndarray:
    """q4_matmul (op.rs:86-137): x [B,M,K] host f32 -> [B,M,N] host f32 (upload, kernel, download)."""
    x = _f32(x)
    if x.ndim != 3:
        raise VoxtralError(1, "Input must be 3D [B, M, K]")
    b, m, k = x.shape
    n, wk = weights.shape()
    if k != wk:
        raise VoxtralError(1, f"K dimension mismatch: input has {k}, weights have {wk}")
    y = np.empty((b, m, n), np.float32)
    bp = None
    if bias is not None:
        bias = _f32(bias)
        if bias.size != n:
            raise VoxtralError(1, f"bias has {bias.size} elements, expected {n}")
        bp = _ptr(bias)
    _check(lib().vox_q4_matmul_host(weights._h, _ptr(x), _ptr(y), b, m, bp))
    return y


EPILOGUES = {"none": 0, "residual": 1, "silu_mul": 2, "gelu": 3}   # include/voxtral.h VOX_EPI_*


def q4_linear(weights: Q4Tensor, x, epi: str = "none", *, bias=None, res=None, gamma=None, eps: float = 1e-5,
              ada=None, ada_m: int = 1, ssq_in=None, want_ssq_out: bool = False, ldy: int | None = None,
              y_rows: int | None = None, sentinel: float = float("nan"), in_place: bool = False):
    """One fused linear layer (vox_q4_linear) on host arrays: y[r] = epi(norm(x[r]) . W^T + bias) (+ res[r]).

    x [rows, K].  ada: [streams, K], row r takes ada[r // ada_m].  res [rows, N] (residual only).  ssq_in
    [ceil(K/16), rows].  y is a [y_rows, ldy] device buffer (defaults: rows, and N or N/2 for SiLU*up) pre-filled with
    `sentinel`, and res is copied into its first rows when in_place (y == res).  Returns y whole, and with
    want_ssq_out the [ceil(N/16), rows] partial sums of squares too."""
    n, k = weights.shape()
    x = _f32(x).reshape(-1, k)
    rows = x.shape[0]
    cols = n // 2 if epi == "silu_mul" else n
    ldy = cols if ldy is None else ldy
    y_rows = rows if y_rows is None else y_rows
    dev = weights.device
    keep = []

    def up(a, dtype=np.float32):
        if a is None:
            return None
        b = DeviceBuffer.from_numpy(np.ascontiguousarray(a, dtype), dev)
        keep.append(b)
        return b.ptr

    y_host = np.full((y_rows, ldy), sentinel, np.float32)
    if res is not None:
        res = _f32(res).reshape(rows, n)
        if in_place:
            y_host[:rows, :n] = res
    y = DeviceBuffer.from_numpy(y_host, dev)
    keep.append(y)
    res_ptr = None
    if res is not None:
        if in_place:
            res_ptr = y.ptr
        else:
            r = np.full((rows, ldy), sentinel, np.float32)
            r[:, :n] = res
            res_ptr = up(r)
    ada_ptr = None
    if ada is not None:
        vecs = [up(v) for v in _f32(ada).reshape(-1, k)]
        ada_ptr = up(np.array([v.value for v in vecs], np.uint64), np.uint64)
    ssq_shape = ((n + 15) // 16, rows)
    ssq_out = DeviceBuffer.from_numpy(np.full(ssq_shape, sentinel, np.float32), dev) if want_ssq_out else None
    _check(lib().vox_q4_linear(weights._h, up(x), y.ptr, rows, ldy, up(bias), res_ptr, EPILOGUES[epi], up(gamma),
                               eps, ada_ptr, ada_m, up(ssq_in), ssq_out.ptr if ssq_out else None, None))
    _check(lib().vox_dev_sync(dev))
    out = y.to_numpy(np.float32, (y_rows, ldy))
    if ssq_out is not None:
        return out, ssq_out.to_numpy(np.float32, ssq_shape)
    return out


ATTN_KERNELS = {"tc": 0, "simt": 1, "stream": 2}   # include/voxtral.h VOX_ATTN_*


class _AttnArgs(C.Structure):
    _fields_ = [("qkv", _P), ("ld", C.c_int32), ("q_off", C.c_int32), ("k_off", C.c_int32), ("v_off", C.c_int32),
                ("b", C.c_int32), ("s", C.c_int32), ("h", C.c_int32), ("hd", C.c_int32), ("seg", _P),
                ("rows", C.c_int32), ("row_slot", _P), ("row_pos", _P), ("k_ring", _P), ("v_ring", _P),
                ("ring", C.c_int32), ("window", C.c_int32), ("scale", C.c_float), ("out", _P)]


def attention(kernel: str, qkv, h: int, hd: int, window: int, scale: float, *, q_off: int = 0, k_off: int = 0,
              v_off: int = 0, b: int = 1, s: int | None = None, seg=None, row_slot=None, row_pos=None, k_ring=None,
              v_ring=None, out_rows: int | None = None, sentinel: float = float("nan"), device: int = 0) -> np.ndarray:
    """One encoder attention launch (vox_attention) on host arrays, on the named kernel ("tc", "simt" or "stream").

    qkv [rows, ld]: for "tc" / "simt" the q, k and v of head hh at columns {q,k,v}_off + hh * hd of each row; b
    streams of s rows each, or the ragged streams seg[t] .. seg[t + 1] - 1 ([b + 1] offsets; s defaults to the longest).
    For "stream", row r is query position row_pos[r] of session row_slot[r], with q at columns hh * hd; k_ring / v_ring
    [slots, ring, h * hd] hold key position p at p % ring.  out is an [out_rows, h * hd] device buffer (default: the
    rows of qkv) pre-filled with `sentinel`, returned whole."""
    qkv = _f32(qkv)
    rows, ld = qkv.shape
    keep = []

    def up(a, dtype):
        if a is None:
            return None
        buf = DeviceBuffer.from_numpy(np.ascontiguousarray(a, dtype), device)
        keep.append(buf)
        return buf.ptr

    a = _AttnArgs(qkv=up(qkv, np.float32), ld=ld, h=h, hd=hd, window=window, scale=scale)
    if kernel == "stream":
        k_ring = _f32(k_ring)
        a.rows, a.ring = rows, k_ring.shape[1]
        a.row_slot, a.row_pos = up(row_slot, np.int32), up(row_pos, np.int32)
        a.k_ring, a.v_ring = up(k_ring, np.float32), up(v_ring, np.float32)
    else:
        a.q_off, a.k_off, a.v_off, a.b = q_off, k_off, v_off, b
        if seg is not None:
            seg = np.asarray(seg, np.int32)
            a.seg = up(seg, np.int32)
            s = int(np.diff(seg).max()) if s is None else s
        a.s = rows // b if s is None else s
    out_rows = rows if out_rows is None else out_rows
    out = DeviceBuffer.from_numpy(np.full((out_rows, h * hd), sentinel, np.float32), device)
    keep.append(out)
    a.out = out.ptr
    _check(lib().vox_attention(device, ATTN_KERNELS[kernel], C.byref(a), None))
    _check(lib().vox_dev_sync(device))
    return out.to_numpy(np.float32, (out_rows, h * hd))


DEC_ATTN_KERNELS = {"fused": 0, "prefill": 1}   # include/voxtral.h VOX_DEC_ATTN_*


class _DecAttnArgs(C.Structure):
    _fields_ = [("qkv", _P), ("ld", C.c_int32), ("b", C.c_int32), ("m", C.c_int32), ("h", C.c_int32),
                ("hkv", C.c_int32), ("hd", C.c_int32), ("kv_dtype", C.c_int32), ("k_pool", _P), ("v_pool", _P),
                ("page_table", _P), ("max_pages", C.c_int32), ("ring", C.c_int32), ("pos", _P), ("cos", _P),
                ("sin", _P), ("rope_rows", C.c_int32), ("window", C.c_int32), ("scale", C.c_float), ("out", _P)]


def dec_attention(kernel: str, qkv, *, b: int, m: int, h: int, hkv: int, hd: int, kv_dtype: str, k_pool, v_pool,
                  page_table, pos, cos, sin, window: int, scale: float, ring: bool = False, out_rows: int | None = None,
                  sentinel: float = float("nan"), device: int = 0):
    """One decoder attention launch (vox_dec_attention) on host arrays, on the named kernel ("fused" or "prefill").

    qkv [b * m, ld] f32; k_pool / v_pool: the cache's pages in their stored form (any dtype, uploaded as bytes);
    page_table [b, max_pages] and pos [b] int32; cos / sin [rope_rows, hd / 2] f32.  out is an [out_rows, h * hd]
    device buffer (default b * m rows) pre-filled with `sentinel`.  Returns (out, qkv, k_pool, v_pool), each as it is on
    the device after the call, in the dtype and shape it was given."""
    qkv = _f32(qkv)
    keep = []

    def up(a):
        buf = DeviceBuffer.from_numpy(a, device)
        keep.append(buf)
        return buf

    page_table = np.ascontiguousarray(page_table, np.int32)
    k_pool, v_pool = np.ascontiguousarray(k_pool), np.ascontiguousarray(v_pool)
    bufs = [up(qkv), up(k_pool), up(v_pool)]
    out_rows = b * m if out_rows is None else out_rows
    out = up(np.full((out_rows, h * hd), sentinel, np.float32))
    a = _DecAttnArgs(qkv=bufs[0].ptr, ld=qkv.shape[1], b=b, m=m, h=h, hkv=hkv, hd=hd, kv_dtype=_kv_dtype(kv_dtype),
                     k_pool=bufs[1].ptr, v_pool=bufs[2].ptr, page_table=up(page_table).ptr,
                     max_pages=page_table.shape[1], ring=int(ring), pos=up(np.ascontiguousarray(pos, np.int32)).ptr,
                     cos=up(_f32(cos)).ptr, sin=up(_f32(sin)).ptr, rope_rows=np.shape(cos)[0], window=window,
                     scale=scale, out=out.ptr)
    _check(lib().vox_dec_attention(device, DEC_ATTN_KERNELS[kernel], C.byref(a), None))
    _check(lib().vox_dev_sync(device))
    return (out.to_numpy(np.float32, (out_rows, h * hd)),
            *(buf.to_numpy(arr.dtype, arr.shape) for buf, arr in zip(bufs, (qkv, k_pool, v_pool))))


class Q4Linear:
    """Q4Linear (linear.rs:17-40)."""

    def __init__(self, weights: Q4Tensor, bias=None):
        self.weights, self.bias = weights, bias

    def forward(self, x) -> np.ndarray:
        return q4_matmul(x, self.weights, self.bias)


def q4_matmul_bench(weights, m: int, iters: int = 200, warmup: int = 20) -> float:
    """Average ms per launch over `iters` launches rotating over `weights` (defeats L2)."""
    n = len(weights)
    arr = (_P * n)(*[w._h for w in weights])
    ms = C.c_float()
    _check(lib().vox_q4_matmul_bench(arr, n, m, iters, warmup, C.byref(ms)))
    return ms.value


# decoder KV cache element types (include/voxtral.h vox_session_create_ex): VOX_DTYPE_F32, VOX_DTYPE_F16, VOX_DTYPE_KV_Q8
KV_DTYPES = {"f32": 0, "f16": 1, "q8": 100}


def _kv_dtype(kv_dtype: str) -> int:
    if kv_dtype not in KV_DTYPES:
        raise ValueError(f"kv_dtype {kv_dtype!r}: one of {sorted(KV_DTYPES)}")
    return KV_DTYPES[kv_dtype]


# ------------------------------------------------------------------------------ model
class Q4VoxtralModel:
    """Q4VoxtralModel (model.rs:759-989) + its session state (LayerCaches, workspace, stream)."""

    def __init__(self, model_handle, device: int, max_batch: int = 1, max_mel_frames: int = 3000,
                 kv_dtype: str = "f32"):
        self._m = model_handle
        self.device = device
        info = _ModelInfo()
        _check(lib().vox_model_get_info(self._m, C.byref(info)))
        self.info = {f[0]: getattr(info, f[0]) for f in _ModelInfo._fields_}
        self._s = _P()
        self.max_batch, self.max_mel_frames = max_batch, max_mel_frames
        self.kv_dtype = kv_dtype
        _check(lib().vox_session_create_ex(self._m, max_batch, max_mel_frames, _kv_dtype(kv_dtype), C.byref(self._s)))

    def device_bytes(self) -> int:
        """Device memory the session holds, in bytes (vox_session_device_bytes)."""
        n = C.c_uint64()
        _check(lib().vox_session_device_bytes(self._s, C.byref(n)))
        return n.value

    def set_delay(self, delay_tokens: float):
        _check(lib().vox_session_set_delay(self._s, delay_tokens))

    def set_delays(self, delays):
        """Stream i of later calls is conditioned on delays[i] (tokens of 80 ms); streams beyond len(delays) keep
        theirs.  Rows at different delays share one decode step."""
        d = _f32(delays).reshape(-1)
        _check(lib().vox_session_set_delays(self._s, _ptr(d), d.size))

    def _mel3(self, mel):
        mel = _f32(mel)
        if mel.ndim == 2:
            mel = mel[None]
        if mel.ndim != 3 or mel.shape[1] != self.info["n_mels"]:
            raise VoxtralError(1, f"mel must be [B,{self.info['n_mels']},T], got {mel.shape}")
        return mel

    def encode_audio(self, mel) -> np.ndarray:
        """mel [B,128,T] -> audio embeds [B, T/16, dec_dim] (model.rs:783-788)."""
        mel = self._mel3(mel)
        b, _, t = mel.shape
        t1 = (t + 2 - 3) // 2 + 1
        s = (t1 + 2 - 3) // 2 + 1
        s4 = s // self.info["reshape_factor"]
        out = np.empty((b, s4, self.info["dec_dim"]), np.float32)
        sl = C.c_int32()
        _check(lib().vox_encode_audio(self._s, _ptr(mel), b, t, _ptr(out), out.size, C.byref(sl)))
        assert sl.value == s4
        return out

    def transcribe_streaming(self, mel, t_embed=None, timings: Timings | None = None):
        """model.rs:873-963.  mel [B,128,T] (or [128,T]); returns list of token ids for B==1
        input given as 2-D/3-D with B==1, else an int32 array [B, n]."""
        mel = self._mel3(mel)
        b, _, t = mel.shape
        cap = b * max(t // 16 + 2, 1)
        out = np.zeros(cap, np.int32)
        n = C.c_int32()
        tm = _Timings()
        _check(lib().vox_transcribe_streaming(self._s, _ptr(mel), b, t, _ptr(out), out.size, C.byref(n), C.byref(tm)))
        self._fill(timings, tm)
        ids = out[: b * n.value].reshape(b, n.value)
        return ids[0].tolist() if b == 1 else ids

    def transcribe_pcm(self, samples, peak_normalize: bool = True, timings: Timings | None = None) -> np.ndarray:
        """Full pipeline for B equal-length streams: samples [B,n] (or [n]) host f32 -> ids [B, n_out]."""
        s = _f32(samples)
        if s.ndim == 1:
            s = s[None]
        b, n = s.shape
        cap = b * (n // 1280 + 120)
        out = np.zeros(cap, np.int32)
        no = C.c_int32()
        tm = _Timings()
        _check(lib().vox_transcribe_pcm(self._s, _ptr(s), b, n, 1 if peak_normalize else 0, _ptr(out), out.size,
                                        C.byref(no), C.byref(tm)))
        self._fill(timings, tm)
        return out[: b * no.value].reshape(b, no.value)

    def transcribe_pcm_ragged(self, streams, peak_normalize: bool = True, timings: Timings | None = None):
        """Streams of different lengths in one call (vox_transcribe_pcm_ragged): a list of 1-D f32 arrays -> a list of
        int32 id arrays, one per stream, each what transcribe_pcm gives that stream alone.  After the call,
        token_scores_ragged() and nbest_ragged() return the per-stream scores and n-best lists."""
        arrs = [_f32(x).reshape(-1) for x in streams]
        if not arrs:
            raise VoxtralError(1, "transcribe_pcm_ragged needs at least one stream")
        lens = np.array([a.size for a in arrs], np.uint64)
        n_out = [stream_n_out(int(n), self.info["reshape_factor"], self.info["prefix_len"]) for n in lens]
        samples = np.concatenate(arrs) if lens.sum() else np.zeros(1, np.float32)
        out = np.zeros(max(sum(n_out), 1), np.int32)
        no = np.zeros(len(arrs), np.int32)
        tm = _Timings()
        _check(lib().vox_transcribe_pcm_ragged(self._s, _ptr(samples), lens.ctypes.data_as(_P), len(arrs),
                                               1 if peak_normalize else 0, _ptr(out), sum(n_out), _ptr(no), C.byref(tm)))
        assert no.tolist() == n_out, (no.tolist(), n_out)
        self._fill(timings, tm)
        self._ragged_n = n_out
        offs = np.concatenate([[0], np.cumsum(n_out)]).astype(int)
        return [out[offs[i]:offs[i + 1]].copy() for i in range(len(arrs))]

    def token_scores_ragged(self):
        """Per stream (top_ids [n_out, k], top_logprobs [n_out, k]) of the last transcribe_pcm_ragged call."""
        n_out = self._ragged_n
        b, n, k = C.c_int32(), C.c_int32(), C.c_int32()
        _check(lib().vox_session_token_scores(self._s, None, None, 0, C.byref(b), C.byref(n), C.byref(k)))
        ids = np.empty((n.value, k.value), np.int32)
        lp = np.empty((n.value, k.value), np.float32)
        _check(lib().vox_session_token_scores(self._s, _ptr(ids), _ptr(lp), max(ids.size, 1), C.byref(b), C.byref(n),
                                              C.byref(k)))
        offs = np.concatenate([[0], np.cumsum(n_out)]).astype(int)
        return [(ids[offs[i]:offs[i + 1]], lp[offs[i]:offs[i + 1]]) for i in range(len(n_out))]

    def nbest_ragged(self):
        """Per stream (ids [W, n_out], scores [W]) of the last transcribe_pcm_ragged call at beam width W > 1."""
        n_out = self._ragged_n
        b, w, n = C.c_int32(), C.c_int32(), C.c_int32()
        _check(lib().vox_session_nbest(self._s, None, None, 0, C.byref(b), C.byref(w), C.byref(n)))
        W = w.value
        ids = np.empty(max(W * n.value, 1), np.int32)
        scores = np.empty((b.value, W), np.float64)
        _check(lib().vox_session_nbest(self._s, _ptr(ids), _ptr(scores), ids.size, C.byref(b), C.byref(w), C.byref(n)))
        out, off = [], 0
        for i, m in enumerate(n_out):
            out.append((ids[off:off + W * m].reshape(W, m), scores[i]))
            off += W * m
        return out

    def transcribe_long(self, samples, max_mel_frames: int = 1200, overlap_frames: int = 0, peak_normalize: bool = True):
        """A recording of any length, as the reference CLI transcribes it (transcribe.rs:187-275): peak-normalise the
        whole recording once, cut it with the chunk plan (vox_chunk_plan), transcribe every chunk on its own -- as
        rows of vox_transcribe_pcm_ragged calls of up to max_batch // W chunks (W the beam width).  Returns
        (per-chunk id arrays, the plan [(start, end, index, is_last)]); join_chunk_texts makes the text."""
        s = _f32(samples).reshape(-1)
        if peak_normalize:
            s = peak_normalize_samples(s)
        plan = chunk_audio(s.size, max_mel_frames, overlap_frames)
        per_call = max(1, self.max_batch // max(1, getattr(self, "_beam", 1)))
        ids = []
        for c0 in range(0, len(plan), per_call):
            group = plan[c0:c0 + per_call]
            ids.extend(self.transcribe_pcm_ragged([s[a:b] for a, b, _, _ in group], peak_normalize=False))
        return ids, plan

    def transcribe_pcm_dev(self, samples_dev: DeviceBuffer, b: int, n: int, timings: Timings | None = None) -> np.ndarray:
        cap = b * (n // 1280 + 120)
        out = np.zeros(cap, np.int32)
        no = C.c_int32()
        tm = _Timings()
        _check(lib().vox_transcribe_pcm_dev(self._s, samples_dev.ptr, b, n, _ptr(out), out.size, C.byref(no),
                                            C.byref(tm)))
        self._fill(timings, tm)
        return out[: b * no.value].reshape(b, no.value)

    @staticmethod
    def _fill(timings, tm):
        if timings is not None:
            for f, _ in _Timings._fields_:
                setattr(timings, f, getattr(tm, f))

    def generate_step_with_cache(self, token_ids) -> np.ndarray:
        """ids [B,M] -> logits [B,M,vocab]; appends to the decoder KV cache (model.rs:857-867)."""
        ids = np.ascontiguousarray(token_ids, dtype=np.int32)
        if ids.ndim == 1:
            ids = ids[None]
        b, m = ids.shape
        out = np.empty((b, m, self.info["vocab"]), np.float32)
        _check(lib().vox_generate_step_with_cache(self._s, _ptr(ids), b, m, _ptr(out), out.size))
        return out

    def forward_streaming(self, mel, token_ids) -> np.ndarray:
        """mel [B,128,T] (or [128,T]), ids [B,S] -> logits [B,S,vocab]: teacher-forced full pass with
        inputs = audio_embeds + embed(ids) (model.rs:801-814)."""
        mel = np.ascontiguousarray(mel, np.float32)
        if mel.ndim == 2:
            mel = mel[None]
        ids = np.ascontiguousarray(token_ids, dtype=np.int32)
        if ids.ndim == 1:
            ids = ids[None]
        b, _, t = mel.shape
        assert ids.shape[0] == b
        out = np.empty((b, ids.shape[1], self.info["vocab"]), np.float32)
        _check(lib().vox_forward_streaming(self._s, _ptr(mel), b, t, _ptr(ids), ids.shape[1], _ptr(out), out.size))
        return out

    def prefill(self, token_ids, add_audio: bool = True) -> np.ndarray:
        """ids [B,M] -> next token per stream [B]; greedy argmax on the device (vox_prefill)."""
        ids = np.ascontiguousarray(token_ids, dtype=np.int32)
        if ids.ndim == 1:
            ids = ids[None]
        b, m = ids.shape
        nxt = np.empty(b, np.int32)
        _check(lib().vox_prefill(self._s, _ptr(ids), b, m, int(add_audio), _ptr(nxt)))
        return nxt

    def decode_step(self, tok=None, batch: int | None = None, add_audio: bool = True, read: bool = True):
        """One decode position.  tok None = device-side feedback of the previous call (vox_decode_step)."""
        if tok is not None:
            tok = np.ascontiguousarray(tok, dtype=np.int32).reshape(-1)
            batch = tok.size
        assert batch is not None
        nxt = np.empty(batch, np.int32) if read else None
        _check(lib().vox_decode_step(self._s, _ptr(tok) if tok is not None else None, batch, int(add_audio),
                                     _ptr(nxt) if read else None))
        return nxt

    def set_top_k(self, k: int):
        """Token confidences for later transcribe / prefill / decode_step calls: the k (<= 8) most likely ids of every
        emitted token and their log-probabilities; 0 turns them off.  The ids do not change."""
        _check(lib().vox_session_set_top_k(self._s, k))

    def token_scores(self):
        """(top_ids [B,n,k] int32, top_logprobs [B,n,k] f32) of the last transcribe call (n = its tokens per stream) or
        of the last prefill / decode_step (n = 1).  top_ids[..., 0] is the emitted id."""
        b, n, k = C.c_int32(), C.c_int32(), C.c_int32()
        _check(lib().vox_session_token_scores(self._s, None, None, 0, C.byref(b), C.byref(n), C.byref(k)))
        ids = np.empty((b.value, n.value, k.value), np.int32)
        lp = np.empty((b.value, n.value, k.value), np.float32)
        _check(lib().vox_session_token_scores(self._s, _ptr(ids), _ptr(lp), ids.size, C.byref(b), C.byref(n), C.byref(k)))
        return ids, lp

    def set_beam(self, w: int):
        """Beam search of width w (1..8) for later transcribe calls; 1 is greedy.  B streams at width w need
        B * w <= max_batch.  The calls return the best hypothesis; nbest() returns all w."""
        _check(lib().vox_session_set_beam(self._s, w))
        self._beam = w

    def nbest(self):
        """(ids [B,W,n] int32, scores [B,W] float64) of the last transcribe call at beam width W > 1, in rank order;
        scores are summed log-probabilities."""
        b, w, n = C.c_int32(), C.c_int32(), C.c_int32()
        _check(lib().vox_session_nbest(self._s, None, None, 0, C.byref(b), C.byref(w), C.byref(n)))
        ids = np.empty((b.value, w.value, n.value), np.int32)
        scores = np.empty((b.value, w.value), np.float64)
        _check(lib().vox_session_nbest(self._s, _ptr(ids), _ptr(scores), ids.size, C.byref(b), C.byref(w), C.byref(n)))
        return ids, scores

    def set_bias(self, phrases, boost, stream: int | None = None):
        """Phrase boosting for greedy decoding: `phrases` is a list of token-id lists (ids >= 1000, up to 16 each, up to
        256 phrases), `boost` one float > 0 (logit units) or one per phrase.  At every emitted position the first id of
        every phrase, and the next id of every phrase whose prefix the stream's recent text ids end in, are boosted; the
        emitted id is the argmax of the boosted logits.  stream None: every stream; an empty list clears.  See
        vox_session_set_bias in include/voxtral.h."""
        _keep, ids, lens, boosts, n = _bias_args(phrases, boost)
        _check(lib().vox_session_set_bias(self._s, -1 if stream is None else stream, ids, lens, boosts, n))

    def set_bias_text(self, phrases, boost, tokenizer: "VoxtralTokenizer", stream: int | None = None):
        """set_bias with the phrases given as words (str, UTF-8): each word boosts its Tekken ids, and those of its
        leading-space form unless it starts with whitespace (vox_session_set_bias_text in include/voxtral.h: the
        expansion runs in the library).  `boost`: one float > 0 or one per word; an empty list clears."""
        _keep, words, boosts, n = _bias_text_args(phrases, boost)
        _check(lib().vox_session_set_bias_text(self._s, -1 if stream is None else stream, _tok_handle(tokenizer), words,
                                               boosts, n))

    def cache_len(self) -> int:
        v = C.c_int32()
        _check(lib().vox_session_cache_len(self._s, C.byref(v)))
        return v.value

    def reset_cache(self):
        _check(lib().vox_session_reset(self._s))

    def debug(self, what: str) -> np.ndarray | None:
        n = C.c_size_t()
        _check(lib().vox_session_debug_read(self._s, what.encode(), None, 0, C.byref(n)))
        if n.value == 0:
            return None
        out = np.empty(n.value, np.float32)
        _check(lib().vox_session_debug_read(self._s, what.encode(), _ptr(out), out.size, C.byref(n)))
        return out

    def launch_count(self) -> int:
        v = C.c_uint64()
        _check(lib().vox_session_launch_count(self._s, C.byref(v)))
        return v.value

    def close(self):
        if getattr(self, "_s", None):
            lib().vox_session_free(self._s)
            self._s = None
        if getattr(self, "_m", None):
            lib().vox_model_free(self._m)
            self._m = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _StreamStats(C.Structure):
    _fields_ = [("gpu_ms", C.c_float), ("live_sessions", C.c_int32), ("mel_frames", C.c_int32), ("encoder_rows", C.c_int32),
                ("prefills", C.c_int32), ("decode_steps", C.c_int32), ("decode_rows", C.c_int32)]


class _StreamSessionInfo(C.Structure):
    _fields_ = [("samples", C.c_int64), ("mel_frames", C.c_int64), ("encoder_frames", C.c_int64), ("audio_embeds", C.c_int64),
                ("first_audio_embed", C.c_int64), ("decoder_positions", C.c_int64), ("ids_emitted", C.c_int64),
                ("kv_pages", C.c_int32)]


class StreamingPool:
    """Live streaming sessions on one GPU worker (vox_stream_*; SURVEY 8(f)-1).  `model` stays owned by the caller
    and must outlive the pool.  max_seconds=None: sessions of any length, with fixed device state (30 s of padded audio
    resident per session; see include/voxtral.h)."""

    def __init__(self, model: "Q4VoxtralModel", max_sessions: int = 8, max_seconds: float | None = 30.0,
                 kv_dtype: str = "f32"):
        """kv_dtype: element type of the decoder KV cache the sessions share, "f32", "f16" or "q8" (include/voxtral.h)."""
        self._model = model
        self._p = _P()
        _check(lib().vox_stream_pool_create_ex(model._m, max_sessions, 0.0 if max_seconds is None else max_seconds,
                                               _kv_dtype(kv_dtype), C.byref(self._p)))
        self.dec_dim = model.info["dec_dim"]
        self.top_k = 0

    def device_bytes(self) -> int:
        """Device memory the pool holds, in bytes (vox_stream_pool_device_bytes)."""
        n = C.c_uint64()
        _check(lib().vox_stream_pool_device_bytes(self._p, C.byref(n)))
        return n.value

    def set_top_k(self, k: int):
        """Token confidences (Q4VoxtralModel.set_top_k) for every session of the pool; only while no session is open."""
        _check(lib().vox_stream_pool_set_top_k(self._p, k))
        self.top_k = k

    def open(self, delay: float | None = None) -> int:
        """A new session, at transcription delay `delay` (tokens of 80 ms; None: the default 6.0)."""
        v = C.c_int32()
        _check(lib().vox_stream_open(self._p, C.byref(v)))
        if delay is not None:
            try:
                self.set_delay(v.value, delay)
            except VoxtralError:
                self.close_session(v.value)
                raise
        return v.value

    def set_delay(self, session: int, delay: float):
        """The session's transcription delay; only before its prefill (session_info()["decoder_positions"] == 0)."""
        _check(lib().vox_stream_set_delay(self._p, session, delay))

    def set_bias(self, session: int, phrases, boost):
        """The session's phrase list (Q4VoxtralModel.set_bias); from its next decoder position.  open() starts a session
        with none."""
        _keep, ids, lens, boosts, n = _bias_args(phrases, boost)
        _check(lib().vox_stream_set_bias(self._p, session, ids, lens, boosts, n))

    def set_bias_text(self, session: int, phrases, boost, tokenizer: "VoxtralTokenizer"):
        """The session's phrase list from words (Q4VoxtralModel.set_bias_text)."""
        _keep, words, boosts, n = _bias_text_args(phrases, boost)
        _check(lib().vox_stream_set_bias_text(self._p, session, _tok_handle(tokenizer), words, boosts, n))

    def push(self, session: int, samples):
        s = _f32(samples).reshape(-1)
        _check(lib().vox_stream_push_pcm(self._p, session, _ptr(s), s.size))

    def finish(self, session: int):
        _check(lib().vox_stream_finish(self._p, session))

    def tick(self) -> dict:
        st = _StreamStats()
        _check(lib().vox_stream_tick(self._p, C.byref(st)))
        return {f[0]: getattr(st, f[0]) for f in _StreamStats._fields_}

    def poll(self, session: int, cap: int = 4096, scores: bool = False):
        """(ids, done) of the tokens emitted since the last poll; with scores=True (after set_top_k(k > 0))
        (ids, done, top_ids [n,k] int32, top_logprobs [n,k] f32)."""
        ids = np.empty(cap, np.int32)
        n, done = C.c_size_t(), C.c_int32()
        if not scores:
            _check(lib().vox_stream_poll_ids(self._p, session, _ptr(ids), cap, C.byref(n), C.byref(done)))
            return ids[:n.value].tolist(), bool(done.value)
        k = max(self.top_k, 1)
        top = np.empty((cap, k), np.int32)
        lp = np.empty((cap, k), np.float32)
        _check(lib().vox_stream_poll_scored(self._p, session, _ptr(ids), _ptr(top), _ptr(lp), cap, C.byref(n),
                                            C.byref(done)))
        return ids[:n.value].tolist(), bool(done.value), top[:n.value].copy(), lp[:n.value].copy()

    def session_info(self, session: int) -> dict:
        info = _StreamSessionInfo()
        _check(lib().vox_stream_session_info(self._p, session, C.byref(info)))
        return {f[0]: getattr(info, f[0]) for f in _StreamSessionInfo._fields_}

    def audio_embeds(self, session: int, first: int | None = None, n: int | None = None) -> np.ndarray:
        """All embeddings so far; or, with `first` and/or `n`, the resident rows [first, first + n) (default: from the
        first resident row to the last one produced)."""
        if first is not None or n is not None:
            info = self.session_info(session)
            first = info["first_audio_embed"] if first is None else first
            n = info["audio_embeds"] - first if n is None else n
            out = np.empty((n, self.dec_dim), np.float32)
            _check(lib().vox_stream_audio_embeds_range(self._p, session, first, n, _ptr(out), out.size))
            return out
        n = C.c_int32()
        _check(lib().vox_stream_audio_embeds(self._p, session, None, 0, C.byref(n)))
        out = np.empty((n.value, self.dec_dim), np.float32)
        _check(lib().vox_stream_audio_embeds(self._p, session, _ptr(out), out.size, C.byref(n)))
        return out

    def mel_range(self, session: int, first: int, n: int) -> np.ndarray:
        """Resident log-mel frames [first, first + n) of the session's padded stream (absolute indices) -> float32
        [n, 128] (vox_stream_mel_range)."""
        out = np.empty((n, 128), np.float32)
        _check(lib().vox_stream_mel_range(self._p, session, first, n, _ptr(out), out.size))
        return out

    def encode_audio_with_cache(self, session: int, mel) -> np.ndarray:
        """mel chunk [128,T] (or [1,128,T]) -> the chunk's audio embeddings [T/16, dec_dim]; the session's encoder
        K/V caches are extended (Q4VoxtralModel::encode_audio_with_cache, model.rs:790-799)."""
        mel = _f32(mel)
        if mel.ndim == 3:
            mel = mel[0]
        t = mel.shape[1]
        t1 = (t + 2 - 3) // 2 + 1
        s = (t1 + 2 - 3) // 2 + 1
        out = np.empty((s // 4 + 1, self.dec_dim), np.float32)
        n = C.c_int32()
        _check(lib().vox_stream_encode_chunk(self._p, session, _ptr(mel), t, _ptr(out), out.size, C.byref(n)))
        return out[:n.value].copy()

    def close_session(self, session: int):
        _check(lib().vox_stream_close(self._p, session))

    def close(self):
        if getattr(self, "_p", None):
            lib().vox_stream_pool_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Q4ModelLoader:
    """Q4ModelLoader (loader.rs:76-128): from_file / from_bytes / from_shards, then load(device)."""

    def __init__(self, reader: GgufReader | None = None, path: str | None = None):
        self._reader, self._path = reader, path

    @staticmethod
    def from_file(path: str) -> "Q4ModelLoader":
        if not os.path.exists(path):
            raise VoxtralError(2, f"Failed to open {path}")
        return Q4ModelLoader(GgufReader.open(path), path)

    @staticmethod
    def from_bytes(data) -> "Q4ModelLoader":
        return Q4ModelLoader(GgufReader.from_bytes(data))

    @staticmethod
    def from_shards(shards) -> "Q4ModelLoader":
        return Q4ModelLoader(GgufReader.from_shards(shards))

    def load(self, device: int = 0, max_batch: int = 1, max_mel_frames: int = 3000,
             kv_dtype: str = "f32") -> Q4VoxtralModel:
        """kv_dtype: element type of the session's decoder KV cache, "f32", "f16" or "q8" (include/voxtral.h)."""
        _kv_dtype(kv_dtype)
        h = _P()
        _check(lib().vox_model_load_gguf_handle(self._reader._h, device, C.byref(h)))
        return Q4VoxtralModel(h, device, max_batch, max_mel_frames, kv_dtype)


# ------------------------------------------------------------------------------ tokenizer
class VoxtralTokenizer:
    """VoxtralTokenizer (tokenizer/mod.rs:56-214), plus the Tekken encoder the reference lacks."""

    def __init__(self, handle):
        self._h = handle

    @staticmethod
    def from_file(path: str) -> "VoxtralTokenizer":
        h = _P()
        _check(lib().vox_tokenizer_from_file(os.fsencode(path), C.byref(h)))
        return VoxtralTokenizer(h)

    @staticmethod
    def from_json(json_str: str) -> "VoxtralTokenizer":
        raw = json_str.encode("utf-8")
        h = _P()
        _check(lib().vox_tokenizer_from_json(raw, len(raw), C.byref(h)))
        return VoxtralTokenizer(h)

    def decode(self, ids) -> str:
        a = np.ascontiguousarray(ids, dtype=np.uint32)
        n = C.c_size_t()
        _check(lib().vox_tokenizer_decode(self._h, _ptr(a), a.size, None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value + 1)
        _check(lib().vox_tokenizer_decode(self._h, _ptr(a), a.size, buf, n.value + 1, C.byref(n)))
        return buf.raw[: n.value].decode("utf-8")

    def decode_token(self, token_id: int):
        n, found = C.c_size_t(), C.c_int32()
        _check(lib().vox_tokenizer_decode_token(self._h, token_id, None, 0, C.byref(n), C.byref(found)))
        if not found.value:
            return None
        buf = C.create_string_buffer(n.value + 1)
        _check(lib().vox_tokenizer_decode_token(self._h, token_id, buf, n.value + 1, C.byref(n), C.byref(found)))
        return buf.raw[: n.value].decode("utf-8")

    def encode(self, text) -> np.ndarray:
        """Text ids (int32, >= 1000) of `text` (str, or bytes that must be UTF-8): mistral_common's
        Tekkenizer.encode(text, bos=False, eos=False)."""
        raw = text.encode("utf-8") if isinstance(text, str) else bytes(text)
        n = C.c_size_t()
        _check(lib().vox_tokenizer_encode(self._h, raw, len(raw), None, 0, C.byref(n)))
        ids = np.empty(n.value, np.int32)
        _check(lib().vox_tokenizer_encode(self._h, raw, len(raw), _ptr(ids), ids.size, C.byref(n)))
        return ids

    def vocab_size(self) -> int:
        n = C.c_size_t()
        _check(lib().vox_tokenizer_vocab_size(self._h, C.byref(n)))
        return n.value

    def __del__(self):
        try:
            if self._h:
                lib().vox_tokenizer_free(self._h)
                self._h = None
        except Exception:
            pass
