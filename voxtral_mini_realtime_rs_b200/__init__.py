"""voxtral_mini_realtime_rs_b200 -- H100-native (sm_90a) Q4_0 Voxtral-Mini-4B streaming-ASR hot path.

Host-side mirror (ctypes over the C ABI in ``include/voxtral.h``) of the reference crate's public
surface for this path (TrevorS/voxtral-mini-realtime-rs, ``src/lib.rs:22-39``):

    GgufReader, Q4ModelLoader, Q4VoxtralModel        src/gguf/{reader,loader,model}.rs
    Q4Tensor, Q4Linear, q4_matmul                    src/gguf/{tensor,linear,op}.rs
    MelSpectrogram, MelConfig, PadConfig, pad_audio  src/audio/{mel,pad}.rs
    peak_normalize, chunk_audio, needs_chunking      src/audio/{io,chunk}.rs
    TimeEmbedding                                    src/models/time_embedding.rs
    VoxtralTokenizer                                 src/tokenizer/mod.rs

All compute runs in ``libvoxtral_b200.so`` (hand-written CUDA); there is no CPU fallback and no
import of the test oracle -- a missing library or missing GPU raises.
"""
from .api import (  # noqa: F401
    VoxtralError, lib, lib_path, device_count,
    GgufReader, Q4ModelLoader, Q4VoxtralModel, Q4Tensor, Q4Linear, q4_matmul,
    MelSpectrogram, PadConfig, pad_audio, peak_normalize, chunk_audio, needs_chunking, stream_progress,
    TimeEmbedding, VoxtralTokenizer, Timings, DeviceBuffer, PinnedArray, q4_matmul_bench, StreamingPool,
)

__all__ = [
    "VoxtralError", "lib", "lib_path", "device_count", "GgufReader", "Q4ModelLoader", "Q4VoxtralModel",
    "Q4Tensor", "Q4Linear", "q4_matmul", "MelSpectrogram", "PadConfig", "pad_audio", "peak_normalize",
    "chunk_audio", "needs_chunking", "stream_progress", "TimeEmbedding", "VoxtralTokenizer", "Timings", "DeviceBuffer",
    "q4_matmul_bench", "PinnedArray", "StreamingPool",
]
