"""Profiling harness: one single-stream (or B-stream) full transcribe on the full-size synthetic
model, with the CUDA profiler API bracketing only the region of interest.  Meant to run under a
profiler that honours cudaProfilerStart/Stop; numbers printed while under a profiler are never
bench values.

    python scripts/profile_decode.py [--streams B] [--region decode|encode|all] [--eager]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import voxtral_mini_realtime_rs_b200 as vx  # noqa: E402
from voxtral_mini_realtime_rs_b200 import synth  # noqa: E402

GGUF = os.environ.get("VOX_BENCH_GGUF", "/dev/shm/voxtral_synth_s42.gguf")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=1)
    ap.add_argument("--seconds", type=float, default=16.0)
    ap.add_argument("--region", default="all", choices=["all", "encode"])
    ap.add_argument("--eager", action="store_true", help="no CUDA graph for the decode loop")
    args = ap.parse_args()
    if not os.path.exists(GGUF):
        synth.write_synthetic_gguf(GGUF, synth.VoxtralConfig(), seed=42)
    B = args.streams
    audio = np.stack([synth.speechlike(args.seconds, seed=1234 + i) for i in range(B)])
    model = vx.Q4ModelLoader.from_file(GGUF).load(0, max_batch=B, max_mel_frames=2400)
    if args.eager:
        model.debug("graph_off")
    tm = vx.Timings()
    model.transcribe_pcm(audio, timings=tm)        # warm-up (also captures the graph)
    vx.lib().vox_profiler_start()
    if args.region == "encode":
        from numpy import float32
        mel = np.zeros((B, 128, 2344), float32)
        model.encode_audio(mel)
    else:
        ids = model.transcribe_pcm(audio, timings=tm)
    vx.lib().vox_profiler_stop()
    print(f"profiled region done: pre {tm.preprocess_ms:.2f} enc {tm.encode_ms:.2f} dec {tm.decode_ms:.2f} ms "
          f"(prefill {tm.prefill_ms:.2f}), tokens {tm.decode_tokens}")


if __name__ == "__main__":
    main()
