#!/usr/bin/env python
"""What phrase boosting costs per decode step, on the full-size synthetic model (seed 42, the weights bench.py runs).

For B = 1 and B = 8 streams of 16 s, transcribe_streaming runs with no list and with a list of 256 four-token phrases
on every stream (random text ids, boost 2.0), the two settings alternating in one run so that both see the same clocks
and neighbours.  Each setting first runs once untimed (it re-captures the decode-step graph), then once timed: the
decode steps after the prefill, replayed from the captured graph, timed by the session's CUDA events (vox_timings:
decode_ms - prefill_ms over n_out - 1 steps).

    python scripts/bias_bench.py [--rounds 5] [--out DIR]

Prints one JSON line with the card's name and power limit; with --out also writes it there.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=16.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import voxtral_mini_realtime_rs_b200 as vx
    from voxtral_mini_realtime_rs_b200 import synth
    from oracle import mel as omel

    if vx.device_count() < 1:
        sys.exit("bias_bench.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": gpu, "rounds": args.rounds, "seconds": args.seconds, "phrases": 256, "phrase_len": 4, "step_ms": {}}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "full.gguf")
        synth.write_synthetic_gguf(path, synth.VoxtralConfig(), seed=42)
        m = vx.Q4ModelLoader.from_file(path).load(0, max_batch=8, max_mel_frames=int(args.seconds * 100) + 1200)
        audio = [omel.peak_normalize(omel.speechlike(args.seconds, 40 + i)) for i in range(8)]
        mels = np.concatenate([omel.mel_tensor_from_audio(a) for a in audio])
        rng = np.random.default_rng(0)
        phrases = rng.integers(1000, m.info["vocab"], size=(256, 4)).tolist()

        def step_ms(B, on):
            m.set_bias(phrases if on else [], 2.0)
            m.transcribe_streaming(mels[:B])                 # re-captures the step graph for this setting
            tm = vx.Timings()
            ids = np.asarray(m.transcribe_streaming(mels[:B], timings=tm)).reshape(B, -1)
            return (tm.decode_ms - tm.prefill_ms) / (ids.shape[1] - 1), ids

        for B in (1, 8):
            off, on = [], []
            step_ms(B, False)                                # warm-up
            flipped = 0
            for _ in range(args.rounds):
                t0, i0 = step_ms(B, False)
                t1, i1 = step_ms(B, True)
                flipped = int(np.sum(i0 != i1))
                off.append(t0)
                on.append(t1)
            med = statistics.median
            res["step_ms"][f"B{B}"] = {"off": med(off), "on": med(on), "off_range": [min(off), max(off)],
                                       "on_range": [min(on), max(on)],
                                       "overhead_pct": 100.0 * (med(on) - med(off)) / med(off), "steps": int(i0.shape[1] - 1),
                                       "ids_changed": flipped}
        m.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "bias_bench.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
