#!/usr/bin/env python
"""What mixing transcription delays in one batch costs, on the full-size synthetic model (seed 42, the weights bench.py
runs).  Alternating in one run, so that both arms see the same clocks and neighbours:

  * decode step, B = 8 (one persistent-kernel launch): every stream at delay 6 against 8 distinct delays (the same
    kernels either way: each row reads its own stream's ffn_norm x ADA vector);
  * pool tick, 8 streaming sessions fed 160 ms each per tick: all at delay 6 against 8 distinct delays.

    python scripts/delay_mix_bench.py [--rounds 10] [--steps 120] [--out DIR]

Decode steps are timed with a host clock around `steps` device-fed steps (no host round trip per step) that end in a
synchronise of the session's stream; ticks by the pool's own device timer (vox_stream_stats.gpu_ms).
Prints one JSON line; with --out also writes it there.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MIXED = [0.5, 1.0, 2.75, 6.0, 8.5, 12.0, 20.5, 30.0]
PREFIX = [1] + [32] * 37


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=120)   # 20 s of audio: 171 positions
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import voxtral_mini_realtime_rs_b200 as vx
    from voxtral_mini_realtime_rs_b200 import synth
    from oracle import mel as omel

    if vx.device_count() < 1:
        sys.exit("delay_mix_bench.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "full.gguf")
        synth.write_synthetic_gguf(path, synth.VoxtralConfig(), seed=42)
        m = vx.Q4ModelLoader.from_file(path).load(0, max_batch=8, max_mel_frames=3000)
        audio = [omel.peak_normalize(omel.speechlike(20.0, 40 + i)) for i in range(8)]
        mels = np.concatenate([omel.mel_tensor_from_audio(a) for a in audio])

        def decode_ms(delays):
            m.set_delays(delays)
            m.encode_audio(mels)
            m.reset_cache()
            m.prefill(np.tile(PREFIX, (8, 1)).astype(np.int32))
            for _ in range(5):
                m.decode_step(batch=8)                    # reading the ids synchronises the session's stream
            t0 = time.perf_counter()
            for _ in range(args.steps - 1):
                m.decode_step(batch=8, read=False)
            m.decode_step(batch=8)
            return (time.perf_counter() - t0) * 1e3 / args.steps

        def tick_ms(delays):
            pool = vx.StreamingPool(m, max_sessions=8, max_seconds=30.0)
            try:
                sids = [pool.open(delay=dl) for dl in delays]
                times = []
                for t in range(args.ticks + 30):
                    for s, a in zip(sids, audio):
                        pool.push(s, a[t * 2560:(t + 1) * 2560])
                    st = pool.tick()
                    if t >= 30 and st["decode_steps"] > 0:   # after the prefills: steady decoding ticks
                        times.append(st["gpu_ms"])
                return statistics.median(times)
            finally:
                pool.close()

        uni, mix, tu, tm = [], [], [], []
        for _ in range(args.rounds):
            uni.append(decode_ms([6.0] * 8))
            mix.append(decode_ms(MIXED))
            tu.append(tick_ms([6.0] * 8))
            tm.append(tick_ms(MIXED))
        m.close()
    med = statistics.median
    res = {"gpu": gpu, "decode_step_ms": {"one_delay": med(uni), "eight_delays": med(mix),
                                          "one_delay_range": [min(uni), max(uni)], "eight_delays_range": [min(mix), max(mix)]},
           "pool_tick_ms": {"one_delay": med(tu), "eight_delays": med(tm),
                            "one_delay_range": [min(tu), max(tu)], "eight_delays_range": [min(tm), max(tm)]},
           "rounds": args.rounds, "steps": args.steps, "ticks": args.ticks, "mixed_delays": MIXED}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "delay_mix_bench.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
