#!/usr/bin/env python
"""What the f16 and 8-bit (q8) decoder KV caches save, on the full-size synthetic model (seed 42, the weights bench.py
runs).

  * Memory: device_bytes of unbounded stream pools of 1 and 2 sessions at f32, f16 and q8; their difference is the
    bytes of one session slot, and (80 GB - the model - the pool's fixed part) / slot the slots that fit in 80 GB.
    Computed from the handles' own counts, never by allocating.
  * Soak: an unbounded pool of 8 sessions, every session fed 160 ms of audio per tick (as scripts/stream_soak.py
    does, without waiting for the wall clock), one pool per --soak-dtypes entry in turn.  Per-tick device time
    (vox_stream_stats.gpu_ms) p50 / p95 over the ticks of the first minute of audio and over the ticks after the
    decoder's 8192-position window has filled.  The decoder advances 6.25 positions per second of audio, so 8192
    positions take about 1310 s: the default --soak-seconds 1500 reaches the window; a shorter soak reports the second
    figure as null.
  * Offline: the 16 s B = 8 and B = 1 decode step, one session per --step-dtypes entry, alternating, --rounds rounds,
    medians and ranges (vox_timings: decode_ms - prefill_ms over the graph-replayed steps), and the share of ids each
    type agrees with the first one on.

    python scripts/kv_half_bench.py [--rounds 5] [--soak-seconds 1500] [--soak-dtypes f16,q8]
                                    [--step-dtypes f16,q8] [--out DIR]

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

TICK_SAMPLES = 2560            # 160 ms at 16 kHz
WINDOW_POSITIONS = 8192


def soak(vx, m, audio, kv_dtype, seconds):
    """Per-tick device times of an 8-session unbounded pool: (first minute, after the window filled) in ms."""
    pool = vx.StreamingPool(m, max_sessions=len(audio), max_seconds=None, kv_dtype=kv_dtype)
    try:
        sids = [pool.open() for _ in audio]
        early, late, fed = [], [], 0
        n_ticks = int(seconds * 16000) // TICK_SAMPLES
        for t in range(n_ticks):
            for s, a in zip(sids, audio):
                pool.push(s, a[(fed % a.size):(fed % a.size) + TICK_SAMPLES])
            fed += TICK_SAMPLES
            st = pool.tick()
            for s in sids:
                pool.poll(s)
            pos = pool.session_info(sids[0])["decoder_positions"]
            if fed <= 60 * 16000:
                early.append(st["gpu_ms"])
            elif pos > WINDOW_POSITIONS:
                late.append(st["gpu_ms"])
        return early, late
    finally:
        pool.close()


def pct(x, q):
    return float(np.percentile(x, q)) if x else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=16.0)
    ap.add_argument("--soak-seconds", type=float, default=1500.0)
    ap.add_argument("--soak-dtypes", default="f16,q8")
    ap.add_argument("--step-dtypes", default="f16,q8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    soak_dtypes, step_dtypes = args.soak_dtypes.split(","), args.step_dtypes.split(",")
    import voxtral_mini_realtime_rs_b200 as vx
    from voxtral_mini_realtime_rs_b200 import synth
    from oracle import mel as omel

    if vx.device_count() < 1:
        sys.exit("kv_half_bench.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": gpu, "rounds": args.rounds, "seconds": args.seconds, "memory": {}, "soak_ms": {}, "step_ms": {}}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "full.gguf")
        synth.write_synthetic_gguf(path, synth.VoxtralConfig(), seed=42)
        loader = vx.Q4ModelLoader.from_file(path)
        m = loader.load(0, max_batch=8, max_mel_frames=int(args.seconds * 100) + 1200)
        sessions = {dt: loader.load(0, max_batch=8, max_mel_frames=int(args.seconds * 100) + 1200, kv_dtype=dt)
                    for dt in step_dtypes}
        model_bytes = int(m.info["device_bytes"])

        for dt in ("f32", "f16", "q8"):
            sizes = []
            for n in (1, 2):
                p = vx.StreamingPool(m, max_sessions=n, max_seconds=None, kv_dtype=dt)
                sizes.append(p.device_bytes())
                p.close()
            slot = sizes[1] - sizes[0]
            fixed = sizes[0] - slot
            res["memory"][dt] = {"slot_bytes": slot, "pool_fixed_bytes": fixed,
                                 "slots_in_80GB": (80 * 10 ** 9 - model_bytes - fixed) // slot}
        res["memory"]["model_bytes"] = model_bytes

        audio = [omel.peak_normalize(omel.speechlike(60.0, 40 + i)).astype(np.float32) for i in range(8)]
        for dt in soak_dtypes:
            early, late = soak(vx, m, audio, dt, args.soak_seconds)
            res["soak_ms"][dt] = {"first_minute_p50": pct(early, 50), "first_minute_p95": pct(early, 95),
                                  "window_full_p50": pct(late, 50), "window_full_p95": pct(late, 95),
                                  "window_full_ticks": len(late)}

        mels = np.concatenate([omel.mel_tensor_from_audio(a[:int(args.seconds * 16000)]) for a in audio])

        def step_ms(model, B):
            model.transcribe_streaming(mels[:B])
            tm = vx.Timings()
            ids = np.asarray(model.transcribe_streaming(mels[:B], timings=tm)).reshape(B, -1)
            return (tm.decode_ms - tm.prefill_ms) / (ids.shape[1] - 1), ids

        for B in (8, 1):
            times, ids = {dt: [] for dt in step_dtypes}, {}
            for dt in step_dtypes:
                step_ms(sessions[dt], B)
            for _ in range(args.rounds):
                for dt in step_dtypes:
                    t, ids[dt] = step_ms(sessions[dt], B)
                    times[dt].append(t)
            med = statistics.median
            row = {}
            for dt in step_dtypes:
                row[dt] = med(times[dt])
                row[f"{dt}_range"] = [min(times[dt]), max(times[dt])]
                a, b = ids[step_dtypes[0]], ids[dt]
                n = min(a.shape[1], b.shape[1])
                row[f"{dt}_ids_agree"] = float(np.mean(a[:, :n] == b[:, :n]))
            res["step_ms"][f"B{B}"] = row
        m.close()
        for s_ in sessions.values():
            s_.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "kv_half_bench.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
