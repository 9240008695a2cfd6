#!/usr/bin/env python
"""Soak of an unbounded streaming pool (max_seconds=None) on the full-size synthetic model.

    python scripts/stream_soak.py [--sessions 8] [--minutes 25] [--piece-ms 160] [--gguf PATH] [--out FILE]

N sessions open together and each gets `piece-ms` of deterministic synthetic audio per tick (160 ms = one decoder
position, so every tick carries one decoder step for every session, as in live captioning).  Prints one JSON line:
per-tick device time (vox_stream_stats.gpu_ms) p50 / p95 during the first minute of audio and after the decoder's
sliding window has filled (dec_window positions of 160 ms, ~21.8 min at 8192), the KV pages each session holds, and
the card's name and power limit read in the same run.  A tick is real-time when it takes less than `piece-ms`.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines()[0].split(", ") + ["?"])[:2] if q.returncode == 0 and q.stdout.strip() else ("?", "?")
    return {"name": name, "power_limit": power}


def pct(v, q):
    return float(np.percentile(v, q)) if len(v) else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, default=8)
    ap.add_argument("--minutes", type=float, default=25.0)
    ap.add_argument("--piece-ms", type=int, default=160)
    ap.add_argument("--gguf", default=os.environ.get("VOX_BENCH_GGUF", "/dev/shm/voxtral_synth_s42.gguf"))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import voxtral_mini_realtime_rs_b200 as vx
    from voxtral_mini_realtime_rs_b200 import synth
    from oracle import mel as omel
    if vx.device_count() < 1:
        raise SystemExit("stream_soak: no CUDA device (times are only measured on the GPU)")
    if not os.path.exists(a.gguf):
        synth.write_synthetic_gguf(a.gguf, synth.VoxtralConfig(), seed=42)
    model = vx.Q4ModelLoader.from_file(a.gguf).load(0, max_batch=1, max_mel_frames=3000)
    dec_window = model.info["dec_window"]
    pool = vx.StreamingPool(model, max_sessions=a.sessions, max_seconds=None)
    sids = [pool.open() for _ in range(a.sessions)]
    piece = 16 * a.piece_ms
    chunk_s = 60.0                                   # audio generated one minute at a time per session
    bufs = [None] * a.sessions
    fed = [0] * a.sessions
    total = int(a.minutes * 60 * 16000)
    early, late, window_s = [], [], dec_window * 0.16
    ids = 0
    t0 = time.time()
    for tick in range(total // piece):
        for i, sid in enumerate(sids):
            off = fed[i] % int(chunk_s * 16000)
            if off == 0:
                bufs[i] = omel.peak_normalize(omel.speechlike(chunk_s, 1000 * i + fed[i] // int(chunk_s * 16000)))
            pool.push(sid, bufs[i][off:off + piece])
            fed[i] += piece
        st = pool.tick()
        for sid in sids:
            ids += len(pool.poll(sid)[0])
        t_audio = fed[0] / 16000.0
        if t_audio <= 60.0:
            early.append(st["gpu_ms"])
        elif t_audio > window_s + 6.0:              # + the left padding: positions count from the padded start
            late.append(st["gpu_ms"])
    infos = [pool.session_info(s) for s in sids]
    res = {
        "sessions": a.sessions, "minutes": a.minutes, "piece_ms": a.piece_ms, "dec_window": dec_window,
        "first_minute_tick_ms": {"p50": pct(early, 50), "p95": pct(early, 95), "ticks": len(early)},
        "window_full_tick_ms": {"p50": pct(late, 50), "p95": pct(late, 95), "ticks": len(late)},
        "kv_pages_per_session": sorted({inf["kv_pages"] for inf in infos}),
        "decoder_positions": infos[0]["decoder_positions"], "ids": ids,
        "wall_s": round(time.time() - t0, 1), "card": card(),
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    pool.close()
    model.close()


if __name__ == "__main__":
    main()
