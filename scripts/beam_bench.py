#!/usr/bin/env python
"""What beam search costs per decode step, on the full-size synthetic model (seed 42, the weights bench.py runs).

For (b streams, W beams) in (1,1), (1,4), (1,8), (2,4), (8,1), transcribe_streaming runs on 16 s streams; every round
runs each configuration once, so greedy and beam configurations alternate and see the same clocks and neighbours.  A
configuration first runs once untimed (it captures the decode-step graph), then once per round timed: the decode steps
after the prefill (and, at W > 1, the position-0 selection), replayed from the captured graph, timed by the session's
CUDA events (vox_timings: decode_ms - prefill_ms over n_out - 1 steps; at W > 1 this includes the one traceback).

Fork bytes per step are computed from shapes: at most b * (W - 1) rows change parent per step, and each copies at most
15 positions x layers x kv heads x head_dim floats of K and of V, plus its page-table entries.

    python scripts/beam_bench.py [--rounds 5] [--out DIR]

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

CONFIGS = [(1, 1), (1, 4), (1, 8), (2, 4), (8, 1)]


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
        sys.exit("beam_bench.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": gpu, "rounds": args.rounds, "seconds": args.seconds, "configs": {}}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "full.gguf")
        synth.write_synthetic_gguf(path, synth.VoxtralConfig(), seed=42)
        m = vx.Q4ModelLoader.from_file(path).load(0, max_batch=8, max_mel_frames=int(args.seconds * 100) + 1200)
        info = m.info
        audio = [omel.peak_normalize(omel.speechlike(args.seconds, 40 + i)) for i in range(8)]
        mels = np.concatenate([omel.mel_tensor_from_audio(a) for a in audio])

        def run(b, W):
            m.set_beam(W)
            tm = vx.Timings()
            ids = np.asarray(m.transcribe_streaming(mels[:b], timings=tm)).reshape(b, -1)
            m.set_beam(1)
            return (tm.decode_ms - tm.prefill_ms) / (ids.shape[1] - 1), ids

        times = {c: [] for c in CONFIGS}
        first = {}
        for c in CONFIGS:
            first[c] = run(*c)[1]                            # captures the step graph of this configuration
        for _ in range(args.rounds):
            for c in CONFIGS:
                t, ids = run(*c)
                assert np.array_equal(ids, first[c]), f"{c}: ids changed between runs"
                times[c].append(t)
        fork_row = 15 * info["dec_layers"] * info["dec_kv_heads"] * info["dec_head_dim"] * 4 * 2
        for (b, W), ts in times.items():
            ms = statistics.median(ts)
            res["configs"][f"b{b}_w{W}"] = {
                "step_ms": ms, "step_ms_range": [min(ts), max(ts)], "tok_s_per_stream": 1000.0 / ms,
                "fork_bytes_per_step_max": b * (W - 1) * fork_row, "steps": int(first[(b, W)].shape[1] - 1)}
        g1 = first[(1, 1)][0]
        for W in (4, 8):
            res["configs"][f"b1_w{W}"]["positions_differing_from_greedy"] = int((first[(1, W)][0] != g1).sum())
        m.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "beam_bench.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
