#!/usr/bin/env python
"""What transcribing streams of different lengths in one call (vox_transcribe_pcm_ragged) saves, on the full-size
synthetic model (seed 42, the weights bench.py runs).  One session (max_batch 8, 2600 mel frames) serves every leg.

A. Eight streams of 4, 6, ..., 18 s:
     ragged   one vox_transcribe_pcm_ragged call;
     singles  the same eight streams as eight single-stream vox_transcribe_pcm calls;
     padded   one equal-length vox_transcribe_pcm call with every stream zero-padded to 18 s -- a cost reference only:
              its ids differ (the padding is transcribed).
   Per leg: encode_ms and decode_ms (the session's CUDA events, summed over the leg's calls), device ms (preprocess +
   encode + decode), host ms (a host clock around the leg, which ends in a synchronise), sum of n_out over device ms,
   and for the ragged call the persistent-kernel launches per decode step.
B. A 10-minute recording cut into 1200-frame chunks (vox_chunk_plan, 50 chunks):
     long     transcribe_long at max_batch 8 (7 ragged calls);
     chunks   one vox_transcribe_pcm call per chunk.
   Host ms per leg.

Every round runs every leg once, so the legs alternate and see the same clocks and neighbours; each leg runs once
untimed first.  Reported: the median over rounds and the range.  Outputs are checked against the first run of the same
leg, and the ragged streams' ids against the single-stream calls (streams whose ids are equal are counted).

    python scripts/ragged_bench.py [--rounds 5] [--out DIR]

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
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SECONDS_A = [4.0 + 2.0 * i for i in range(8)]
LONG_SECONDS = 600.0
CHUNK_FRAMES = 1200


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import voxtral_mini_realtime_rs_b200 as vx
    from voxtral_mini_realtime_rs_b200 import synth

    if vx.device_count() < 1:
        sys.exit("ragged_bench.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": gpu, "rounds": args.rounds, "A": {}, "B": {}}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "full.gguf")
        synth.write_synthetic_gguf(path, synth.VoxtralConfig(), seed=42)
        m = vx.Q4ModelLoader.from_file(path).load(0, max_batch=8, max_mel_frames=2600)
        streams = [vx.peak_normalize(synth.speechlike(s, 50 + i)) for i, s in enumerate(SECONDS_A)]
        n_long = max(a.size for a in streams)
        padded = np.stack([np.concatenate([a, np.zeros(n_long - a.size, np.float32)]) for a in streams])
        n_out = [vx.stream_n_out(a.size) for a in streams]
        rec = synth.speechlike(LONG_SECONDS, 7)
        plan = vx.chunk_audio(rec.size, CHUNK_FRAMES, 0)
        rec_norm = vx.peak_normalize(rec)

        def timed(fn):
            tms = []
            t0 = time.perf_counter()
            out = fn(tms)
            host = (time.perf_counter() - t0) * 1e3
            return out, host, tms

        def leg_ragged(tms):
            tm = vx.Timings()
            before = float(m.debug("mega_epoch")[0])
            ids = m.transcribe_pcm_ragged(streams, peak_normalize=False, timings=tm)
            tms.append(tm)
            tms.append(float(m.debug("mega_epoch")[0]) - before)
            return ids

        def leg_singles(tms):
            ids = []
            for a in streams:
                tm = vx.Timings()
                ids.append(m.transcribe_pcm(a, peak_normalize=False, timings=tm)[0])
                tms.append(tm)
            return ids

        def leg_padded(tms):
            tm = vx.Timings()
            ids = m.transcribe_pcm(padded, peak_normalize=False, timings=tm)
            tms.append(tm)
            return list(ids)

        def leg_long(tms):
            return m.transcribe_long(rec, max_mel_frames=CHUNK_FRAMES)[0]

        def leg_chunks(tms):
            return [m.transcribe_pcm(rec_norm[a:b], peak_normalize=False)[0] for a, b, _, _ in plan]

        legs = {"ragged": leg_ragged, "singles": leg_singles, "padded": leg_padded, "long": leg_long, "chunks": leg_chunks}
        first = {k: timed(f)[0] for k, f in legs.items()}
        samples = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, f in legs.items():
                out, host, tms = timed(f)
                assert all(np.array_equal(x, y) for x, y in zip(out, first[k])), f"{k}: ids changed between runs"
                samples[k].append((host, tms))

        def med(xs):
            return {"median": statistics.median(xs), "range": [min(xs), max(xs)]}

        for k in ("ragged", "singles", "padded"):
            rows = samples[k]
            tm_lists = [[t for t in tms if isinstance(t, vx.Timings)] for _, tms in rows]
            enc = [sum(t.encode_ms for t in tl) for tl in tm_lists]
            dec = [sum(t.decode_ms for t in tl) for tl in tm_lists]
            dev = [sum(t.preprocess_ms + t.encode_ms + t.decode_ms for t in tl) for tl in tm_lists]
            toks = sum(len(x) for x in first[k])
            res["A"][k] = {"encode_ms": med(enc), "decode_ms": med(dec), "device_ms": med(dev),
                           "host_ms": med([h for h, _ in rows]), "tokens": toks,
                           "tok_per_device_s": toks / (statistics.median(dev) / 1e3)}
        launches = samples["ragged"][0][1][1]
        res["A"]["ragged"]["mega_launches_per_step"] = launches / (max(n_out) - 1)
        res["A"]["n_out"] = n_out
        res["A"]["ragged_streams_equal_to_singles"] = int(sum(np.array_equal(x, y) for x, y in
                                                             zip(first["ragged"], first["singles"])))
        for k in ("long", "chunks"):
            res["B"][k] = {"host_ms": med([h for h, _ in samples[k]])}
        res["B"]["chunks"]["n"] = len(plan)
        res["B"]["recording_s"] = LONG_SECONDS
        res["B"]["chunks_equal"] = int(sum(np.array_equal(x, y) for x, y in zip(first["long"], first["chunks"])))
        res["B"]["tokens"] = int(sum(len(x) for x in first["long"]))
        m.close()
    line = json.dumps(res, default=float)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "ragged_bench.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
