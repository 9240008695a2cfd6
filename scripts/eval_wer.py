#!/usr/bin/env python
"""WER evaluation through the C ABI (the role of the reference's scripts/eval_wer.py, which shells out to its
`voxtral-transcribe` binary; here the model is loaded once in-process and utterances are batched per GPU step).

    python scripts/eval_wer.py --gguf models/voxtral-q4.gguf --tokenizer models/voxtral/tekken.json \
        --manifest utts.jsonl [--batch 8] [--delay 6] [--streaming | --beam W]

`utts.jsonl`: one {"id", "audio": path to a 16 kHz mono WAV (PCM16/float32), "text": reference} per line -- datasets
cannot be downloaded in the build environment, so the loader is a manifest, not HF `datasets`.  Needs the REAL weights
and tokenizer (absent offline: SURVEY F3); `--streaming` feeds every utterance through vox_stream_* in 80 ms pieces
instead of vox_transcribe_pcm and must give the same hypotheses.
Word error rate = word-level Levenshtein distance / reference words after the same normalisation for both sides
(lower-case, punctuation stripped) -- what jiwer computes for the reference's report.  Next to each utterance's WER
the report gives its mean log-probability over the emitted text tokens (ids >= 1000; vox_session_set_top_k): the
utterances the model was least sure of are the ones to review first.  `--beam W` transcribes with beam search of width
W (the best hypothesis, with each token's log-probability in the distribution it was chosen from).  Like the rest of
this script it needs the real weights; the beam option has not been run on real speech.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import struct
import sys
import time
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def read_wav(path: str) -> np.ndarray:
    with wave.open(path, "rb") as w:
        assert w.getframerate() == 16000, f"{path}: resample to 16 kHz first (the reference uses rubato)"
        n, ch, sw = w.getnframes(), w.getnchannels(), w.getsampwidth()
        raw = w.readframes(n)
    if sw == 2:
        a = np.frombuffer(raw, "<i2").astype(np.float32) / 32768.0
    elif sw == 4:
        a = np.frombuffer(raw, "<f4").astype(np.float32)
    else:
        raise ValueError(f"{path}: unsupported sample width {sw}")
    return a.reshape(-1, ch).mean(axis=1).astype(np.float32)


def normalise(text: str) -> list[str]:
    return re.sub(r"[^\w\s']", " ", text.lower()).split()


def edit_distance(a: list[str], b: list[str]) -> int:
    prev = list(range(len(b) + 1))
    for i, x in enumerate(a, 1):
        cur = [i]
        for j, y in enumerate(b, 1):
            cur.append(min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (x != y)))
        prev = cur
    return prev[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gguf", required=True)
    ap.add_argument("--tokenizer", required=True)
    ap.add_argument("--manifest", required=True)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--delay", type=float, default=6.0)
    ap.add_argument("--max-seconds", type=float, default=30.0)
    ap.add_argument("--streaming", action="store_true")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--beam", type=int, default=1, help="beam width (offline only; 1 = greedy)")
    args = ap.parse_args()
    import voxtral_mini_realtime_rs_b200 as vx

    assert args.beam == 1 or not args.streaming, "streaming pools decode greedily"
    utts = [json.loads(l) for l in open(args.manifest) if l.strip()]
    tok = vx.VoxtralTokenizer.from_file(args.tokenizer)
    max_mel = int(args.max_seconds * 100) + 1200
    model = vx.Q4ModelLoader.from_file(args.gguf).load(args.device, max_batch=max(args.batch, args.beam),
                                                        max_mel_frames=max_mel)
    model.set_delay(args.delay)
    model.set_beam(args.beam)
    model.set_top_k(max(1, args.beam))   # each emitted token's log-probability (at W > 1: among its parent's W best)
    errs = words = 0
    audio_s = 0.0
    t0 = time.time()
    out = []

    def decode(ids):
        return tok.decode([int(t) for t in ids if t >= 1000])       # control tokens filtered as transcribe.rs:309-318

    def mean_logprob(ids, lp):   # over the emitted text tokens: the utterance's confidence
        text = np.asarray(ids) >= 1000
        return float(np.mean(lp[text])) if text.any() else None

    if args.streaming:
        pool = vx.StreamingPool(model, max_sessions=args.batch, max_seconds=args.max_seconds)
        pool.set_top_k(1)
    for u in utts:
        a = vx.peak_normalize(read_wav(u["audio"]))
        audio_s += a.size / 16000.0
        if args.streaming:
            sid = pool.open(delay=args.delay)   # a pool session has its own delay (default 6), not the model's
            ids, lps = [], []

            def poll():
                got, _, _, lp = pool.poll(sid, scores=True)
                ids.extend(got)
                lps.append(lp[:, 0])
            for p in range(0, a.size, 1280):
                pool.push(sid, a[p:p + 1280]); pool.tick(); poll()
            pool.finish(sid); pool.tick(); poll()
            pool.close_session(sid)
            lp = np.concatenate(lps)
        else:
            ids = model.transcribe_pcm(a, peak_normalize=False)[0]
            top_ids, top_lp = (x[0] for x in model.token_scores())
            lp = top_lp[np.arange(len(ids)), np.argmax(top_ids == np.asarray(ids)[:, None], axis=1)]
        hyp = decode(ids)
        r, h = normalise(u["text"]), normalise(hyp)
        e = edit_distance(r, h)
        errs += e
        words += len(r)
        out.append({"id": u.get("id"), "wer": e / max(1, len(r)), "mean_logprob": mean_logprob(ids, lp), "hypothesis": hyp})
    wall = time.time() - t0
    print(json.dumps({"utterances": len(utts), "wer": errs / max(1, words), "audio_seconds": audio_s, "wall_seconds": wall,
                      "rtf": wall / max(audio_s, 1e-9), "delay_tokens": args.delay, "results": out}, indent=1))


if __name__ == "__main__":
    main()
