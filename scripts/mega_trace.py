"""Phase trace of the persistent decode-step kernel (CTA 0): where one step's time goes.

    python scripts/mega_trace.py [--streams B]      (GPU box)
Prints per op class the mean microseconds spent staging, in the op body (weight stream / attention) and
in the grid barrier, and the step total, from SM-clock stamps the kernel leaves behind.
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
    args = ap.parse_args()
    if not os.path.exists(GGUF):
        synth.write_synthetic_gguf(GGUF, synth.VoxtralConfig(), seed=42)
    B = args.streams
    audio = np.stack([synth.speechlike(16.0, seed=1234 + i) for i in range(B)])
    model = vx.Q4ModelLoader.from_file(GGUF).load(0, max_batch=B, max_mel_frames=2400)
    tm = vx.Timings()
    model.debug("mega_on")
    model.transcribe_pcm(audio, timings=tm)
    model.transcribe_pcm(audio, timings=tm)
    tr = model.debug("mega_trace")
    if tr is None:
        print("no trace (persistent kernel not in use)")
        return
    tr = tr.reshape(-1, 6)
    n = tr.shape[0]
    per_layer = ["qkv", "attn", "wo", "w13", "w2"]
    names = ["embed"] + per_layer * ((n - 3) // len(per_layer)) + ["lm_head", "argmax"]
    agg = {}
    for i, nm in enumerate(names):
        t0, t1, t2, t3, t4, t5 = tr[i]
        if i == n - 1:
            t3 = t2
        a = agg.setdefault(nm, [0] + [0.0] * 6)
        a[0] += 1
        a[1] += t1 - t0            # staging (matvec) / q and the first K tile landed (attention)
        a[2] += t4 - t1            # wait for the first weight stage / KV walk
        a[3] += t5 - t4            # weight loop (matvec)
        a[4] += t2 - max(t5, t4)   # last reduce + epilogue / softmax merge
        a[5] += t3 - t2            # grid barrier
        a[6] += t3 - t0
    step = (tm.decode_ms - tm.prefill_ms) / max(1, tm.decode_tokens - 1)
    print(f"B={B}: step (graph) {step:.3f} ms; traced kernel span {tr[n - 1][2] - tr[0][0]:.1f} us")
    print(f"{'op':8s} {'n':>3s} {'stage':>7s} {'w-wait':>7s} {'loop':>7s} {'tail':>7s} {'barrier':>7s} | {'sum':>7s}  (mean us)  total us")
    for nm, (c, s, w, l, t, g, tot) in agg.items():
        print(f"{nm:8s} {c:3d} {s / c:7.2f} {w / c:7.2f} {l / c:7.2f} {t / c:7.2f} {g / c:7.2f} | {tot / c:7.2f}   {tot:9.1f}")


if __name__ == "__main__":
    main()
